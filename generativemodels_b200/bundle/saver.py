"""``NiftiSaver`` of the brain-LDM bundle (model-zoo/models/brain_image_synthesis_latent_diffusion_model/scripts/
saver.py:8-33): crop the decoded volume, min-max normalise to uint8 and write ``<name>.nii.gz``; and ``JPGSaver`` of
the chest X-ray bundle (below).

The reference delegates the file format to ``nibabel`` (not vendored under /root/reference and not installed in this
image); the writer below restates the published NIfTI-1 single-file layout (348-byte header, 4-byte extension flag,
voxel data x-fastest) with the fields ``nibabel.Nifti1Image(data, affine, Nifti1Header())`` is documented to fill:
sform = the affine with code 2 ("aligned"), quaternion parameters of the same affine with qform_code 0, unit zooms,
``scl_slope``/``scl_inter`` = NaN (no scaling), magic ``n+1``.  tests/test_bundle.py reads the file back through the
standard's byte offsets — parity with nibabel itself is unpinned.

The crop / normalise / quantise arithmetic runs on the device the sample lives on (three fp32 IEEE operations per
voxel, the same ones numpy performs in the reference, so the bytes are identical) and only the uint8 volume crosses
PCIe — 4x less than the reference's fp32 ``.cpu()``.
"""
from __future__ import annotations

import gzip
import math
import struct

import numpy as np
import torch


def _quaternion(affine: np.ndarray):
    """(qfac, b, c, d) of the affine's rotation part (NIfTI-1 standard, 'METHOD 2')."""
    R = affine[:3, :3].astype(np.float64)
    zooms = np.sqrt((R * R).sum(axis=0))
    zooms[zooms == 0] = 1.0
    R = R / zooms
    qfac = 1.0
    if np.linalg.det(R) < 0:
        R[:, 2] = -R[:, 2]
        qfac = -1.0
    tr = 1.0 + R[0, 0] + R[1, 1] + R[2, 2]
    if tr > 0.5:
        a = 0.5 * math.sqrt(tr)
        b = 0.25 * (R[2, 1] - R[1, 2]) / a
        c = 0.25 * (R[0, 2] - R[2, 0]) / a
        d = 0.25 * (R[1, 0] - R[0, 1]) / a
    else:                                                   # near a 180 degree rotation: solve for the largest term
        xd = 1.0 + R[0, 0] - (R[1, 1] + R[2, 2])
        yd = 1.0 + R[1, 1] - (R[0, 0] + R[2, 2])
        zd = 1.0 + R[2, 2] - (R[0, 0] + R[1, 1])
        if xd > 1.0:
            b = 0.5 * math.sqrt(xd)
            c, d, a = 0.25 * (R[0, 1] + R[1, 0]) / b, 0.25 * (R[0, 2] + R[2, 0]) / b, 0.25 * (R[2, 1] - R[1, 2]) / b
        elif yd > 1.0:
            c = 0.5 * math.sqrt(yd)
            b, d, a = 0.25 * (R[0, 1] + R[1, 0]) / c, 0.25 * (R[1, 2] + R[2, 1]) / c, 0.25 * (R[0, 2] - R[2, 0]) / c
        else:
            d = 0.5 * math.sqrt(zd)
            b, c, a = 0.25 * (R[0, 2] + R[2, 0]) / d, 0.25 * (R[1, 2] + R[2, 1]) / d, 0.25 * (R[1, 0] - R[0, 1]) / d
        if a < 0:
            b, c, d = -b, -c, -d
    return qfac, b, c, d, zooms


def nifti1_bytes(volume_u8: np.ndarray, affine: np.ndarray) -> bytes:
    """Single-file NIfTI-1 image of a 3-D uint8 array indexed [x, y, z]."""
    if volume_u8.dtype != np.uint8 or volume_u8.ndim != 3:
        raise ValueError("expected a 3-D uint8 volume")
    qfac, qb, qc, qd, zooms = _quaternion(affine)
    nan = float("nan")
    hdr = bytearray(348)
    struct.pack_into("<i", hdr, 0, 348)                                         # sizeof_hdr
    hdr[38:39] = b"r"                                                           # regular
    struct.pack_into("<8h", hdr, 40, 3, *volume_u8.shape, 1, 1, 1, 1)           # dim
    struct.pack_into("<hh", hdr, 70, 2, 8)                                      # datatype DT_UINT8, bitpix
    struct.pack_into("<8f", hdr, 76, qfac, *zooms, 1.0, 1.0, 1.0, 1.0)          # pixdim
    struct.pack_into("<f", hdr, 108, 352.0)                                     # vox_offset
    struct.pack_into("<ff", hdr, 112, nan, nan)                                 # scl_slope, scl_inter: no scaling
    struct.pack_into("<hh", hdr, 252, 0, 2)                                     # qform_code unknown, sform_code aligned
    struct.pack_into("<6f", hdr, 256, qb, qc, qd, *affine[:3, 3])               # quatern_b/c/d, qoffset_x/y/z
    struct.pack_into("<12f", hdr, 280, *affine[0], *affine[1], *affine[2])      # srow_x, srow_y, srow_z
    hdr[344:348] = b"n+1\0"
    return bytes(hdr) + b"\0\0\0\0" + np.asfortranarray(volume_u8).tobytes(order="F")


class NiftiSaver:
    def __init__(self, output_dir: str) -> None:
        super().__init__()
        self.output_dir = output_dir
        self.affine = np.array(                                 # saver.py:12-19 (the bundle's template space)
            [
                [-1.0, 0.0, 0.0, 96.48149872],
                [0.0, 1.0, 0.0, -141.47715759],
                [0.0, 0.0, 1.0, -156.55375671],
                [0.0, 0.0, 0.0, 1.0],
            ]
        )

    @staticmethod
    def quantise(image_data: torch.Tensor) -> np.ndarray:
        """saver.py:22-25 on the sample's own device: crop, min-max normalise, scale to [0, 255], truncate to uint8."""
        v = image_data[0, 0, 5:-5, 5:-5, :-15].float()
        lo, hi = v.min(), v.max()
        v = (v - lo) / (hi - lo)
        return (v * 255).to(torch.uint8).cpu().numpy()

    def save(self, image_data: torch.Tensor, file_name: str) -> None:
        payload = nifti1_bytes(self.quantise(image_data), self.affine)
        with gzip.open(f"{str(self.output_dir)}/{file_name}.nii.gz", "wb") as f:
            f.write(payload)


class JPGSaver:
    """``JPGSaver`` of the chest X-ray bundle (model-zoo/models/cxr_image_synthesis_latent_diffusion_model/scripts/
    saver.py:8-17): clip the decoded image to [0, 1], scale by 255, truncate to uint8 and write plane ``[0, 0]`` as
    ``<output_dir>/<file_name>.jpg`` through PIL.

    The clip / scale / truncate runs on the sample's device in its own dtype — the IEEE operations numpy performs in the
    reference, so the array handed to PIL is identical — and only the uint8 plane crosses PCIe.  PIL is needed only
    to write the file: a missing PIL raises ``ImportError`` at ``save``, not at import."""

    def __init__(self, output_dir: str) -> None:
        super().__init__()
        self.output_dir = output_dir

    @staticmethod
    def quantise(image_data: torch.Tensor) -> np.ndarray:
        """saver.py:14-16 up to the PIL call: ``(clip(x, 0, 1) * 255).astype(uint8)`` of plane [0, 0]."""
        v = image_data[0, 0]
        if v.dtype not in (torch.float16, torch.float32, torch.float64):
            v = v.float()
        return (v.clamp(0, 1) * 255).to(torch.uint8).cpu().numpy()

    def save(self, image_data: torch.Tensor, file_name: str) -> None:
        try:
            from PIL import Image
        except ImportError as e:
            raise ImportError("JPGSaver writes its .jpg through Pillow (PIL), which is not installed: "
                              "pip install pillow") from e
        Image.fromarray(self.quantise(image_data)).save(f"{str(self.output_dir)}/{file_name}.jpg")
