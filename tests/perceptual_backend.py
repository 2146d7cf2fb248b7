"""TEST-ONLY CPU stand-in for the perceptual entry points of libb200gen.so (include/b200gen_perceptual.h), on HOST
pointers: tests/fid_backend.FidFakeLib extended by b200_perceptual_prep, b200_perceptual_distance and
b200_perceptual_mean, each viewing its pointers as host tensors and storing what the float64 reading of the contract
(tests/perceptual_emulator.py) computes.  install() routes the product's C-ABI calls to it, the ResNet-50's
convolutions included."""
import ctypes as C

import torch

from generativemodels_b200 import _lib, ops
from tests import fid_backend
from tests import igemm_emulator as IE
from tests import perceptual_emulator as E
from tests.cpu_backend import _np, _strided, bf16, f32, rows16


class PerceptualFakeLib(fid_backend.FidFakeLib):
    def b200_perceptual_prep(self, x, xdt, xs, y, ydt, ys, C_, S, OH, OW, idx, n_out, out_x, out_y, stream):
        ids = None if not idx else torch.from_numpy(_np(idx, n_out, C.c_int64).copy())
        N_ = (int(ids.max()) // S + 1) if ids is not None else n_out
        for ptr, dt, st, out in ((x, xdt, xs, out_x), (y, ydt, ys, out_y)):
            src = _strided(ptr, dt, list(st[:5]), [N_, C_, S, OH, OW])
            z = E.prep(E.gather(src, S, ids))
            o = torch.zeros(n_out, OH, OW, 8, dtype=ops.H16)
            o[..., :3] = z.permute(0, 2, 3, 1).to(ops.H16)
            bf16(out, o.numel()).copy_(o.reshape(-1))
        return 0

    def b200_perceptual_distance(self, x, y, dt, B, HW, C_, pitch, pixel, image, image32, stream):
        if dt == _lib.DT_F32:
            fx, fy = (f32(p, B * HW * pitch).view(B, HW, pitch)[..., :C_] for p in (x, y))
        else:
            fx, fy = (rows16(p, B * HW, pitch, C_).reshape(B, HW, C_) for p in (x, y))
        v = E.distance(fx, fy)
        _np(image, B, C.c_double)[:] = v.numpy()
        if image32:
            f32(image32, B).copy_(v.float())
        return 0

    def b200_perceptual_mean(self, image, n_groups, counts, means, loss, stream):
        cnt = [counts[g] for g in range(n_groups)]
        img = torch.from_numpy(_np(image, sum(cnt), C.c_double).copy())
        m = E.mean(img, cnt)
        _np(means, n_groups + 1, C.c_double)[:] = m.numpy()
        f32(loss, 1)[0] = float(m[-1])
        return 0


def install(monkeypatch):
    """fid_backend.install with the stand-in that also serves the perceptual entry points (tests only)."""
    fid_backend.install(monkeypatch)
    fake = PerceptualFakeLib()
    monkeypatch.setattr(_lib, "require_device", lambda: fake)
    monkeypatch.setattr(ops, "igemm_raw", lambda p, split_k=True: IE.emulate(p))
    import generativemodels_b200.losses.perceptual as P
    monkeypatch.setattr(P, "require_cuda", lambda x, m: None)
    return fake
