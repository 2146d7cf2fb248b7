"""Pre-packed weight cache file (SURVEY.md §8f rank 4: ``state_dict`` → packed-weight file).

Every convolution / linear layer is repacked once into the K-major h16 tap matrices the wgmma implicit-GEMM kernel
reads (ops.PackedConv and friends) the first time the network runs.  ``save_packed`` writes those packed objects of a
*warm* network to one file; ``load_packed`` installs them into a freshly constructed network whose ``state_dict`` has
the same fingerprint, so a serving process goes from ``load_state_dict`` to its first sample without the repacking
pass.  A file whose fingerprint does not match the live weights is refused (returns False) — the network then packs
lazily as usual; nothing is ever computed from stale weights.

    model(x, t)                                   # or one sampler step: populates the per-module caches
    save_packed(model, "unet.packed.pt")
    ...
    model = DiffusionModelUNet(**kw).cuda().eval(); model.load_state_dict(sd)
    load_packed(model, "unet.packed.pt")          # True: first forward launches kernels only
"""
from __future__ import annotations

import hashlib

import torch
import torch.nn as nn

from ..networks._holders import LinearHolder, _key

_FORMAT = 1
_INT_VIEW = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def fingerprint(model: nn.Module) -> str:
    """Names, shapes, dtypes and two exact integer checksums (plain and position-weighted sum of the raw bit
    patterns, computed on the tensor's own device) of every ``state_dict`` entry."""
    h = hashlib.sha256()
    sums = []
    for name, t in model.state_dict().items():
        h.update(f"{name}|{tuple(t.shape)}|{t.dtype};".encode())
        if t.numel() == 0:
            continue
        bits = t.detach().contiguous().view(-1).view(_INT_VIEW[t.element_size()]).to(torch.int64)
        ramp = torch.arange(bits.numel(), device=bits.device, dtype=torch.int64) % 251 + 1
        sums.append(torch.stack([bits.sum(), (bits * ramp).sum()]).cpu())
    if sums:
        h.update(torch.stack(sums).numpy().tobytes())
    return h.hexdigest()


def _move(obj, device):
    """Packed objects are plain attribute bags of tensors / nested lists and tuples."""
    if torch.is_tensor(obj):
        return obj.to(device)
    if isinstance(obj, list):
        return [_move(v, device) for v in obj]
    if isinstance(obj, tuple):
        return tuple(_move(v, device) for v in obj)
    if hasattr(obj, "__dict__") and type(obj).__module__.startswith("generativemodels_b200"):
        clone = object.__new__(type(obj))
        clone.__dict__.update({k: _move(v, device) for k, v in obj.__dict__.items()})
        return clone
    return obj


def _param_names(module: nn.Module, key) -> list[str | None]:
    """Names (within ``module``) of the parameters a cache key was built from, matched by data_ptr."""
    by_ptr = {p.data_ptr(): n for n, p in module.named_parameters()}
    return [None if k is None else by_ptr.get(k[0], "?") for k in key]


def save_packed(model: nn.Module, path: str) -> int:
    """Write every packed weight currently cached in ``model``; returns the number of entries."""
    entries = []
    for mname, m in model.named_modules():
        for extra, (k, obj) in m.__dict__.get("_pack_cache", {}).items():
            entries.append(dict(module=mname, kind="pack", extra=extra, params=_param_names(m, k[1]),
                                obj=_move(obj, "cpu")))
        for lname, holder in m.__dict__.get("_lin_holders", {}).items():
            for extra, (k, obj) in holder.__dict__.get("_pack_cache", {}).items():
                entries.append(dict(module=mname, kind="lin", name=lname, extra=extra,
                                    params=_param_names(holder.lin, k[1]), obj=_move(obj, "cpu")))
    if any("?" in e["params"] for e in entries):
        raise RuntimeError("a cached packed weight no longer matches the module's parameters")
    torch.save(dict(format=_FORMAT, fingerprint=fingerprint(model), entries=entries), path)
    return len(entries)


def load_packed(model: nn.Module, path: str) -> bool:
    """Install the packed weights of ``path`` into ``model``.  False (and nothing installed) if the file was written
    for different weights or by another format version.  The file is a pickle of this package's packed-weight objects
    (``torch.load(weights_only=False)``): load only files you wrote yourself, like any ``torch.load`` checkpoint."""
    blob = torch.load(path, map_location="cpu", weights_only=False)
    if blob.get("format") != _FORMAT or blob.get("fingerprint") != fingerprint(model):
        return False
    modules = dict(model.named_modules())
    staged = []
    for e in blob["entries"]:
        m = modules.get(e["module"])
        if m is None:
            return False
        if e["kind"] == "lin":
            lin = getattr(m, e["name"]) if "." not in e["name"] else m.get_submodule(e["name"])
            owner, source = LinearHolder(lin), lin
        else:
            owner, source = m, m
        named = dict(source.named_parameters())
        if any(n is not None and n not in named for n in e["params"]):
            return False
        params = [None if n is None else named[n] for n in e["params"]]
        device = next((p.device for p in params if p is not None), torch.device("cpu"))
        staged.append((m, e, owner, (e["extra"], _key(*params)), _move(e["obj"], device)))
    for m, e, owner, key, obj in staged:
        if e["kind"] == "lin":
            m.__dict__.setdefault("_lin_holders", {})[e["name"]] = owner
        owner.__dict__.setdefault("_pack_cache", {})[e["extra"]] = (key, obj)
    return True
