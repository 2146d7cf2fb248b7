"""Reference fixtures written by the unmodified reference (make_golden*.py).  A fixture is one dict; save() stores it
as a head file <stem>.pt whose tensors are packed, flattened and cut where needed, into part files
<stem>.part<k>.pt of at most PART_BYTES each, so that no stored file exceeds 1 MB.  load() restores the dict exactly
(same dtypes, shapes and values); a plain torch.save file without parts loads as is."""
from pathlib import Path

import torch

GOLD = Path(__file__).resolve().parent
PART_BYTES = 768 * 1024


def save(obj, stem: str) -> None:
    parts, cur, cur_bytes = [], {}, 0

    def put(t):
        nonlocal cur, cur_bytes
        flat = t.detach().reshape(-1)
        per = max(1, PART_BYTES // t.element_size())
        refs = []
        for i in range(0, max(flat.numel(), 1), per):
            piece = flat[i:i + per].clone()
            if cur and cur_bytes + piece.nbytes > PART_BYTES:
                parts.append(cur)
                cur, cur_bytes = {}, 0
            key = f"t{len(cur)}"
            cur[key] = piece
            cur_bytes += piece.nbytes
            refs.append((len(parts), key))
        return {"__golden_part__": refs, "shape": tuple(t.shape)}

    def walk(o):
        if torch.is_tensor(o):
            return put(o)
        if isinstance(o, dict):
            return {k: walk(v) for k, v in o.items()}
        if isinstance(o, (list, tuple)):
            return type(o)(walk(v) for v in o)
        return o

    head = walk(obj)
    if cur:
        parts.append(cur)
    for old in GOLD.glob(f"{stem}.part*.pt"):
        old.unlink()
    torch.save({"head": head, "n_parts": len(parts)}, GOLD / f"{stem}.pt")
    for k, p in enumerate(parts):
        torch.save(p, GOLD / f"{stem}.part{k}.pt")


def load(stem: str):
    f = torch.load(GOLD / f"{stem}.pt", weights_only=False)
    if not (isinstance(f, dict) and set(f) == {"head", "n_parts"}):
        return f
    parts = [torch.load(GOLD / f"{stem}.part{k}.pt", weights_only=True) for k in range(f["n_parts"])]

    def walk(o):
        if isinstance(o, dict) and "__golden_part__" in o:
            return torch.cat([parts[p][k] for p, k in o["__golden_part__"]]).reshape(o["shape"])
        if isinstance(o, dict):
            return {k: walk(v) for k, v in o.items()}
        if isinstance(o, (list, tuple)):
            return type(o)(walk(v) for v in o)
        return o

    return walk(f["head"])
