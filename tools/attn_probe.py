"""Dev probe: one full-length attention call (T = S = 89 600, d = 512), timed with CUDA events."""
import math, sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch
from generativemodels_b200 import ops
T = S = 89600
dh = 512
torch.manual_seed(0)
q = (torch.randn(1, T, dh, device="cuda") * 0.5).to(ops.H16)
k = (torch.randn(1, S, dh, device="cuda") * 0.5).to(ops.H16)
vt = torch.randn(1, dh, S, device="cuda").to(ops.H16)
for i in range(6):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    o = ops.attention(q, k, None, 1, dh, 1 / math.sqrt(dh), vt=vt)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    print(f"flash attention T=S={T} d={dh}: {ms:.2f} ms, {4*T*S*dh/ms/1e9:.0f} TFLOP/s algorithmic")
