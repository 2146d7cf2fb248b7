"""TEST-ONLY CPU stand-in for the sampler entry point of libb200gen.so (include/b200gen_samplers.h), on HOST pointers:
tests/cpu_backend.FakeLib extended by b200_dpm_solver_step, which views its pointers as host tensors and stores what
the float64 reading of the contract (tests/dpm_solver_emulator.abi_step) computes.  install() routes the product's
C-ABI calls to it."""
from generativemodels_b200 import _lib
from tests import cpu_backend
from tests import dpm_solver_emulator as E
from tests.cpu_backend import _obj, f32, store32


class SamplersFakeLib(cpu_backend.FakeLib):
    def b200_dpm_solver_step(self, m, s, hist, n_hist, nz, c, prev, x0o, n, stream):
        assert 0 <= n_hist <= _lib.DPM_MAX_HIST and prev and x0o
        rp, rx = E.abi_step(f32(m, n), f32(s, n), [f32(hist[k], n) for k in range(n_hist)], f32(nz, n), _obj(c), n)
        store32(prev, rp)
        store32(x0o, rx)
        return 0


def install(monkeypatch):
    """cpu_backend.install with the stand-in that also serves the sampler entry point (tests only)."""
    cpu_backend.install(monkeypatch)
    fake = SamplersFakeLib()
    monkeypatch.setattr(_lib, "require_device", lambda: fake)
    import generativemodels_b200.networks.schedulers.dpm_solver as D
    monkeypatch.setattr(D, "_prep", lambda *ts: [None if t is None else t.float().contiguous() for t in ts])
    return fake
