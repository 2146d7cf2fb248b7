"""TEST-ONLY CPU stand-in for the SA-Solver entry point of libb200gen.so (include/b200gen_samplers.h), on HOST
pointers: tests/samplers_backend.SamplersFakeLib extended by b200_sa_solver_step, which views its pointers as host
tensors and stores what the float64 reading of the contract (tests/sa_solver_emulator.abi_step) computes.  install()
routes the product's C-ABI calls to it."""
from generativemodels_b200 import _lib
from tests import cpu_backend, samplers_backend
from tests import sa_solver_emulator as E
from tests.cpu_backend import _obj, f32, store32


class SASolverFakeLib(samplers_backend.SamplersFakeLib):
    def b200_sa_solver_step(self, m, s, last, zl, hist, n_hist, z, c, prev, x0o, xco, n, stream):
        assert 0 <= n_hist <= _lib.SA_SOLVER_MAX_HIST and prev and x0o and xco and (last or not zl)
        rp, rx, rc = E.abi_step(f32(m, n), f32(s, n), f32(last, n), f32(zl, n),
                                [f32(hist[k], n) for k in range(n_hist)], f32(z, n), _obj(c), n)
        store32(prev, rp)
        store32(x0o, rx)
        store32(xco, rc)
        return 0


def install(monkeypatch):
    """cpu_backend.install with the stand-in that also serves the sampler entry points (tests only)."""
    cpu_backend.install(monkeypatch)
    fake = SASolverFakeLib()
    monkeypatch.setattr(_lib, "require_device", lambda: fake)
    import generativemodels_b200.networks.schedulers.dpm_solver as D
    import generativemodels_b200.networks.schedulers.sa_solver as S
    for mod in (D, S):
        monkeypatch.setattr(mod, "_prep", lambda *ts: [None if t is None else t.float().contiguous() for t in ts])
    return fake
