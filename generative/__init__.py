"""``generative`` — the reference's import path, served by the H100-native implementation.

SURVEY.md section 8(b): callers of MONAI-GenerativeModels import ``generative.networks.nets``,
``generative.networks.layers``, ``generative.networks.schedulers``, ``generative.networks.blocks``,
``generative.inferers`` and ``generative.utils`` (reference: generative/networks/nets/__init__.py:14-22,
generative/inferers/__init__.py:14-20, generative/networks/schedulers/__init__.py:14-17).  With this repository's root
on ``sys.path`` those imports resolve here, and every ``generative.<x>`` module *is* the ``generativemodels_b200.<x>``
module of the same relative name (one module object under two names, so classes, ``isinstance`` checks and pickles
agree) — a tutorial's sampling cell or a reference test runs with only ``sys.path`` changed.

The discriminators (``PatchDiscriminator``, ``MultiScalePatchDiscriminator``) are provided as forward-only,
inference-mode networks.  The training-side parts of the reference (``generative.losses``, ``generative.metrics``,
``generative.engines``) are not provided: importing them raises ``ModuleNotFoundError`` naming this scope
(SURVEY.md section 8, out of scope), rather than silently resolving to something else.
"""
from __future__ import annotations

import importlib
import importlib.abc
import importlib.util
import sys

_SRC = "generativemodels_b200"
_OUT_OF_SCOPE = ("generative.losses", "generative.metrics", "generative.engines")


class _AliasFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    """``generative.a.b`` -> the already-importable module ``generativemodels_b200.a.b`` (same object)."""

    def find_spec(self, fullname, path=None, target=None):
        if not fullname.startswith("generative."):
            return None
        if fullname.startswith(_OUT_OF_SCOPE):
            raise ModuleNotFoundError(
                f"{fullname}: this package provides the reference's sampling path only (networks, schedulers, "
                "inferers, utils); losses / metrics / engines are out of scope (SURVEY.md section 8)", name=fullname)
        real = _SRC + fullname[len("generative"):]
        try:
            spec = importlib.util.find_spec(real)
        except ModuleNotFoundError:
            return None
        if spec is None:
            return None
        return importlib.util.spec_from_loader(fullname, self, is_package=spec.submodule_search_locations is not None)

    def create_module(self, spec):
        real = importlib.import_module(_SRC + spec.name[len("generative"):])
        self._specs[id(real)] = real.__spec__
        return real

    def exec_module(self, module):       # the real module is already executed; keep its own spec
        spec = self._specs.pop(id(module), None)
        if spec is not None:
            module.__spec__ = spec

    _specs: dict = {}


if not any(isinstance(f, _AliasFinder) for f in sys.meta_path):
    sys.meta_path.insert(0, _AliasFinder())

from generativemodels_b200 import __version__ as __version__  # noqa: E402
