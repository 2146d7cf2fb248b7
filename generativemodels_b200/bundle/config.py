"""Just enough of the MONAI-bundle configuration language to run the reference's own
``model-zoo/models/brain_image_synthesis_latent_diffusion_model/configs/inference.json`` unmodified on this package.

The bundle is driven by ``python -m monai.bundle run <id> --config_file configs/inference.json --age 0.7 ...``
(the bundle's docs/README.md); MONAI is not part of the reference repository, so the subset of its published
``ConfigParser`` semantics that file uses is restated here:

* ``"imports"``: a list of ``"$import x"`` / ``"$from x import y"`` statements that populate the expression globals;
* ``"$<python expression>"``: evaluated lazily, at most once; ``@id`` inside it is replaced by the resolved item;
* ``"@id"``: reference to another item (``#`` or ``::`` descend into dicts and lists);
* ``{"_target_": "pkg.mod.Class", "_requires_": ..., "_disabled_": ..., **kwargs}``: resolve ``_requires_`` first,
  then instantiate ``Class(**resolved kwargs)``;
* anything else is a literal, resolved recursively.

``_target_`` paths are remapped so the unmodified file lands on this package's classes:
``generative.…`` → ``generativemodels_b200.…`` and the bundle's ``scripts.sampler.Sampler`` / ``scripts.saver.
NiftiSaver`` → :mod:`generativemodels_b200.bundle`.  Nothing here touches the GPU; it is the thin app edge of
SURVEY.md §8f rank 4, not a re-implementation of MONAI's bundle machinery (no ``_mode_``, no macros ``%``, no YAML).

The chest X-ray bundle (``model-zoo/models/cxr_image_synthesis_latent_diffusion_model``) runs the same way with
``bundle="cxr"``: its ``scripts.sampler.Sampler`` is the guided sampler of :mod:`.cxr_sampler` and its
``scripts.saver.JPGSaver`` the JPEG writer of :mod:`.saver`.  Items resolve lazily, so running ``save_jpg`` with an
overridden ``prompt_embeds`` never builds the file's ``tokenizer`` / ``text_encoder``; only its ``imports`` still name
``transformers`` and can be overridden where that package is absent.
"""
from __future__ import annotations

import importlib
import json
import os
import re
from pathlib import Path
from typing import Any

TARGET_MAP = {
    "scripts.sampler.Sampler": "generativemodels_b200.bundle.sampler.Sampler",
    "scripts.saver.NiftiSaver": "generativemodels_b200.bundle.saver.NiftiSaver",
}
CXR_TARGET_MAP = {
    "scripts.sampler.Sampler": "generativemodels_b200.bundle.cxr_sampler.Sampler",
    "scripts.saver.JPGSaver": "generativemodels_b200.bundle.saver.JPGSaver",
}
# Both bundles name their scripts ``scripts.sampler.Sampler``, so the ``scripts.*`` map is chosen per bundle:
# short name -> (the bundle's directory name in the reference's model zoo, its script map).
BUNDLES = {
    "brain": ("brain_image_synthesis_latent_diffusion_model", TARGET_MAP),
    "cxr": ("cxr_image_synthesis_latent_diffusion_model", CXR_TARGET_MAP),
}
DEFAULT_BUNDLE = "brain"
_PREFIX_MAP = (("generative.", "generativemodels_b200."),)
_REF = re.compile(r"@((?:\w+)(?:(?:#|::)\w+)*)")
_SPECIAL = ("_target_", "_requires_", "_disabled_", "_desc_")


def _locate(path: str, target_map: dict = TARGET_MAP):
    path = target_map.get(path, path)
    for old, new in _PREFIX_MAP:
        if path.startswith(old):
            path = new + path[len(old):]
    module, _, name = path.rpartition(".")
    if not module:
        raise ValueError(f"_target_ '{path}' is not a dotted path")
    return getattr(importlib.import_module(module), name)


def detect_bundle(config_path: str | os.PathLike | None) -> str:
    """Short name of the bundle whose directory (its model-zoo name) contains ``config_path``; the brain bundle when
    none does (or there is no path)."""
    if config_path is not None:
        parts = Path(os.path.abspath(config_path)).parts
        for name, (dirname, _) in BUNDLES.items():
            if dirname in parts:
                return name
    return DEFAULT_BUNDLE


class BundleConfig:
    """A bundle's ``inference.json`` (a path or the parsed dict) with ``overrides`` applied.  ``bundle`` ("brain" or
    "cxr") selects the map of the bundle's ``scripts.*`` targets; by default it is detected from the config path and
    is the brain bundle otherwise."""

    def __init__(self, config: dict | str, overrides: dict | None = None, bundle: str | None = None) -> None:
        if bundle is None:
            bundle = detect_bundle(config if isinstance(config, (str, os.PathLike)) else None)
        if bundle not in BUNDLES:
            raise ValueError(f"unknown bundle {bundle!r}; expected one of {sorted(BUNDLES)}")
        self.bundle = bundle
        self.target_map = BUNDLES[bundle][1]
        if isinstance(config, (str, os.PathLike)):
            with open(config) as f:
                config = json.load(f)
        self.config = dict(config)
        for k, v in (overrides or {}).items():
            self[k] = v
        self._resolved: dict[str, Any] = {}
        self._resolving: list[str] = []
        self._globals: dict[str, Any] | None = None

    # -- raw access ----------------------------------------------------------------------------------------------
    def __setitem__(self, id: str, value: Any) -> None:
        keys = re.split(r"#|::", id)
        node = self.config
        for k in keys[:-1]:
            node = node[int(k)] if isinstance(node, list) else node[k]
        if isinstance(node, list):
            node[int(keys[-1])] = value
        else:
            node[keys[-1]] = value
        self._resolved = {}

    def _raw(self, id: str) -> Any:
        node = self.config
        for k in re.split(r"#|::", id):
            try:
                node = node[int(k)] if isinstance(node, list) else node[k]
            except (KeyError, IndexError, ValueError):
                raise KeyError(f"config item '{id}' does not exist") from None
        return node

    # -- evaluation ----------------------------------------------------------------------------------------------
    def _expr_globals(self) -> dict:
        if self._globals is None:
            g: dict[str, Any] = {}
            for stmt in self.config.get("imports", []):
                if not (isinstance(stmt, str) and stmt.startswith("$")):
                    raise ValueError(f"'imports' entries must be '$import ...' statements, got {stmt!r}")
                exec(stmt[1:], g)                                   # noqa: S102 - the config is the program
            self._globals = g
        return self._globals

    def _eval(self, expr: str) -> Any:
        refs: dict[str, Any] = {}

        def sub(m):
            refs[m.group(1)] = self.get(m.group(1))
            return f"__refs__[{m.group(1)!r}]"
        code = _REF.sub(sub, expr)
        # the references go into a copy of the GLOBALS: names used inside comprehensions / lambdas of the expression are
        # looked up there, not in the eval locals (NameError on Python < 3.12 otherwise)
        return eval(code, {**self._expr_globals(), "__refs__": refs})   # noqa: S307

    def _resolve(self, node: Any) -> Any:
        if isinstance(node, str):
            if node.startswith("$"):
                return self._eval(node[1:])
            if node.startswith("@") and _REF.fullmatch(node):
                return self.get(node[1:])
            return node
        if isinstance(node, list):
            return [self._resolve(v) for v in node]
        if isinstance(node, dict):
            if "_target_" not in node:
                return {k: self._resolve(v) for k, v in node.items()}
            requires = node.get("_requires_", [])
            for r in requires if isinstance(requires, list) else [requires]:
                self._resolve(r)
            if self._resolve(node.get("_disabled_", False)) in (True, "true", "True"):
                return None
            kwargs = {k: self._resolve(v) for k, v in node.items() if k not in _SPECIAL}
            return _locate(node["_target_"], self.target_map)(**kwargs)
        return node

    def get(self, id: str) -> Any:
        """Resolved value of item ``id`` (instantiated / evaluated once, then cached)."""
        if id in self._resolved:
            return self._resolved[id]
        if id in self._resolving:
            raise ValueError("circular reference: " + " -> ".join(self._resolving + [id]))
        self._resolving.append(id)
        try:
            value = self._resolve(self._raw(id))
        finally:
            self._resolving.pop()
        self._resolved[id] = value
        return value

    def run(self, *ids: str) -> list:
        return [self.get(i) for i in ids]


def parse_cli_value(text: str) -> Any:
    """``--age 0.7`` → 0.7, ``--load_diffusion '$None'`` stays an expression, anything unparsable stays a string."""
    try:
        return json.loads(text)
    except json.JSONDecodeError:
        return text
