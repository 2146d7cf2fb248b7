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
SURVEY.md §8f rank 4, not a re-implementation of MONAI's bundle machinery (no ``_mode_``, no macros ``%``).

The chest X-ray bundle (``model-zoo/models/cxr_image_synthesis_latent_diffusion_model``) runs the same way with
``bundle="cxr"``: its ``scripts.sampler.Sampler`` is the guided sampler of :mod:`.cxr_sampler` and its
``scripts.saver.JPGSaver`` the JPEG writer of :mod:`.saver`.  Items resolve lazily, so running ``save_jpg`` with an
overridden ``prompt_embeds`` never builds the file's ``tokenizer`` / ``text_encoder``; only its ``imports`` still name
``transformers`` and can be overridden where that package is absent.

The MedNIST DDPM bundle (``model-zoo/models/mednist_ddpm``, ``bundle="mednist_ddpm"``) keeps its configs as YAML split
over several files: inference is ``common.yaml`` + ``infer.yaml``, with ``metadata.json`` passed as the meta file.  So
``config`` may also be

* a ``.yaml`` / ``.yml`` path (read with PyYAML's ``safe_load``; PyYAML is needed only then);
* a sequence of paths, JSON and YAML mixed, merged as MONAI's ``read_config`` merges a list: the files are read in
  order and a top-level key of a later file replaces the same key of an earlier one (no deeper merge).

``meta_file`` (a path or a dict) is stored under the ``_meta_`` key, as MONAI's ``read_meta`` does.  A ``_target_``
without a dot (``Compose``, ``ScaleIntensity``, ``ToTensor``, ``SaveImage`` in that bundle's ``save_trans``) is looked
up the way MONAI's component locator does, among the imported ``monai.*`` modules; MONAI's transforms are host-side
post-processing this package does not restate, so such a target needs MONAI installed.  The bundle's ``scripts``
package only holds a training helper, so it needs no remapping; ``$import scripts`` resolves to the bundle's own (or
any importable) ``scripts`` package.
"""
from __future__ import annotations

import importlib
import inspect
import json
import os
import re
import sys
from collections.abc import Sequence
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
    # its scripts package only defines a training helper (inv_metric_cmp_fn): nothing to remap
    "mednist_ddpm": ("mednist_ddpm", {}),
}
DEFAULT_BUNDLE = "brain"
_PREFIX_MAP = (("generative.", "generativemodels_b200."),)
_REF = re.compile(r"@((?:\w+)(?:(?:#|::)\w+)*)")
_SPECIAL = ("_target_", "_requires_", "_disabled_", "_desc_")
META_KEY = "_meta_"


def _locate_monai(name: str):
    """A dotless ``_target_`` the way MONAI's ComponentLocator finds it: the class or function ``name`` defined in an
    imported ``monai.*`` module (the first such module in import order)."""
    try:
        importlib.import_module("monai")            # MONAI's __init__ imports its submodules
    except ImportError as e:
        raise ModuleNotFoundError(f"_target_ '{name}' has no module path; MONAI looks such names up among its monai.* "
                                  f"modules, and MONAI is not installed (pip install monai)") from e
    for modname, mod in list(sys.modules.items()):
        if mod is None or not (modname == "monai" or modname.startswith("monai.")):
            continue
        obj = getattr(mod, name, None)
        if (inspect.isclass(obj) or inspect.isfunction(obj)) and obj.__module__ == modname:
            return obj
    raise ValueError(f"_target_ '{name}' is not defined in any imported monai.* module")


def _locate(path: str, target_map: dict = TARGET_MAP):
    path = target_map.get(path, path)
    for old, new in _PREFIX_MAP:
        if path.startswith(old):
            path = new + path[len(old):]
    module, _, name = path.rpartition(".")
    if not module:
        return _locate_monai(path)
    return getattr(importlib.import_module(module), name)


def load_config_file(path: str | os.PathLike) -> dict:
    """One config file: JSON, or YAML for a ``.yaml`` / ``.yml`` suffix."""
    with open(path) as f:
        if Path(path).suffix.lower() in (".yaml", ".yml"):
            try:
                import yaml
            except ImportError as e:
                raise ImportError(f"reading {os.fspath(path)!r} needs PyYAML (pip install pyyaml)") from e
            return yaml.safe_load(f)
        return json.load(f)


def load_config_files(files: str | os.PathLike | Sequence) -> dict:
    """One path or a sequence of paths merged as MONAI's ``read_config`` merges a list: read in order, a top-level key
    of a later file replacing the same key of an earlier one."""
    if isinstance(files, (str, os.PathLike)):
        files = [files]
    merged: dict = {}
    for f in files:
        merged.update(load_config_file(f))
    return merged


def _is_paths(config) -> bool:
    return isinstance(config, (str, os.PathLike)) or (
        isinstance(config, Sequence) and len(config) > 0 and all(isinstance(c, (str, os.PathLike)) for c in config))


def detect_bundle(config_path: str | os.PathLike | Sequence | None) -> str:
    """Short name of the bundle whose directory (its model-zoo name) contains ``config_path`` (the first path of a
    sequence); the brain bundle when none does (or there is no path)."""
    if config_path is not None and not isinstance(config_path, (str, os.PathLike)):
        config_path = config_path[0] if len(config_path) else None
    if config_path is not None:
        parts = Path(os.path.abspath(config_path)).parts
        for name, (dirname, _) in BUNDLES.items():
            if dirname in parts:
                return name
    return DEFAULT_BUNDLE


class BundleConfig:
    """A bundle's config (the parsed dict, a JSON or YAML path, or a sequence of paths merged in order, later
    top-level keys winning) with ``overrides`` applied.  ``meta_file`` (a path or a dict) is stored under ``_meta_``.
    ``bundle`` ("brain", "cxr" or "mednist_ddpm") selects the map of the bundle's ``scripts.*`` targets; by default it
    is detected from the (first) config path and is the brain bundle otherwise."""

    def __init__(self, config: dict | str | Sequence, overrides: dict | None = None, bundle: str | None = None,
                 meta_file: dict | str | os.PathLike | None = None) -> None:
        paths = _is_paths(config)
        if bundle is None:
            bundle = detect_bundle(config if paths else None)
        if bundle not in BUNDLES:
            raise ValueError(f"unknown bundle {bundle!r}; expected one of {sorted(BUNDLES)}")
        self.bundle = bundle
        self.target_map = BUNDLES[bundle][1]
        if paths:
            config = load_config_files(config)
        if meta_file is not None:
            # MONAI's read_meta then read_config: the meta goes in first, a config's own _meta_ key replaces it
            meta = meta_file if isinstance(meta_file, dict) else load_config_file(meta_file)
            config = {META_KEY: meta, **config}
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
