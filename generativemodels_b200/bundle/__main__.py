"""``python -m generativemodels_b200.bundle run <id> [<id> ...] --config_file <file | list of files>
[--meta_file configs/metadata.json] [--bundle brain|cxr|mednist_ddpm] [--key value ...]``

Mirrors ``python -m monai.bundle run`` for the reference's model-zoo bundles (their docs/README.md): resolves the
requested items of the bundle's unmodified configs on this package's classes.  ``--config_file`` is one JSON / YAML
file or, as MONAI's CLI receives it, a Python list of files merged in order (later top-level keys win):
``"['configs/common.yaml', 'configs/infer.yaml']"`` or ``"'configs/common.yaml', 'configs/infer.yaml'"``.
``--meta_file`` is stored under the ``_meta_`` key.  ``--bundle`` picks the bundle's ``scripts.*`` classes: ``brain``
(the brain-LDM bundle, the default), ``cxr`` (the chest X-ray text-to-image bundle) or ``mednist_ddpm`` (the MedNIST
DDPM bundle); without it the bundle is detected from the (first) config path's directory name.  ``--key value``
overrides a config item (JSON value or ``$expression``), e.g. ``--age 0.7 --brain_vol 0.5``; with no checkpoint files
at hand, ``--load_autoencoder '$None' --load_diffusion '$None'`` samples from randomly initialised networks.  For the
chest X-ray bundle without a CLIP download, ``--prompt_embeds '$torch.load("emb.pt").to(@device)'`` supplies the
(2, 77, 1024) embeddings of the empty and the user's prompt.  The MedNIST bundle runs as its notebook calls it:
``run testing --meta_file configs/metadata.json --config_file "'configs/common.yaml', 'configs/infer.yaml'"
--ckpt_path model.pt --bundle_root . --out_file test.pt``, plus ``--imports`` without ``$import monai`` where MONAI is
not installed.
"""
from __future__ import annotations

import ast
import os
import sys

from .config import BUNDLES, BundleConfig, parse_cli_value


def parse_config_file(value: str):
    """An existing file as is; otherwise a Python list / tuple literal of files (MONAI's CLI form)."""
    if os.path.isfile(value):
        return value
    try:
        files = ast.literal_eval(value)
    except (ValueError, SyntaxError):
        return value                                # a missing file: open() reports it
    if isinstance(files, str):
        return files
    if isinstance(files, (list, tuple)) and files and all(isinstance(f, str) for f in files):
        return list(files)
    return value


def main(argv: list[str]) -> int:
    if not argv or argv[0] != "run":
        print(__doc__)
        return 2
    ids, overrides, config_file, bundle, meta_file = [], {}, None, None, None
    it = iter(argv[1:])
    for a in it:
        if a.startswith("--"):
            try:
                value = next(it)
            except StopIteration:
                print(f"option {a} needs a value")
                return 2
            if a == "--config_file":
                config_file = parse_config_file(value)
            elif a == "--meta_file":
                meta_file = value
            elif a == "--bundle":
                bundle = value
            else:
                overrides[a[2:]] = parse_cli_value(value)
        else:
            ids.append(a)
    if config_file is None or not ids:
        print(__doc__)
        return 2
    if bundle is not None and bundle not in BUNDLES:
        print(f"unknown --bundle {bundle!r}; expected one of {', '.join(sorted(BUNDLES))}")
        return 2
    BundleConfig(config_file, overrides, bundle=bundle, meta_file=meta_file).run(*ids)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
