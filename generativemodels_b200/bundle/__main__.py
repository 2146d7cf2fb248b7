"""``python -m generativemodels_b200.bundle run <id> [<id> ...] --config_file configs/inference.json [--key value ...]``

Mirrors ``python -m monai.bundle run`` for the brain-LDM bundle (its docs/README.md): resolves the requested items of
the bundle's unmodified ``inference.json`` on this package's classes.  ``--key value`` overrides a config item (JSON value
or ``$expression``), e.g. ``--age 0.7 --brain_vol 0.5``; with no checkpoint files at hand,
``--load_autoencoder '$None' --load_diffusion '$None'`` samples from randomly initialised networks.
"""
from __future__ import annotations

import sys

from .config import BundleConfig, parse_cli_value


def main(argv: list[str]) -> int:
    if not argv or argv[0] != "run":
        print(__doc__)
        return 2
    ids, overrides, config_file = [], {}, None
    it = iter(argv[1:])
    for a in it:
        if a.startswith("--"):
            try:
                value = next(it)
            except StopIteration:
                print(f"option {a} needs a value")
                return 2
            if a == "--config_file":
                config_file = value
            else:
                overrides[a[2:]] = parse_cli_value(value)
        else:
            ids.append(a)
    if config_file is None or not ids:
        print(__doc__)
        return 2
    BundleConfig(config_file, overrides).run(*ids)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
