"""``python -m generativemodels_b200.bundle run <id> [<id> ...] --config_file configs/inference.json [--bundle brain|cxr]
[--key value ...]``

Mirrors ``python -m monai.bundle run`` for the reference's two latent-diffusion bundles (their docs/README.md):
resolves the requested items of the bundle's unmodified ``inference.json`` on this package's classes.  ``--bundle``
picks the bundle's ``scripts.*`` classes: ``brain`` (the brain-LDM bundle, the default) or ``cxr`` (the chest X-ray
text-to-image bundle); without it the bundle is detected from the config path's directory name.  ``--key value``
overrides a config item (JSON value or ``$expression``), e.g. ``--age 0.7 --brain_vol 0.5``; with no checkpoint files
at hand, ``--load_autoencoder '$None' --load_diffusion '$None'`` samples from randomly initialised networks.  For the
chest X-ray bundle without a CLIP download, ``--prompt_embeds '$torch.load("emb.pt").to(@device)'`` supplies the
(2, 77, 1024) embeddings of the empty and the user's prompt.
"""
from __future__ import annotations

import sys

from .config import BUNDLES, BundleConfig, parse_cli_value


def main(argv: list[str]) -> int:
    if not argv or argv[0] != "run":
        print(__doc__)
        return 2
    ids, overrides, config_file, bundle = [], {}, None, None
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
    BundleConfig(config_file, overrides, bundle=bundle).run(*ids)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
