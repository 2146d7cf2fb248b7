"""Import the UNMODIFIED reference (a checkout of the reference project, REFERENCE_DIR or /root/reference) as
`generative`, on top of oracle/monai_shim when real MONAI is absent.  Only usable where such a checkout is present and
readable: used to validate oracle/torch_oracle.py and by tests/golden/make_golden*.py to generate the committed
fixtures."""
import os
import sys
from pathlib import Path

REF_ROOT = Path(os.environ.get("REFERENCE_DIR", "/root/reference"))
_SHIM = Path(__file__).resolve().parent / "monai_shim"


def available() -> bool:
    try:
        return (REF_ROOT / "generative" / "__init__.py").is_file()
    except OSError:           # a checkout this user may not read counts as absent
        return False


def import_reference():
    if not available():
        raise ImportError(f"{REF_ROOT} is not present or not readable; use the committed golden vectors")
    try:
        import monai  # noqa: F401
    except Exception:
        if str(_SHIM) not in sys.path:
            sys.path.insert(0, str(_SHIM))
    if str(REF_ROOT) not in sys.path:
        sys.path.insert(0, str(REF_ROOT))
    import generative  # noqa: F401
    from generative import inferers, networks  # noqa: F401
    from generative.networks import nets, schedulers  # noqa: F401
    return generative
