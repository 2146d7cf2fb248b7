from .encoder_modules import SpatialRescaler  # noqa: F401
from .selfattention import SABlock  # noqa: F401
from .spade_norm import SPADE, SegPyramid  # noqa: F401
from .transformerblock import TransformerBlock  # noqa: F401
