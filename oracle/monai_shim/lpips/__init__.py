"""Stand-in for the `lpips` package, which the reference's generative/losses/perceptual.py imports at module level:
importing it works, constructing an LPIPS network raises (its weights are a download).  Lets the unmodified reference
losses import offline for the resnet50 network type."""


class LPIPS:
    def __init__(self, *args, **kwargs):
        raise RuntimeError("lpips is not installed here: the LPIPS networks are not available offline")
