"""nope_b200 -- H100-native implementation of the NOPE (nv-nguyen/nope) inference hot
path: pose-conditioned UNet sweep over a pose grid + template scoring + top-k."""
from ._lib import NopeError, load as load_library  # noqa: F401

__all__ = ["NopeError", "load_library"]
