"""sr3_b200 -- H100-native SR3 diffusion hot path (UNet forward + p_sample loop) behind the reference's
`model.networks.define_G` / `GaussianDiffusion` interface.  The compute lives in lib/libsr3_b200.so
(hand-written sm_90a CUDA, C ABI in include/sr3_b200.h); this package is the thin host-side mirror of the
reference's Python interface.  There is no CPU / eager fallback: without the library or an H100 the ops raise."""
from . import _native  # noqa: F401
from .model import networks  # noqa: F401
from .model.networks import define_G  # noqa: F401
from .model.sr3_modules.diffusion import GaussianDiffusion  # noqa: F401
from .model.sr3_modules.unet import UNet  # noqa: F401
from .optim import FusedAdam  # noqa: F401

__all__ = ["define_G", "networks", "GaussianDiffusion", "UNet", "FusedAdam"]
__version__ = "0.1.0"
