"""yolact_b200 -- H100-native (sm_90a) YOLACT inference path behind the reference's
Yolact.forward() / Detect() / postprocess() surface.  See DESIGN.md and INTEGRATION.md."""
from .config import cfg, set_cfg, CONFIGS, MEANS, STD  # noqa: F401

__all__ = ["cfg", "set_cfg", "CONFIGS", "Yolact", "Detect", "postprocess", "FastBaseTransform"]


def __getattr__(name):  # lazy: importing the package must not require torch/CUDA
    if name == "Yolact":
        from .yolact import Yolact
        return Yolact
    if name == "Detect":
        from .detection import Detect
        return Detect
    if name == "postprocess":
        from .output_utils import postprocess
        return postprocess
    if name == "FastBaseTransform":
        from .augmentations import FastBaseTransform
        return FastBaseTransform
    raise AttributeError(name)
