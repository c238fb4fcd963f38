"""Drop-in for the reference's `losses` package (losses/__init__.py:1-2) when `make-a-scene_b200/` precedes the reference
root on sys.path: `losses.discriminator` (the PatchGAN discriminator) and `losses.lpips` (the LPIPS perceptual loss) are
ours, on the sm_90a kernels; every other module (`loss_img`, `loss_seg`, `lpips_with_object`, ...) resolves to the
reference's own file through the extended package path, so `loss_img.py`'s `from .discriminator import Discriminator,
weights_init` and `lpips_with_object.py`'s `from .lpips import LPIPS` pick up this package's modules.

The reference's re-exports are resolved lazily: importing `losses.discriminator` does not import LPIPS or torchvision."""
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)

_EXPORTS = {"BCELossWithQuant": "loss_seg", "VQVAEWithBCELoss": "loss_seg", "VQLPIPSWithDiscriminator": "loss_img"}


def __getattr__(name):
    mod = _EXPORTS.get(name)
    if mod is None:
        raise AttributeError("module %r has no attribute %r" % (__name__, name))
    import importlib
    return getattr(importlib.import_module("." + mod, __name__), name)
