"""Drop-in for the reference's `losses` package (losses/__init__.py:1-2) when `make-a-scene_b200/` precedes the reference
root on sys.path: `losses.discriminator` (the PatchGAN discriminator), `losses.lpips` (the LPIPS perceptual loss) and
`losses.face_loss` (the VGGFace2 face loss) are ours, on the sm_90a kernels, as are `losses.object_loss` (the
object-aware loss, which the reference has no module for) and `losses.scene_loss` (kernel forms of `loss_seg.py`'s two
VQ-SEG objectives, under a module name of its own); every other module (`loss_img`, `loss_seg`,
`lpips_with_object`, ...) resolves to the reference's own file through the extended package path, so `loss_img.py`'s
`from .discriminator import Discriminator, weights_init` and `from .face_loss import FaceLoss`, and
`lpips_with_object.py`'s `from .lpips import LPIPS` pick up this package's modules.

The reference's re-exports are resolved lazily: importing one of the three modules imports neither of the other two, nor
torchvision."""
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)

_EXPORTS = {"BCELossWithQuant": "loss_seg", "VQVAEWithBCELoss": "loss_seg", "VQLPIPSWithDiscriminator": "loss_img"}


def __getattr__(name):
    mod = _EXPORTS.get(name)
    if mod is None:
        raise AttributeError("module %r has no attribute %r" % (__name__, name))
    import importlib
    return getattr(importlib.import_module("." + mod, __name__), name)
