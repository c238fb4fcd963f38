"""Object-aware perceptual loss: LPIPS over the object boxes of each image, on the sm_90a kernels in libmas_b200.so.

The value is the per-box loop that the reference's loss_img.py leaves commented out, with LPIPS as the crop loss:

    L = sum_b 1 / (n_b + 1) * sum_k LPIPS(crop(img_b, box_bk), crop(rec_b, box_bk))

A box is (x0, y0, x1, y1, ...), read with int(); crop is torchvision's (top y0, left x0, height y1 - y0, width x1 - x0,
zeros outside the image). `bbox_obj` holds one entry per image: a list of boxes or an [n, >= 4] tensor.

Boxes under 16 pixels on a side are dropped and do not count in n_b: four 2x2 max-pools leave nothing of them (the
reference's loop fails on such a box inside max_pool2d). A box with zero or negative extent raises ValueError.

Instead of one VGG16 pass per box, every box goes to a size class (per side the next power of two, at least 16) and each
class runs as one batch of canvases with the activations outside each crop held at zero (DESIGN §3.10), so the number of
kernel launches depends on the number of classes, not of boxes."""
import torch
import torch.nn as nn

from mas_b200 import ops


class ObjectLoss(nn.Module):
    """ObjectLoss(lpips=None): `lpips` is the losses.lpips.LPIPS whose weights the crops are scored with, typically the
    perceptual loss's own (`ObjectLoss(self.perceptual_loss)`). A given instance is shared, not registered as a submodule,
    so the owner's state_dict does not list its weights twice. With None an LPIPS() is built and owned."""

    def __init__(self, lpips=None):
        super().__init__()
        if lpips is None:
            from .lpips import LPIPS
            self.lpips = LPIPS().eval()
        else:
            self._shared = (lpips,)

    @property
    def scorer(self):
        shared = getattr(self, "_shared", None)
        return shared[0] if shared is not None else self.lpips

    def _parts(self):
        m = self.scorer
        m.check()
        return (m.scaling_layer.shift, m.scaling_layer.scale, m.vgg.convs(), [lin.model[1].weight for lin in m.lins])

    def forward(self, images, reconstructions, bbox_obj):
        """-> 0-dim fp32 loss; images.new_tensor(0) when no box counts (no kernel runs)."""
        parts = self._parts()
        plan = ops.ObjectPlan(images.shape, reconstructions.shape, bbox_obj)
        if plan.K == 0:
            return images.new_tensor(0)
        keep = torch.is_grad_enabled() and (images.requires_grad or reconstructions.requires_grad)
        return ops.ObjectLossFn.apply(images, reconstructions, plan, *parts, keep)

    @torch.no_grad()
    def per_box(self, images, reconstructions, bbox_obj):
        """(LPIPS of every counted box [K] in box order, the plan) from the same kernels as forward(); None without boxes."""
        parts = self._parts()
        plan = ops.ObjectPlan(images.shape, reconstructions.shape, bbox_obj)
        if plan.K == 0:
            return None, plan
        r = ops.object_forward_raw(images.contiguous(), reconstructions.contiguous(), plan, *parts, False)
        return r["p"], plan
