"""VQ-SEG training objectives of the reference's losses/loss_seg.py on the sm_90a kernels in libmas_b200.so.

`BCELossWithQuant` (loss_seg.py:6-22) and `VQVAEWithBCELoss` (loss_seg.py:25-41) with the reference's constructor,
`weight` buffer (pos_weight 20 on channels 153..157, so the state_dict is the same) and `forward(qloss, target,
prediction)`. The loss term runs as ops.BCELogitsFn / ops.BCEMSELogitsFn: one kernel for the forward and one for the
backward, which writes the gradient straight into the padded channels-last buffer the decoder's last convolution
returns. `target` is the dense fp32 [B, 159, H, W] map or the compact uint8 [B, 4, H, W] map of mas_b200.scene; both give
the same loss and gradient bit for bit. The result is that loss plus `codebook_weight * qloss`, as in the reference.

With `make-a-scene_b200/` ahead of the reference root on sys.path, a yaml `loss._target_` of
`losses.scene_loss.VQVAEWithBCELoss` (or `.BCELossWithQuant`) is the whole integration; `losses.BCELossWithQuant` and
`losses.VQVAEWithBCELoss` still name the reference's own classes."""
import torch
import torch.nn as nn

from mas_b200 import ops, scene

__all__ = ["BCELossWithQuant", "VQVAEWithBCELoss"]


def _on_device(t):
    return t.is_cuda


def _check(weight, qloss, target, prediction):
    """ValueError unless the operands are what the kernels take, before anything is launched."""
    if not isinstance(prediction, torch.Tensor) or not isinstance(target, torch.Tensor):
        raise ValueError("prediction and target must be tensors")
    if not _on_device(prediction) or prediction.dtype != torch.float32 or prediction.dim() != 4:
        raise ValueError("prediction must be a 4-D float32 CUDA tensor, got %s %s on %s"
                         % (tuple(prediction.shape), prediction.dtype, prediction.device))
    n, c, h, w = prediction.shape
    if c != weight.numel():
        raise ValueError("prediction has %d channels, the loss was built for image_channels=%d" % (c, weight.numel()))
    if weight.device != prediction.device:
        raise ValueError("the loss's weight buffer is on %s, prediction on %s: move the loss with .to(device)"
                         % (weight.device, prediction.device))
    if target.device != prediction.device:
        raise ValueError("target is on %s, prediction on %s" % (target.device, prediction.device))
    if target.dtype == torch.uint8:
        if c != scene.CHANNELS or tuple(target.shape) != (n, scene.PLANES, h, w):
            raise ValueError("a compact scene map [%d, %d, %d, %d] is the target of %d-channel predictions, got %s for %s"
                             % (n, scene.PLANES, h, w, scene.CHANNELS, tuple(target.shape), tuple(prediction.shape)))
    elif target.dtype == torch.float32:
        if target.shape != prediction.shape:
            raise ValueError("target shape %s != prediction shape %s" % (tuple(target.shape), tuple(prediction.shape)))
    else:
        raise ValueError("target must be a dense float32 map or a compact uint8 scene map, got %s" % target.dtype)
    if isinstance(qloss, torch.Tensor) and qloss.device != prediction.device:
        raise ValueError("qloss is on %s, prediction on %s" % (qloss.device, prediction.device))


class _SegLoss(nn.Module):
    _fn = None

    def __init__(self, image_channels=159, codebook_weight=1.0):
        super().__init__()
        self.codebook_weight = codebook_weight
        self.register_buffer(
            "weight",
            torch.ones(image_channels).index_fill(0, torch.arange(153, 158), 20),
        )

    def forward(self, qloss, target, prediction):
        _check(self.weight, qloss, target, prediction)
        return self._fn.apply(prediction, target, self.weight) + self.codebook_weight * qloss


class BCELossWithQuant(_SegLoss):
    """binary_cross_entropy_with_logits(prediction, target, pos_weight=weight) + codebook_weight * qloss
    (loss_seg.py:15-22), on mas_bce_* (ops.BCELogitsFn)."""
    _fn = ops.BCELogitsFn


class VQVAEWithBCELoss(_SegLoss):
    """mse_loss(prediction.sigmoid(), target) + binary_cross_entropy_with_logits(prediction, target, pos_weight=weight)
    + codebook_weight * qloss (loss_seg.py:34-41), on mas_bce_mse_* (ops.BCEMSELogitsFn): the two means are one mean over
    N*C*H*W, computed in one pass."""
    _fn = ops.BCEMSELogitsFn
