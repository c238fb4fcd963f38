"""Reconstruction quality of images on the device: per-image PSNR and SSIM (mas_image_quality, csrc/image_quality.cu).

A VQ-IMG tokenizer's round trip and its score are

    rec = vq_img.decode_code(vq_img.encode_code(x))
    psnr, ssim = image.quality(rec, x)
"""
from __future__ import annotations

import torch

from . import _lib as L

WINDOW = 11            # SSIM window taps; H and W must be at least this
GRID_LIMIT = 65535     # largest B and C of one launch


def _kernel_device(t):
    """Whether t lives where the kernels run."""
    return t.is_cuda


def quality(rec, ref):
    """PSNR and SSIM of each image of rec against ref -> (psnr, ssim), two fp32 [B] tensors on the inputs' device.

    rec, ref: fp32 CUDA tensors [B, C, H, W] of one shape on one device, in any layout (NCHW, channels-last, views); they are
    read through their strides, never copied.  The definition (include/mas_b200.h, mas_image_quality):
      - every value is clamped to [-1, 1] and mapped to [0, 1] by v -> (v + 1) / 2 (the decoder's range; a saved image is
        clamped the same way);
      - a NaN anywhere in an image makes that image's PSNR and SSIM NaN;
      - psnr[b] = 10 log10(1 / MSE_b), MSE_b over all C*H*W mapped elements; +inf when MSE_b = 0;
      - SSIM (Wang et al. 2004) per channel: an 11-tap Gaussian window, sigma = 1.5, normalised to sum 1 in fp64 and rounded
        once to fp32; C1 = 0.01^2, C2 = 0.03^2; mu_x = G*x, population moments sigma_x^2 = G*x^2 - mu_x^2,
        sigma_xy = G*(xy) - mu_x mu_y; the map ((2 mu_x mu_y + C1)(2 sigma_xy + C2)) / ((mu_x^2 + mu_y^2 + C1)(sigma_x^2 +
        sigma_y^2 + C2)) at the (H - 10)(W - 10) pixels whose window lies inside the image; ssim[b] is the mean over
        channels of each channel's mean.  This is scikit-image's structural_similarity(gaussian_weights=True, sigma=1.5,
        use_sample_covariance=False, data_range=1, channel_axis=0);
      - every call returns the same bits, whatever the strides.
    Runs under no_grad.  Raises ValueError, before any launch, on a non-tensor, a tensor not on CUDA, a dtype other than
    float32, a rank other than 4, a shape mismatch, two devices, H or W below 11, an empty batch or B or C above 65535."""
    for name, t in (("rec", rec), ("ref", ref)):
        if not isinstance(t, torch.Tensor):
            raise ValueError("%s: expected a tensor, got %s" % (name, type(t).__name__))
        if not _kernel_device(t):
            raise ValueError("%s: expected a CUDA tensor, got one on %s" % (name, t.device))
        if t.dtype != torch.float32:
            raise ValueError("%s: expected float32, got %s" % (name, t.dtype))
        if t.dim() != 4:
            raise ValueError("%s: expected a [B, C, H, W] tensor, got shape %s" % (name, tuple(t.shape)))
    if rec.shape != ref.shape:
        raise ValueError("rec %s and ref %s differ in shape" % (tuple(rec.shape), tuple(ref.shape)))
    if rec.device != ref.device:
        raise ValueError("rec (%s) and ref (%s) are on different devices" % (rec.device, ref.device))
    b, c, h, w = rec.shape
    if h < WINDOW or w < WINDOW:
        raise ValueError("quality needs H and W of at least %d (the SSIM window), got shape %s" % (WINDOW, tuple(rec.shape)))
    if not (0 < b <= GRID_LIMIT and 0 < c <= GRID_LIMIT):
        raise ValueError("quality needs 1 <= B, C <= %d, got shape %s" % (GRID_LIMIT, tuple(rec.shape)))
    with torch.no_grad():
        psnr = torch.empty(b, dtype=torch.float32, device=rec.device)
        ssim = torch.empty(b, dtype=torch.float32, device=rec.device)
        nb = int(L.query("mas_image_quality_ws_bytes", b, c, h, w))
        ws = L.workspace(nb, rec.device)
        L.call("mas_image_quality", rec, L.t4(rec), ref, L.t4(ref), psnr, ssim, ws, nb)
    return psnr, ssim
