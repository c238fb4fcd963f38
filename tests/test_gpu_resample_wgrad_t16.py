"""GPU: the phase-decomposed Upsample / Downsample weight gradients (wgrad_t16<128, 1 / 2> + conv_wgrad_fold16 /
conv_wgrad_reduce, csrc/conv_tma.cu) through ops.Conv3x3Fn. dW and db are checked against an fp64 product of the same fp16
operands (the layer's x shadow and dy shadow, dequantised, through F.conv2d's weight gradient on the nearest-x2 / padded
map), against the fp64 reference layer on the fp32 operands, and against the register-staged route (MAS_CONV_PHASE=0).
Shapes: every Upsample / Downsample of the VQ-IMG model at batch 2, plus small maps with odd tile counts, batch 1 and 3,
bias on and off."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

MODEL = [("up", 512, 16, 16, 2, True), ("up", 512, 32, 32, 2, True), ("up", 256, 64, 64, 2, True), ("up", 128, 128, 128, 2, True),
         ("down", 128, 256, 256, 2, True), ("down", 128, 128, 128, 2, True), ("down", 256, 64, 64, 2, True),
         ("down", 512, 32, 32, 2, True)]
SMALL = [("up", 128, 16, 8, 3, False), ("up", 256, 32, 16, 1, True), ("down", 128, 32, 16, 3, True), ("down", 256, 64, 32, 1, False)]


def _ref_wgrad(kind, x, dy, c):
    if kind == "up":
        return torch.nn.grad.conv2d_weight(F.interpolate(x, scale_factor=2.0, mode="nearest"), (c, c, 3, 3), dy, padding=1)
    return torch.nn.grad.conv2d_weight(F.pad(x, (0, 1, 0, 1)), (c, c, 3, 3), dy, stride=2)


def _run(kind, x, w, b, dy):
    from mas_b200 import _lib as L, ops
    wg = w.clone().requires_grad_(True)
    bg = b.clone().requires_grad_(True) if b is not None else None
    y = ops.Conv3x3Fn.apply(x, wg, bg, None, L.CONV_UP if kind == "up" else L.CONV_S2, False)
    y.backward(dy)
    return wg.grad, (bg.grad if bg is not None else None)


def _err(a, ref):
    return (a.double() - ref).abs().max().item() / ref.abs().max().item()


@pytest.mark.parametrize("kind,c,h,w,n,bias", MODEL + SMALL)
def test_phase_wgrad(kind, c, h, w, n, bias, monkeypatch):
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(3 * c + h + n)
    # fp16-exact input: its scaled shadow dequantises to x itself
    x = torch.randn(n, c, h, w, device=dev, generator=g).half().float().contiguous(memory_format=torch.channels_last)
    wt = torch.randn(c, c, 3, 3, device=dev, generator=g) / (3.0 * c ** 0.5)
    b = torch.randn(c, device=dev, generator=g) if bias else None
    ho, wo = (2 * h, 2 * w) if kind == "up" else (h // 2, w // 2)
    dy = (torch.randn(n, c, ho, wo, device=dev, generator=g) * 1e-3).contiguous(memory_format=torch.channels_last)

    monkeypatch.setenv("MAS_CONV_PHASE", "1")
    assert ops.phase_mode(x, c, L.CONV_UP if kind == "up" else L.CONV_S2) is not None
    t0 = L.tc_launch_count()
    L.profile_start()
    dw, db = _run(kind, x, wt, b, dy)
    calls = {k.split("|")[0] for k in L.profile_report()}
    assert L.tc_launch_count() > t0
    assert "mas_conv3x3_phase_wgrad_tc16" in calls, calls
    for gone in ("mas_space_to_depth", "mas_s2d_unpack_wgrad", "mas_conv3x3_wgrad_tc16", "mas_conv3x3_wgrad"):
        assert gone not in calls, calls
    assert (db is not None) == bias

    # the exact product of the same fp16 operands: dy has no shadow here, so the layer converts it with amax(dy)
    am = ops.amax(dy)
    dyq = ops.to_half(dy, am).double() * 2.0 ** -(14 - math.floor(math.log2(am.item())))
    xq = x.double()
    dw_q = _ref_wgrad(kind, xq, dyq, c)
    e = _err(dw, dw_q)
    print("%s %d %dx%d n%d: max |dw - fp64(fp16 operands)| / max |dw| = %.2e" % (kind, c, h, w, n, e))
    assert e <= 2e-5
    if bias:
        assert _err(db, dyq.sum(dim=(0, 2, 3))) <= 1e-5

    # the reference layer in fp64 on the fp32 operands (fp16 rounding of dy bounds this one)
    dw_r = _ref_wgrad(kind, xq, dy.double(), c)
    assert _err(dw, dw_r) < 3e-3, _err(dw, dw_r)
    if bias:
        assert _err(db, dy.double().sum(dim=(0, 2, 3))) < 3e-3

    monkeypatch.setenv("MAS_CONV_PHASE", "0")
    dw0, db0 = _run(kind, x, wt, b, dy)
    assert _err(dw, dw0.double()) < 2e-3, _err(dw, dw0.double())
    if bias:
        assert _err(db, db0.double()) < 2e-3
