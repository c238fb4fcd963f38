"""GPU: the phase-decomposed Upsample / Downsample convolutions (shift_gemm_t16 phase-out / phase-in, csrc/conv_tma.cu).
Forward and data gradient through ops.Conv3x3Fn are checked against an fp64 evaluation of the reference layer
(nearest x2 then 3x3 / (0,1,0,1) pad then 3x3 stride 2) on the same fp16-exact input, and against the register-staged
route (MAS_CONV_PHASE=0). Shapes: every Upsample / Downsample of the VQ-IMG model at batch 2, plus small maps with an odd
tile count (the pair kernel's missing second tile), batch 3 and bias on / off; image borders are part of every map."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

MODEL = [("up", 512, 16, 16, 2, True), ("up", 512, 32, 32, 2, True), ("up", 256, 64, 64, 2, True), ("up", 128, 128, 128, 2, True),
         ("down", 128, 256, 256, 2, True), ("down", 128, 128, 128, 2, True), ("down", 256, 64, 64, 2, True),
         ("down", 512, 32, 32, 2, True)]
SMALL = [("up", 128, 16, 8, 3, False), ("up", 256, 32, 16, 1, True), ("down", 128, 32, 16, 3, True), ("down", 256, 64, 32, 1, False)]


def _ref(kind, x, w, b):
    if kind == "up":
        return F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, b, padding=1)
    return F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _run(kind, x, w, b, dy):
    from mas_b200 import _lib as L, ops
    xg = x.clone().requires_grad_(True)
    y = ops.Conv3x3Fn.apply(xg, w, b, None, L.CONV_UP if kind == "up" else L.CONV_S2, False)
    y.backward(dy)
    return y.detach(), xg.grad


@pytest.mark.parametrize("kind,c,h,w,n,bias", MODEL + SMALL)
def test_phase_route(kind, c, h, w, n, bias, monkeypatch):
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(c + h + n)
    # fp16-exact input: the shadow holds the same values (up to a power-of-two scale)
    x = torch.randn(n, c, h, w, device=dev, generator=g).half().float().contiguous(memory_format=torch.channels_last)
    wt = torch.randn(c, c, 3, 3, device=dev, generator=g) / (3.0 * c ** 0.5)
    b = torch.randn(c, device=dev, generator=g) if bias else None
    ho, wo = (2 * h, 2 * w) if kind == "up" else (h // 2, w // 2)
    dy = (torch.randn(n, c, ho, wo, device=dev, generator=g) * 1e-3).contiguous(memory_format=torch.channels_last)
    monkeypatch.setenv("MAS_CONV_PHASE", "1")
    assert ops.phase_mode(x, c, L.CONV_UP if kind == "up" else L.CONV_S2) is not None
    y, dx = _run(kind, x, wt, b, dy)

    xd = x.double().requires_grad_(True)
    yr = _ref(kind, xd, wt.double(), None if b is None else b.double())
    yr.backward(dy.double())
    # fp16 weights (for the Upsample, per-phase sums rounded once) and fp16 dy: ~1e-3 of the norm at most
    assert _rel(y, yr) < 2e-3, _rel(y, yr)
    assert _rel(dx, xd.grad) < 2e-3, _rel(dx, xd.grad)

    monkeypatch.setenv("MAS_CONV_PHASE", "0")
    y0, dx0 = _run(kind, x, wt, b, dy)
    assert _rel(y, y0) < 2e-3 and _rel(dx, dx0) < 2e-3, (_rel(y, y0), _rel(dx, dx0))
