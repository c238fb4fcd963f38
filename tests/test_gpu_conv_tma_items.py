"""shift_gemm_t16 (csrc/conv_tma.cu) on the item counts its ping-pong schedule distinguishes: the two MMA warpgroups of a CTA
take its 64-output-channel work items alternately, so the cases are CTAs with one item (the second warpgroup idle), CTAs with
an odd number of items, four items per pixel unit (Cout = 256), channel tiles beyond the stored channels, and the phase forms
with an odd number of items per CTA. Launches with at most two items per CTA and the deep phase layers run on the
cooperative form (both warpgroups on one 128-channel item), which some cases cover too.
Checked against F.conv2d on the same fp16-rounded operands."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


SHAPES = [  # n, cin, cout, h, w (ping-pong from 2 x 132 + 1 items; fewer run the cooperative form)
    (1, 128, 128, 32, 32),     # 8 items: the cooperative form
    (1, 64, 4, 16, 8),         # cooperative form, 4 stored channels of a 128-channel tile
    (2, 128, 128, 352, 72),    # 198 32 x 8 units, 396 items: three per CTA on 132 SMs
    (4, 128, 256, 128, 64),    # four 64-channel items per unit, 512 items
    (3, 128, 192, 48, 264),    # pairs of 16 x 8 tiles (the last one half empty), 149 units x three channel tiles of which
                               # the last is stored: 447 items, odd counts per CTA; the fourth tile is never computed
    (1, 128, 128, 48, 1056),   # pairs of 16 x 8 tiles, 198 units, 396 items: three per CTA on 132 SMs
]


@pytest.mark.parametrize("shape", SHAPES)
def test_conv_tma_item_schedule(shape):
    from mas_b200 import _lib as L, ops
    n, cin, cout, h, w = shape
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(cin + cout + h)
    x = _cl(torch.randn(n, cin, h, w, generator=g).to(dev))
    wt = (torch.randn(cout, cin, 3, 3, generator=g) * (1.0 / (3.0 * cin ** 0.5))).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    ops.set_operand_format("f16")
    x16 = ops.to_half(x)
    cp = (cout + 127) // 128 * 128           # weights / bias padded to the 128-wide tile, the output stores cout channels
    wp = torch.zeros(cp, cin, 3, 3, device=dev)
    wp[:cout] = wt
    bp = torch.zeros(cp, device=dev)
    bp[:cout] = b
    y = ops.empty_nhwc(n, cout, h, w, x)
    pk = torch.empty(9 * cp * cin, dtype=torch.float16, device=dev)
    L.call("mas_pack_conv3x3_tc16", wp, pk, None, cp, cin, 0)
    L.call("mas_conv3x3_fprop_tc16h", x16, L.t4(x16), pk, bp, None, y, L.t4(y), None, None)
    ref = F.conv2d(x16.float(), wt.half().float(), b, padding=1)
    err = (y - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-4, err


def test_conv_tma_residual_statistics_odd_items():
    """conv2's form (residual and GroupNorm-statistics epilogues) with three items per CTA."""
    from mas_b200 import ops
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(17)
    n, c, h, w = 2, 128, 352, 72
    x = _cl(torch.randn(n, c, h, w, generator=g).to(dev))
    wt = (torch.randn(c, c, 3, 3, generator=g) * 0.03).to(dev)
    b = torch.randn(c, generator=g).to(dev)
    res = _cl(torch.randn(n, c, h, w, generator=g).to(dev))
    ops.set_operand_format("f16")
    x16 = ops.to_half(x)
    y, st = ops.conv3x3_h_raw(x16, wt, b, res, want_stats=True)
    ref = F.conv2d(x16.float(), wt.half().float(), b, padding=1) + res
    assert (y - ref).abs().max().item() / ref.abs().max().item() < 1e-4
    m, r = ops.gn_stats(y)
    assert torch.allclose(st[0], m, rtol=1e-4, atol=1e-6) and torch.allclose(st[1], r, rtol=1e-4)


PHASE = [  # kind, c, h, w, n: the low-resolution extent
    ("up", 128, 32, 64, 5),      # 40 units x 2 channel tiles x 4 output phases = 320 items: two or three per CTA
    ("up", 128, 16, 8, 1),       # 1 unit (half empty), 8 items: the second warpgroup of every CTA idle
    ("down", 128, 32, 400, 3),   # 150 units x 2 channel tiles = 300 items: two or three per CTA
    ("down", 128, 16, 40, 1),    # pairs of 16 x 8 tiles, 3 units x 2 channel tiles = 6 items
    ("down", 256, 16, 40, 1),    # the cooperative form (phase-in from 256 channels), pairs of 16 x 8 tiles
    ("up", 512, 16, 8, 3),       # the cooperative form (phase-out from 512 channels)
]


@pytest.mark.parametrize("kind,c,h,w,n", PHASE)
def test_conv_tma_phase_item_schedule(kind, c, h, w, n):
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(c + h + w + n)
    hs, ws = (h, w) if kind == "up" else (2 * h, 2 * w)
    x = _cl(torch.randn(n, c, hs, ws, device=dev, generator=g).half().float())
    wt = torch.randn(c, c, 3, 3, device=dev, generator=g) / (3.0 * c ** 0.5)
    b = torch.randn(c, device=dev, generator=g)
    ops.set_operand_format("f16")
    x16 = ops.to_half(x)
    y = ops.conv3x3_phase_raw(x16, wt, b, L.CONV_UP_PHASE if kind == "up" else L.CONV_S2_PHASE)
    xd = x.double()
    if kind == "up":
        ref = F.conv2d(F.interpolate(xd, scale_factor=2.0, mode="nearest"), wt.double(), b.double(), padding=1)
    else:
        ref = F.conv2d(F.pad(xd, (0, 1, 0, 1)), wt.double(), b.double(), stride=2)
    assert _rel(y, ref) < 2e-3, _rel(y, ref)   # fp16 weights (Upsample: per-phase sums rounded once)
