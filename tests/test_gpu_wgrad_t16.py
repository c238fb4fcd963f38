"""GPU: the shadow-fed 3x3 weight-gradient kernel wgrad_t16 (csrc/conv_tma.cu). Its activation operand is one MN-major
N = 128 wgmma operand made of two 64-channel swizzle atoms (the two halo boxes), pinned here with a one-MMA probe; the
kernel is checked against the register-staged kernel on the same fp16 operands and against an fp64 product of them."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _desc(lbo, sbo, layout_type):
    return ((lbo >> 4) << 16) | ((sbo >> 4) << 32) | (1 << 46) | (layout_type << 61)


def _idesc16(n, b_mn):
    return ((1 << 16) if b_mn else 0) | ((n >> 3) << 17)


def _mn_sw128_half_index(n, k, lbo, sbo, off):
    """Half the tensor core reads for B element (n, k) of an MN-major operand under the 128-byte swizzle: 64-channel atoms
    LBO bytes apart, 8-row K groups SBO bytes apart, 128-byte rows; the 16-byte chunk is XORed with address bits 7-9."""
    atom, nn = divmod(n, 64)
    kg, kr = divmod(k, 8)
    a = off + atom * lbo + kg * sbo + kr * 128 + (nn // 8) * 16
    a ^= ((a >> 7) & 7) << 4
    return a // 2 + nn % 8


PROBE = [  # lbo, sbo, start offset: the two-atom operand, plain / shifted by one and two 128-byte rows (the dx taps), K groups
    (2048, 1024, 0),   # one atom apart or five rows apart (the kernel's halo rows are ten rows apart)
    (2048, 640, 128),
    (2048, 640, 256),
]


@pytest.mark.parametrize("lbo,sbo,off", PROBE)
def test_mn_major_two_atom_operand(lbo, sbo, off):
    from mas_b200 import _lib as L
    dev = torch.device("cuda:0")
    D = torch.full((128, 128), float("nan"), device=dev)
    L.call("mas_tc_probe16", D, _desc(lbo, sbo, 2), _idesc16(128, 1), off)
    got = D[:16].t().cpu().long()         # [n][k]
    want = torch.tensor([[_mn_sw128_half_index(n, k, lbo, sbo, off) for k in range(16)] for n in range(128)])
    assert want.max().item() < 2048          # inside the probe's indexed region
    assert torch.equal(got, want), (got[62:66], want[62:66])


SHAPES = [  # n, cin, cout, h, w, bias
    (3, 64, 128, 16, 16, True),
    (1, 128, 128, 8, 8, True),
    (3, 128, 256, 16, 16, False),
    (2, 256, 128, 8, 8, True),
    (1, 512, 256, 16, 16, True),
    (3, 512, 128, 8, 8, False),
    (5, 256, 256, 32, 24, True),
    (3, 128, 160, 16, 16, True),
    (1, 64, 160, 8, 8, False),
]


@pytest.mark.parametrize("shape", SHAPES, ids=["n%d_ci%d_co%d_%dx%d_%s" % (s[:5] + ("bias" if s[5] else "nobias",)) for s in SHAPES])
def test_wgrad_t16_matches_reference(shape):
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(29)
    ops.set_operand_format("f16")
    n, cin, cout, h, w, bias = shape
    x = torch.randn(n, cin, h, w, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    dy = (torch.randn(n, cout, h, w, generator=g) * 3e-6).to(dev).contiguous(memory_format=torch.channels_last)
    bound = ops.amax(dy) * 1.7
    dy16 = ops.to_half(dy, bound)
    x16 = ops.to_half(x)
    rows = (cout + 127) // 128 * 128
    t0 = L.tc_launch_count()
    dw, db = ops.conv3x3_wgrad_raw(x16, dy16, rows, cin, L.CONV_S1, want_bias=bias, dy_amax=bound)
    torch.cuda.synchronize()
    assert L.tc_launch_count() > t0
    assert (db is not None) == bias

    # the exact product of the same fp16 operands
    inv = 2.0 ** -(14 - math.floor(math.log2(bound.item())))
    xq = x16.cpu().double()
    dyq = dy16.cpu().double() * inv
    dw_ref = torch.nn.grad.conv2d_weight(xq, (cout, cin, 3, 3), dyq, padding=1)
    scale = dw_ref.abs().max().item()
    err = (dw[:cout].cpu().double() - dw_ref).abs().max().item()
    print("%s: max |dw - fp64| / max |dw| = %.2e" % (shape, err / scale))
    assert err <= 2e-5 * scale
    if rows != cout:
        assert dw[cout:].abs().max().item() == 0.0
    if bias:
        db_ref = dyq.sum(dim=(0, 2, 3))
        assert (db[:cout].cpu().double() - db_ref).abs().max().item() <= 1e-5 * db_ref.abs().max().item()
        if rows != cout:
            assert db[cout:].abs().max().item() == 0.0

    if rows == cout:
        # fp32 dy through the register-staged kernel with the same scale: same fp16 MMA operands, different summation order
        # (its bias gradient sums the unrounded fp32 dy, so the bias is checked against the fp64 sum above instead)
        dw0, _ = ops.conv3x3_wgrad_raw(x16, dy, cout, cin, L.CONV_S1, want_bias=bias, dy_amax=bound)
        assert (dw - dw0).abs().max().item() <= 2e-5 * dw0.abs().max().item()

    # and fp32 autograd on the unrounded tensors (the fp16 rounding of both operands bounds this one)
    xr = x.clone().requires_grad_(True)
    wr = torch.zeros(cout, cin, 3, 3, device=dev, requires_grad=True)
    F.conv2d(xr, wr, None, padding=1).backward(dy)
    assert (dw[:cout] - wr.grad).abs().max().item() / wr.grad.abs().max().item() < 3e-3
