"""GPU: conv2's form of shift_gemm_t16 (csrc/conv_tma.cu), whose residual the copy engine stages into shared-memory slabs, is the
bias-only form plus the residual bit for bit, with the same GroupNorm statistics. Shapes run the ping-pong kernel (more than
2 x 132 items): 32 x 8 units, pairs of 16 x 8 tiles with a half-empty last unit, and four channel tiles per unit."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [  # n, cin, cout, h, w
    (2, 128, 128, 256, 256),   # the model's 256^2 block at batch 2: 32 x 8 units, 1024 items
    (3, 128, 128, 48, 264),    # pairs of 16 x 8 tiles, the last pair half empty: 149 units, 298 items
    (4, 128, 256, 128, 64),    # four 64-channel items per unit
]


@pytest.mark.parametrize("shape", SHAPES)
def test_residual_epilogue_is_bias_form_plus_residual(shape):
    from mas_b200 import ops
    n, cin, cout, h, w = shape
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(cin + cout + h + w)
    x = torch.randn(n, cin, h, w, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    wt = torch.randn(cout, cin, 3, 3, device=dev, generator=g) * 0.03
    b = torch.randn(cout, device=dev, generator=g)
    res = torch.randn(n, cout, h, w, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    ops.set_operand_format("f16")
    x16 = ops.to_half(x)
    y0 = ops.conv3x3_h_raw(x16, wt, b, None)
    y1, (m1, r1) = ops.conv3x3_h_raw(x16, wt, b, res, want_stats=True)
    assert torch.equal(y1, y0 + res)
    m, r = ops.gn_stats(y1)
    assert torch.allclose(m1, m, rtol=1e-4, atol=1e-6) and torch.allclose(r1, r, rtol=1e-4)
