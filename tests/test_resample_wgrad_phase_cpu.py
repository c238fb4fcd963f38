"""CPU: the phase decomposition of the Upsample / Downsample weight gradients that wgrad_t16<128, 1 / 2> and
conv_wgrad_fold16 compute (csrc/conv_tma.cu), restated in fp64 torch and checked against F.conv2d's weight gradient on the
nearest-x2 map / the (0,1,0,1)-padded map. Maps are small, so image borders and the Downsample pad take part everywhere."""
import pytest
import torch
import torch.nn.functional as F


def _shifted(x, oy, ox, h, w):
    """x[:, :, i + oy, j + ox] for i < h, j < w, zero outside the image (the copy engine's out-of-image fill)."""
    xp = F.pad(x, (2, 2 + w, 2, 2 + h))
    return xp[:, :, 2 + oy:2 + oy + h, 2 + ox:2 + ox + w]


def _corr(dy, xs):
    """sum over images and pixels of dy[co] * xs[ci]: one partial tap, [Cout][Cin]."""
    return torch.einsum("nohw,nihw->oi", dy, xs)


def _up_set(ph, a):
    """Weight taps of one dimension summed into tap a of output phase ph (phase_table(up = true, transpose = false))."""
    return ({0}, {1, 2})[a] if ph == 0 else ({0, 1}, {2})[a]


def up_wgrad_phase(x, dy):
    """16 partial taps (g = 2 py + px, a, b): dy's phase plane g against the low-resolution x at offset (py - 1 + a,
    px - 1 + b), then folded into the nine taps in the kernel's order (k = 4 g + 2 a + b ascending)."""
    n, ci, h, w = x.shape
    dw = torch.zeros(dy.shape[1], ci, 3, 3, dtype=x.dtype)
    for g in range(4):
        py, px = g >> 1, g & 1
        plane = dy[:, :, py::2, px::2]
        for a in range(2):
            for b in range(2):
                part = _corr(plane, _shifted(x, py - 1 + a, px - 1 + b, h, w))
                for ty in _up_set(py, a):
                    for tx in _up_set(px, b):
                        dw[:, :, ty, tx] += part
    return dw


DOWN_ROWS = [(0, 0), (0, 1), (1, 0), (1, 1), (2, 0), (3, 0)]   # (tap group, kernel row) pairs the kernel launches


def down_wgrad_phase(x, dy):
    """12 correlations (six (g, a) rows x b = 0, 1) of dy against phase plane g of x at offset (a, b); partial (g, a, b) is
    weight tap (py + 2 a, px + 2 b), and tx = 3 (odd px, b = 1) is dropped."""
    ho, wo = dy.shape[2], dy.shape[3]
    dw = torch.zeros(dy.shape[1], x.shape[1], 3, 3, dtype=x.dtype)
    hits = torch.zeros(3, 3, dtype=torch.int64)
    for g, a in DOWN_ROWS:
        py, px = g >> 1, g & 1
        plane = x[:, :, py::2, px::2]
        for b in range(2):
            ty, tx = py + 2 * a, px + 2 * b
            part = _corr(dy, _shifted(plane, a, b, ho, wo))
            if tx > 2:
                continue
            dw[:, :, ty, tx] += part
            hits[ty, tx] += 1
    assert torch.equal(hits, torch.ones(3, 3, dtype=torch.int64))   # every tap has exactly one producer
    return dw


@pytest.mark.parametrize("n,ci,co,h,w", [(1, 3, 2, 2, 2), (2, 5, 4, 4, 6), (3, 2, 3, 5, 3)])
def test_upsample_wgrad_phase_decomposition(n, ci, co, h, w):
    g = torch.Generator().manual_seed(n * 100 + h * 10 + w)
    x = torch.randn(n, ci, h, w, generator=g, dtype=torch.float64)
    dy = torch.randn(n, co, 2 * h, 2 * w, generator=g, dtype=torch.float64)
    ref = torch.nn.grad.conv2d_weight(F.interpolate(x, scale_factor=2.0, mode="nearest"), (co, ci, 3, 3), dy, padding=1)
    got = up_wgrad_phase(x, dy)
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12), (got - ref).abs().max()


@pytest.mark.parametrize("n,ci,co,h,w", [(1, 3, 2, 2, 2), (2, 5, 4, 8, 6), (3, 2, 3, 6, 10)])
def test_downsample_wgrad_phase_decomposition(n, ci, co, h, w):
    g = torch.Generator().manual_seed(n * 100 + h * 10 + w + 1)
    x = torch.randn(n, ci, h, w, generator=g, dtype=torch.float64)
    dy = torch.randn(n, co, h // 2, w // 2, generator=g, dtype=torch.float64)
    ref = torch.nn.grad.conv2d_weight(F.pad(x, (0, 1, 0, 1)), (co, ci, 3, 3), dy, stride=2)
    got = down_wgrad_phase(x, dy)
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12), (got - ref).abs().max()
