"""Per-image PSNR and SSIM without a GPU: the definition of mas_image_quality (include/mas_b200.h) restated in fp64 numpy with
direct 11 x 11 sliding windows, checked against a second, separable restatement through scipy.ndimage.correlate1d and against
closed forms; the C entry's workspace query and refusals on the real library (no launch); and the host logic of
image.quality above an emulated C-ABI (the pointers, strides and workspace it passes, no aten arithmetic, every ValueError
before any call).  The kernel is tested on the GPU (tests/test_gpu_image_quality.py)."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import ndimage

from test_host_logic_vq_cpu import _addr, _f32, _view4
from test_seg_mse_loss_cpu import PLUMBING, TorchOps

C1, C2 = 0.01 ** 2, 0.03 ** 2


def taps():
    """The window: a Gaussian, sigma 1.5, k = -5..5, normalised to sum 1 in fp64 and rounded once to fp32 (as fp64)."""
    k = np.arange(-5, 6, dtype=np.float64)
    g = np.exp(-k * k / (2 * 1.5 ** 2))
    return (g / g.sum()).astype(np.float32).astype(np.float64)


def mapped(x):
    """Clamp to [-1, 1] (NaN stays NaN) and map to [0, 1], in fp64."""
    return (np.clip(np.asarray(x, dtype=np.float64), -1.0, 1.0) + 1.0) / 2.0


def _psnr(X, Y):
    mse = ((X - Y) ** 2).mean(axis=(1, 2, 3))
    with np.errstate(divide="ignore"):
        return 10.0 * np.log10(1.0 / mse)


def _ssim_map(mx, my, xx, yy, xy):
    vx, vy, cxy = xx - mx * mx, yy - my * my, xy - mx * my
    return ((2 * mx * my + C1) * (2 * cxy + C2)) / ((mx * mx + my * my + C1) * (vx + vy + C2))


def quality_np(rec, ref):
    """The definition on [B, C, H, W] arrays -> (psnr, ssim) float64 [B]: every 11 x 11 window inside the image taken
    directly, as the weighted sum over its 121 offsets."""
    X, Y = mapped(rec), mapped(ref)
    _, _, h, w = X.shape
    hv, wv = h - 10, w - 10
    w2 = np.outer(taps(), taps())
    mom = [np.zeros(X.shape[:2] + (hv, wv)) for _ in range(5)]
    for i in range(11):
        for j in range(11):
            x, y = X[..., i:i + hv, j:j + wv], Y[..., i:i + hv, j:j + wv]
            for m, v in zip(mom, (x, y, x * x, y * y, x * y)):
                m += w2[i, j] * v
    return _psnr(X, Y), _ssim_map(*mom).mean(axis=(2, 3)).mean(axis=1)


def quality_scipy(rec, ref):
    """The same definition, separably: scipy.ndimage.correlate1d along H then W, cropped to the windows inside the image."""
    X, Y = mapped(rec), mapped(ref)
    g = taps()

    def blur(a):
        return ndimage.correlate1d(ndimage.correlate1d(a, g, axis=2, mode="constant"), g, axis=3, mode="constant")[..., 5:-5, 5:-5]

    s = _ssim_map(blur(X), blur(Y), blur(X * X), blur(Y * Y), blur(X * Y))
    return _psnr(X, Y), s.mean(axis=(2, 3)).mean(axis=1)


def _images(seed, b=2, c=3, h=23, w=31, lo=-1.0, hi=1.0):
    return np.random.default_rng(seed).uniform(lo, hi, (b, c, h, w))


def _cases():
    rng = np.random.default_rng(11)
    x = _images(1)
    yield "random", x, _images(2)
    yield "noisy copy", x, x + 0.05 * rng.standard_normal(x.shape)
    yield "constant", np.full((2, 3, 17, 13), 0.3), np.full((2, 3, 17, 13), -0.2)
    near = 0.4 + 1e-3 * rng.standard_normal((2, 1, 19, 25))
    yield "near-constant", near, near + 1e-3 * rng.standard_normal(near.shape)
    yield "offset", x, x + 0.1
    yield "clamped range", 1.5 * _images(3), 1.4 * _images(4)


@pytest.mark.parametrize("name,rec,ref", list(_cases()), ids=[c[0] for c in _cases()])
def test_direct_windows_match_the_separable_restatement(name, rec, ref):
    p1, s1 = quality_np(rec, ref)
    p2, s2 = quality_scipy(rec, ref)
    # fp64 G*x^2 - mu^2 still cancels on flat images (~1e-17), which C2 = 9e-4 scales up to ~1e-13
    assert np.allclose(p1, p2, rtol=1e-13, atol=0) and np.allclose(s1, s2, rtol=0, atol=1e-12), name


def test_identical_images_give_one_and_infinity():
    x = _images(5, b=3, c=1, h=11, w=40)
    psnr, ssim = quality_np(x, x.copy())
    assert np.all(psnr == np.inf) and np.allclose(ssim, 1.0, rtol=0, atol=1e-15)


def test_constant_pair_closed_form():
    a, b = 0.3, -0.2                                          # mapped: p = 0.65, q = 0.4
    p, q = (a + 1) / 2, (b + 1) / 2
    psnr, ssim = quality_np(np.full((1, 3, 15, 12), a), np.full((1, 3, 15, 12), b))
    assert psnr[0] == pytest.approx(10 * np.log10(1 / (p - q) ** 2), rel=1e-14)
    s = taps().sum() ** 2                                     # the fp32 window sums to 1 only up to its rounding
    mx, my, vx, vy, cxy = p * s, q * s, p * p * s * (1 - s), q * q * s * (1 - s), p * q * s * (1 - s)
    want = ((2 * mx * my + C1) * (2 * cxy + C2)) / ((mx * mx + my * my + C1) * (vx + vy + C2))
    assert ssim[0] == pytest.approx(want, rel=1e-12)
    assert ssim[0] == pytest.approx((2 * p * q + C1) / (p * p + q * q + C1), rel=1e-6)    # sigma = 0 up to that rounding


def test_values_outside_the_range_score_as_their_clamped_values():
    x, y = 2.0 * _images(6), 2.0 * _images(7)
    x[0, 0, 3, 4], y[1, 2, 5, 6] = 1e30, -np.inf
    got = quality_np(x, y)
    want = quality_np(np.clip(x, -1, 1), np.clip(y, -1, 1))
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    x[1, 1, 0, 0] = np.nan                                    # a NaN: that image only
    p, s = quality_np(x, y)
    assert np.isnan(p[1]) and np.isnan(s[1]) and p[0] == want[0][0] and s[0] == want[1][0]


# ------------------------------------------------------------------------------------------------ the C entry on this host
def test_workspace_query_and_refusals_need_no_launch():
    """The size query, and every refusal of mas_image_quality, run on the host before any CUDA call."""
    from mas_b200 import _lib
    lib = _lib.load()
    assert lib.mas_image_quality_ws_bytes(2, 3, 37, 53) == 2 * 3 * 2 * 2 * 16       # one fp64 pair per 32 x 32 tile
    assert lib.mas_image_quality_ws_bytes(1, 1, 11, 11) == 16
    assert lib.mas_image_quality_ws_bytes(1, 1, 10, 11) == 0 and lib.mas_image_quality_ws_bytes(0, 1, 11, 11) == 0
    T = _lib.Tensor4

    def t4(b, c, h, w):
        return T(b, h, w, c, c * h * w, w, 1, h * w)

    fake, ws = ctypes.c_void_p(256), ctypes.c_void_p(512)
    ok = t4(2, 3, 37, 53)
    n0 = _lib.launch_count()
    for args in ((None, ok, fake, ok, fake, fake, ws, 1 << 20),
                 (fake, ok, fake, ok, fake, None, ws, 1 << 20),
                 (fake, ok, fake, ok, fake, fake, None, 1 << 20),
                 (fake, t4(2, 3, 10, 53), fake, t4(2, 3, 10, 53), fake, fake, ws, 1 << 20),
                 (fake, t4(2, 3, 37, 10), fake, t4(2, 3, 37, 10), fake, fake, ws, 1 << 20),
                 (fake, t4(0, 3, 37, 53), fake, t4(0, 3, 37, 53), fake, fake, ws, 1 << 20),
                 (fake, t4(2, 0, 37, 53), fake, t4(2, 0, 37, 53), fake, fake, ws, 1 << 20),
                 (fake, ok, fake, t4(2, 3, 37, 52), fake, fake, ws, 1 << 20),
                 (fake, t4(65536, 1, 11, 11), fake, t4(65536, 1, 11, 11), fake, fake, ws, 1 << 30),
                 (fake, t4(1, 65536, 11, 11), fake, t4(1, 65536, 11, 11), fake, fake, ws, 1 << 30),
                 (fake, ok, fake, ok, fake, fake, ws, 383)):
        assert lib.mas_image_quality(*args, None) == -1
        assert b"image_quality" in lib.mas_last_error()
    assert _lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------ host logic over the C-ABI
class QualityEmu:
    """mas_image_quality by its definition, through the pointers and strides it is given."""

    def __init__(self):
        self.names, self.calls = [], []

    def __call__(self, name, *a):
        self.names.append(name)
        getattr(self, name)(*a)

    def mas_image_quality(self, rec, rs, ref, fs, psnr, ssim, ws, ws_bytes):
        self.calls.append(dict(rec=_addr(rec), ref=_addr(ref), psnr=_addr(psnr), ssim=_addr(ssim), ws=ws, ws_bytes=ws_bytes,
                               rs=tuple(getattr(rs, f) for f in ("n", "h", "w", "c", "sn", "sh", "sw", "sc")),
                               fs=tuple(getattr(fs, f) for f in ("n", "h", "w", "c", "sn", "sh", "sw", "sc"))))
        p, s = quality_np(_view4(rec, rs).transpose(0, 3, 1, 2), _view4(ref, fs).transpose(0, 3, 1, 2))
        _f32(psnr, rs.n)[:] = p
        _f32(ssim, rs.n)[:] = s


def _ws_bytes(b, c, h, w):
    return 7 * b * c * h + w                                  # any size: the test checks that it is the one passed


@pytest.fixture
def iq_emu(monkeypatch):
    from mas_b200 import image
    e = QualityEmu()
    queries = []

    def query(name, *a):
        assert name == "mas_image_quality_ws_bytes"
        queries.append(a)
        return _ws_bytes(*a)

    monkeypatch.setattr(image.L, "call", e)
    monkeypatch.setattr(image.L, "query", query)
    monkeypatch.setattr(image, "_kernel_device", lambda t: True)
    e.queries = queries
    return e


def _layouts(x):
    """The same values as NCHW, channels-last and a crop of a larger tensor."""
    b, c, h, w = x.shape
    big = torch.full((b, c + 2, h + 5, w + 7), float("nan"))
    big[:, 1:c + 1, 2:h + 2, 3:w + 3] = x
    return {"nchw": x.contiguous(), "channels_last": x.contiguous(memory_format=torch.channels_last),
            "crop": big[:, 1:c + 1, 2:h + 2, 3:w + 3]}


def test_quality_host_logic(iq_emu):
    from mas_b200 import image
    g = torch.Generator().manual_seed(3)
    ref = torch.rand(2, 3, 14, 19, generator=g) * 2.2 - 1.1
    rec = ref + 0.1 * torch.randn(2, 3, 14, 19, generator=g)
    want = quality_np(rec.numpy(), ref.numpy())
    for name, r in _layouts(rec).items():
        for fname, f in _layouts(ref).items():
            first = len(iq_emu.names)
            with TorchOps() as ops:
                psnr, ssim = image.quality(r, f)
            assert ops.ops <= PLUMBING, ops.ops - PLUMBING
            assert iq_emu.names[first:] == ["mas_image_quality"], (name, fname)
            call = iq_emu.calls[-1]
            assert call["rec"] == r.data_ptr() and call["ref"] == f.data_ptr()                 # as they are: no copy
            for key, t in (("rs", r), ("fs", f)):
                sn, sc, sh, sw = t.stride()
                assert call[key] == (2, 14, 19, 3, sn, sh, sw, sc)
            assert call["psnr"] == psnr.data_ptr() and call["ssim"] == ssim.data_ptr()
            assert iq_emu.queries[-1] == (2, 3, 14, 19) and call["ws_bytes"] == _ws_bytes(2, 3, 14, 19)
            assert call["ws"].numel() >= call["ws_bytes"]
            assert psnr.dtype == ssim.dtype == torch.float32 and psnr.shape == ssim.shape == (2,)
            assert np.allclose(psnr.numpy(), want[0], rtol=1e-6) and np.allclose(ssim.numpy(), want[1], rtol=0, atol=1e-6)


def test_every_value_error_fires_before_any_call(iq_emu, monkeypatch):
    from mas_b200 import image
    x = torch.zeros(2, 3, 16, 16)
    cases = [lambda: image.quality(x.numpy(), x), lambda: image.quality(x, [x]),
             lambda: image.quality(x.double(), x), lambda: image.quality(x, x.half()),
             lambda: image.quality(x[0], x[0]), lambda: image.quality(x[None], x[None]),
             lambda: image.quality(x, x[:1]), lambda: image.quality(x, x[:, :1]), lambda: image.quality(x, x[..., :15]),
             lambda: image.quality(x, torch.zeros(2, 3, 16, 16, device="meta")),
             lambda: image.quality(x[:, :, :10], x[:, :, :10]), lambda: image.quality(x[..., :10], x[..., :10]),
             lambda: image.quality(x[:0], x[:0]), lambda: image.quality(x[:, :0], x[:, :0]),
             lambda: image.quality(torch.zeros(1, 1, 11, 11).expand(65536, 1, 11, 11), torch.zeros(1, 1, 11, 11).expand(65536, 1, 11, 11)),
             lambda: image.quality(torch.zeros(1, 1, 11, 11).expand(1, 65536, 11, 11), torch.zeros(1, 1, 11, 11).expand(1, 65536, 11, 11))]
    for f in cases:
        with pytest.raises(ValueError):
            f()
    monkeypatch.setattr(image, "_kernel_device", lambda t: t.is_cuda)
    with pytest.raises(ValueError):                                                           # CPU tensors
        image.quality(x, x)
    assert iq_emu.names == [] and iq_emu.queries == []
