"""Per-image PSNR and SSIM on the H100 (image.quality, mas_image_quality) against the fp64 restatement of the definition
(tests/test_image_quality_cpu.py): seeded images at 11 x 11 to 512 x 512, constant and near-constant images, exact results
for identical images, NaN confined to its image, the same bits on every layout and call, a second device, and the VQ-IMG
round trip decode_code(encode_code(x))."""
import os

import numpy as np
import pytest
import torch

from test_image_quality_cpu import quality_np

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SSIM_ATOL, PSNR_RTOL = 1e-5, 1e-5
MEASURED = {}   # case -> (largest |ssim error|, largest relative psnr error), printed with -s


def _check(name, rec, ref):
    from mas_b200 import image
    psnr, ssim = image.quality(rec, ref)
    assert psnr.shape == ssim.shape == (rec.shape[0],) and psnr.dtype == ssim.dtype == torch.float32
    assert psnr.device == ssim.device == rec.device
    p, s = quality_np(rec.detach().cpu().numpy(), ref.detach().cpu().numpy())
    gp, gs = psnr.cpu().double().numpy(), ssim.cpu().double().numpy()
    es, ep = float(np.abs(gs - s).max()), float((np.abs(gp - p) / np.abs(p)).max())
    MEASURED[name] = (es, ep)
    print("%-28s max |ssim err| %.2e  max psnr rel err %.2e  (ssim %.6f, psnr %.3f)" % (name, es, ep, s.mean(), p.mean()))
    assert es <= SSIM_ATOL and ep <= PSNR_RTOL, (name, es, ep)
    return psnr, ssim


def _pair(b, c, h, w, seed, noise=0.1):
    """A reference beyond [-1, 1] in places and a noisy reconstruction of it."""
    g = torch.Generator().manual_seed(seed)
    ref = torch.rand(b, c, h, w, generator=g) * 2.2 - 1.1
    return (ref + noise * torch.randn(b, c, h, w, generator=g)).to(DEV), ref.to(DEV)


SHAPES = [(2, 1, 11, 11), (1, 3, 11, 11), (2, 1, 37, 53), (3, 3, 37, 53), (8, 3, 256, 256), (2, 1, 256, 256), (2, 3, 512, 512)]


@pytest.mark.parametrize("b,c,h,w", SHAPES)
def test_matches_the_fp64_definition(b, c, h, w):
    rec, ref = _pair(b, c, h, w, seed=b * 7 + c * 13 + h + w)
    _check("random %dx%dx%dx%d" % (b, c, h, w), rec, ref)
    noise = torch.randn(ref.shape, generator=torch.Generator().manual_seed(h * w)).to(DEV)
    _check("close %dx%dx%dx%d" % (b, c, h, w), ref + 0.003 * noise, ref)


def test_constant_and_near_constant_images():
    g = torch.Generator().manual_seed(9)
    b, c, h, w = 4, 3, 45, 70
    vals = torch.tensor([0.3, -0.97, 0.0, 0.99]).view(4, 1, 1, 1)
    const = vals.expand(b, c, h, w).contiguous()
    _check("constant pair", const.to(DEV), (const - 0.25).to(DEV))
    _check("constant vs itself + 1e-6", const.to(DEV), (const + 1e-6).to(DEV))
    near = const + 1e-3 * torch.randn(b, c, h, w, generator=g)
    _check("near-constant", near.to(DEV), (near + 1e-3 * torch.randn(b, c, h, w, generator=g)).to(DEV))
    _check("near-constant offset", near.to(DEV), (near + 0.02).to(DEV))
    flat_edge = const.clone()
    flat_edge[..., w // 2:] += 0.5                                        # two flat halves: a tile far from its own mean
    _check("flat halves", (flat_edge + 1e-4 * torch.randn(b, c, h, w, generator=g)).to(DEV), flat_edge.to(DEV))


def test_identical_images_are_exact():
    from mas_b200 import image
    rec, _ = _pair(3, 3, 40, 29, seed=1)
    for other in (rec, rec.clone(), rec.contiguous(memory_format=torch.channels_last)):
        psnr, ssim = image.quality(rec, other)
        assert torch.all(ssim == 1.0) and torch.all(psnr == float("inf"))


def test_nan_stays_in_its_image():
    from mas_b200 import image
    rec, ref = _pair(3, 3, 64, 64, seed=2)
    clean = image.quality(rec, ref)
    for where in ((0, 0), (63, 63), (31, 40)):
        for which in ("rec", "ref"):
            r, f = rec.clone(), ref.clone()
            (r if which == "rec" else f)[1, 2, where[0], where[1]] = float("nan")
            psnr, ssim = image.quality(r, f)
            assert torch.isnan(psnr[1]) and torch.isnan(ssim[1]), (where, which)
            for i in (0, 2):
                assert psnr[i].view(torch.int32) == clean[0][i].view(torch.int32)
                assert ssim[i].view(torch.int32) == clean[1][i].view(torch.int32)


def _same_bits(a, b):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


def test_every_layout_and_call_gives_the_same_bits():
    from mas_b200 import image
    rec, ref = _pair(4, 3, 96, 77, seed=3)
    big = torch.randn(4, 5, 110, 100, device=DEV)
    big[:, 1:4, 7:103, 11:88] = rec
    layouts = [rec, rec.contiguous(memory_format=torch.channels_last), big[:, 1:4, 7:103, 11:88]]
    assert not layouts[2].is_contiguous() and layouts[1].stride(1) == 1
    want = image.quality(rec, ref)
    for r in layouts:
        for f in (ref, ref.contiguous(memory_format=torch.channels_last)):
            assert _same_bits(image.quality(r, f), want)
    assert _same_bits(image.quality(rec, ref), want)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_runs_on_the_tensors_device():
    from mas_b200 import image
    rec, ref = _pair(2, 3, 40, 40, seed=4)
    want = image.quality(rec, ref)
    d1 = torch.device("cuda:1")
    assert torch.cuda.current_device() == 0
    got = image.quality(rec.to(d1), ref.to(d1))
    assert got[0].device == got[1].device == d1 and _same_bits([g.cpu() for g in got], [w.cpu() for w in want])


def test_vqimg_round_trip():
    """A seeded VQBASE at img_config's channels and 64 x 64: decode_code(encode_code(x)) scored against x."""
    import yaml
    from conftest import PKG
    from models import VQBASE
    cfg = yaml.safe_load(open(os.path.join(PKG, "conf", "img_config.yaml")))["model"]
    dd = dict(cfg["ddconfig"], resolution=64)
    torch.manual_seed(0)
    m = VQBASE(dd, cfg["n_embed"], cfg["embed_dim"], 10, 100)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    m = m.to(DEV).eval()
    x = (torch.rand(3, 3, 64, 64, generator=torch.Generator().manual_seed(5)) * 2 - 1).to(DEV)
    rec = m.decode_code(m.encode_code(x))
    assert rec.shape == x.shape
    _check("vqimg round trip", rec, x)
