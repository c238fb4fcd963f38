"""Per-image PSNR and SSIM on the device: image.quality (mas_image_quality) against a torch statement of the same definition
(clamp and map, grouped F.conv2d with the separable 11-tap Gaussian over x, y, x^2, y^2 and xy, the SSIM map and the MSE),
checked to agree, and placed beside VQ-IMG's decode_code at the same batch (img_config model, seeded).

    python tools/bench_image_quality.py [--batch 32] [--size 256] [--iters 20] [--rounds 5]

CUDA events over --iters calls per arm after a warm-up, the arms alternated over --rounds rounds; medians (min / max) of the
rounds.  The kernel's GB/s are over the 2*B*C*H*W*4 bytes it must read, against the H100 SXM data-sheet 3.35 TB/s.  Prints
the card, its power limit and max SM clock first.  The torch arm runs its convolutions in full fp32 (no TF32)."""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200"), os.path.join(ROOT, "tools")]

from bench_scene_decode import card, compare, report  # noqa: E402

C1, C2 = 0.01 ** 2, 0.03 ** 2


def window(dev):
    k = torch.arange(-5, 6, dtype=torch.float64)
    g = torch.exp(-k * k / (2 * 1.5 ** 2))
    return (g / g.sum()).float().to(dev)


def torch_quality(rec, ref, g):
    x, y = (rec.clamp(-1, 1) + 1) / 2, (ref.clamp(-1, 1) + 1) / 2
    b, c, h, w = x.shape
    mse = (x - y).square().mean((1, 2, 3))
    prods = torch.cat([x, y, x * x, y * y, x * y], 1)
    n = 5 * c
    blur = F.conv2d(F.conv2d(prods, g.view(1, 1, 11, 1).expand(n, 1, 11, 1), groups=n), g.view(1, 1, 1, 11).expand(n, 1, 1, 11), groups=n)
    mx, my, xx, yy, xy = blur.split(c, 1)
    vx, vy, cxy = xx - mx * mx, yy - my * my, xy - mx * my
    s = ((2 * mx * my + C1) * (2 * cxy + C2)) / ((mx * mx + my * my + C1) * (vx + vy + C2))
    return -10 * torch.log10(mse), s.mean((2, 3)).mean(1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    torch.backends.cudnn.allow_tf32 = False
    import yaml
    from mas_b200 import image
    from models import VQBASE
    dev = torch.device("cuda:0")
    b, r = a.batch, a.size
    print("card:", card())
    print("batch %d, 3 x %d x %d, NCHW fp32" % (b, r, r))

    gen = torch.Generator(device=dev).manual_seed(0)
    ref = torch.rand((b, 3, r, r), device=dev, generator=gen) * 2.2 - 1.1
    rec = ref + 0.1 * torch.randn((b, 3, r, r), device=dev, generator=gen)
    g = window(dev)
    (kp, ks), (tp, ts) = image.quality(rec, ref), torch_quality(rec, ref, g)
    dp, ds = float(((kp.double() - tp.double()).abs() / tp.double().abs()).max()), float((ks.double() - ts.double()).abs().max())
    print("agreement with the torch statement: max psnr rel diff %.2e, max |ssim diff| %.2e" % (dp, ds))
    assert dp < 1e-5 and ds < 1e-4, "the kernel and the torch statement disagree"
    res = compare({"image.quality (kernel)": lambda: image.quality(rec, ref), "torch conv2d statement": lambda: torch_quality(rec, ref, g)},
                  a.iters, a.rounds)
    report("PSNR + SSIM", res, 2 * b * 3 * r * r * 4)
    k, t = res["image.quality (kernel)"][0], res["torch conv2d statement"][0]
    print("  torch / kernel: %.1fx" % (t / k))
    del ref, rec

    cfg = yaml.safe_load(open(os.path.join(ROOT, "make-a-scene_b200", "conf", "img_config.yaml")))["model"]
    torch.manual_seed(0)
    m = VQBASE(cfg["ddconfig"], cfg["n_embed"], cfg["embed_dim"], 10, 100)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    m = m.to(dev).eval()
    tok = torch.randint(0, cfg["n_embed"], (b, r // 16, r // 16), device=dev, generator=gen)
    with torch.no_grad():
        x = m.decode_code(tok).clone()
        res = compare({"decode_code": lambda: m.decode_code(tok), "decode_code + image.quality": lambda: image.quality(m.decode_code(tok), x)},
                      max(1, a.iters // 4), a.rounds)
    report("beside the img_config decoder (tokens %d x %d)" % (r // 16, r // 16), res)
    print("  image.quality alone is %.2f %% of decode_code" % (100 * k / res["decode_code"][0]))


if __name__ == "__main__":
    main()
