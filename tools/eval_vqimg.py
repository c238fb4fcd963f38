"""Reconstruction quality of a VQ-IMG checkpoint's round trip, decode_code(encode_code(x)) against x, over the images of a
directory, and the codebook usage on them.

    python tools/eval_vqimg.py --checkpoint vq_img.pt --data DIR [--config make-a-scene_b200/conf/img_config.yaml]
                               [--batch 16] [--size 256] [--limit N] [--lpips]

The checkpoint is handled as in tools/eval_vqseg.py (a VQBASE state_dict, or the "model" entry of a resumable one).  Every
.jpg / .jpeg / .png file under DIR is read with PIL, resized so that its shorter side is --size (antialiased bicubic),
centre-cropped to --size x --size and mapped to [-1, 1].  Per batch the tool runs codes = encode_code(x),
rec = decode_code(codes) and image.quality(rec, x) on the device, and adds the codes to a host histogram over n_embed.
Prints mean and median PSNR, mean SSIM, with --lpips the mean LPIPS distance (losses.lpips.LPIPS, which needs its weight
file), the number of codes used, the codebook perplexity exp(-sum p log p) and the five worst images by PSNR.  A recipe:
nothing runs it on real data in the test suite."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]

from eval_vqseg import load_model  # noqa: E402  (tools/ is the script's directory)

EXTENSIONS = (".jpg", ".jpeg", ".png")


def find_images(data):
    out = []
    for folder, _, files in os.walk(data):
        out += [os.path.join(folder, f) for f in files if f.lower().endswith(EXTENSIONS)]
    return sorted(out)


def load_image(path, size):
    """One image as fp32 [3, size, size] in [-1, 1] (CPU): the shorter side resized to `size`, then a centre crop."""
    from PIL import Image
    im = Image.open(path).convert("RGB")
    w, h = im.size
    if min(w, h) != size:
        w, h = max(size, round(w * size / min(w, h))), max(size, round(h * size / min(w, h)))
        im = im.resize((w, h), Image.Resampling.BICUBIC)
    left, top = (w - size) // 2, (h - size) // 2
    a = np.asarray(im.crop((left, top, left + size, top + size)), dtype=np.float32)
    return torch.from_numpy(a).permute(2, 0, 1) / 127.5 - 1.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--checkpoint", required=True)
    ap.add_argument("--data", required=True)
    ap.add_argument("--config", default=os.path.join(ROOT, "make-a-scene_b200", "conf", "img_config.yaml"))
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--limit", type=int, default=0)
    ap.add_argument("--lpips", action="store_true", help="also the mean LPIPS distance (needs LPIPS's weight file)")
    a = ap.parse_args()
    from mas_b200 import image
    dev = torch.device("cuda:0")
    m = load_model(a.config, a.checkpoint, dev)
    n_embed = m.quantize.embedding.weight.shape[0]
    paths = find_images(a.data)
    if a.limit:
        paths = paths[:a.limit]
    if not paths:
        raise SystemExit("no .jpg / .png images under %s" % a.data)
    lp = None
    if a.lpips:
        from losses.lpips import LPIPS
        lp = LPIPS().eval().to(dev)
    psnr, ssim, dist = [], [], []
    hist = np.zeros(n_embed, dtype=np.int64)
    with torch.no_grad():
        for i in range(0, len(paths), a.batch):
            x = torch.stack([load_image(p, a.size) for p in paths[i:i + a.batch]]).to(dev)
            codes = m.encode_code(x)
            rec = m.decode_code(codes)
            p, s = image.quality(rec, x)
            psnr.append(p.cpu())
            ssim.append(s.cpu())
            if lp is not None:
                dist.append(lp(x, rec).flatten().cpu())
            hist += np.bincount(codes.flatten().cpu().numpy(), minlength=n_embed)
    psnr, ssim = torch.cat(psnr).double().numpy(), torch.cat(ssim).double().numpy()
    prob = hist[hist > 0] / hist.sum()
    print("%d images, %d x %d, %s" % (len(paths), a.size, a.size, a.checkpoint))
    print("  PSNR  mean %.3f dB   median %.3f dB" % (psnr.mean(), np.median(psnr)))
    print("  SSIM  mean %.4f" % ssim.mean())
    if lp is not None:
        print("  LPIPS mean %.4f" % torch.cat(dist).double().mean())
    print("  codes used %d / %d   perplexity %.1f" % (prob.size, n_embed, float(np.exp(-(prob * np.log(prob)).sum()))))
    print("  worst by PSNR: %s" % ", ".join("%s %.2f" % (os.path.relpath(paths[k], a.data), psnr[k]) for k in np.argsort(psnr)[:5]))


if __name__ == "__main__":
    main()
