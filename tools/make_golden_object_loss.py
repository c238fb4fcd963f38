"""Writes tests/golden/object_loss.pt from the REAL reference LPIPS (losses/lpips.py of a reference checkout) and the per-box
loop that the reference's loss_img.py leaves commented out, on the CPU in fp32:

    python tools/make_golden_object_loss.py --reference <reference checkout>

The LPIPS module is loaded offline and filled exactly as tools/make_golden_lpips.py fills it (oracle.seeded.fill_seeded,
then that tool's adjust()), so no weights are stored; the tests apply the same two steps to the drop-in module. The loop
crops with torchvision's `crop` (zeros outside the image) and runs one LPIPS per box:

    object_loss = sum over (img, rec, bboxes) of  sum_k LPIPS(crop(img, box_k), crop(rec, box_k)).mean() / (len(bboxes) + 1)

Boxes under 16 pixels on a side fail inside the reference's max_pool2d; the loop runs on the list without them, and the
fixture records which boxes were dropped.

Cases (boxes are [x0, y0, x1, y1]):
  a: two 256x256 images: mixed sizes and aspect ratios, the whole image, one box crossing the right / bottom edge, one crossing
     the left edge, two overlapping boxes, and one 10-pixel-wide box (dropped);
  b: three 72x72 images, the second with no boxes.
Recorded per case: the boxes, the kept boxes and the dropped ones, the per-box p in kept order, the per-image terms, the loss,
and d loss / d rec (the full tensor at 72x72; norm and seeded samples at 256x256).
"""
import argparse
import importlib.util
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "object_loss.pt")
MIN_SIDE = 16
CASES = {
    "a": dict(seed=41, size=256, batch=2,
              boxes=[[[10, 20, 110, 90], [60, 50, 160, 170], [200, 180, 290, 250], [40, 100, 72, 120], [5, 5, 15, 100]],
                     [[0, 0, 256, 256], [100, 120, 133, 137], [-10, 30, 50, 100]]]),
    "b": dict(seed=42, size=72, batch=3,
              boxes=[[[5, 5, 45, 60], [20, 30, 72, 72]], [], [[0, 0, 72, 72], [10, 10, 27, 40]]]),
}


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


lpips_tool = _tool("make_golden_lpips")


def split(boxes):
    """(kept boxes per image, dropped (image, box)) under the 16-pixel rule."""
    kept, dropped = [], []
    for b, bb in enumerate(boxes):
        kept.append([])
        for box in bb:
            x0, y0, x1, y1 = (int(v) for v in box[:4])
            if y1 - y0 < MIN_SIDE or x1 - x0 < MIN_SIDE:
                dropped.append((b, [x0, y0, x1, y1]))
            else:
                kept[-1].append([x0, y0, x1, y1])
    return kept, dropped


def loop(model, images, recs, kept):
    """loss_img.py's commented-out object loss, with `self.object_loss` = model -> (loss, per-image terms, per-box p)."""
    from torchvision.transforms.functional import crop
    total, terms, ps = images.new_tensor(0), [], []
    for img, rec, bboxes in zip(images, recs, kept):
        img_loss = img.new_tensor(0)
        for bbox in bboxes:
            top, left, height, width = bbox[1], bbox[0], bbox[3] - bbox[1], bbox[2] - bbox[0]
            p = model(crop(img, top, left, height, width).unsqueeze(0).contiguous(),
                      crop(rec, top, left, height, width).unsqueeze(0).contiguous()).mean()
            ps.append(p)
            img_loss = img_loss + p
        term = img_loss / (len(bboxes) + 1)
        terms.append(term)
        total = total + term
    return total, terms, ps


def run_case(ref, fill_seeded, seed, size, batch, boxes):
    model = ref.LPIPS().eval()
    checks = fill_seeded(model, seed)
    lpips_tool.adjust(model, 0.0)
    img, rec = lpips_tool.images(seed, size, batch)
    kept, dropped = split(boxes)
    r = rec.clone().requires_grad_(True)
    loss, terms, ps = loop(model, img, r, kept)
    loss.backward()
    return {"seed": seed, "size": size, "batch": batch, "fill_checks": checks, "images_sha256": lpips_tool.sha(torch.cat([img, rec])),
            "boxes": boxes, "kept": kept, "dropped": dropped, "p": torch.stack([p.detach() for p in ps]),
            "terms": [float(t.detach()) for t in terms], "loss": float(loss.detach()),
            "drec": lpips_tool.record(r.grad, seed + 101, size <= 72)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="root of a reference checkout (holds losses/lpips.py)")
    a = ap.parse_args()
    import torchvision
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from seeded import fill_seeded
    spec = importlib.util.spec_from_file_location("_ref_lpips", os.path.join(a.reference, "losses", "lpips.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    with tempfile.TemporaryDirectory() as td:
        empty = os.path.join(td, "vgg.pth")
        torch.save({}, empty)
        ref.vgg16 = lambda pretrained=True: torchvision.models.vgg16(weights=None)
        ref.get_ckpt_path = lambda name, root: empty
        torch.set_num_threads(max(1, os.cpu_count() or 1))
        out = {name: run_case(ref, fill_seeded, **kw) for name, kw in CASES.items()}
    torch.save(out, OUT)
    for name, c in out.items():
        print(name, "p", [round(v, 5) for v in c["p"].tolist()], "terms", c["terms"], "loss", c["loss"], "dropped", c["dropped"],
              "|d rec|", c["drec"]["norm"])
    print("wrote", OUT, "%.1f KiB" % (os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
