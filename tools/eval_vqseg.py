"""Mean IoU of a VQ-SEG checkpoint's round trip, decode_scene(encode_code(labels)) against labels, over the scene maps of a
directory of the reference's preprocessed .npz files (Data/dataset_preprocessor.py: <name>_panoptic.npz with seg_panoptic
and edges, <name>_human.npz with seg_human and edges, <name>_face.npz with seg_face, under DIR or DIR/segmentations).

    python tools/eval_vqseg.py --checkpoint vq_seg.pt --data DIR [--config make-a-scene_b200/conf/seg_config.yaml]
                               [--batch 16] [--size 256] [--limit N]

The checkpoint is a VQBASE state_dict (train.py's checkpoint.pt / final.pt, or the "model" entry of a resumable one).  Maps
are packed with mas_b200.scene.pack, nearest-resized so that the shorter side is --size and centre-cropped to --size x
--size, as the reference's loader does with a random crop (a resize and a crop commute with the packing), and counted on
the device with scene.confusion; the counts of all batches are summed before scene.iou.  Prints per-group mean IoU and the
worst classes of each group.  A recipe: nothing runs it on real data in the test suite."""
import argparse
import glob
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]


def find_maps(data):
    folder = os.path.join(data, "segmentations") if os.path.isdir(os.path.join(data, "segmentations")) else data
    names = sorted(p[:-len("_panoptic.npz")] for p in glob.glob(os.path.join(folder, "*_panoptic.npz")))
    return [n for n in names if os.path.exists(n + "_human.npz") and os.path.exists(n + "_face.npz")]


def load_planes(name, size):
    """One image's compact planes [4, size, size] (uint8 CPU), through scene.pack."""
    from mas_b200 import scene
    pan, hum, face = (np.load("%s_%s.npz" % (name, k)) for k in ("panoptic", "human", "face"))
    lab = scene.pack(pan["seg_panoptic"], hum["seg_human"], face["seg_face"],
                     pan["edges"].astype(np.int64) + hum["edges"].astype(np.int64))
    h, w = lab.shape[-2:]
    if min(h, w) != size:            # the shorter side to `size` (the reference loader's SmallestMaxSize), nearest labels
        h, w = max(size, round(h * size / min(h, w))), max(size, round(w * size / min(h, w)))
        lab = F.interpolate(lab[None].float(), size=(h, w), mode="nearest")[0].to(torch.uint8)
    top, left = (h - size) // 2, (w - size) // 2   # a centre crop where the loader's RandomCrop takes a random one
    return lab[:, top:top + size, left:left + size].contiguous()


def load_model(config, checkpoint, dev):
    """The VQBASE of a yaml config's model block with a checkpoint's weights, in eval mode on dev.  The checkpoint is a
    state_dict (train.py's checkpoint.pt / final.pt) or a resumable checkpoint with a "model" entry."""
    import yaml
    from mas_b200 import scene
    from models import VQBASE
    cfg = yaml.safe_load(open(config))["model"]
    cfg.pop("_target_", None)
    cfg["ddconfig"].setdefault("out_channels", cfg["ddconfig"].get("out_ch", scene.CHANNELS))   # seg_config omits it
    m = VQBASE(**cfg)
    sd = torch.load(checkpoint, map_location="cpu", weights_only=False)
    m.load_state_dict(sd["model"] if "model" in sd else sd)
    return m.to(dev).eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--checkpoint", required=True)
    ap.add_argument("--data", required=True)
    ap.add_argument("--config", default=os.path.join(ROOT, "make-a-scene_b200", "conf", "seg_config.yaml"))
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--limit", type=int, default=0)
    a = ap.parse_args()
    from mas_b200 import scene
    dev = torch.device("cuda:0")
    m = load_model(a.config, a.checkpoint, dev)
    names = find_maps(a.data)
    if a.limit:
        names = names[:a.limit]
    if not names:
        raise SystemExit("no <name>_panoptic/_human/_face.npz triples under %s" % a.data)
    conf = None
    for i in range(0, len(names), a.batch):
        labels = torch.stack([load_planes(n, a.size) for n in names[i:i + a.batch]]).to(dev)
        c = scene.confusion(m.decode_scene(m.encode_code(labels)), labels)
        conf = c if conf is None else {k: conf[k] + c[k] for k in c}
    r = scene.iou(conf)
    print("%d scene maps, %d x %d" % (len(names), a.size, a.size))
    for g in scene.GROUPS:
        per = r[g]["iou"]
        worst = [(k, per[k]) for k in np.argsort(np.nan_to_num(per, nan=2.0)) if k > 0 and not np.isnan(per[k])][:5]
        print("  %-9s mIoU %.4f   worst: %s" % (g, r[g]["miou"], ", ".join("%d: %.3f" % kv for kv in worst)))


if __name__ == "__main__":
    main()
