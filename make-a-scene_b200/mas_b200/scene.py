"""Compact scene maps: the VQ-SEG input as four uint8 label planes per pixel instead of the 159-channel fp32 one-hot stack.

The reference's preprocessing stores, per image, one panoptic class, one human part and one face part per pixel plus two
edge maps (`seg_panoptic`, `seg_human`, `seg_face`, `edges` in its .npz files); PreprocessedDataset.load_segmentation
(Data/dataset_preprocessor.py:61-86) expands them on the CPU into the dense [H, W, 159] map.  `pack` keeps them as

    plane 0  panoptic  seg_panoptic + 1          0 = none, k = 1..133 -> dense channel k - 1
    plane 1  human     seg_human + 1             0 = none, k = 1..20  -> dense channel 132 + k
    plane 2  face      seg_face                  0 = none, k = 1..5   -> dense channel 152 + k
    plane 3  edges     edges_panoptic + edges_human (0..2)            -> dense channel 158 = the count

and the kernels expand them on the GPU (mas_scene_expand, mas_bce_scene_*, include/mas_b200.h) into exactly the dense
map load_segmentation would have built: 4 bytes a pixel cross the bus instead of 636.  Nearest-neighbour resizes and
crops commute with the expansion, so a loader transforms the 4 planes in place of the 159 channels.

`VQBASE(...)(labels)` and `ops.BCELogitsFn.apply(dec, labels, pos_weight)` take the batched planes, a [B, 4, H, W]
uint8 CUDA tensor (contiguous NCHW; other strides are made contiguous first).

The output side runs the other way.  `decode` turns VQ-SEG logits (or a dense map) into planes on the device by the BCE
decision boundary: a channel is on when its logit is > 0, and each one-hot plane is 1 + the argmax of its group when that
maximum is > 0, else 0 (mas_scene_decode, include/mas_b200.h).  `unpack` is the host inverse of `pack`.  `confusion` counts
target x prediction cells per plane on the device (mas_scene_confusion) and `iou` turns the counts into per-class IoU.
`VQBASE.decode_scene(tokens)` is `decode(decode_code(tokens))`, so a tokenizer's round trip and its quality are

    rec = vq_seg.decode_scene(vq_seg.encode_code(labels))
    scores = scene.iou(scene.confusion(rec, labels))
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib as L

PANOPTIC_CLASSES, HUMAN_PARTS, FACE_PARTS = 133, 20, 5
PLANES = 4
CHANNELS = PANOPTIC_CLASSES + HUMAN_PARTS + FACE_PARTS + 1     # 159
GROUPS = ("panoptic", "human", "face", "edges")
CLASSES = (PANOPTIC_CLASSES + 1, HUMAN_PARTS + 1, FACE_PARTS + 1, 2)    # per plane, "none" (0) included
CONFUSION_LEN = sum(k * k for k in CLASSES) + 1                 # the four matrices and the out-of-range count


def _array(name, a):
    if isinstance(a, torch.Tensor):
        if a.device.type != "cpu":
            raise ValueError("%s: expected a CPU array, got a %s tensor" % (name, a.device.type))
        a = a.numpy()
    a = np.asarray(a)
    if a.dtype != np.bool_ and not np.issubdtype(a.dtype, np.integer):
        raise ValueError("%s: expected an integer or bool array, got %s" % (name, a.dtype))
    return a


def pack(seg_panoptic, seg_human, seg_face, edges):
    """The four label planes of one image ([H, W] arrays, as stored in the reference's .npz files) or of a batch ([B, H, W])
    -> uint8 torch tensor [4, H, W] / [B, 4, H, W] (CPU; pin and copy it to the GPU like any batch).

    seg_panoptic: -1 (none) .. 132; seg_human: -1 (none) .. 19; seg_face: 0 (none) .. 5; edges: the sum of the
    panoptic and human edge maps, 0 .. 2.  Raises ValueError on any other value, a non-integer dtype or mismatched shapes:
    the kernels never index out of bounds whatever the bytes, but a map outside these ranges is not one the reference
    could have built."""
    arrays = [_array(n, a) for n, a in (("seg_panoptic", seg_panoptic), ("seg_human", seg_human), ("seg_face", seg_face),
                                         ("edges", edges))]
    shape = arrays[0].shape
    if len(shape) not in (2, 3) or 0 in shape:
        raise ValueError("seg_panoptic: expected a non-empty [H, W] or [B, H, W] array, got shape %s" % (shape,))
    for name, a in zip(("seg_human", "seg_face", "edges"), arrays[1:]):
        if a.shape != shape:
            raise ValueError("%s: shape %s differs from seg_panoptic's %s" % (name, a.shape, shape))
    out = np.empty(shape[:-2] + (PLANES,) + shape[-2:], dtype=np.uint8)
    for p, (name, a, lo, hi, off) in enumerate((("seg_panoptic", arrays[0], -1, PANOPTIC_CLASSES - 1, 1),
                                                ("seg_human", arrays[1], -1, HUMAN_PARTS - 1, 1),
                                                ("seg_face", arrays[2], 0, FACE_PARTS, 0),
                                                ("edges", arrays[3], 0, 2, 0))):
        a = a.astype(np.int64)
        amin, amax = int(a.min()), int(a.max())
        if amin < lo or amax > hi:
            raise ValueError("%s: values must lie in [%d, %d], got [%d, %d]" % (name, lo, hi, amin, amax))
        out[..., p, :, :] = a + off
    return torch.from_numpy(out)


def unpack(planes):
    """The inverse of `pack`: compact planes [4, H, W] / [B, 4, H, W] (a CPU uint8 array or tensor) -> (seg_panoptic,
    seg_human, seg_face, edges) as int64 numpy arrays [H, W] / [B, H, W] in pack's value conventions (-1 = none for the
    panoptic and human planes, 0 = none for the face plane, edges 0..2).  unpack(pack(*a)) == a for every map pack accepts.
    Raises ValueError on a byte outside its plane's range, a dtype other than uint8 or a wrong shape."""
    if isinstance(planes, torch.Tensor):
        if planes.device.type != "cpu":
            raise ValueError("planes: expected a CPU array, got a %s tensor" % planes.device.type)
        planes = planes.numpy()
    a = np.asarray(planes)
    if a.dtype != np.uint8:
        raise ValueError("planes: expected uint8, got %s" % a.dtype)
    if a.ndim not in (3, 4) or a.shape[-3] != PLANES or 0 in a.shape:
        raise ValueError("planes: expected a non-empty [4, H, W] or [B, 4, H, W] array, got shape %s" % (a.shape,))
    out = []
    for p, (name, hi, off) in enumerate((("panoptic", PANOPTIC_CLASSES, 1), ("human", HUMAN_PARTS, 1), ("face", FACE_PARTS, 0),
                                         ("edges", 2, 0))):
        v = a[..., p, :, :].astype(np.int64)
        amax = int(v.max())
        if amax > hi:
            raise ValueError("planes: %s codes must lie in [0, %d], got %d" % (name, hi, amax))
        out.append(v - off)
    return tuple(out)


def _kernel_device(t):
    """Whether t lives where the kernels run."""
    return t.is_cuda


def decode(logits):
    """VQ-SEG logits (model(seg)[0], decode_code(tokens)) or a dense scene map -> compact planes, uint8 [B, 4, H, W] on the
    same device, by the rule of mas_scene_decode: per one-hot plane 1 + the argmax of its channel group when that maximum is
    > 0 (sigma > 0.5, the BCE decision boundary), else 0 ("none"); edges 1 when the edge logit is > 0.  Ties go to the
    lowest channel, a NaN never wins and is never > 0.  A dense map decodes to the planes `pack` made, an edge count of 2
    becoming 1.

    logits: a CUDA fp32 [B, 159, H, W] tensor in any layout; the decoder's padded channels-last view is the fast case.  Runs
    under no_grad.  Raises ValueError, before any launch, on another device, dtype, shape, or on B or H of 0 or above 65535."""
    if not isinstance(logits, torch.Tensor) or logits.dim() != 4 or logits.shape[1] != CHANNELS:
        raise ValueError("decode expects [B, %d, H, W] logits, got %s" % (
            CHANNELS, str(tuple(logits.shape)) if isinstance(logits, torch.Tensor) else type(logits).__name__))
    if not _kernel_device(logits):
        raise ValueError("decode needs a CUDA tensor, got one on %s" % logits.device)
    if logits.dtype != torch.float32:
        raise ValueError("decode takes float32 logits, got %s" % logits.dtype)
    b, _, h, w = logits.shape
    if not (0 < b <= 65535 and 0 < h <= 65535 and w > 0):
        raise ValueError("decode needs 1 <= B, H <= 65535 and W >= 1, got shape %s" % (tuple(logits.shape),))
    with torch.no_grad():
        out = torch.empty((b, PLANES, h, w), dtype=torch.uint8, device=logits.device)
        L.call("mas_scene_decode", logits, L.t4(logits), out)
    return out


def confusion(pred, target):
    """Per-plane confusion matrices of compact maps pred and target (uint8 [B, 4, H, W] of one shape on one CUDA device):
    {"panoptic": [134, 134], "human": [21, 21], "face": [6, 6], "edges": [2, 2]} int64 tensors on that device, row = target
    code, column = predicted code (an edge count of 1 or 2 is an edge), plus "out_of_range": the number of pixels with a plane
    counted in no cell because its target or predicted byte lies outside the plane's range (once per pixel; its other planes
    are counted; always 0 for maps from `pack` and `decode`).  The counts are
    exact integers, the same on every call.  Raises ValueError, before any launch, on a wrong device, dtype or shape."""
    for name, t in (("pred", pred), ("target", target)):
        if not isinstance(t, torch.Tensor) or t.dim() != 4 or t.shape[1] != PLANES or 0 in t.shape:
            raise ValueError("%s: expected a non-empty [B, %d, H, W] compact map, got %s" % (
                name, PLANES, str(tuple(t.shape)) if isinstance(t, torch.Tensor) else type(t).__name__))
        if t.dtype != torch.uint8:
            raise ValueError("%s: expected uint8, got %s" % (name, t.dtype))
        if not _kernel_device(t):
            raise ValueError("%s: expected a CUDA tensor, got one on %s" % (name, t.device))
    if pred.shape != target.shape:
        raise ValueError("pred %s and target %s differ in shape" % (tuple(pred.shape), tuple(target.shape)))
    if pred.device != target.device:
        raise ValueError("pred (%s) and target (%s) are on different devices" % (pred.device, target.device))
    b, _, h, w = pred.shape
    if b > 2 ** 31 - 1:
        raise ValueError("confusion takes at most 2^31 - 1 images, got %d" % b)
    pred, target = pred.contiguous(), target.contiguous()
    conf = torch.empty(CONFUSION_LEN, dtype=torch.int64, device=pred.device)
    nb = int(L.query("mas_scene_confusion_ws_bytes", h * w, b))
    ws = L.workspace(nb, pred.device) if nb else None
    L.call("mas_scene_confusion", pred, target, h * w, b, conf, ws, nb)
    out, o = {}, 0
    for g, k in zip(GROUPS, CLASSES):
        out[g] = conf[o:o + k * k].view(k, k)
        o += k * k
    out["out_of_range"] = conf[o]
    return out


def iou(conf):
    """Per-class IoU from `confusion`'s matrices (host arithmetic; tensors or arrays): for each group, "iou" = TP / (TP + FP
    + FN) per class as a float64 numpy array (NaN where the union is empty, "none" included as class 0) and "miou", the mean
    over the classes other than "none" whose union is non-empty (NaN when there is none).  For edges, class 1 is "edge"."""
    res = {}
    for g, k in zip(GROUPS, CLASSES):
        m = conf[g]
        m = (m.cpu().numpy() if isinstance(m, torch.Tensor) else np.asarray(m)).astype(np.int64)
        if m.shape != (k, k):
            raise ValueError("%s: expected a [%d, %d] matrix, got shape %s" % (g, k, k, m.shape))
        tp = np.diag(m).astype(np.float64)
        union = m.sum(0) + m.sum(1) - np.diag(m)
        with np.errstate(invalid="ignore", divide="ignore"):
            per = np.where(union > 0, tp / np.maximum(union, 1), np.nan)
        valid = per[1:][union[1:] > 0]
        res[g] = {"iou": per, "miou": float(valid.mean()) if valid.size else float("nan")}
    return res
