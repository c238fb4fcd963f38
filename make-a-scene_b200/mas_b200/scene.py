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
"""
from __future__ import annotations

import numpy as np
import torch

PANOPTIC_CLASSES, HUMAN_PARTS, FACE_PARTS = 133, 20, 5
PLANES = 4
CHANNELS = PANOPTIC_CLASSES + HUMAN_PARTS + FACE_PARTS + 1     # 159


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
