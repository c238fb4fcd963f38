"""Writes tests/golden/seg_mse_loss.pt from the REAL reference VQVAEWithBCELoss (losses/loss_seg.py:25-41), on the CPU in
fp32, from the copy of loss_seg.py that oracle/vendor_ref.py stages under oracle/_ref/ (run `python oracle/vendor_ref.py`
first, or build()):

    python tools/make_golden_seg_mse_loss.py

The target is a dense 159-channel scene map expanded from seeded compact label planes (mas_b200.scene's layout: panoptic
code 0..133, human 0..20, face 0..5, edge count 0..2) by a restatement of the reference's load_segmentation
(Data/dataset_preprocessor.py:61-86); the planes are stored too, so the compact route is checked against the same numbers.
The first pixels of the batch hold every code of every plane, edge counts of 2 included. The logits are seeded normals
times 3 with a few saturating values (+-30, +-90). W = 32 so the padded channels-last view takes the tiled kernels.

Recorded: labels (uint8 [2, 4, 4, 32]), target (the dense map, stored as uint8: its values are 0, 1 and 2), pred, qloss,
loss and d loss / d pred."""
import importlib.util
import os

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "seg_mse_loss.pt")
LOSS_SEG = os.path.join(ROOT, "oracle", "_ref", "losses", "loss_seg.py")
N, H, W = 2, 4, 32


def labels(seed=17):
    g = torch.Generator().manual_seed(seed)
    planes = [torch.randint(0, hi + 1, (N, H, W), generator=g) for hi in (133, 20, 5, 2)]
    lab = torch.stack(planes, 1).to(torch.uint8)
    flat = lab.transpose(0, 1).reshape(4, -1)
    for p, hi in enumerate((133, 20, 5, 2)):
        flat[p, :hi + 1] = torch.arange(hi + 1, dtype=torch.uint8)
    lab = flat.view(4, N, H, W).transpose(0, 1).contiguous()
    lab[1, 3, 1] = 2                                       # a whole row of edge count 2
    return lab


def load_segmentation(lab):
    """Data/dataset_preprocessor.py:61-86 on the packed planes -> NCHW [N, 159, H, W] float32."""
    lab = lab.long()
    seg = torch.cat([F.one_hot(lab[:, 0], num_classes=134)[..., 1:], F.one_hot(lab[:, 1], num_classes=21)[..., 1:],
                     F.one_hot(lab[:, 2], num_classes=6)[..., 1:], lab[:, 3].unsqueeze(-1)], dim=-1)
    return seg.float().permute(0, 3, 1, 2).contiguous()


def main():
    if not os.path.exists(LOSS_SEG):
        raise SystemExit("%s is missing: run `python oracle/vendor_ref.py` where the reference checkout exists" % LOSS_SEG)
    spec = importlib.util.spec_from_file_location("_ref_loss_seg", LOSS_SEG)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    lab = labels()
    target = load_segmentation(lab)
    assert target[:, 158].max() == 2
    g = torch.Generator().manual_seed(18)
    pred = torch.randn(N, 159, H, W, generator=g) * 3
    pred[0, :4, 0, 0] = torch.tensor([30.0, -30.0, 90.0, -90.0])
    pred[1, 158, 1, :4] = torch.tensor([30.0, -30.0, 90.0, -90.0])   # saturated logits at edge count 2
    pred.requires_grad_(True)
    qloss = torch.tensor(0.37)
    loss_fn = ref.VQVAEWithBCELoss(image_channels=159)
    loss = loss_fn(qloss, target, pred)
    loss.backward()
    torch.save(dict(labels=lab, target=target.to(torch.uint8), pred=pred.detach().clone(), qloss=qloss, loss=loss.detach(),
                    grad=pred.grad.clone()), OUT)
    print("wrote", OUT, "loss", float(loss.detach()))


if __name__ == "__main__":
    main()
