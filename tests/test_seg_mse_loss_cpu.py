"""VQVAEWithBCELoss on the CPU: the oracle against the fixture made from the real reference (tools/make_golden_seg_mse_loss.py),
and the host logic of ops.BCEMSELogitsFn and losses.scene_loss above the emulated C-ABI of tests/test_scene_maps_cpu.py, with
fp64 numpy restatements of the mas_bce_mse_* entries (include/mas_b200.h).  The kernels are tested on the GPU
(tests/test_gpu_seg_mse_loss.py)."""
import os

import numpy as np
import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode

from conftest import GOLDEN, rel_err
from test_host_logic_vq_cpu import _f32, _view4, vq_emu  # noqa: F401  (vq_emu: fixture)
from test_scene_maps_cpu import SceneEmu, expand_np


def _golden():
    return torch.load(os.path.join(GOLDEN, "seg_mse_loss.pt"), weights_only=False)


def _pos_weight(c=159):
    return torch.ones(c).index_fill(0, torch.arange(153, 158), 20)


def bce_mse_np(X, T, pw):
    """fp64 restatement of the entries' loss terms and d/dx of one element (include/mas_b200.h), [..., C] arrays."""
    s = 1.0 / (1.0 + np.exp(-X))
    coef = 1.0 + (pw - 1.0) * T
    lterm = coef * np.logaddexp(0.0, -X) + (1.0 - T) * X + (s - T) ** 2
    dterm = coef * s - pw * T + 2.0 * (s - T) * s * (1.0 - s)
    return lterm, dterm


class SegEmu(SceneEmu):
    """SceneEmu plus the mas_bce_mse_* entries and mas_scale_by."""

    def mas_bce_mse_cl_forward(self, logits, target, pos_weight, N, C, CP, H, W, loss_out, ws, ws_bytes):
        X, T = self._bce_views(logits, target, N, C, CP, H, W)
        lterm, _ = bce_mse_np(X, T, _f32(pos_weight, C).astype(np.float64))
        _f32(loss_out, 1)[0] = lterm.mean()

    def mas_bce_mse_cl_backward(self, logits, target, pos_weight, g, N, C, CP, H, W, grad):
        X, T = self._bce_views(logits, target, N, C, CP, H, W)
        _, dterm = bce_mse_np(X, T, _f32(pos_weight, C).astype(np.float64))
        gg = float(_f32(g, 1)[0]) if g is not None else 1.0
        out = np.zeros((N, H, W, CP), dtype=np.float32)           # pad channels written as zeros
        out[..., :C] = gg * dterm / (N * C * H * W)
        _f32(grad, N * H * W * CP)[...] = out.reshape(-1)

    def mas_bce_mse_scene_forward(self, logits, labels, pos_weight, N, CP, H, W, loss_out, ws, ws_bytes):
        self.mas_bce_mse_cl_forward(logits, self._dense_target(labels, N, H, W), pos_weight, N, 159, CP, H, W, loss_out, ws, ws_bytes)

    def mas_bce_mse_scene_backward(self, logits, labels, pos_weight, g, N, CP, H, W, grad):
        self.mas_bce_mse_cl_backward(logits, self._dense_target(labels, N, H, W), pos_weight, g, N, 159, CP, H, W, grad)

    def mas_bce_mse_logits(self, logits, ls, target, ts, pos_weight, loss_out, grad, gs, grad_scale, ws, ws_bytes):
        X, T = _view4(logits, ls).astype(np.float64), _view4(target, ts).astype(np.float64)
        lterm, dterm = bce_mse_np(X, T, _f32(pos_weight, ls.c).astype(np.float64))
        _f32(loss_out, 1)[0] = lterm.mean()
        if grad is not None:
            _view4(grad, gs)[...] = grad_scale * dterm

    def mas_scale_by(self, x, g, y, n):
        _f32(y, n)[...] = _f32(x, n) * _f32(g, 1)[0]


@pytest.fixture
def seg_emu(vq_emu, monkeypatch):  # noqa: F811
    from losses import scene_loss
    from mas_b200 import ops
    e = SegEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x, dtype=None: None)
    monkeypatch.setattr(scene_loss, "_on_device", lambda t: True)
    return e


class TorchOps(TorchDispatchMode):
    """Records the aten operators that run inside the block."""

    def __init__(self):
        super().__init__()
        self.ops = set()

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        self.ops.add(func.overloadpacket.__name__)
        return func(*args, **(kwargs or {}))


# allocation, views and copies: nothing that computes a term of the loss or of its gradient
PLUMBING = {"empty", "empty_like", "empty_strided", "permute", "slice", "view", "alias", "detach", "as_strided", "contiguous",
            "clone", "_to_copy", "copy_", "select", "transpose", "expand", "ones_like", "new_empty", "new_empty_strided",
            "zeros_like", "fill_", "lift_fresh"}


def _labels(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randint(0, hi + 1, (n, h, w), generator=g) for hi in (133, 20, 5, 2)], 1).to(torch.uint8)


def _padded(lo, cp=160):
    n, c, h, w = lo.shape
    base = torch.zeros(n, h, w, cp)
    base[..., :c] = lo.permute(0, 2, 3, 1)
    return base.permute(0, 3, 1, 2)[:, :c]


def _ref64(lo, tg, g=1.0):
    """The reference expression (losses/loss_seg.py:34-41) in fp64 torch: loss and g * d loss / d logits."""
    import torch.nn.functional as F
    x = lo.double().clone().requires_grad_(True)
    t = tg.double()
    loss = F.mse_loss(x.sigmoid(), t) + F.binary_cross_entropy_with_logits(
        x.permute(0, 2, 3, 1), t.permute(0, 2, 3, 1), pos_weight=_pos_weight(x.shape[1]).double())
    (g * loss).backward()
    return loss.detach(), x.grad


def vqvae_with_bce_loss(qloss, target, prediction, image_channels=159, codebook_weight=1.0):
    """CPU restatement of losses/loss_seg.py:25-41: mse_loss(sigmoid(prediction), target) + the weighted BCE of
    oracle.vqgan_oracle.bce_loss_with_quant + codebook_weight * qloss, summed in the reference's order."""
    import torch.nn.functional as F
    bce = F.binary_cross_entropy_with_logits(prediction.permute(0, 2, 3, 1), target.permute(0, 2, 3, 1),
                                             pos_weight=_pos_weight(image_channels))
    return (F.mse_loss(prediction.sigmoid(), target) + bce) + codebook_weight * qloss


def test_oracle_reproduces_fixture():
    """The restatement above reproduces the fixture the real reference class wrote, and the fixture's dense target is the
    expansion of its compact labels."""
    g = _golden()
    pred = g["pred"].clone().requires_grad_(True)
    loss = vqvae_with_bce_loss(g["qloss"], g["target"].float(), pred)
    loss.backward()
    assert abs(float(loss.detach()) - float(g["loss"])) < 1e-6
    assert rel_err(pred.grad, g["grad"]) < 1e-6
    assert g["target"][:, 158].max() == 2
    assert torch.equal(torch.from_numpy(expand_np(g["labels"].numpy())).permute(0, 3, 1, 2), g["target"].float())


@pytest.mark.parametrize("layout", ["padded_cl", "padded_cl_w48", "nchw", "strided"])
def test_routes_and_values_host_logic(seg_emu, layout):
    """Padded channels-last logits (W % 32 == 0) go to mas_bce_mse_cl_* with a dense target and mas_bce_mse_scene_* with a
    compact one; every other layout to mas_bce_mse_logits, a compact target expanded by mas_scene_expand first, the backward
    a mas_scale_by of the gradient it wrote. Loss and gradient equal the fp64 reference expression, and no aten operator
    that computes anything runs in the forward or the backward."""
    from mas_b200 import ops
    n, h = 2, 4
    w = 48 if layout == "padded_cl_w48" else 32
    lab = _labels(n, h, w, seed=w)
    dense = torch.from_numpy(expand_np(lab.numpy())).permute(0, 3, 1, 2).contiguous()
    lo = torch.randn(n, 159, h, w, generator=torch.Generator().manual_seed(1)) * 3
    ref_loss, ref_grad = _ref64(lo, dense, 3.0)
    pw = _pos_weight()
    out = []
    for t in (dense, lab):
        if layout == "nchw":
            logits = lo.clone()
        elif layout == "strided":
            big = torch.zeros(n, 159, h, 2 * w)
            big[..., ::2] = lo
            logits = big[..., ::2]
        else:
            logits = _padded(lo)
        logits.requires_grad_(True)
        first = len(seg_emu.names)
        rec, g3 = TorchOps(), torch.tensor(3.0)
        with rec:
            loss = ops.BCEMSELogitsFn.apply(logits, t, pw)
            loss.backward(g3)
        names = seg_emu.names[first:]
        assert not (rec.ops - PLUMBING), rec.ops
        assert abs(float(loss) - float(ref_loss)) < 1e-6 * float(ref_loss)
        assert rel_err(logits.grad, ref_grad) < 1e-6
        out.append((names, loss.detach(), logits.grad))
    (nd, ld, gd), (nc, lc, gc) = out
    assert torch.equal(ld, lc) and torch.equal(gd, gc)
    if layout.startswith("padded_cl") and w % 32 == 0:
        assert nd == ["mas_bce_mse_cl_forward", "mas_bce_mse_cl_backward"]
        assert nc == ["mas_bce_mse_scene_forward", "mas_bce_mse_scene_backward"]
    else:
        assert nd == ["mas_bce_mse_logits", "mas_scale_by"]
        assert nc == ["mas_scene_expand", "mas_bce_mse_logits", "mas_scale_by"]


def test_compact_target_saves_only_labels(seg_emu):
    from mas_b200 import ops
    lab = _labels(2, 4, 32, seed=3)
    logits = _padded(torch.randn(2, 159, 4, 32)).requires_grad_(True)
    loss = ops.BCEMSELogitsFn.apply(logits, lab, _pos_weight())
    saved = loss.grad_fn.saved_tensors
    assert [t.dtype for t in saved] == [torch.float32, torch.uint8, torch.float32]
    assert saved[1].shape == lab.shape


def test_scene_loss_modules_against_fixture(seg_emu):
    """Both modules run end to end on the emulated entries: VQVAEWithBCELoss reproduces the reference's fixture from the
    dense and the compact target (loss and d loss / d pred), BCELossWithQuant is BCELogitsFn + qloss."""
    from losses import scene_loss
    from mas_b200 import ops
    g = _golden()
    m = scene_loss.VQVAEWithBCELoss()
    for t in (g["target"].float(), g["labels"]):
        for layout in ("padded", "nchw"):
            pred = (_padded(g["pred"]) if layout == "padded" else g["pred"].clone()).requires_grad_(True)
            loss = m(g["qloss"], t, pred)
            loss.backward()
            assert abs(float(loss) - float(g["loss"])) < 1e-6
            assert rel_err(pred.grad, g["grad"]) < 1e-6
    first = len(seg_emu.names)
    pred = _padded(g["pred"])
    b = scene_loss.BCELossWithQuant()(g["qloss"], g["labels"], pred)
    assert torch.equal(b, ops.BCELogitsFn.apply(pred, g["labels"], _pos_weight()) + g["qloss"])
    assert seg_emu.names[first:] == ["mas_bce_scene_forward"] * 2


def test_scene_loss_state_dict_is_the_references():
    from losses import scene_loss
    for cls in (scene_loss.BCELossWithQuant, scene_loss.VQVAEWithBCELoss):
        for kw in ({}, dict(image_channels=159, codebook_weight=0.5)):
            m = cls(**kw)
            sd = m.state_dict()
            assert list(sd) == ["weight"] and sd["weight"].dtype == torch.float32
            assert torch.equal(sd["weight"], torch.ones(159).index_fill(0, torch.arange(153, 158), 20))
            assert m.codebook_weight == kw.get("codebook_weight", 1.0) and not list(m.parameters())
    ref = os.path.join(os.path.dirname(GOLDEN), "..", "oracle", "_ref", "losses", "loss_seg.py")
    if os.path.exists(ref):                                   # the reference's own classes, where build() staged them
        import importlib.util
        spec = importlib.util.spec_from_file_location("_ref_loss_seg_cpu", ref)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        for name in ("BCELossWithQuant", "VQVAEWithBCELoss"):
            a, b = getattr(mod, name)().state_dict(), getattr(scene_loss, name)().state_dict()
            assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
            getattr(scene_loss, name)().load_state_dict(a)


def test_losses_package_still_resolves_loss_seg_to_the_reference():
    import losses
    assert losses._EXPORTS["BCELossWithQuant"] == losses._EXPORTS["VQVAEWithBCELoss"] == "loss_seg"
    here = os.path.dirname(os.path.abspath(losses.__file__))
    assert not os.path.exists(os.path.join(here, "loss_seg.py"))


def test_scene_loss_refuses_bad_operands_before_any_launch(seg_emu, monkeypatch):
    from losses import scene_loss
    n, h, w = 2, 4, 32
    pred = torch.randn(n, 159, h, w)
    dense = torch.zeros(n, 159, h, w)
    lab = _labels(n, h, w, seed=1)
    q = torch.tensor(0.1)
    bad = [
        (pred.double(), dense), (pred.half(), dense), (pred[0], dense[0]),               # prediction dtype / rank
        (pred, dense.double()), (pred, dense.long()), (pred, lab.long()),                # target dtype
        (pred, dense[:, :158]), (pred, dense[..., :16]), (pred, dense[:1]),              # dense shapes
        (pred, lab[:, :3]), (pred, lab[..., :16]), (pred, lab[:1]),                      # compact shapes
        (pred[:, :158], lab), (pred[:, :158], dense[:, :158]),                           # channels != image_channels
        ("pred", dense), (pred, None),
    ]
    for cls in (scene_loss.BCELossWithQuant, scene_loss.VQVAEWithBCELoss):
        m = cls()
        for p, t in bad:
            with pytest.raises(ValueError):
                m(q, t, p)
        with pytest.raises(ValueError):
            cls(image_channels=158)(q, lab, pred[:, :158])                              # compact map of 158 channels
    assert seg_emu.names == []
    monkeypatch.undo()                                                                     # the real device check
    for m in (scene_loss.BCELossWithQuant(), scene_loss.VQVAEWithBCELoss()):
        with pytest.raises(ValueError):
            m(q, dense, pred)                                                              # CPU tensors
        with pytest.raises(ValueError):
            m(q, lab, pred)
