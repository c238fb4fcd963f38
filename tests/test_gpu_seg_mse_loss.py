"""VQVAEWithBCELoss on the H100: the mas_bce_mse_* kernels (ops.BCEMSELogitsFn) against the fixture made from the real
reference and against fp64 torch of the reference expression on every route, compact targets against dense ones bit for
bit, and whole VQ-SEG training steps through losses.scene_loss against the same steps fed the dense map and against the
reference's own classes (the copy of losses/loss_seg.py that build() stages under oracle/_ref/)."""
import copy
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, ROOT, rel_err

pytestmark = pytest.mark.gpu

# mas_vq_backward accumulates the codebook gradient with fp32 atomics, so its last bits vary from run to run whatever the
# input (tests/test_gpu_scene_maps.py); it is compared within this bound, every other result bit for bit.
ATOMIC_GRADS = {"quantize.embedding.weight": 1e-6}
TC_DD = dict(z_channels=64, in_channels=159, out_channels=159, channels=[128, 128], num_res_blocks=1, resolution=64,
             attn_resolutions=[], dropout=0.0)


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _pw(dev=None):
    return torch.ones(159, device=dev).index_fill(0, torch.arange(153, 158, device=dev), 20)


def _ref_loss_seg():
    path = os.path.join(ROOT, "oracle", "_ref", "losses", "loss_seg.py")
    assert os.path.exists(path), "build() stages the reference's losses/loss_seg.py under oracle/_ref/"
    spec = importlib.util.spec_from_file_location("_ref_loss_seg_gpu", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_segmentation(lab):
    """Data/dataset_preprocessor.py:61-86 restated on the packed planes -> NCHW [N, 159, H, W] float32."""
    lab = lab.long()
    seg = torch.cat([F.one_hot(lab[:, 0], num_classes=134)[..., 1:], F.one_hot(lab[:, 1], num_classes=21)[..., 1:],
                     F.one_hot(lab[:, 2], num_classes=6)[..., 1:], lab[:, 3].unsqueeze(-1).float()], dim=-1)
    return seg.float().permute(0, 3, 1, 2).contiguous()


def _labels(n, h, w, seed):
    """Random valid planes, about half of each one-hot plane empty, edge counts 0..2."""
    g = torch.Generator().manual_seed(seed)
    planes = []
    for hi in (133, 20, 5):
        code = torch.randint(1, hi + 1, (n, h, w), generator=g)
        planes.append(torch.where(torch.rand(n, h, w, generator=g) < 0.5, code, torch.zeros_like(code)))
    planes.append(torch.randint(0, 3, (n, h, w), generator=g))
    return torch.stack(planes, 1).to(torch.uint8)


def _padded(lo, cp=160):
    """lo as the padded channels-last view the decoder's last convolution returns (pitch cp, pad channels zero)."""
    n, c, h, w = lo.shape
    base = torch.zeros(n, h, w, cp, device=lo.device)
    base[..., :c] = lo.permute(0, 2, 3, 1)
    return base.permute(0, 3, 1, 2)[:, :c]


def _ref64(lo, tg, g=1.0):
    """losses/loss_seg.py:34-41 (without qloss) in fp64 torch on the device: loss and g * d loss / d logits."""
    x = lo.detach().double().requires_grad_(True)
    t = tg.double()
    loss = F.mse_loss(x.sigmoid(), t) + F.binary_cross_entropy_with_logits(
        x.permute(0, 2, 3, 1), t.permute(0, 2, 3, 1), pos_weight=_pw(x.device).double())
    (g * loss).backward()
    return loss.detach(), x.grad


def _run(logits_fn, t, g=1.0):
    """BCEMSELogitsFn on fresh logits: loss, d loss / d logits, the padded buffer the gradient lives in (or None), entries."""
    from mas_b200 import _lib as L, ops
    logits = logits_fn().requires_grad_(True)
    seen = {}
    logits.register_hook(lambda gr: seen.update(base=getattr(gr, "_mas_pad_base", None)))
    L.profile_start()
    loss = ops.BCEMSELogitsFn.apply(logits, t, _pw(logits.device))
    (g * loss).backward() if g != 1.0 else loss.backward()
    names = L.profile_report(lambda k: k.split("|")[0])
    return loss.detach(), logits.grad, seen.get("base"), set(names)


def test_against_reference_fixture():
    """scene_loss.VQVAEWithBCELoss against the reference's own numbers: loss within 1e-5 and gradient within 1e-5 relative
    (the bars test_gpu_parity.py holds BCELogitsFn to), from the dense and the compact target, tiled and generic routes."""
    from losses import scene_loss
    g = torch.load(os.path.join(GOLDEN, "seg_mse_loss.pt"), weights_only=False)
    dev = _dev()
    m = scene_loss.VQVAEWithBCELoss().to(dev)
    q = g["qloss"].to(dev)
    for t in (g["target"].float().to(dev), g["labels"].to(dev)):
        for layout in ("padded", "nchw"):
            pred = (_padded(g["pred"].to(dev)) if layout == "padded" else g["pred"].to(dev)).requires_grad_(True)
            loss = m(q, t, pred)
            assert abs(float(loss.detach()) - float(g["loss"])) < 1e-5
            loss.backward()
            assert rel_err(pred.grad, g["grad"]) < 1e-5


@pytest.mark.parametrize("n,hw", [(2, 64), (8, 64), (2, 256), (8, 256)])
def test_padded_view_vs_fp64(n, hw):
    """The model's padded channels-last view (mas_bce_mse_cl_* / _scene_*) against fp64 of the reference expression, at
    g = 3: pad channels of the gradient buffer exactly 0; the compact target equal to the dense one bit for bit."""
    dev = _dev()
    lab = _labels(n, hw, hw, seed=n * hw).to(dev)
    dense = load_segmentation(lab)
    lo = torch.randn(n, 159, hw, hw, generator=torch.Generator().manual_seed(hw)).to(dev) * 3
    ref_loss, ref_grad = _ref64(lo, dense, 3.0)
    ld, gd, bd, nd = _run(lambda: _padded(lo), dense, 3.0)
    lc, gc, bc, nc = _run(lambda: _padded(lo), lab, 3.0)
    assert nd == {"mas_bce_mse_cl_forward", "mas_bce_mse_cl_backward"}
    assert nc == {"mas_bce_mse_scene_forward", "mas_bce_mse_scene_backward"}
    assert abs(float(ld) - float(ref_loss)) < 1e-5 * float(ref_loss)
    assert rel_err(gd, ref_grad) < 1e-5
    for base in (bd, bc):
        assert base is not None and base.shape == (n, 160, hw, hw) and not base[:, 159:].any()
    assert torch.equal(lc, ld) and torch.equal(gc, gd)
    del ref_grad, gd, gc, bd, bc


@pytest.mark.parametrize("layout", ["nchw", "strided", "padded_w48"])
def test_generic_route_vs_fp64(layout):
    """NCHW-contiguous, odd-strided and W % 32 != 0 logits take mas_bce_mse_logits (a compact target expanded first by
    mas_scene_expand): against fp64 at g = 3, and compact equal to dense bit for bit."""
    dev = _dev()
    n, h, w = 2, 24, 48
    lab = _labels(n, h, w, seed=7).to(dev)
    dense = load_segmentation(lab)
    lo = torch.randn(n, 159, h, w, generator=torch.Generator().manual_seed(8)).to(dev) * 3

    def make():
        if layout == "nchw":
            return lo.clone()
        if layout == "strided":                                   # every other column of a wider, channels-last tensor
            big = torch.zeros(n, 159, h, 2 * w + 1, device=dev).contiguous(memory_format=torch.channels_last)
            big[..., 1::2] = lo
            return big[..., 1::2]
        return _padded(lo)
    ref_loss, ref_grad = _ref64(lo, dense, 3.0)
    ld, gd, _, nd = _run(make, dense, 3.0)
    lc, gc, _, nc = _run(make, lab, 3.0)
    assert "mas_bce_mse_logits" in nd and "mas_bce_mse_logits" in nc and "mas_scene_expand" in nc
    assert not any(k.startswith("mas_bce_mse_cl") or k.startswith("mas_bce_mse_scene") for k in nd | nc)
    assert abs(float(ld) - float(ref_loss)) < 1e-5 * float(ref_loss)
    assert rel_err(gd, ref_grad) < 1e-5
    assert torch.equal(lc, ld) and torch.equal(gc, gd)


def test_repeatable_bits():
    """Two calls give the same loss and gradient bits on every route (fixed-order fp64 reduction, no atomics)."""
    dev = _dev()
    lab = _labels(4, 64, 64, seed=3).to(dev)
    dense = load_segmentation(lab)
    lo = torch.randn(4, 159, 64, 64, generator=torch.Generator().manual_seed(4)).to(dev) * 3
    for make in (lambda: _padded(lo), lambda: lo.clone()):
        for t in (dense, lab):
            a, b = _run(make, t, 0.5), _run(make, t, 0.5)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def _model(dev):
    from models import VQBASE
    torch.manual_seed(0)
    m = VQBASE(TC_DD, 128, 64, 10, 100)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    m.quantize.q_counter = 10 ** 6
    return m.train().to(dev)


def _step(m, loss_fn, x):
    m.zero_grad(set_to_none=True)
    dec, diff = m(x)
    loss = loss_fn(diff, x, dec)
    loss.backward()
    out = {"loss": loss.detach().clone(), "dec": dec.detach().clone()}
    out.update({"grad." + k: p.grad.clone() for k, p in m.named_parameters()})
    return out


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        tol = ATOMIC_GRADS.get(k[5:]) if k.startswith("grad.") else None
        if tol is None:
            assert torch.equal(a[k], b[k]), k
        else:
            assert rel_err(a[k], b[k]) < tol, k


@pytest.mark.parametrize("name", ["VQVAEWithBCELoss", "BCELossWithQuant"])
def test_vqseg_step_compact_dense_and_reference(name):
    """A seg-config VQBASE at 64 x 64 stepped with losses.scene_loss.<name>: the compact map gives the dense map's step
    bit for bit (loss, dec and every parameter gradient); the dense step agrees with the reference's own class on the same
    decoder output (loss within 1e-5, d loss / d dec within 1e-5 relative); and BCELossWithQuant is BCELogitsFn + qloss bit
    for bit."""
    from losses import scene_loss
    from mas_b200 import ops
    dev = _dev()
    lab = _labels(2, 64, 64, seed=5).to(dev)
    seg = load_segmentation(lab)
    loss_fn = getattr(scene_loss, name)().to(dev)
    ref_fn = getattr(_ref_loss_seg(), name)().to(dev)
    assert loss_fn.state_dict().keys() == ref_fn.state_dict().keys()
    assert torch.equal(loss_fn.weight, ref_fn.weight)
    m = _model(dev)
    state = copy.deepcopy(m.state_dict())
    dense = _step(m, loss_fn, seg)
    m.load_state_dict(state)
    compact = _step(m, loss_fn, lab)
    _assert_same(compact, dense)
    if name == "BCELossWithQuant":
        m.load_state_dict(state)
        direct = _step(m, lambda q, t, p: ops.BCELogitsFn.apply(p, t, _pw(dev)) + q, lab)
        _assert_same(direct, compact)
    m.load_state_dict(state)
    m.zero_grad(set_to_none=True)
    dec, diff = m(seg)
    lk = loss_fn(diff, seg, dec)
    lr = ref_fn(diff, seg, dec)
    assert abs(float(lk.detach()) - float(lr.detach())) < 1e-5 * float(lr.detach())
    gk, = torch.autograd.grad(lk, dec, retain_graph=True)
    gr, = torch.autograd.grad(lr, dec)
    assert rel_err(gk, gr) < 1e-5
