"""Compact scene maps on the H100: mas_scene_expand against a torch restatement of the reference's one-hot stack, the
label-reading weighted BCE (mas_bce_scene_*) against mas_bce_cl_* on the expanded target, and whole VQ-SEG training steps
fed the compact map against the same steps fed its dense expansion - bit for bit - plus the memory the compact input
frees and the captured CUDA-graph step."""
import copy

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu

# The codebook gradient of mas_vq_backward is accumulated with fp32 atomics: its summation order, and so its last bits,
# vary from run to run whatever the input. It is compared within this bound; every other result bit for bit.
ATOMIC_GRADS = {"quantize.embedding.weight": 1e-6}


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def load_segmentation(lab):
    """Data/dataset_preprocessor.py:61-86 restated on the packed planes (codes = the .npz arrays + their offsets):
    one_hot(134)[1:], one_hot(21)[1:], one_hot(6)[1:], edges_panoptic + edges_human -> NCHW [N, 159, H, W] float32."""
    lab = lab.long()
    seg = torch.cat([F.one_hot(lab[:, 0], num_classes=134)[..., 1:], F.one_hot(lab[:, 1], num_classes=21)[..., 1:],
                     F.one_hot(lab[:, 2], num_classes=6)[..., 1:], lab[:, 3].unsqueeze(-1).float()], dim=-1)
    return seg.float().permute(0, 3, 1, 2).contiguous()


def _labels(n, h, w, seed=0):
    """Random valid planes with about half of each one-hot plane empty; the first pixels of image 0 hold every code of every
    plane (edges 0, 1, 2 included) and the first row of the last image is empty in every plane."""
    g = torch.Generator().manual_seed(seed)
    planes = []
    for hi in (133, 20, 5):
        code = torch.randint(1, hi + 1, (n, h, w), generator=g)
        planes.append(torch.where(torch.rand(n, h, w, generator=g) < 0.5, code, torch.zeros_like(code)))
    planes.append(torch.randint(0, 3, (n, h, w), generator=g))
    lab = torch.stack(planes, 1).to(torch.uint8)
    flat = lab[0].reshape(4, -1)
    for p, hi in enumerate((133, 20, 5, 2)):
        k = min(hi + 1, flat.shape[1])
        flat[p, :k] = torch.arange(k, dtype=torch.uint8)
    lab[0] = flat.view(4, h, w)
    lab[-1, :, 0] = 0
    return lab


SHAPES = [(2, 64, 64), (3, 16, 96), (1, 17, 45), (2, 30, 33)]     # the last two: W % 32 != 0 and H % 16 != 0


@pytest.mark.parametrize("n,h,w", SHAPES)
def test_scene_expand_matches_load_segmentation(n, h, w):
    from mas_b200 import ops
    dev = _dev()
    lab = _labels(n, h, w, seed=h * w)
    ref = load_segmentation(lab)
    assert ref[:, 158].max() == 2 and (ref[-1, :, 0] == 0).all()
    labd = lab.to(dev)
    dense = ops.scene_expand(labd)
    assert dense.shape == (n, 159, h, w) and dense.is_contiguous()
    assert torch.equal(dense.cpu(), ref)
    for cp in (160, 192):
        padded = ops.scene_expand(labd, cp)
        assert padded.shape == (n, cp, h, w) and ops._cl_pitch(padded) == cp
        assert torch.equal(padded[:, :159].cpu(), ref) and not padded[:, 159:].any()
        assert torch.equal(padded, ops.pad_nhwc(ref.to(dev), cp))       # the operand the dense map's route builds
    empty = ops.scene_expand(torch.zeros_like(labd), 160)
    assert not empty.any()


def test_out_of_range_codes_expand_to_nothing_and_leave_the_loss():
    """Every byte above a plane's range (134..255, 21..255, 6..255, 3..255) sets no channel: written at pixels that are empty
    in the valid map, it changes neither the expansion nor the loss and gradient."""
    from mas_b200 import ops
    dev = _dev()
    n, h, w = 2, 16, 64
    lab = _labels(n, h, w, seed=7)
    lab[:, :, 4:12] = 0                                                   # rows left empty in every plane
    bad = lab.clone()
    for p, lo in enumerate((134, 21, 6, 3)):
        vals = torch.arange(lo, 256, dtype=torch.int32)
        bad[:, p, 4:12] = vals[torch.arange(n * 8 * w) % len(vals)].view(n, 8, w).to(torch.uint8)
    labd, badd = lab.to(dev), bad.to(dev)
    for cp in (None, 160):
        assert torch.equal(ops.scene_expand(badd, cp), ops.scene_expand(labd, cp))
    g = torch.Generator().manual_seed(3)
    base = torch.zeros(n, h, w, 160, device=dev)
    base[..., :159] = torch.randn(n, h, w, 159, generator=g).to(dev) * 2
    pw = torch.ones(159, device=dev)
    pw[153:158] = 20
    out = []
    for t in (labd, badd):
        logits = base.permute(0, 3, 1, 2)[:, :159].detach().requires_grad_(True)
        loss = ops.BCELogitsFn.apply(logits, t, pw)
        loss.backward()
        out.append((loss.detach(), logits.grad))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


@pytest.mark.parametrize("layout", ["padded_cl", "padded_cl_w48", "nchw"])
def test_bce_compact_target_bit_identical_to_dense(layout):
    """Loss and gradient with the compact target equal those with its dense expansion bit for bit: on the tiled fast path
    (padded channels-last logits, W % 32 == 0: mas_bce_scene_* against mas_bce_cl_*, the gradient in the padded buffer) and on
    the generic path (W % 32 != 0, or NCHW logits: the expanded target through mas_bce_logits)."""
    from mas_b200 import _lib as L, ops
    dev = _dev()
    n, h, w = 2, 16, 48 if layout == "padded_cl_w48" else 64
    lab = _labels(n, h, w, seed=11).to(dev)
    dense = load_segmentation(lab.cpu()).to(dev)
    g = torch.Generator().manual_seed(9)
    lo = torch.randn(n, 159, h, w, generator=g).to(dev) * 2
    pw = torch.ones(159, device=dev)
    pw[153:158] = 20
    out = []
    for t in (dense, lab):
        if layout == "nchw":
            logits = lo.clone().requires_grad_(True)
        else:
            base = torch.zeros(n, h, w, 160, device=dev)
            base[..., :159] = lo.permute(0, 2, 3, 1)
            logits = base.permute(0, 3, 1, 2)[:, :159].requires_grad_(True)
        seen = {}
        logits.register_hook(lambda gr: seen.update(base=getattr(gr, "_mas_pad_base", None)))
        L.profile_start()
        loss = ops.BCELogitsFn.apply(logits, t, pw)
        (loss * 0.7).backward()
        names = L.profile_report(lambda k: k.split("|")[0])
        out.append((loss.detach(), logits.grad, names, seen["base"]))
    (ld, gd, nd, _), (lc, gc, nc, pad_base) = out
    assert torch.equal(lc, ld) and torch.equal(gc, gd)
    if layout == "padded_cl":
        assert set(nd) == {"mas_bce_cl_forward", "mas_bce_cl_backward"}
        assert set(nc) == {"mas_bce_scene_forward", "mas_bce_scene_backward"}
        # the gradient is a view of the padded buffer conv_out's backward takes without a copy
        assert pad_base is not None and pad_base.shape == (n, 160, h, w) and not pad_base[:, 159:].any()
    else:
        assert "mas_bce_logits" in nd and "mas_bce_logits" in nc and "mas_scene_expand" in nc


def _model(dd, dev):
    from models import VQBASE
    torch.manual_seed(0)
    m = VQBASE(dd, 128, 64, 10, 100)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    m.quantize.q_counter = 10 ** 6
    return m.train().to(dev)


def _step(m, x, pw):
    """One training step; returns what it computed and the C-ABI entries it called (name -> calls)."""
    from mas_b200 import _lib as L, ops
    cb, seen = m.quantize, {}
    fwd = type(cb).forward

    def rec(z):
        zq, loss, idx = fwd(cb, z)
        seen["idx"] = idx
        return zq, loss, idx
    cb.forward = rec
    m.zero_grad(set_to_none=True)
    L.profile_start()
    dec, diff = m(x)
    loss = ops.BCELogitsFn.apply(dec, x, pw) + diff
    loss.backward()
    names = L.profile_report(lambda k: k.split("|")[0])
    del cb.forward
    out = {"dec": dec.detach().clone(), "diff": diff.detach().clone(), "idx": seen["idx"].clone(), "loss": loss.detach().clone()}
    out.update({"grad." + k: p.grad.clone() for k, p in m.named_parameters()})
    out.update({k: v.clone() for k, v in m.state_dict().items() if "running" in k})
    return out, {k: c for k, (c, _) in names.items()}


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        tol = ATOMIC_GRADS.get(k[5:]) if k.startswith("grad.") else None
        if tol is None:
            assert torch.equal(a[k], b[k]), k
        else:
            assert rel_err(a[k], b[k]) < tol, k


TC_DD = dict(z_channels=64, in_channels=159, out_channels=159, channels=[128, 128], num_res_blocks=1, resolution=64,
             attn_resolutions=[], dropout=0.0)              # the shape of test_vqseg_tensor_path_step_vs_oracle
GENERAL_DD = dict(z_channels=64, in_channels=159, out_channels=159, channels=[32, 32, 64], num_res_blocks=1, resolution=64,
                  attn_resolutions=[32], dropout=0.0)       # 32-channel conv_in: off the 128-wide output tile


@pytest.mark.parametrize("case", ["tensor", "general", "tf32"])
def test_compact_step_bit_identical_to_dense_step(case):
    """A segmentation-shaped VQBASE stepped with the compact map and with its dense expansion from identical weights and state:
    dec, diff, codebook indices, loss, every parameter gradient and the BatchNorm running statistics agree bit for bit.
    tensor: conv_in on the padded tensor route (the gradient reaches conv_out's backward in the loss kernel's padded buffer, no
    pad copy); general: a conv_in shape off the tensor tiles; tf32: TF32 operands, which send conv_in to the general route."""
    from mas_b200 import ops
    dev = _dev()
    dd = GENERAL_DD if case == "general" else TC_DD
    lab = _labels(2, 64, 64, seed=5).to(dev)
    seg = load_segmentation(lab.cpu()).to(dev)
    pw = torch.ones(159, device=dev)
    pw[153:158] = 20
    m = _model(dd, dev)
    state = copy.deepcopy(m.state_dict())
    old = ops.get_operand_format()
    ops.set_operand_format("tf32" if case == "tf32" else "f16")
    try:
        dense, nd = _step(m, seg, pw)
        m.load_state_dict(state)
        compact, nc = _step(m, lab, pw)
    finally:
        ops.set_operand_format(old)
    _assert_same(compact, dense)
    fast = "mas_bce_logits" not in nd                      # the loss on the tiled kernels (channels-last logits, W % 32 == 0)
    assert ("mas_bce_logits" in nc) == (not fast) and not any(k.startswith("mas_bce_cl") for k in nc)
    # expanded for conv_in's forward and its weight gradient (and for the generic loss kernel); never the dense pad copy
    assert nc.get("mas_scene_expand") == (2 if fast else 3) and "mas_nchw_to_nhwc_pad" not in nc
    if fast:
        assert nc.get("mas_bce_scene_forward") == 1 and nc.get("mas_bce_scene_backward") == 1
    if case == "tensor":
        assert fast and nd.get("mas_nchw_to_nhwc_pad") == 1   # the dense map's padded copy, in conv_in's forward only


def test_compact_input_lowers_peak_memory():
    """One training step at 128 x 128, batch 8, on a 128-wide trunk down to 16 x 16: the dense input and conv_in's padded copy
    of it (held from the forward to the last backward kernel) are gone; the labels are re-expanded only for conv_in's weight
    gradient at the end of the backward, after the peak."""
    from mas_b200 import ops
    dev = _dev()
    n, h, w = 8, 128, 128
    dd = dict(TC_DD, channels=[128, 128, 128, 128], resolution=128)
    lab = _labels(n, h, w, seed=1).to(dev)
    pw = torch.ones(159, device=dev)
    pw[153:158] = 20
    m = _model(dd, dev)
    state = copy.deepcopy(m.state_dict())
    peaks = {}
    for name in ("dense", "compact", "dense2", "compact2"):     # the first of each sizes the library's workspace
        m.load_state_dict(state)
        m.zero_grad(set_to_none=True)
        x = ops.scene_expand(lab) if name.startswith("dense") else lab
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        dec, diff = m(x)
        (ops.BCELogitsFn.apply(dec, x, pw) + diff).backward()
        del dec, diff
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated(dev) - base + (x.numel() * x.element_size())
        del x
    saving = peaks["dense2"] - peaks["compact2"]
    expected = n * h * w * (159 + 160) * 4
    print("peak allocated: dense %.1f MB, compact %.1f MB, saving %.1f MB (dense input + padded copy: %.1f MB)"
          % (peaks["dense2"] / 2 ** 20, peaks["compact2"] / 2 ** 20, saving / 2 ** 20, expected / 2 ** 20))
    # measured on an H100 80GB HBM3 (700 W): 159.0 of 159.5 MB; the re-expansion for conv_in's weight gradient is off the peak
    assert saving >= 0.99 * expected


def test_graphed_compact_step_matches_eager():
    """GraphedStep captures and replays a step fed a compact batch (its static input a uint8 clone): loss and gradients equal
    the eager compact step's bit for bit, for the example batch and a new one."""
    from mas_b200 import ops
    from mas_b200.graph import GraphedStep
    dev = _dev()
    pw = torch.ones(159, device=dev)
    pw[153:158] = 20
    xs = [_labels(2, 64, 64, seed=s).to(dev) for s in (21, 22)]

    def loss_fn(m, x):
        dec, diff = m(x)
        return ops.BCELogitsFn.apply(dec, x, pw) + diff
    me, mg = _model(TC_DD, dev), _model(TC_DD, dev)
    gs = GraphedStep(mg, loss_fn, xs[0], warmup=2)
    assert gs.static_in.dtype == torch.uint8
    try:
        for x in xs:
            me.zero_grad(set_to_none=True)
            le = loss_fn(me, x)
            le.backward()
            lg = gs(x)
            torch.cuda.synchronize()
            assert torch.equal(lg, le.detach())
            for (k, pe), (_, pg) in zip(me.named_parameters(), mg.named_parameters()):
                if k in ATOMIC_GRADS:
                    assert rel_err(pg.grad, pe.grad) < ATOMIC_GRADS[k], k
                else:
                    assert torch.equal(pg.grad, pe.grad), k
    finally:
        gs.close()
