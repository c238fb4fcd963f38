"""GPU parity tests (run on an H100): every call goes through the C-ABI (ctypes -> libmas_b200.so) and is
compared with (a) fixtures generated from the REAL reference and (b) the CPU oracle on seeded inputs.

Tolerances: VQ indices bit-exact (or fp64-tie-explained on the tie-heavy sets); floating point within 1e-3
relative (norm-wise) for the TF32 tensor path, 1e-4 for the fp32 SIMT path — north_star's stated bar is 1e-3.
"""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_err

pytestmark = pytest.mark.gpu

TOL_FWD = 1e-3
TOL_GRAD = 3e-3


def _dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _w(y):
    return torch.linspace(-1, 1, y.numel(), device=y.device).view(y.shape)


@pytest.fixture(params=["auto", "simt"])
def impl(request):
    from mas_b200 import _lib, ops
    ops.set_impl(_lib.IMPL_AUTO if request.param == "auto" else _lib.IMPL_SIMT)
    yield request.param
    ops.set_impl(_lib.IMPL_AUTO)


# ------------------------------------------------------------------------------------------------ codebook
def test_codebook_sets_vs_reference():
    from models.modules import Codebook
    from oracle import vqgan_oracle as O
    sets = _load("codebook_sets.pt")
    dev = _dev()
    for name, s in sets.items():
        cb = Codebook(256, 64, beta=0.25, init_steps=10, reservoir_size=100).to(dev).eval()
        with torch.no_grad():
            cb.embedding.weight.copy_(s["E"])
        z = s["z"].to(dev).requires_grad_(True)
        z_q, loss, idx = cb(z)
        assert idx.dtype == torch.int64 and idx.shape == s["idx"].shape
        bad = torch.nonzero(idx.cpu() != s["idx"]).flatten()
        if name in ("trained", "clustered", "duplicated"):
            # duplicated rows are bit-identical codes => exact ties => first index must win, bit-exactly
            assert bad.numel() == 0, (name, bad)
        else:
            zf = s["z"].permute(0, 2, 3, 1).reshape(-1, 64)
            gap, ulp = O.codebook_gap_fp64(zf, s["E"], idx.cpu(), s["idx"])
            assert bool((gap[bad] <= 4 * ulp[bad]).all()), name
        ok = (idx.cpu() == s["idx"])
        zq_rows = z_q.detach().cpu().permute(0, 2, 3, 1).reshape(-1, 64)
        ref_rows = s["z_q"].permute(0, 2, 3, 1).reshape(-1, 64)
        assert torch.allclose(zq_rows[ok], ref_rows[ok], atol=1e-6), name
        if bad.numel() == 0:
            assert abs(float(loss) - float(s["loss"])) <= 1e-5 * abs(float(s["loss"])) + 1e-9
            ((z_q * _w(z_q)).sum() + loss).backward()
            assert rel_err(z.grad, s["grad_z"]) < 1e-5, name
            assert rel_err(cb.embedding.weight.grad, s["grad_E"]) < 1e-4, name
            ent = cb.get_codebook_entry(idx, (3, 4, 4, 64))
            assert torch.equal(ent.cpu().contiguous(), s["entry"])


def test_codebook_full_size_properties():
    """K=8192, D=256, 8192 rows (BASELINE config 2/3): size-independent properties + sampled exact check."""
    from mas_b200 import ops
    from oracle import vqgan_oracle as O
    dev = _dev()
    g = torch.Generator().manual_seed(1234)
    z = torch.randn(32, 256, 16, 16, generator=g)
    E = torch.randn(8192, 256, generator=torch.Generator().manual_seed(4321))
    zd, Ed = z.to(dev), E.to(dev)
    zq, loss, idx = ops.VQFn.apply(zd, Ed, 0.25)
    idx_c = idx.cpu()
    assert int(idx_c.min()) >= 0 and int(idx_c.max()) < 8192
    # oracle on a sample of rows (numpy fp32 restatement) — bit-exact on margin-safe data
    zf = z.permute(0, 2, 3, 1).reshape(-1, 256)
    rows = torch.arange(0, 8192, 17)
    ref = torch.from_numpy(O.codebook_argmin_numpy(zf[rows].numpy(), E.numpy()))
    bad = torch.nonzero(idx_c[rows] != ref).flatten()
    if bad.numel():
        gap, ulp = O.codebook_gap_fp64(zf[rows], E, idx_c[rows], ref)
        assert bool((gap[bad] <= 4 * ulp[bad]).all())
    # optimality: no code is closer (fp64) than the chosen one by more than rounding noise
    d_best = ((zf.double() - E[idx_c].double()) ** 2).sum(1)
    probe = torch.randint(0, 8192, (8192, 64), generator=g)
    d_probe = ((zf.double()[:, None, :] - E[probe].double()) ** 2).sum(2)
    assert bool((d_best[:, None] <= d_probe + 1e-3).all())
    # idempotence: quantising the code vectors returns the same indices and zero loss
    e_img = E[idx_c].view(32, 16, 16, 256).permute(0, 3, 1, 2).contiguous().to(dev)
    zq2, loss2, idx2 = ops.VQFn.apply(e_img, Ed, 0.25)
    assert torch.equal(idx2.cpu(), idx_c) and float(loss2) < 1e-10
    # loss value
    ref_loss = 1.25 * float(d_best.sum() / zf.numel())
    assert abs(float(loss) - ref_loss) < 1e-5 * ref_loss
    # first-index tie-break at full size: duplicate the codebook's first half into its second half
    E2 = torch.cat([E[:4096], E[:4096]], 0).to(dev)
    _, _, idx3 = ops.VQFn.apply(zd, E2, 0.25)
    assert int(idx3.max()) < 4096


@pytest.fixture
def vq_paths():
    from mas_b200 import ops
    yield ops.vq_select_path
    ops.vq_select_path(True)


@pytest.mark.parametrize("R_img,K,D,kind", [(32, 8192, 256, "randn"), (5, 8192, 256, "randn"), (3, 1000, 64, "randn"),
                                            (2, 512, 128, "clustered"), (2, 512, 32, "duplicated"), (2, 300, 64, "fresh"),
                                            (4, 8192, 256, "scaled_small"), (4, 2048, 256, "scaled_big")])
def test_codebook_tensor_core_filter_is_bit_identical_to_exact_kernel(R_img, K, D, kind, vq_paths):
    """The tensor-core filter + exact re-evaluation path (csrc/vq_tc.cu, the default) against the all-pairs exact-fp32
    FFMA kernel on the same inputs: identical int64 indices, identical z_q and loss - on ordinary data, on clustered /
    duplicated / tie-heavy codebooks (every row undecided: the filter must hand them all to the exact kernel) and on
    operands far outside the fp16 range (the power-of-two operand scales)."""
    from mas_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(K + D + R_img)
    E = torch.randn(K, D, generator=g)
    z = torch.randn(R_img, D, 16, 16, generator=g)
    if kind == "clustered":
        j = torch.randint(0, K, (R_img * 256,), generator=g)
        z = (E[j] + 0.3 * torch.randn(R_img * 256, D, generator=g)).view(R_img, 16, 16, D).permute(0, 3, 1, 2).contiguous()
    elif kind == "duplicated":
        E = torch.cat([E[:K // 2], E[:K // 2]], 0)
    elif kind == "fresh":
        E = (torch.rand(K, D, generator=g) * 2 - 1) / K
    elif kind == "scaled_small":
        E, z = E * 3e-6, z * 3e-6
    elif kind == "scaled_big":
        E, z = E * 4e4, z * 4e4
    zd, Ed = z.to(dev), E.to(dev)
    vq_paths(False)
    zq0, loss0, idx0 = ops.VQFn.apply(zd, Ed, 0.25)
    vq_paths(True)
    zq1, loss1, idx1 = ops.VQFn.apply(zd, Ed, 0.25)
    assert torch.equal(idx0, idx1), (kind, int((idx0 != idx1).sum()))
    assert torch.equal(zq0, zq1) and float(loss0) == float(loss1)


def test_codebook_tensor_core_filter_accuracy_and_margin():
    """The error model of the filter (vq_margin in csrc/vq.cu): on BASELINE-sized random data the 2 x fp16 split distances
    agree with fp64 far inside the margin, and only a small fraction of rows needs the exact re-evaluation."""
    from mas_b200 import _lib as L, ops
    dev = _dev()
    g = torch.Generator().manual_seed(11)
    z = torch.randn(8, 256, 16, 16, generator=g)
    E = torch.randn(8192, 256, generator=g)
    zd, Ed = z.to(dev), E.to(dev)
    before = L.tc_launch_count()
    _, _, idx = ops.VQFn.apply(zd, Ed, 0.25)
    assert L.tc_launch_count() == before + 1            # the filter kernel ran
    zf = z.permute(0, 2, 3, 1).reshape(-1, 256).double()
    d = (zf * zf).sum(1, keepdim=True) + (E.double() ** 2).sum(1)[None] - 2 * zf @ E.double().t()
    top2 = d.topk(2, dim=1, largest=False).values
    assert torch.equal(idx.cpu(), d.argmin(1)) or bool(((top2[:, 1] - top2[:, 0])[idx.cpu() != d.argmin(1)] < 1e-3).all())
    # the margin the resolve kernel uses for this data (|z| ~ 16, |e|max ~ 18.5): a few percent of the rows fall inside it
    margin = 2.5e-4 * zf.norm(dim=1) * E.double().norm(dim=1).max()
    frac = float(((top2[:, 1] - top2[:, 0]) < margin).double().mean())
    assert frac < 0.25, frac


def test_codebook_ragged_rows():
    """R not a multiple of the 64-row tile, K not a multiple of the 128-code tile."""
    from mas_b200 import ops
    from oracle import vqgan_oracle as O
    dev = _dev()
    g = torch.Generator().manual_seed(3)
    z = torch.randn(1, 32, 7, 11, generator=g)
    E = torch.randn(200, 32, generator=g)
    zq, loss, idx = ops.VQFn.apply(z.to(dev), E.to(dev), 0.25)
    zq_o, loss_o, idx_o = O.codebook_forward(z, E)
    assert torch.equal(idx.cpu(), idx_o)
    assert torch.allclose(zq.cpu(), zq_o, atol=1e-6) and abs(float(loss) - float(loss_o)) < 1e-6


# ------------------------------------------------------------------------------------------------ blocks vs reference fixtures
def _run_block(name, b, impl):
    from models import modules as M
    dev = _dev()
    kind = name.split("_")[0]
    sd = b["state_dict"]
    if kind == "res":
        cin, cout = sd["conv1.weight"].shape[1], sd["conv1.weight"].shape[0]
        mod = M.ResnetBlock(in_channels=cin, out_channels=cout, dropout=0.0)
    elif kind == "attn":
        mod = M.AttnBlock(sd["q.weight"].shape[0])
    elif kind == "down":
        mod = M.Downsample(sd["conv.weight"].shape[0], True)
    else:
        mod = M.Upsample(sd["conv.weight"].shape[0], True)
    mod.load_state_dict(sd)
    mod.to(dev)
    x = b["x"].to(dev).requires_grad_(True)
    y = mod(x)
    assert y.shape == b["y"].shape
    tf, tg = (TOL_FWD, TOL_GRAD) if impl == "auto" else (1e-4, 5e-4)
    assert rel_err(y, b["y"]) < tf, name
    (y * _w(y)).sum().backward()
    assert rel_err(x.grad, b["grad_x"]) < tg, name
    for k, gv in b["grads"].items():
        if k == "k.bias":
            continue  # softmax over keys is invariant to a per-query constant: the true gradient is exactly zero
        p = dict(mod.named_parameters())[k]
        assert rel_err(p.grad, gv) < tg, (name, k)


def test_blocks_vs_reference(impl):
    blocks = _load("blocks.pt")
    for name, b in blocks.items():
        _run_block(name, b, impl)


# ------------------------------------------------------------------------------------------------ whole model, tiny
def test_vqbase_tiny_vs_reference(impl):
    from models import VQBASE
    g = _load("vqbase_tiny.pt")
    dev = _dev()
    m = VQBASE(g["ddconfig"], g["n_embed"], g["embed_dim"], 10, 100)
    m.load_state_dict(g["state_dict"])
    m.quantize.q_counter = 10 ** 6
    m.train().to(dev)
    x = g["x"].to(dev)
    dec, diff = m(x)
    assert dec.shape == g["dec"].shape and dec.is_contiguous() and diff.dim() == 0
    tf, tg = (TOL_FWD, TOL_GRAD) if impl == "auto" else (1e-4, 1e-3)
    assert rel_err(dec, g["dec"]) < tf
    assert abs(float(diff) - float(g["diff"])) < tf * abs(float(g["diff"]))
    loss = (x - dec).abs().mean() + diff
    loss.backward()
    for k, gv in g["grads"].items():
        p = dict(m.named_parameters())[k]
        assert p.grad is not None, k
        assert rel_err(p.grad, gv) < max(tg, 2e-3), k
    # running statistics of the (Sync)BatchNorm update like the reference's
    assert rel_err(m.quant_conv[1].running_mean, g["running_mean"]) < 1e-4
    assert rel_err(m.quant_conv[1].running_var, g["running_var"]) < 1e-4
    assert int(m.quant_conv[1].num_batches_tracked) == 1


def test_vqbase_tiny_modes():
    from models import VQBASE
    g = _load("vqbase_tiny.pt")
    mo = _load("vqbase_tiny_modes.pt")
    dev = _dev()
    m = VQBASE(g["ddconfig"], g["n_embed"], g["embed_dim"], 10, 100)
    m.load_state_dict(g["state_dict"])
    m.train().to(dev)
    dec, diff = m(g["x"].to(dev))            # q_counter=1 < q_init: warm-up bypass (modules.py:482-484)
    assert float(diff) == 0.0 and rel_err(dec, mo["dec_bypass"]) < TOL_FWD
    m.load_state_dict(g["state_dict"])
    m.eval()
    dec, diff = m(g["x"].to(dev))
    assert rel_err(dec, mo["dec_eval"]) < TOL_FWD
    assert abs(float(diff) - float(mo["diff_eval"])) < TOL_FWD * abs(float(mo["diff_eval"]))


def test_graphed_step_matches_eager():
    """mas_b200.graph.GraphedStep: the captured step replays to the same loss / gradients as eager launches, for changing
    inputs, and keeps the host-side codebook state (q_counter, reservoir) advancing like eager steps do."""
    from models import VQBASE
    from mas_b200.graph import GraphedStep
    g = _load("vqbase_tiny.pt")
    dev = _dev()

    def make():
        m = VQBASE(g["ddconfig"], g["n_embed"], g["embed_dim"], 10, 100)
        m.load_state_dict(g["state_dict"])
        m.quantize.q_counter = 10 ** 6
        return m.train().to(dev)

    def loss_fn(m, x):
        dec, diff = m(x)
        return (x - dec).abs().mean() + diff
    xs = [g["x"].to(dev), (g["x"] * 0.5 + 0.25).to(dev), g["x"].flip(0).contiguous().to(dev)]
    me, mg = make(), make()
    gs = GraphedStep(mg, loss_fn, xs[0], warmup=2)
    for _ in range(2):                       # the two eager warm-up steps inside GraphedStep advance BN statistics too
        me.zero_grad(set_to_none=True)
        loss_fn(me, xs[0]).backward()
    assert mg.quantize.q_counter == me.quantize.q_counter
    for x in xs:
        me.zero_grad(set_to_none=True)
        le = loss_fn(me, x)
        le.backward()
        lg = gs(x)
        assert abs(float(lg) - float(le)) <= 1e-6 * abs(float(le)) + 1e-9
        for (k, pe), (_, pg) in zip(me.named_parameters(), mg.named_parameters()):
            assert pg.grad is not None and rel_err(pg.grad, pe.grad) < 1e-6, k
        assert mg.quantize.q_counter == me.quantize.q_counter
        assert mg.quantize.reservoir.shape == me.quantize.reservoir.shape
    assert rel_err(mg.quant_conv[1].running_mean, me.quant_conv[1].running_mean) < 1e-6
    gs.close()
    mg.zero_grad(set_to_none=True)
    loss_fn(mg, xs[0]).backward()            # eager stepping works again after close()
    assert mg.decoder.model[-1].weight.grad is not None


def test_graphed_step_trains_with_optimizer_and_zero_grad():
    """optimizer.step() + zero_grad(set_to_none=True) between replays (the usual loop): the static gradient buffers are
    re-attached after every replay, so the graphed loop follows the eager one; a larger eager call while the graph is
    alive must not disturb it (the captured scratch buffer stays allocated)."""
    from models import VQBASE
    from mas_b200 import ops
    from mas_b200.graph import GraphedStep
    g = _load("vqbase_tiny.pt")
    dev = _dev()

    def make():
        m = VQBASE(g["ddconfig"], g["n_embed"], g["embed_dim"], 10, 100)
        m.load_state_dict(g["state_dict"])
        m.quantize.q_counter = 10 ** 6
        return m.train().to(dev)

    def loss_fn(m, x):
        dec, diff = m(x)
        return (x - dec).abs().mean() + diff
    x = g["x"].to(dev)
    me, mg = make(), make()
    oe = torch.optim.Adam(me.parameters(), lr=1e-3, betas=(0.5, 0.9))
    og = torch.optim.Adam(mg.parameters(), lr=1e-3, betas=(0.5, 0.9))
    gs = GraphedStep(mg, loss_fn, x, warmup=2)
    for _ in range(2):
        me.zero_grad(set_to_none=True)
        loss_fn(me, x).backward()
    big = torch.randn(64, 64, 64, 64, device=dev).contiguous(memory_format=torch.channels_last)
    losses_e, losses_g = [], []
    for step in range(4):
        oe.zero_grad()                       # set_to_none=True is the default
        le = loss_fn(me, x)
        le.backward()
        oe.step()
        og.zero_grad()
        lg = gs(x)
        assert all(p.grad is not None for p in mg.parameters())
        og.step()
        losses_e.append(float(le)); losses_g.append(float(lg))
        if step == 1:
            ops.gn_stats(big)                # an eager call needing far more scratch than the captured step did
    for a, b in zip(losses_e, losses_g):
        assert abs(a - b) <= 2e-5 * abs(a), (losses_e, losses_g)
    assert losses_e[-1] != losses_e[0]       # the parameters did move
    gs.close()


def test_reentrant_backward_last_layer():
    """loss_img.py:57-60 runs autograd.grad(..., last_layer.weight, retain_graph=True) twice before backward()."""
    from models import VQBASE
    g = _load("vqbase_tiny.pt")
    dev = _dev()
    m = VQBASE(g["ddconfig"], g["n_embed"], g["embed_dim"], 10, 100)
    m.load_state_dict(g["state_dict"])
    m.quantize.q_counter = 10 ** 6
    m.train().to(dev)
    x = g["x"].to(dev)
    dec, diff = m(x)
    last = m.decoder.model[-1].weight
    l1 = (x - dec).abs().mean()
    g1 = torch.autograd.grad(l1, last, retain_graph=True)[0]
    g2 = torch.autograd.grad(dec.square().mean(), last, retain_graph=True)[0]
    (l1 + diff).backward()
    assert rel_err(g1, g["grads"]["decoder.model.%d.weight" % (len(m.decoder.model) - 1)]) < 5e-3
    assert torch.isfinite(g2).all() and last.grad is not None


# ------------------------------------------------------------------------------------------------ tensor-path blocks vs reference
def _sampled_err(t, fx, norm):
    """Fixture entries stored as (strided sample, stride): error on that sample relative to the tensor's norm."""
    smp, stride = fx
    got = t.detach().reshape(-1)[::stride].double().cpu()
    scale = norm * (smp.numel() / t.numel()) ** 0.5
    return float((got - smp.double()).norm() / max(scale, 1e-30))


TC_BLOCKS = ["res_128_128", "res_128_256", "res_512_512", "attn_512", "attn_res_512", "res_res_attn_512", "up_128", "down_128",
             "up_512"]


@pytest.mark.parametrize("name", TC_BLOCKS)
def test_tensor_path_blocks_vs_reference(name):
    """Blocks at widths / extents the tensor-core kernels take (fused GroupNorm prologue, statistics epilogue and its
    take_stats hand-off between modules, AttnBlock at C=512 / HW=256, Up/Downsample on the tensor kernels) against
    outputs and gradients of the REAL reference (tests/golden/blocks_tc.pt; weights / inputs regenerated from seeds)."""
    from mas_b200 import _lib as L
    from models import modules as M
    from oracle.seeded import assert_same_fill, fill_seeded, seeded_input
    from test_oracle import build_tc_block
    dev = _dev()
    b = _load("blocks_tc.pt")[name]
    mod = build_tc_block(name, M)
    assert_same_fill(fill_seeded(mod, b["seed_w"]), b["param_checks"])
    mod.to(dev)
    x = seeded_input(b["shape"], b["seed_x"], 1.5, 0.3).to(dev).requires_grad_(True)
    before = L.launch_count()
    y = mod(x)
    assert _sampled_err(y, b["y"], b["y_norm"]) < TOL_FWD, name
    (y * _w(y)).sum().backward()
    assert L.launch_count() > before
    assert _sampled_err(x.grad, b["grad_x"], b["grad_x_norm"]) < TOL_GRAD, name
    named = dict(mod.named_parameters())
    for k, gv in b["grads"].items():
        if k.endswith("k.bias"):
            continue  # softmax over keys is invariant to a per-query constant: the true gradient is exactly zero
        g = named[k].grad
        e = _sampled_err(g, gv, b["grad_norms"][k]) if isinstance(gv, tuple) else rel_err(g, gv)
        assert e < TOL_GRAD, (name, k, e)


def test_tensor_path_blocks_use_tensor_kernels():
    """The fixtures above are only meaningful if those shapes are tensor-path eligible."""
    from mas_b200 import _lib as L, ops
    dev = _dev()
    for (n, c, h, w), cout, mode in [((2, 128, 32, 32), 128, L.CONV_S1), ((2, 128, 32, 32), 256, L.CONV_S1),
                                     ((2, 512, 16, 16), 512, L.CONV_S1), ((2, 128, 16, 16), 128, L.CONV_UP)]:
        x = torch.empty((n, c, h, w), device=dev).contiguous(memory_format=torch.channels_last)
        assert ops.conv_tc_eligible(x, cout, mode), (c, h, cout)


# ------------------------------------------------------------------------------------------------ img_config widths
def _img_model(g, dev):
    from models import VQBASE
    torch.manual_seed(0)
    m = VQBASE(g["ddconfig"], 8192, 256, 3000, 12500)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    m.quantize.q_counter = 10 ** 6
    return m.train().to(dev)


def _explain_index_mismatches(z_ours, E, idx_ours, idx_ref):
    """Rows whose code differs from the reference's: ours must be the fp64 arg-min of OUR latent (up to fp32 rounding of
    the distance), i.e. the encoder-side TF32 drift moved the latent across a Voronoi boundary, not a VQ error.
    Returns the number of mismatching rows."""
    bad = torch.nonzero(idx_ours != idx_ref).flatten()
    if bad.numel():
        zb = z_ours[bad].double()
        d = (zb * zb).sum(1, keepdim=True) + (E.double() ** 2).sum(1)[None] - 2 * zb @ E.double().t()
        best = d.min(1).values
        mine = d.gather(1, idx_ours[bad][:, None]).squeeze(1)
        ulp = torch.finfo(torch.float32).eps * d.abs().max(1).values
        assert bool((mine - best <= 4 * ulp).all()), (bad, mine - best)
    return int(bad.numel())


def _forced_indices(m, idx_ref):
    """Pin the quantiser's decision to the reference's indices (product kernels: mas_vq_forward_given + mas_vq_backward),
    so decoder outputs and ALL gradients are comparable element for element even when TF32 drift flips a few codes."""
    from mas_b200 import ops
    cb = m.quantize

    def fwd(z):
        zq, loss = ops.VQGivenFn.apply(z, cb.embedding.weight, cb.beta, idx_ref.to(z.device))
        return zq, loss, idx_ref.to(z.device)
    cb.forward = fwd


def test_vqbase_img_config_64px_vs_reference():
    """The 95M-parameter img_config model with seeded init (bit-identical to the reference's init, see
    tests/test_abi.py) on 2x3x64x64: outputs, indices and gradients against the reference fixture."""
    g = _load("vqbase_img_64.pt")
    dev = _dev()
    m = _img_model(g, dev)
    x = g["x"].to(dev)
    h = {}
    hk = m.quant_conv.register_forward_hook(lambda _m, _i, o: h.__setitem__("q", o.detach()))
    hi = m.quantize.register_forward_hook(lambda _m, _i, o: h.__setitem__("idx", o[2].detach()))
    m(x)
    hk.remove(); hi.remove()
    e_q = rel_err(h["q"], g["quant_in"])
    assert e_q < 3e-3, e_q          # end-to-end TF32 drift through 23 layers (reported, SURVEY.md 7.3 #3)
    zf = h["q"].permute(0, 2, 3, 1).reshape(-1, 256).cpu()
    mism = _explain_index_mismatches(zf, m.quantize.embedding.weight.detach().cpu(), h["idx"].cpu(), g["idx"])
    assert mism <= 2, mism
    # second pass with the decision pinned to the reference's codes: decoder output and every gradient, unconditionally
    m.quant_conv[1].reset_running_stats()
    _forced_indices(m, g["idx"])
    m.zero_grad(set_to_none=True)
    dec, diff = m(x)
    assert rel_err(dec, g["dec"]) < 5e-3
    assert abs(float(diff) - float(g["diff"])) < 5e-3 * abs(float(g["diff"]))
    ((x - dec).abs().mean() + diff).backward()
    named = dict(m.named_parameters())
    for k, gv in g["grads_small"].items():
        assert rel_err(named[k].grad, gv) < 2e-2, k
    # gradient norms of all 348 tensors; tensors whose true gradient is ~0 (biases feeding a GroupNorm with
    # one channel per group, key biases of the attention) are compared on an absolute scale
    worst = max(((abs(float(named[k].grad.double().norm()) - v) / max(v, 1e-4 * named[k].numel() ** 0.5)), k)
                for k, v in g["grad_norms"].items())
    assert worst[0] < 5e-2, worst


def test_vqbase_img_config_256px_vs_reference():
    """BASELINE's own resolution: the img_config model on 2x3x256x256 (every production kernel at its production shape:
    128-channel 256x256 convolutions, HW=256 AttnBlocks with the statistics epilogue, space-to-depth Downsample, fused
    Upsample) against the REAL reference's forward and backward (tests/golden/vqbase_img_256.pt)."""
    g = _load("vqbase_img_256.pt")
    dev = _dev()
    m = _img_model(g, dev)
    x = torch.rand(g["x_shape"], generator=torch.Generator().manual_seed(g["x_seed"]))
    assert abs(float(x.double().sum()) - g["x_sum"]) < 1e-6
    x = x.to(dev)
    h = {}
    hk = m.quant_conv.register_forward_hook(lambda _m, _i, o: h.__setitem__("q", o.detach()))
    hi = m.quantize.register_forward_hook(lambda _m, _i, o: h.__setitem__("idx", o[2].detach()))
    m(x)
    hk.remove(); hi.remove()
    e_q = rel_err(h["q"], g["quant_in"])
    assert e_q < 3e-3, e_q
    zf = h["q"].permute(0, 2, 3, 1).reshape(-1, 256).cpu()
    mism = _explain_index_mismatches(zf, m.quantize.embedding.weight.detach().cpu(), h["idx"].cpu(), g["idx"])
    assert mism <= 26, mism         # 5 % of 512 rows: each one verified above to be a boundary crossing of OUR latent
    _forced_indices(m, g["idx"])
    m.zero_grad(set_to_none=True)
    def keep(_m, _i, o):
        o.retain_grad()
        h["qg"] = o
    hq = m.quant_conv.register_forward_hook(keep)
    dec, diff = m(x)
    hq.remove()
    assert _sampled_err(dec, g["dec_sample"], g["dec_norm"]) < 5e-3
    assert abs(float(diff) - float(g["diff"])) < 5e-3 * abs(float(g["diff"]))
    loss = (x - dec).abs().mean() + diff
    assert abs(float(loss) - float(g["loss"])) < 2e-3 * abs(float(g["loss"]))
    loss.backward()
    assert _sampled_err(h["qg"].grad, g["g_quant_in"], g["g_quant_in_norm"]) < 2e-2
    named = dict(m.named_parameters())
    worst_n = max(((abs(float(named[k].grad.double().norm()) - v) / max(v, 1e-4 * named[k].numel() ** 0.5)), k)
                  for k, v in g["grad_norms"].items())
    assert worst_n[0] < 5e-2, worst_n
    errs = sorted(((_sampled_err(named[k].grad, g["grad_samples"][k], max(v, 1e-4 * named[k].numel() ** 0.5)), k)
                   for k, v in g["grad_norms"].items()), reverse=True)
    assert errs[0][0] < 5e-2, errs[:5]
    assert errs[len(errs) // 2][0] < 1e-2, errs[len(errs) // 2]     # median over the 348 tensors


# ------------------------------------------------------------------------------------------------ op-level vs oracle
@pytest.mark.parametrize("c,hw", [(32, 8), (64, 12), (128, 16), (256, 8), (512, 4)])
def test_groupnorm_swish_vs_oracle(c, hw):
    from models import modules as M
    from oracle import vqgan_oracle as O
    dev = _dev()
    g = torch.Generator().manual_seed(c + hw)
    x = (torch.randn(3, c, hw, hw, generator=g) * 2 + 0.5)
    gn = M.Normalize(c)
    with torch.no_grad():
        gn.weight.copy_(torch.randn(c, generator=g))
        gn.bias.copy_(torch.randn(c, generator=g))
    sd = {"n.weight": gn.weight.detach().clone().requires_grad_(True), "n.bias": gn.bias.detach().clone().requires_grad_(True)}
    xo = x.clone().requires_grad_(True)
    yo = O.swish(O.normalize(xo, sd, "n"))
    (yo * _w(yo)).sum().backward()
    gn.to(dev)
    xd = x.to(dev).requires_grad_(True)
    y = gn(xd, silu=True)
    (y * _w(y)).sum().backward()
    assert rel_err(y, yo) < 1e-5
    assert rel_err(xd.grad, xo.grad) < 1e-4
    assert rel_err(gn.weight.grad, sd["n.weight"].grad) < 1e-4 and rel_err(gn.bias.grad, sd["n.bias"].grad) < 1e-4


@pytest.mark.parametrize("shape,cl", [((3, 32, 9, 7), False), ((2, 64, 8, 8), True), ((5, 7), False)])
def test_standalone_swish_vs_torch(shape, cl):
    """nonlinearity / Swish modules on their own (modules.py:35-37,194-196): mas_silu_forward / mas_silu_backward."""
    from models import modules as M
    dev = _dev()
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(*shape, generator=g) * 3
    xo = x.clone().requires_grad_(True)
    yo = xo * torch.sigmoid(xo)
    (yo * _w(yo)).sum().backward()
    xd = x.to(dev)
    if cl:
        xd = xd.contiguous(memory_format=torch.channels_last)
    xd = xd.requires_grad_(True)
    y = M.Swish()(xd) if len(shape) == 4 else M.nonlinearity(xd)
    (y * _w(yo).to(dev)).sum().backward()
    assert rel_err(y, yo) < 1e-6 and rel_err(xd.grad, xo.grad) < 1e-6


@pytest.mark.parametrize("cin,cout,h,w,mode", [(3, 32, 9, 7, "s1"), (32, 3, 8, 8, "s1"), (64, 64, 16, 16, "s1"),
                                               (128, 128, 32, 32, "s1"), (128, 256, 8, 24, "s1"), (256, 128, 16, 16, "s1"),
                                               (512, 512, 16, 16, "s1"), (64, 64, 16, 16, "s2"), (128, 128, 32, 32, "s2"),
                                               (64, 64, 8, 8, "up"), (128, 128, 16, 16, "up"), (159, 128, 8, 8, "s1"),
                                               # register-tiled edge kernels (wide side % 128 == 0), ragged strips / tiles
                                               (3, 128, 19, 37, "s1"), (3, 256, 9, 7, "s1"), (128, 3, 21, 35, "s1"),
                                               (256, 3, 8, 8, "s1"), (3, 128, 32, 64, "s1"), (128, 3, 32, 64, "s1")])
def test_conv3x3_family_vs_oracle(cin, cout, h, w, mode, impl):
    import torch.nn.functional as F
    from mas_b200 import _lib as L, ops
    dev = _dev()
    g = torch.Generator().manual_seed(cin * 7 + cout + h)
    x = torch.randn(2, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 3, 3, generator=g) / (3 * cin ** 0.5)
    b = torch.randn(cout, generator=g)
    xo, wo, bo = x.clone().requires_grad_(True), wt.clone().requires_grad_(True), b.clone().requires_grad_(True)
    if mode == "s1":
        yo = F.conv2d(xo, wo, bo, padding=1)
        md = L.CONV_S1
    elif mode == "s2":
        yo = F.conv2d(F.pad(xo, (0, 1, 0, 1)), wo, bo, stride=2)
        md = L.CONV_S2
    else:
        yo = F.conv2d(F.interpolate(xo, scale_factor=2.0, mode="nearest"), wo, bo, padding=1)
        md = L.CONV_UP
    (yo * _w(yo)).sum().backward()
    xd = x.to(dev)
    if (cin + cout) % 2 == 0:      # channels-last input: tensor-core eligible when the shape allows
        xd = xd.contiguous(memory_format=torch.channels_last)
    xd, wd, bd = xd.requires_grad_(True), wt.to(dev).requires_grad_(True), b.to(dev).requires_grad_(True)
    y = ops.Conv3x3Fn.apply(xd, wd, bd, None, md, False)      # NCHW-strided inputs exercise the generic-stride path
    (y * _w(y)).sum().backward()
    tf, tg = (TOL_FWD, TOL_GRAD) if impl == "auto" else (2e-5, 1e-4)
    assert rel_err(y, yo) < tf
    assert rel_err(xd.grad, xo.grad) < tg
    assert rel_err(wd.grad, wo.grad) < tg
    assert rel_err(bd.grad, bo.grad) < 1e-4


@pytest.mark.parametrize("M,N,K,batch,ta,tb", [(64, 64, 64, 1, 0, 1), (256, 256, 512, 4, 0, 1), (256, 512, 256, 3, 0, 0),
                                               (256, 512, 256, 2, 1, 0), (100, 36, 52, 2, 1, 1), (8192, 512, 512, 1, 0, 1),
                                               (77, 130, 19, 1, 0, 0)])
def test_gemm_vs_oracle(M, N, K, batch, ta, tb, impl):
    from mas_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(batch, *((K, M) if ta else (M, K)), generator=g)
    B = torch.randn(batch, *((N, K) if tb else (K, N)), generator=g)
    bias = torch.randn(N, generator=g)
    res = torch.randn(batch, M, N, generator=g)
    ref = 0.5 * torch.bmm(A.transpose(1, 2) if ta else A, B.transpose(1, 2) if tb else B) + bias + res
    Ad, Bd, Cd = A.to(dev), B.to(dev), torch.empty(batch, M, N, device=dev)
    ops.gemm(Ad, Bd, Cd, M, N, K, batch=batch, lda=A.shape[2], ldb=B.shape[2], ldc=N, sa=A.shape[1] * A.shape[2],
             sb=B.shape[1] * B.shape[2], sc=M * N, ta=bool(ta), tb=bool(tb), alpha=0.5, bias=bias.to(dev), residual=res.to(dev))
    assert rel_err(Cd, ref) < (TOL_FWD if impl == "auto" else 2e-5)


@pytest.mark.parametrize("cin,cout,hw,n", [(512, 512, 16, 4), (256, 128, 32, 2), (128, 256, 16, 3), (64, 32, 8, 2), (256, 256, 16, 32)])
def test_conv1x1_vs_oracle(cin, cout, hw, n, impl):
    import torch.nn.functional as F
    from mas_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(cin + cout)
    x = torch.randn(n, cin, hw, hw, generator=g)
    wt = torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5
    b = torch.randn(cout, generator=g)
    xo, wo, bo = x.clone().requires_grad_(True), wt.clone().requires_grad_(True), b.clone().requires_grad_(True)
    yo = F.conv2d(xo, wo, bo)
    (yo * _w(yo)).sum().backward()
    xd, wd, bd = x.to(dev).requires_grad_(True), wt.to(dev).requires_grad_(True), b.to(dev).requires_grad_(True)
    y = ops.Conv1x1Fn.apply(xd, wd, bd)
    (y * _w(y)).sum().backward()
    tf, tg = (TOL_FWD, TOL_GRAD) if impl == "auto" else (2e-5, 1e-4)
    assert rel_err(y, yo) < tf
    assert rel_err(xd.grad, xo.grad) < tg
    assert rel_err(wd.grad, wo.grad) < tg and rel_err(bd.grad, bo.grad) < 1e-4


def test_tensor_path_full_resolution_linearity():
    """BASELINE-size conv (128->128 @256x256, batch 4 here) on the tensor-core kernel: compared with the exact-fp32 SIMT
    kernel on the same inputs, plus linearity conv(a*x1 + x2) = a*conv(x1) + conv(x2) (bias-free)."""
    from mas_b200 import _lib as L, ops
    dev = _dev()
    g = torch.Generator().manual_seed(99)
    x1 = torch.randn(4, 128, 256, 256, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    x2 = torch.randn(4, 128, 256, 256, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(128, 128, 3, 3, generator=g) * 0.03).to(dev)
    b = torch.randn(128, generator=g).to(dev)
    ops.set_impl(L.IMPL_TC)
    try:
        y_tc = ops.conv3x3_raw(x1, w, b, x2, L.CONV_S1)
        l1 = ops.conv3x3_raw(2.0 * x1 + x2, w, None, None, L.CONV_S1)
        l2 = 2.0 * ops.conv3x3_raw(x1, w, None, None, L.CONV_S1) + ops.conv3x3_raw(x2, w, None, None, L.CONV_S1)
        d_tc = ops.conv3x3_dgrad_raw(x1, w, L.CONV_S1)
        gw_tc, gb_tc = ops.conv3x3_wgrad_raw(x1, x2, 128, 128, L.CONV_S1)
    finally:
        ops.set_impl(L.IMPL_SIMT)
    y_ref = ops.conv3x3_raw(x1, w, b, x2, L.CONV_S1)
    d_ref = ops.conv3x3_dgrad_raw(x1, w, L.CONV_S1)
    gw_ref, gb_ref = ops.conv3x3_wgrad_raw(x1, x2, 128, 128, L.CONV_S1)
    ops.set_impl(L.IMPL_AUTO)
    assert rel_err(y_tc, y_ref) < TOL_FWD
    assert rel_err(d_tc, d_ref) < TOL_FWD
    assert rel_err(gw_tc, gw_ref) < TOL_FWD and rel_err(gb_tc, gb_ref) < 1e-4
    assert rel_err(l1, l2) < TOL_FWD


def test_fused_groupnorm_prologue_and_stats_epilogue():
    """The tensor-path fusions against the unfused kernels: conv(act(GN(x))) with the prologue table == conv of the
    materialised activation; epilogue statistics == mas_gn_stats of the stored output; same for the weight gradient."""
    from mas_b200 import _lib as L, ops
    dev = _dev()
    g = torch.Generator().manual_seed(21)
    x = (torch.randn(3, 128, 32, 32, generator=g) * 1.5 + 0.3).to(dev).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(3, 256, 32, 32, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(256, 128, 3, 3, generator=g) * 0.03).to(dev)
    b = torch.randn(256, generator=g).to(dev)
    gamma, beta = torch.randn(128, generator=g).to(dev), torch.randn(128, generator=g).to(dev)
    m, r = ops.gn_stats(x)
    a = ops.gn_apply(x, m, r, gamma, beta, True)
    tab = ops.gn_table(m, r, gamma, beta, 3, 128)
    y_ref = ops.conv3x3_raw(a, w, b, None, L.CONV_S1)
    y, st = ops.conv3x3_raw(x, w, b, None, L.CONV_S1, table=tab, want_stats=True)
    assert rel_err(y, y_ref) < 1e-5          # same kernel, same operands up to the activation's rounding
    m2, r2 = ops.gn_stats(y)
    assert st is not None and rel_err(st[0], m2) < 1e-5 and rel_err(st[1], r2) < 1e-5
    gw_ref, gb_ref = ops.conv3x3_wgrad_raw(a, dy, 256, 128, L.CONV_S1)
    gw, gb = ops.conv3x3_wgrad_raw(x, dy, 256, 128, L.CONV_S1, table=tab)
    assert rel_err(gw, gw_ref) < 1e-5 and rel_err(gb, gb_ref) < 1e-6


def test_seg_loss_vs_reference():
    from mas_b200 import ops
    g = _load("seg_loss.pt")
    dev = _dev()
    pred = g["pred"].to(dev).requires_grad_(True)
    pw = torch.ones(159, device=dev)
    pw[153:158] = 20
    loss = ops.BCELogitsFn.apply(pred, g["target"].to(dev), pw) + g["qloss"].to(dev)
    assert abs(float(loss) - float(g["loss"])) < 1e-5
    loss.backward()
    assert rel_err(pred.grad, g["grad"]) < 1e-5


@pytest.mark.parametrize("cin,cout,h,w", [(159, 128, 32, 32), (128, 159, 32, 64), (100, 256, 16, 16), (64, 200, 16, 24)])
def test_conv3x3_padded_channel_counts_vs_oracle(cin, cout, h, w):
    """Channel counts off the tensor tiles (VQ-SEG's 159-channel input / output layers): zero-padded to the 16-wide K step /
    the 128-wide output tile inside Conv3x3Fn, run on the fp16 tensor-core kernels; the 159-wide output comes back as a
    channels-last view. Forward and all gradients against F.conv2d (fp32, CPU)."""
    import torch.nn.functional as F
    from mas_b200 import _lib as L, ops
    dev = _dev()
    g = torch.Generator().manual_seed(cin + cout)
    x = torch.randn(2, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 3, 3, generator=g) / (3 * cin ** 0.5)
    b = torch.randn(cout, generator=g)
    xo, wo, bo = x.clone().requires_grad_(True), wt.clone().requires_grad_(True), b.clone().requires_grad_(True)
    yo = F.conv2d(xo, wo, bo, padding=1)
    (yo * _w(yo)).sum().backward()
    xd = x.to(dev)
    if cin % 16 == 0:
        xd = xd.contiguous(memory_format=torch.channels_last)
    xd, wd, bd = xd.requires_grad_(True), wt.to(dev).requires_grad_(True), b.to(dev).requires_grad_(True)
    before = L.tc_launch_count()
    y = ops.Conv3x3Fn.apply(xd, wd, bd, None, L.CONV_S1, False)
    assert L.tc_launch_count() > before and y.shape == yo.shape
    (y * _w(yo).to(dev)).sum().backward()
    # (the gradients join the forward on the tensor cores when their own extents fit: 160 padded input channels do, 112 do not)
    assert rel_err(y, yo) < TOL_FWD
    assert rel_err(xd.grad, xo.grad) < TOL_GRAD
    assert rel_err(wd.grad, wo.grad) < TOL_GRAD
    assert rel_err(bd.grad, bo.grad) < 1e-4


def test_seg_loss_fast_path_and_padded_gradient():
    """Weighted BCE on the VQ-SEG step's layouts: channels-last logits with channel pitch 160 (the view the padded decoder
    head returns) x NCHW target -> loss and gradient against torch's own binary_cross_entropy_with_logits on the CPU; the
    gradient comes back as a view of a padded channels-last tensor (pad channel exactly zero), scaled by the upstream gradient."""
    import torch.nn.functional as F
    from mas_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(9)
    n, c, h, w = 2, 159, 16, 64
    lo = torch.randn(n, c, h, w, generator=g) * 2
    tg = (torch.rand(n, c, h, w, generator=g) > 0.9).float()
    pw = torch.ones(c)
    pw[153:158] = 20
    lr = lo.clone().requires_grad_(True)
    ref = F.binary_cross_entropy_with_logits(lr.permute(0, 2, 3, 1), tg.permute(0, 2, 3, 1), pos_weight=pw)
    (ref * 0.7).backward()
    base = torch.zeros(n, h, w, 160, device=dev)
    base[..., :c] = lo.permute(0, 2, 3, 1).to(dev)
    logits = base.permute(0, 3, 1, 2)[:, :c].requires_grad_(True)
    loss = ops.BCELogitsFn.apply(logits, tg.to(dev), pw.to(dev))
    assert abs(float(loss) - float(ref)) < 1e-5 * abs(float(ref))
    (loss * 0.7).backward()
    assert rel_err(logits.grad, lr.grad) < 1e-5


def test_vqseg_tensor_path_step_vs_oracle():
    """Segmentation-shaped VQBASE whose 159-channel edge layers take the padded tensor-core paths (128-wide trunk, 64x64
    one-hot-like maps): forward, weighted-BCE + codebook loss and every gradient against the CPU oracle."""
    from mas_b200 import _lib as L, ops
    from models import VQBASE
    from oracle import vqgan_oracle as O
    dev = _dev()
    dd = dict(z_channels=64, in_channels=159, out_channels=159, channels=[128, 128], num_res_blocks=1, resolution=64,
              attn_resolutions=[], dropout=0.0)
    torch.manual_seed(0)
    m = VQBASE(dd, 128, 64, 10, 100)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    m.quantize.q_counter = 10 ** 6
    m.train()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    params = {k: v.requires_grad_(True) for k, v in sd.items() if v.is_floating_point() and "running" not in k}
    sd.update(params)
    seg = (torch.rand(2, 159, 64, 64, generator=torch.Generator().manual_seed(5)) > 0.9).float()
    dec_o, diff_o, idx_o = O.vqbase_forward(sd, dd, seg)
    lo = O.bce_loss_with_quant(diff_o, seg, dec_o)
    lo.backward()
    m.to(dev)
    pw = torch.ones(159, device=dev)
    pw[153:158] = 20
    segd = seg.to(dev)
    before = L.tc_launch_count()
    _forced_indices(m, idx_o)          # the quantiser's decision pinned to the oracle's (the VQ kernels have their own tests)
    dec, diff = m(segd)
    assert dec.shape == (2, 159, 64, 64) and ops._cl_pitch(dec) == 160
    loss = ops.BCELogitsFn.apply(dec, segd, pw) + diff
    loss.backward()
    assert L.tc_launch_count() - before >= 20
    assert rel_err(dec, dec_o) < 2e-3
    assert abs(float(loss) - float(lo)) < 2e-3 * abs(float(lo))
    named = dict(m.named_parameters())
    for k, pr in params.items():
        assert rel_err(named[k].grad, pr.grad) < 1e-2, k


def test_native_library_is_the_path_that_ran():
    from mas_b200 import _lib
    assert _lib.launch_count() > 0
    assert os.path.exists(_lib.LIB_PATH)


def test_vqseg_plumbing_three_adam_steps_vs_oracle():
    """BASELINE configs[0] (the reference's CPU plumbing case, here on the GPU): seg-config-shaped VQBASE (159 input /
    output channels, 64x64, batch 2), weighted BCE + codebook loss (losses/loss_seg.py:15-22), Adam lr 4.5e-6 betas
    (0.5,0.9), three steps — loss trajectory against the CPU oracle driven by the same weights."""
    from mas_b200 import ops
    from models import VQBASE
    from oracle import vqgan_oracle as O
    dev = _dev()
    dd = dict(z_channels=64, in_channels=159, out_channels=159, channels=[32, 32, 64], num_res_blocks=1, resolution=64,
              attn_resolutions=[32], dropout=0.0)
    torch.manual_seed(0)
    m = VQBASE(dd, 128, 64, 10, 100)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    m.quantize.q_counter = 10 ** 6
    m.train()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    params = {k: v.requires_grad_(True) for k, v in sd.items() if v.is_floating_point() and "running" not in k}
    sd.update(params)
    seg = (torch.rand(2, 159, 64, 64, generator=torch.Generator().manual_seed(5)) > 0.9).float()
    # Adam: lr and betas of conf/seg_config.yaml:34-39 (lr raised so that three steps move the loss measurably)
    opt_o = torch.optim.Adam(list(params.values()), lr=1e-3, betas=(0.5, 0.9))
    m.to(dev)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.5, 0.9))
    pw = torch.ones(159, device=dev)
    pw[153:158] = 20
    segd = seg.to(dev)
    for step in range(3):
        opt_o.zero_grad()
        dec_o, diff_o, _ = O.vqbase_forward(sd, dd, seg)
        lo = O.bce_loss_with_quant(diff_o, seg, dec_o)
        lo.backward()
        opt_o.step()
        opt.zero_grad()
        dec, diff = m(segd)
        loss = ops.BCELogitsFn.apply(dec, segd, pw) + diff
        loss.backward()
        opt.step()
        assert abs(float(loss) - float(lo)) < 2e-3 * abs(float(lo)), (step, float(loss), float(lo))


def test_kmeans_update_step_vs_torch():
    """mas_kmeans_update (segmented mean, empty clusters keep their centre, centre shift) against index_add_ in torch."""
    from mas_b200 import _lib as L
    dev = _dev()
    g = torch.Generator().manual_seed(5)
    n, K, D = 5000, 96, 32
    x = torch.randn(n, D, generator=g).to(dev)
    idx = torch.randint(0, K - 6, (n,), generator=g).to(dev)          # the last six clusters stay empty
    old = torch.randn(K, D, generator=g).to(dev)
    new = torch.empty_like(old)
    shift = torch.empty(1, device=dev)
    ws = L.workspace(L.query("mas_kmeans_ws_bytes", K, D), dev)
    L.call("mas_kmeans_update", x, idx, n, K, D, old, new, shift, ws, ws.numel())
    sums = torch.zeros(K, D, device=dev, dtype=torch.float64).index_add_(0, idx, x.double())
    cnt = torch.zeros(K, device=dev, dtype=torch.float64).index_add_(0, idx, torch.ones(n, device=dev, dtype=torch.float64))
    ref = torch.where(cnt[:, None] > 0, sums / cnt.clamp_min(1)[:, None], old.double()).float()
    assert torch.allclose(new, ref, rtol=1e-6, atol=1e-7)
    assert torch.equal(new[K - 6:], old[K - 6:])
    assert abs(float(shift) - float((ref - old).norm())) < 1e-4 * float((ref - old).norm())


def test_kmeans_reinit_runs_and_reduces_quantisation_error():
    """Codebook re-initialisation from the reservoir (modules.py:487-499) with the seeded Lloyd iterations that replace
    the absent fast_pytorch_kmeans: the assignment step is the VQ kernel; the error must not increase."""
    from models.modules import Codebook
    dev = _dev()
    torch.manual_seed(1)
    cb = Codebook(64, 32, beta=0.25, init_steps=10, reservoir_size=4000).to(dev)
    centers = torch.randn(64, 32, device=dev) * 3
    cb.reservoir = (centers[torch.randint(0, 64, (4000,), device=dev)] + 0.1 * torch.randn(4000, 32, device=dev))
    z = cb.reservoir[:512].view(2, 16, 16, 32).permute(0, 3, 1, 2).contiguous()
    cb.eval()
    _, loss0, _ = cb(z)
    cb._kmeans_reinit(iters=10)
    _, loss1, idx = cb(z)
    assert torch.isfinite(cb.embedding.weight).all() and cb.embedding.weight.shape == (64, 32)
    # random-point initialisation leaves a few of the 64 tight clusters merged: a local optimum, but far below the start
    assert float(loss1) < 0.4 * float(loss0)
