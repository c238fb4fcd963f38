"""GPU parity of the tier-2 token transformer drop-in (models/transformer.py) against fixtures from the REAL reference:
logits, cross-entropy loss and every parameter gradient (tiny: fp32 SIMT path; wide: tensor-core Linear layers)."""
import os

import pytest
import torch

from conftest import GOLDEN, rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tag,tol_f,tol_g", [("tiny", 1e-3, 5e-3), ("wide", 1e-3, 5e-3)])
def test_make_a_scene_forward_backward_vs_reference(tag, tol_f, tol_g):
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, f"transformer_{tag}.pt"), weights_only=False)
    dev = torch.device("cuda:0")
    m = MakeAScene(**g["cfg"])
    assert list(m.state_dict().keys()) == list(g["state_dict"].keys())
    m.load_state_dict(g["state_dict"])
    m.to(dev)
    m.device = dev
    logits = m(g["text"].to(dev), g["seg"].to(dev), g["img"].to(dev))
    assert logits.shape == g["logits"].shape
    assert rel_err(logits, g["logits"]) < tol_f
    loss = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), g["img"].to(dev).reshape(-1))
    assert abs(float(loss) - float(g["loss"])) < tol_f * max(1.0, float(g["loss"]))
    loss.backward()
    named = dict(m.named_parameters())
    for k, gv in g["grads"].items():
        assert named[k].grad is not None, k
        assert rel_err(named[k].grad, gv) < tol_g, (tag, k)
    for k, v in g["grad_norms"].items():
        got = float(named[k].grad.double().norm())
        assert abs(got - v) <= 2e-2 * max(v, 1e-4 * named[k].numel() ** 0.5), (tag, k, got, v)


# ------------------------------------------------------------------------------------------------ sampling (SURVEY 8f-3)
def _load_model(tag):
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, f"transformer_{tag}.pt"), weights_only=False)
    dev = torch.device("cuda:0")
    m = MakeAScene(**g["cfg"])
    m.load_state_dict(g["state_dict"])
    m.to(dev).eval()
    m.device = dev
    return m, g, dev


@pytest.mark.parametrize("tag", ["tiny", "wide"])
def test_generate_teacher_forced_matches_reference_logits(tag):
    """KV-cached decoding fed the fixture's image tokens reproduces, position by position, the logits the REAL reference's
    non-cached forward produced (the only specification the reference offers for this path). Tolerance 2e-3: the prefix
    runs on the TF32 Linear kernels when the widths allow, the decode steps are strict fp32."""
    m, g, dev = _load_model(tag)
    img = g["img"].to(dev)
    toks, lg = m.generate(g["text"].to(dev), g["seg"].to(dev), img_tokens=img, return_logits=True)
    assert toks.shape == img.shape and bool((toks == img).all())
    assert lg.shape == g["logits"].shape
    assert rel_err(lg, g["logits"]) < 2e-3


def test_generate_guidance_greedy_and_seeded_sampling():
    m, g, dev = _load_model("tiny")
    text, seg, img = g["text"].to(dev), g["seg"].to(dev), g["img"].to(dev)
    with torch.no_grad():
        cond = m(text, seg, img)
        uncond = m(torch.zeros_like(text), seg, img)
    s = 2.5
    _, lg = m.generate(text, seg, guidance_scale=s, img_tokens=img, return_logits=True)
    assert rel_err(lg, uncond + s * (cond - uncond)) < 2e-3
    # greedy decoding follows its own arg-max chain
    toks, lg = m.generate(text, seg, guidance_scale=s, temperature=0, return_logits=True)
    assert bool((toks == lg.argmax(-1)).all())
    # seeded sampling: reproducible, in range, top-k respected
    V = g["cfg"]["image_vocab_size"]
    a = m.generate(text, seg, temperature=0.9, top_k=5, generator=torch.Generator(device=dev).manual_seed(7))
    b, lgb = m.generate(text, seg, temperature=0.9, top_k=5, generator=torch.Generator(device=dev).manual_seed(7), return_logits=True)
    assert a.shape == img.shape and a.dtype == torch.int64 and int(a.min()) >= 0 and int(a.max()) < V
    assert bool((a == b).all())
    kth = lgb.topk(5, dim=-1).values[..., -1]
    assert bool((lgb.gather(-1, b.unsqueeze(-1)).squeeze(-1) >= kth).all())


def test_generate_with_cuda_graphs_matches_eager():
    """generate(use_graphs=True): first call captures one graph per position, later calls replay them; both reproduce the
    reference logits under teacher forcing and the eager path's samples under a fixed seed."""
    m, g, dev = _load_model("tiny")
    text, seg, img = g["text"].to(dev), g["seg"].to(dev), g["img"].to(dev)
    for _ in range(2):                       # capture, then replay
        toks, lg = m.generate(text, seg, img_tokens=img, return_logits=True, use_graphs=True)
        assert bool((toks == img).all()) and rel_err(lg, g["logits"]) < 2e-3
    other = img.flip(1).contiguous()         # different tokens through the same graphs
    _, lg_g = m.generate(text, seg, img_tokens=other, return_logits=True, use_graphs=True)
    _, lg_e = m.generate(text, seg, img_tokens=other, return_logits=True)
    assert torch.equal(lg_g, lg_e)
    a = m.generate(text, seg, guidance_scale=2.0, temperature=1.0, top_k=8, generator=torch.Generator(device=dev).manual_seed(3))
    b = m.generate(text, seg, guidance_scale=2.0, temperature=1.0, top_k=8, generator=torch.Generator(device=dev).manual_seed(3),
                   use_graphs=True)   # 4 rows now: a new decoder is captured
    assert bool((a == b).all())
    m.reset_sampler()


@pytest.mark.parametrize("R,N,K,act", [(1, 37, 132, 0), (3, 64, 1024, 1), (8, 130, 4 * 257, 0), (2, 8192, 1024, 0),
                                       (2, 1024, 4096, 0), (5, 37, 2052, 1), (8, 2, 4096, 0)])   # last three: K-split variant
def test_linear_small_vs_torch(R, N, K, act):
    from mas_b200 import ops
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(R * 1000 + N)
    x = torch.randn(R, K, generator=gen)
    w = torch.randn(N, K, generator=gen) / K ** 0.5
    b = torch.randn(N, generator=gen)
    ref = torch.nn.functional.linear(x.double(), w.double(), b.double())
    if act:
        ref = 0.5 * ref * (1.0 + torch.tanh(0.7978845608028654 * ref * (1.0 + 0.044715 * ref * ref)))
    y = ops.linear_small(x.to(dev), w.to(dev), b.to(dev), act=act)
    assert rel_err(y, ref.float()) < 1e-5


@pytest.mark.parametrize("R,H,res", [(1, 1024, True), (2, 1024, False), (8, 4096, True), (3, 132, True), (64, 64, False)])
def test_layernorm_few_rows_vs_torch(R, H, res):
    """The block-per-row LayerNorm the decode steps use (R <= 64 rows)."""
    from mas_b200 import ops
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(R + H)
    x = torch.randn(R, H, generator=gen) * 3 + 0.5
    w, b = torch.randn(H, generator=gen), torch.randn(H, generator=gen)
    r = torch.randn(R, H, generator=gen) if res else None
    ref = torch.nn.functional.layer_norm(x.double(), (H,), w.double(), b.double(), 1e-5)
    if res:
        ref = ref + r.double()
    y = ops.LayerNormFn.apply(x.to(dev), w.to(dev), b.to(dev), r.to(dev) if res else None, 1e-5)
    assert rel_err(y, ref.float()) < 1e-5


@pytest.mark.parametrize("heads,hd,length,tmax", [(4, 16, 5, 37), (2, 64, 130, 640), (3, 32, 257, 300), (1, 128, 640, 640)])
def test_kv_append_and_attn_decode_vs_torch(heads, hd, length, tmax):
    from mas_b200 import ops
    dev = torch.device("cuda:0")
    R, H = 3, heads * hd
    gen = torch.Generator().manual_seed(hd + length)
    qkv_all = torch.randn(R, length, 3 * H, generator=gen)
    kc = torch.zeros(R, heads, tmax, hd, device=dev)
    vc = torch.zeros_like(kc)
    ops.kv_append(qkv_all[:, :length - 1].to(dev), kc, vc, 0)                 # prefix in one call
    ops.kv_append(qkv_all[:, length - 1:].to(dev), kc, vc, length - 1)        # the current token
    k = qkv_all[..., H:2 * H].view(R, length, heads, hd).permute(0, 2, 1, 3)
    v = qkv_all[..., 2 * H:].view(R, length, heads, hd).permute(0, 2, 1, 3)
    assert torch.equal(kc[:, :, :length].cpu(), k) and torch.equal(vc[:, :, :length].cpu(), v)
    q = qkv_all[:, -1, :H].view(R, heads, 1, hd)
    p = torch.softmax((q.double() @ k.double().transpose(-1, -2)) / hd ** 0.5, -1)
    ref = (p @ v.double()).reshape(R, H).float()
    ctx = ops.attn_decode(qkv_all[:, -1].contiguous().to(dev), kc, vc, length)
    assert rel_err(ctx, ref) < 1e-5
    # the fused form: the token's k / v are appended by the attention kernel itself
    kc2 = torch.zeros_like(kc)
    vc2 = torch.zeros_like(vc)
    ops.kv_append(qkv_all[:, :length - 1].to(dev), kc2, vc2, 0)
    ctx2 = ops.attn_decode_append(qkv_all[:, -1].contiguous().to(dev), kc2, vc2, length - 1)
    assert torch.equal(kc2, kc) and torch.equal(vc2, vc)
    assert rel_err(ctx2, ref) < 1e-5 and rel_err(ctx2, ctx) < 1e-6


@pytest.mark.parametrize("R,H,res", [(1, 1024, True), (2, 1024, False), (8, 4096, True), (3, 132, True)])
def test_layernorm_pair_vs_torch(R, H, res):
    """mas_layernorm2_forward: y1 = residual + LN1(x), y2 = LN2(y1) (the two chained LayerNorms of a decode step)."""
    from mas_b200 import ops
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(7 * R + H)
    x = torch.randn(R, H, generator=gen) * 3 + 0.5
    ln1, ln2 = torch.nn.LayerNorm(H, eps=1e-5), torch.nn.LayerNorm(H, eps=1e-5)
    with torch.no_grad():
        for ln in (ln1, ln2):
            ln.weight.copy_(torch.randn(H, generator=gen))
            ln.bias.copy_(torch.randn(H, generator=gen))
    r = torch.randn(R, H, generator=gen) if res else None
    with torch.no_grad():
        ref1 = ln1.double()(x.double())
        if res:
            ref1 = ref1 + r.double()
        ref2 = ln2.double()(ref1)
    ln1.float().to(dev)
    ln2.float().to(dev)
    y1, y2 = ops.layernorm2(x.to(dev), ln1, r.to(dev) if res else None, ln2)
    assert rel_err(y1, ref1.float()) < 1e-5 and rel_err(y2, ref2.float()) < 1e-5


def test_causal_attention_on_tensor_cores_matches_fp32_kernels(monkeypatch):
    """transformer.py:77-103 at the paper's extents (640 tokens, 16 heads of 64): QK^T / PV and their four gradients on the
    3xTF32 wgmma GEMM against the exact-fp32 FFMA kernels (which the reference fixtures pin at small extents)."""
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(3)
    qkv = torch.randn(2, 640, 3 * 1024, generator=g).to(dev)
    w = torch.randn(2, 640, 1024, generator=g).to(dev)
    out = {}
    monkeypatch.setenv("MAS_ATTN_FUSED", "0")      # the GEMM / softmax / GEMM sequence (the fused core has its own test below)
    for name, impl in (("tc", L.IMPL_AUTO), ("simt", L.IMPL_SIMT)):
        ops.set_impl(impl)
        try:
            x = qkv.clone().requires_grad_(True)
            before = L.tc_launch_count()
            y = ops.CausalAttentionFn.apply(x, 16)
            (y * w).sum().backward()
            out[name] = (y.detach(), x.grad.detach(), L.tc_launch_count() - before)
        finally:
            ops.set_impl(L.IMPL_AUTO)
    assert out["tc"][2] == 6 and out["simt"][2] == 0     # one launch per contraction over all (sequence, head) pairs
    assert rel_err(out["tc"][0], out["simt"][0]) < 2e-5
    assert rel_err(out["tc"][1], out["simt"][1]) < 2e-5


# ------------------------------------------------------------------------------------------------ fused cross-entropy / sampler
@pytest.mark.parametrize("R,V,pitch", [(7, 33, 33), (512, 8192, 8192), (64, 1000, 1024)])
def test_cross_entropy_vs_torch(R, V, pitch):
    """mas_ce_forward / mas_ce_backward against F.cross_entropy (fp64 on the CPU): loss, gradient, ignored rows, row pitch."""
    from mas_b200 import ops
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(R + V)
    full = torch.randn(R, pitch, generator=g) * 3
    tgt = torch.randint(0, V, (R,), generator=g)
    tgt[R // 3] = -100                                      # F.cross_entropy's default ignore_index
    ref_in = full[:, :V].double().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(ref_in, tgt)
    (ref * 1.7).backward()
    x = full.to(dev)[:, :V].requires_grad_(True)            # a strided view when pitch > V
    loss = ops.cross_entropy(x, tgt.to(dev))
    (loss * 1.7).backward()
    assert abs(float(loss) - float(ref)) < 1e-5 * max(1.0, abs(float(ref)))
    assert rel_err(x.grad, ref_in.grad.float()) < 1e-5
    assert float(x.grad[R // 3].abs().max()) == 0.0


@pytest.mark.parametrize("tag", ["tiny", "wide"])
def test_make_a_scene_loss_entry_matches_reference(tag):
    """MakeAScene.loss (forward + fused cross-entropy) against the REAL reference's loss and gradients (train.py:150-153)."""
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, f"transformer_{tag}.pt"), weights_only=False)
    dev = torch.device("cuda:0")
    m = MakeAScene(**g["cfg"])
    m.load_state_dict(g["state_dict"])
    m.to(dev)
    m.device = dev
    loss = m.loss(g["text"].to(dev), g["seg"].to(dev), g["img"].to(dev))
    assert abs(float(loss) - float(g["loss"])) < 1e-3 * max(1.0, float(g["loss"]))
    loss.backward()
    named = dict(m.named_parameters())
    for k, gv in g["grads"].items():
        assert rel_err(named[k].grad, gv) < 5e-3, (tag, k)


def test_sample_topk_kernel():
    """mas_sample_topk: greedy when top_k = 1, the inverse CDF of the top-k softmax at the caller's uniforms otherwise,
    and the right distribution over many rows."""
    from mas_b200 import ops
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(11)
    lg = torch.randn(8, 8192, generator=g) * 2
    u = torch.rand(8, generator=g)
    tok = ops.sample_topk(lg.to(dev), 0.8, 1, u.to(dev)).cpu()
    assert torch.equal(tok, lg.argmax(-1))
    for k in (5, 100, None):
        tok = ops.sample_topk(lg.to(dev), 0.8, k, u.to(dev)).cpu()
        z = lg.double() / 0.8
        if k is not None:
            kth = z.topk(k, -1).values[:, -1:]
            z = torch.where(z < kth, torch.full_like(z, float("-inf")), z)
        cdf = torch.softmax(z, -1).cumsum(-1)
        for r in range(8):
            t = int(tok[r])
            assert z[r, t] > float("-inf")
            lo = float(cdf[r, t - 1]) if t > 0 else 0.0
            assert lo - 1e-5 <= float(u[r]) <= float(cdf[r, t]) + 1e-5, (k, r, t)
    # distribution: 20000 rows of the same 50 logits, top 10
    row = torch.randn(50, generator=g)
    R = 20000
    tok = ops.sample_topk(row.expand(R, 50).contiguous().to(dev), 1.3, 10, torch.rand(R, generator=g).to(dev)).cpu()
    z = row.double() / 1.3
    keep = z >= z.topk(10).values[-1]
    p = torch.softmax(torch.where(keep, z, torch.full_like(z, float("-inf"))), -1)
    freq = torch.bincount(tok, minlength=50).double() / R
    assert float(freq[~keep].sum()) == 0.0
    assert float((freq - p).abs().max()) < 5 * float((p * (1 - p) / R).sqrt().max())


@pytest.mark.parametrize("B,S,heads", [(1, 128, 1), (2, 640, 16), (3, 256, 2)])
def test_fused_causal_attention_core_matches_fp32_kernels(B, S, heads, monkeypatch):
    """csrc/attn_causal.cu (scores -> causal softmax -> P v in one tensor-core kernel, 2 x fp16 operand split) against the
    exact-fp32 FFMA sequence: ctx, the saved probabilities (incl. the zeros above the diagonal) and the gradients."""
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(S + heads)
    qkv = (torch.randn(B, S, 3 * heads * 64, generator=g) * 1.5).to(dev)
    w = torch.randn(B, S, heads * 64, generator=g).to(dev)
    out = {}
    for name, impl, fused in (("fused", L.IMPL_AUTO, "1"), ("gemm", L.IMPL_AUTO, "0"), ("simt", L.IMPL_SIMT, "0")):
        monkeypatch.setenv("MAS_ATTN_FUSED", fused)
        ops.set_impl(impl)
        try:
            x = qkv.clone().requires_grad_(True)
            before = L.launch_count()
            y = ops.CausalAttentionFn.apply(x, heads)
            fwd_launches = L.launch_count() - before
            P = y.grad_fn.saved_tensors[1].clone()
            (y * w).sum().backward()
            out[name] = (y.detach(), x.grad.detach(), P, fwd_launches)
        finally:
            ops.set_impl(L.IMPL_AUTO)
    assert out["fused"][3] == 2 and out["gemm"][3] == 3        # amax + the fused core vs GEMM, softmax, GEMM
    for other in ("simt", "gemm"):
        assert rel_err(out["fused"][0], out[other][0]) < 2e-5, other
        assert rel_err(out["fused"][2], out[other][2]) < 2e-5, other
        assert rel_err(out["fused"][1], out[other][1]) < 2e-5, other
    P = out["fused"][2]
    assert float(P.triu(1).abs().max()) == 0.0
    assert float((P.sum(-1) - 1).abs().max()) < 1e-5


@pytest.mark.parametrize("R,K,N", [(256, 128, 128), (5120, 1024, 3072), (1000, 4096, 1024), (77, 128, 256), (2048, 1024, 8192)])
def test_linear_on_tma_fed_f16_row_gemm(R, K, N, monkeypatch):
    """csrc/gemm_tma.cu (TMA-fed fp16 operands, N = 256 MMAs) behind ops.LinearFn: forward, data gradient and weight gradient against
    fp64 torch; the operands carry 11 significant bits like the TF32 path (tolerance 1e-3), row tails are zero-filled by the copy
    engine, the weight images are cached per parameter version."""
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(R + K + N)
    x = (torch.randn(R, K, generator=g) * 2 + 0.3)
    w = torch.randn(N, K, generator=g) * 0.05
    b = torch.randn(N, generator=g)
    dy = torch.randn(R, N, generator=g) * 1e-4          # gradient-sized values: the power-of-two operand scale matters
    xr, wr, br = x.double().requires_grad_(True), w.double().requires_grad_(True), b.double().requires_grad_(True)
    yr = torch.nn.functional.linear(xr, wr, br)
    yr.backward(dy.double())
    monkeypatch.setenv("MAS_LINEAR_F16", "1")
    xd = x.to(dev).requires_grad_(True)
    wd = torch.nn.Parameter(w.to(dev))
    bd = torch.nn.Parameter(b.to(dev))
    before = L.tc_launch_count()
    y = ops.LinearFn.apply(xd, wd, bd)
    y.backward(dy.to(dev))
    assert L.tc_launch_count() - before == 3          # forward, data gradient, weight gradient
    assert rel_err(y, yr.float()) < 1e-3
    assert rel_err(xd.grad, xr.grad.float()) < 1e-3
    assert rel_err(wd.grad, wr.grad.float()) < 2e-3 and rel_err(bd.grad, br.grad.float()) < 5e-4   # sums of the fp16-rounded dy
    ent = ops._pack_entry(wd)
    assert ("lin16", False) in ent and ("lin16", True) in ent
    # the register-staged TF32 kernel on the same problem agrees to operand-rounding level
    monkeypatch.setenv("MAS_LINEAR_F16", "0")
    x2 = x.to(dev).requires_grad_(True)
    y2 = ops.LinearFn.apply(x2, wd, bd)
    assert rel_err(y, y2) < 1e-3


@pytest.mark.parametrize("R,H,res", [(5, 132, True), (640, 1024, True), (100, 4096, False), (33, 256, False), (7, 8192, False)])
def test_layernorm_forward_backward_vs_torch(R, H, res):
    """LayerNormFn (warp-per-row and block-per-row kernels of both directions) against fp64 torch: output, dx, dgamma, dbeta and
    the residual pass-through."""
    from mas_b200 import ops
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(R * 7 + H)
    x = torch.randn(R, H, generator=g) * 2 + 0.7
    w, b = torch.randn(H, generator=g), torch.randn(H, generator=g)
    r = torch.randn(R, H, generator=g) if res else None
    dy = torch.randn(R, H, generator=g)
    xr, wr, br = x.double().requires_grad_(True), w.double().requires_grad_(True), b.double().requires_grad_(True)
    rr = r.double().requires_grad_(True) if res else None
    yr = torch.nn.functional.layer_norm(xr, (H,), wr, br, 1e-5)
    if res:
        yr = yr + rr
    yr.backward(dy.double())
    xd, wd, bd = x.to(dev).requires_grad_(True), w.to(dev).requires_grad_(True), b.to(dev).requires_grad_(True)
    rd = r.to(dev).requires_grad_(True) if res else None
    y = ops.LayerNormFn.apply(xd, wd, bd, rd, 1e-5)
    y.backward(dy.to(dev))
    assert rel_err(y, yr.float()) < 1e-5
    assert rel_err(xd.grad, xr.grad.float()) < 2e-5
    assert rel_err(wd.grad, wr.grad.float()) < 1e-5 and rel_err(bd.grad, br.grad.float()) < 1e-5
    if res:
        assert torch.equal(rd.grad.cpu(), dy)
