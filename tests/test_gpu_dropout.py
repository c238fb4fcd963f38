"""GPU: dropout of the token transformer (include/mas_b200.h, dropout). The kernels' masks against the numpy restatement of
tests/test_dropout_cpu.py bit for bit, the dropout units against fp64 torch driven by the same masks, the whole model with
dropout against an fp64 restatement of the reference (transformer.py:90-91, 114, 139) driven by the recorded masks, seeding,
eval mode, sampling and CUDA-graph replay."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, rel_err
from test_dropout_cpu import keep_mask

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

# S = 48 + 4^2 + 8^2 = 128 tokens and head dim 64: the fused attention core (csrc/attn_causal.cu) runs
FUSED_CFG = dict(num_layers=2, hidden_dim=128, num_attn_heads=2, image_vocab_size=64, seg_vocab_size=32, text_vocab_size=80,
                 image_tokens_per_dim=8, seg_tokens_per_dim=4, text_length=48)


def _seed(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


def _mask(seed, shape, p, scale=1.0):
    """keep * scale materialised by mas_dropout with x = NULL."""
    from mas_b200 import _lib as L
    y = torch.empty(shape, dtype=torch.float32, device=DEV)
    L.call("mas_dropout", None, None, y, y.numel(), float(p), float(scale), seed)
    return y


@pytest.fixture
def seeds(monkeypatch):
    """Records every seed ops.dropout_seed draws (the device tensors themselves), in draw order."""
    from mas_b200 import ops
    got = []
    orig = ops.dropout_seed

    def record(device):
        s = orig(device)
        got.append(s)
        return s
    monkeypatch.setattr(ops, "dropout_seed", record)
    return got


@pytest.mark.parametrize("n", [1, 7, 4099, (1 << 20) + 3])
@pytest.mark.parametrize("p", [0.0, 0.1, 0.5, 1.0])
def test_mask_equals_numpy_restatement(n, p):
    for s in (0, -1, 987654321987654321):
        got = _mask(_seed(s), (n,), p, 1.0 / (1.0 - p) if p < 1 else 0.0).cpu().numpy()
        want = np.where(keep_mask(s, n, p), np.float32(1.0 / (1.0 - p) if p < 1 else 0.0), np.float32(0.0))
        assert np.array_equal(got, want), (n, p, s)


def test_keep_fraction_is_binomial():
    n, p = 1 << 24, 0.1
    kept = float(_mask(_seed(20261017), (n,), p).sum())
    sigma = (n * p * (1 - p)) ** 0.5
    assert abs(kept - n * (1 - p)) < 6 * sigma


@pytest.mark.parametrize("offset", [0, 1])
def test_dropout_with_residual_and_its_backward(offset, seeds):
    """DropoutFn: residual + x * keep / (1 - p) and its backward; offset 1 runs the unaligned (scalar) path."""
    from mas_b200 import ops
    g = torch.Generator().manual_seed(offset)
    base = torch.randn(3 * 77 * 64 + offset, generator=g).to(DEV)
    x = base[offset:].view(3, 77, 64).requires_grad_(True)
    r = torch.randn(3, 77, 64, generator=g).to(DEV).requires_grad_(True)
    y = ops.DropoutFn.apply(x, 0.3, r)
    w = torch.randn(3, 77, 64, generator=g).to(DEV)
    (y * w).sum().backward()
    k = _mask(seeds[0], x.shape, 0.3)
    sc = np.float32(1 / 0.7)
    assert torch.equal(y.detach(), r.detach() + torch.where(k > 0, x.detach() * float(sc), 0.0))
    assert torch.equal(x.grad, torch.where(k > 0, w * float(sc), 0.0)) and torch.equal(r.grad, w)
    assert 0.6 < float(k.mean()) < 0.8


@pytest.mark.parametrize("R,H,res", [(5, 64, True), (300, 1024, True), (130, 256, False)])
def test_layernorm_dropout_forward_backward(R, H, res, seeds):
    from mas_b200 import ops
    g = torch.Generator().manual_seed(R + H)
    a = (torch.randn(R, H, generator=g) * 2 + 0.5).to(DEV)
    gam = (torch.rand(H, generator=g) + 0.5).to(DEV)
    bet = torch.randn(H, generator=g).to(DEV)
    resid = torch.randn(R, H, generator=g).to(DEV) if res else None
    w = torch.randn(R, H, generator=g).to(DEV)
    ins = [t.clone().requires_grad_(True) for t in (a, gam, bet)] + [resid.clone().requires_grad_(True) if res else None]
    y = ops.LayerNormFn.apply(ins[0], ins[1], ins[2], ins[3], 1e-5, 0.25)
    (y * w).sum().backward()
    k = _mask(seeds[0], (R, H), 0.25).double()
    ref_in = [t.double().requires_grad_(True) for t in (a, gam, bet)] + [resid.double().requires_grad_(True) if res else None]
    yr = F.layer_norm(ref_in[0] * k / 0.75, (H,), ref_in[1], ref_in[2], 1e-5)
    if res:
        yr = yr + ref_in[3]
    (yr * w.double()).sum().backward()
    assert rel_err(y, yr) < 1e-5
    for i in range(3 + res):
        assert rel_err(ins[i].grad, ref_in[i].grad) < 1e-5, i


def _attention_ref(qkv, heads, keep, p):
    B, S, H3 = qkv.shape
    H = H3 // 3
    hd = H // heads
    q, k, v = [t.view(B, S, heads, hd).permute(0, 2, 1, 3) for t in qkv.split(H, dim=-1)]
    s = (q @ k.transpose(-1, -2)) / hd ** 0.5
    s = s.masked_fill(~torch.tril(torch.ones(S, S, dtype=torch.bool, device=qkv.device)), float("-inf"))
    return ((torch.softmax(s, -1) * keep / (1 - p)) @ v).permute(0, 2, 1, 3).reshape(B, S, H)


@pytest.mark.parametrize("B,S,heads,hd", [(1, 128, 1, 64), (2, 640, 16, 64), (3, 256, 2, 64), (2, 40, 3, 16), (1, 200, 2, 64)])
def test_causal_attention_dropout_against_fp64(B, S, heads, hd, seeds, monkeypatch):
    """Fused shapes (S % 128 == 0, hd = 64) and fallback shapes: ctx and dqkv against fp64 torch with the materialised mask;
    for the fused shapes also the fallback (GEMM / softmax / mas_dropout / GEMM) with the same seed."""
    from mas_b200 import ops
    g = torch.Generator().manual_seed(S + heads)
    qkv = (torch.randn(B, S, 3 * heads * hd, generator=g) * 1.5).to(DEV)
    w = torch.randn(B, S, heads * hd, generator=g).to(DEV)
    p = 0.2
    fused = S % 128 == 0 and hd == 64
    out = {}
    for name in (("fused", "gemm") if fused else ("gemm",)):
        monkeypatch.setenv("MAS_ATTN_FUSED", "1" if name == "fused" else "0")
        torch.manual_seed(11)
        x = qkv.clone().requires_grad_(True)
        y = ops.CausalAttentionFn.apply(x, heads, p)
        P = y.grad_fn.saved_tensors[1]
        (y * w).sum().backward()
        out[name] = (y.detach(), x.grad, P.clone(), seeds[-1])
    assert len(seeds) == len(out) and all(torch.equal(s, seeds[0]) for s in seeds)     # same torch seed, same mask seed
    keep = _mask(seeds[0], (B, heads, S, S), p).double()
    r = qkv.double().requires_grad_(True)
    ref = _attention_ref(r, heads, keep, p)
    (ref * w.double()).sum().backward()
    for name, (y, dq, P, _) in out.items():
        assert rel_err(y, ref) < 2e-5, (name, rel_err(y, ref))
        assert rel_err(dq, r.grad) < 2e-5, (name, rel_err(dq, r.grad))
        assert float(P.triu(1).abs().max()) == 0.0 and float((P.sum(-1) - 1).abs().max()) < 1e-5      # P is stored undropped
    if fused:
        assert rel_err(out["fused"][0], out["gemm"][0]) < 2e-5 and rel_err(out["fused"][1], out["gemm"][1]) < 2e-5


def _fixture_model(tag, p_attn, p_out):
    from models.transformer import MakeAScene
    if tag == "fused":
        torch.manual_seed(2)
        m = MakeAScene(**FUSED_CFG, attn_dropout_prob=p_attn, out_dropout_prob=p_out)
        gen = torch.Generator().manual_seed(3)
        c = FUSED_CFG
        g = dict(cfg=c, state_dict={k: v.clone() for k, v in m.state_dict().items()},
                 text=torch.randint(0, c["text_vocab_size"], (2, c["text_length"]), generator=gen),
                 seg=torch.randint(0, c["seg_vocab_size"], (2, c["seg_tokens_per_dim"] ** 2), generator=gen),
                 img=torch.randint(0, c["image_vocab_size"], (2, c["image_tokens_per_dim"] ** 2), generator=gen))
    else:
        g = torch.load(os.path.join(GOLDEN, f"transformer_{tag}.pt"), weights_only=False)
        m = MakeAScene(**g["cfg"], attn_dropout_prob=p_attn, out_dropout_prob=p_out)
        m.load_state_dict(g["state_dict"])
    m.to(DEV).train()
    return m, g


def _reference_loss(g, masks, p_attn, p_out, monkeypatch):
    """fp64 restatement of the reference forward (oracle/transformer_oracle.py) with the three dropout sites of each layer
    applying the recorded masks; returns (loss, {parameter name: gradient})."""
    from oracle import transformer_oracle as O
    queue = list(masks)

    def drop(x, p):
        return x if p == 0 else x * queue.pop(0) / (1 - p)

    def layer(x, sd, pre, heads, mask):
        b, s, h = x.shape
        hd = h // heads
        qkv = O.linear(O.layer_norm(x, sd, pre + ".ln_in"), sd, pre + ".attn.qkv")
        q, k, v = [t.view(b, s, heads, hd).permute(0, 2, 1, 3) for t in torch.split(qkv, h, dim=-1)]
        sc = torch.matmul(q / hd ** 0.5, k.transpose(-1, -2))
        sc = sc.masked_fill(mask == 0, float("-inf"))                      # [B, 1, S, S], plain causal
        ctx = torch.matmul(drop(torch.softmax(sc, -1), p_attn), v).permute(0, 2, 1, 3).reshape(b, s, h)
        a = drop(O.linear(ctx, sd, pre + ".attn.out_proj"), p_out)
        x = x + O.layer_norm(a, sd, pre + ".first_ln_sandwich")
        m = drop(O.linear(O.gelu(O.linear(O.layer_norm(x, sd, pre + ".ln_out"), sd, pre + ".mlp.lin1")), sd, pre + ".mlp.lin2"), p_out)
        return x + O.layer_norm(m, sd, pre + ".second_ln_sandwich")
    monkeypatch.setattr(O, "transformer_layer", layer)
    sd = {k: v.detach().double().cpu().requires_grad_(v.is_floating_point() and k != "transformer.mask")
          for k, v in g["state_dict"].items()}
    logits = O.make_a_scene_forward(sd, g["cfg"], g["text"], g["seg"], g["img"])
    loss = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), g["img"].reshape(-1))
    loss.backward()
    assert not queue
    return loss, {k: v.grad for k, v in sd.items() if v.grad is not None}


@pytest.mark.parametrize("tag,tol_f,tol_g", [("tiny", 1e-3, 5e-3), ("wide", 1e-3, 5e-3), ("fused", 1e-3, 5e-3)])
def test_model_with_dropout_matches_reference_under_recorded_masks(tag, tol_f, tol_g, seeds, monkeypatch):
    p_attn, p_out = 0.15, 0.1
    m, g = _fixture_model(tag, p_attn, p_out)
    torch.manual_seed(7)
    loss = m.loss(g["text"].to(DEV), g["seg"].to(DEV), g["img"].to(DEV))
    loss.backward()
    cfg = g["cfg"]
    S = cfg["text_length"] + cfg["seg_tokens_per_dim"] ** 2 + cfg["image_tokens_per_dim"] ** 2
    B, H, heads = g["text"].shape[0], cfg["hidden_dim"], cfg["num_attn_heads"]
    assert len(seeds) == 3 * cfg["num_layers"]
    shapes = [(B, heads, S, S), (B, S, H), (B, S, H)] * cfg["num_layers"]
    masks = [_mask(s, shp, p).double().cpu() for s, shp, p in zip(seeds, shapes, [p_attn, p_out, p_out] * cfg["num_layers"])]
    rl, rgrads = _reference_loss(g, masks, p_attn, p_out, monkeypatch)
    assert abs(float(loss) - float(rl)) < tol_f * max(1.0, float(rl)), (float(loss), float(rl))
    named = dict(m.named_parameters())
    for k, gv in rgrads.items():
        assert rel_err(named[k].grad, gv) < tol_g, (tag, k, rel_err(named[k].grad, gv))


def _step(m, g):
    m.zero_grad(set_to_none=True)
    loss = m.loss(g["text"].to(DEV), g["seg"].to(DEV), g["img"].to(DEV))
    loss.backward()
    return loss.detach().clone(), {k: p.grad.clone() for k, p in m.named_parameters()}


def test_manual_seed_repeats_a_step():
    """The same torch seed repeats a training step bit for bit (the embedding tables' gradients are summed with atomics, so
    they are compared to rounding); another seed draws other masks."""
    m, g = _fixture_model("fused", 0.1, 0.1)
    torch.manual_seed(5)
    l1, g1 = _step(m, g)
    torch.manual_seed(5)
    l2, g2 = _step(m, g)
    assert torch.equal(l1, l2)
    for k in g1:
        if "embedding" in k:
            assert torch.allclose(g1[k], g2[k], rtol=1e-5, atol=1e-7), k
        else:
            assert torch.equal(g1[k], g2[k]), k
    torch.manual_seed(6)
    l3, _ = _step(m, g)
    assert not torch.equal(l1, l3)


@pytest.mark.parametrize("tag", ["tiny", "fused"])
def test_eval_mode_and_generate_apply_no_dropout(tag, seeds):
    m0, g = _fixture_model(tag, 0.0, 0.0)
    m1, _ = _fixture_model(tag, 0.3, 0.2)
    text, seg, img = g["text"].to(DEV), g["seg"].to(DEV), g["img"].to(DEV)
    m0.eval()
    m1.eval()
    with torch.no_grad():
        assert torch.equal(m0(text, seg, img), m1(text, seg, img))
    m1.train()
    a = m0.generate(text, seg, img_tokens=img, return_logits=True)
    b = m1.generate(text, seg, img_tokens=img, return_logits=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    ta = m0.generate(text, seg, temperature=1.0, top_k=8, generator=torch.Generator(device=DEV).manual_seed(4))
    tb = m1.generate(text, seg, temperature=1.0, top_k=8, generator=torch.Generator(device=DEV).manual_seed(4))
    assert torch.equal(ta, tb)
    assert not seeds


def test_graph_replays_draw_new_masks(seeds):
    """A captured CausalAttentionFn forward draws a fresh seed at each replay; each replay equals eager execution with the
    seed it drew."""
    from mas_b200 import ops
    g = torch.Generator().manual_seed(9)
    qkv = torch.randn(2, 256, 3 * 2 * 64, generator=g).to(DEV)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ops.CausalAttentionFn.apply(qkv, 2, 0.3)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = ops.CausalAttentionFn.apply(qkv, 2, 0.3)
        gseed = seeds[-1]
        runs = []
        for _ in range(2):
            graph.replay()
            torch.cuda.synchronize()
            runs.append((out.clone(), gseed.clone()))
        assert not torch.equal(runs[0][1], runs[1][1]) and not torch.equal(runs[0][0], runs[1][0])
        for ctx, sd in runs:
            orig = ops.dropout_seed
            ops.dropout_seed = lambda device: sd
            try:
                eager = ops.CausalAttentionFn.apply(qkv, 2, 0.3)
            finally:
                ops.dropout_seed = orig
            assert torch.equal(ctx, eager)
