"""GPU: causal attention that stores no probabilities (csrc/attn_causal.cu: mas_attn_causal_forward_stats and
mas_attn_causal_backward, ops.CausalAttentionFn(recompute=True), MakeAScene(recompute_attention=True)): the kernels against
fp64 torch under the numpy restatement of the dropout mask, ctx bit-identical to the P-writing kernel, a deterministic
backward, nothing S x S saved and the memory it frees, and the whole model against the stored-P route and the fp64
reference."""
import pytest
import torch

from conftest import rel_err
from test_dropout_cpu import keep_mask
from test_gpu_dropout import FUSED_CFG, _fixture_model, _mask, _reference_loss, seeds  # noqa: F401 (seeds: fixture)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SHAPES = [(1, 128, 1), (3, 256, 2), (2, 640, 16), (1, 1408, 16)]


def _inputs(B, S, heads):
    g = torch.Generator().manual_seed(S + 7 * heads)
    qkv = (torch.randn(B, S, 3 * heads * 64, generator=g) * 1.5).to(DEV)
    w = torch.randn(B, S, heads * 64, generator=g).to(DEV)
    return qkv, w


def _forward(qkv, heads, p, recompute, seed):
    """(x, ctx) of one call with its autograd graph, the dropout seed fixed."""
    from mas_b200 import ops
    orig = ops.dropout_seed
    ops.dropout_seed = lambda device: seed.clone()
    try:
        x = qkv.clone().requires_grad_(True)
        return x, ops.CausalAttentionFn.apply(x, heads, p, recompute)
    finally:
        ops.dropout_seed = orig


def _grad(x, y, w):
    return torch.autograd.grad(y, x, w, retain_graph=True)[0]


@pytest.mark.parametrize("p", [0.0, 0.2])
@pytest.mark.parametrize("B,S,heads", SHAPES)
def test_recompute_kernels_against_fp64(B, S, heads, p):
    qkv, w = _inputs(B, S, heads)
    seed = torch.tensor([S * 1000003 + heads], dtype=torch.int64, device=DEV)
    x, y = _forward(qkv, heads, p, True, seed)
    dq = _grad(x, y, w)
    stats = y.grad_fn.saved_tensors[2]
    keep = torch.from_numpy(keep_mask(int(seed), B * heads * S * S, p).reshape(B, heads, S, S)).to(DEV)
    H = heads * 64
    r = qkv.double().requires_grad_(True)
    q, k, v = [t.view(B, S, heads, 64).permute(0, 2, 1, 3) for t in r.split(H, dim=-1)]
    s = (q @ k.transpose(-1, -2)) / 8.0
    s = s.masked_fill(~torch.tril(torch.ones(S, S, dtype=torch.bool, device=DEV)), float("-inf"))
    ref = ((torch.softmax(s, -1) * keep / (1.0 - p)) @ v).permute(0, 2, 1, 3).reshape(B, S, H)
    (ref * w.double()).sum().backward()
    assert rel_err(y, ref) < 2e-5, rel_err(y, ref)
    assert rel_err(dq, r.grad) < 2e-5, rel_err(dq, r.grad)
    with torch.no_grad():
        m_ref = s.amax(-1)
        l_ref = torch.exp(s - m_ref[..., None]).sum(-1)
    assert rel_err(stats[0], m_ref) < 1e-6 and rel_err(stats[1], l_ref) < 1e-6, (rel_err(stats[0], m_ref), rel_err(stats[1], l_ref))


@pytest.mark.parametrize("p", [0.0, 0.2])
@pytest.mark.parametrize("B,S,heads", SHAPES)
def test_ctx_identical_to_the_p_writing_kernel_and_backward_deterministic(B, S, heads, p):
    qkv, w = _inputs(B, S, heads)
    seed = torch.tensor([-987654321 - S], dtype=torch.int64, device=DEV)
    x0, y0 = _forward(qkv, heads, p, False, seed)
    x1, y1 = _forward(qkv, heads, p, True, seed)
    assert torch.equal(y0, y1)
    dq0, dq1, dq2 = _grad(x0, y0, w), _grad(x1, y1, w), _grad(x1, y1, w)
    assert rel_err(dq1, dq0) < 2e-5, rel_err(dq1, dq0)
    assert torch.equal(dq1, dq2)


def test_nothing_s_by_s_is_saved():
    B, S, heads = 2, 640, 16
    qkv, w = _inputs(B, S, heads)
    seed = torch.tensor([5], dtype=torch.int64, device=DEV)
    for p in (0.0, 0.2):
        shapes = []

        def pack(t):
            shapes.append(tuple(t.shape))
            return t
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            x, y = _forward(qkv, heads, p, True, seed)
        assert shapes
        for shp in shapes:
            n = 1
            for d in shp:
                n *= d
            assert n < B * heads * S * S // 2 and shp[-2:] != (S, S), shp
        _grad(x, y, w)


def _train_peak(recompute, cfg, B):
    from models.transformer import MakeAScene
    torch.manual_seed(0)
    m = MakeAScene(**cfg, recompute_attention=recompute).to(DEV).train()
    g = torch.Generator().manual_seed(1)
    text = torch.randint(1, cfg["text_vocab_size"], (B, cfg["text_length"]), generator=g).to(DEV)
    seg = torch.randint(0, cfg["seg_vocab_size"], (B, cfg["seg_tokens_per_dim"] ** 2), generator=g).to(DEV)
    img = torch.randint(0, cfg["image_vocab_size"], (B, cfg["image_tokens_per_dim"] ** 2), generator=g).to(DEV)
    m.loss(text, seg, img).backward()          # first step: weight images, workspaces
    m.zero_grad(set_to_none=False)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss = m.loss(text, seg, img)
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del m
    torch.cuda.empty_cache()
    return peak


def test_memory_drop_at_s1408():
    """4 layers, 16 heads of 64, S = 128 + 16^2 + 32^2 = 1408: the stored-P route holds every layer's P [B,16,S,S], and one dP
    during the backward. Without them the peak moves to where the MLP backward's temporaries live and the recompute route
    saves ctx for D = dO . ctx, so the peak drops by less than P + dP (measured on an H100 80 GB HBM3 at 700 W: 1882 -> 800 MB,
    85 % of the 1269 MB of P + dP); it must drop by at least 90 % of the stored P alone."""
    cfg = dict(num_layers=4, hidden_dim=1024, num_attn_heads=16, image_vocab_size=1024, seg_vocab_size=256, text_vocab_size=1024,
               image_tokens_per_dim=32, seg_tokens_per_dim=16, text_length=128)
    B, S = 2, 1408
    stored = _train_peak(False, cfg, B)
    rec = _train_peak(True, cfg, B)
    p_bytes = (cfg["num_layers"] + 1) * B * cfg["num_attn_heads"] * S * S * 4
    print("peak above the parameters: stored P %.1f MB, recomputed %.1f MB, P + dP %.1f MB" % (stored / 1e6, rec / 1e6, p_bytes / 1e6))
    assert stored - rec >= 0.9 * p_bytes * cfg["num_layers"] / (cfg["num_layers"] + 1), (stored, rec, p_bytes)


def test_model_recompute_matches_stored_route_and_reference(seeds, monkeypatch):
    """Train mode with attention and residual dropout, the same torch seed: the loss is the same bits as the stored-P route,
    the gradients agree with it and with the fp64 reference under the recorded masks (test_gpu_dropout's tolerances)."""
    from models.transformer import MakeAScene
    p_attn, p_out = 0.15, 0.1
    m0, g = _fixture_model("fused", p_attn, p_out)
    m1 = MakeAScene(**FUSED_CFG, attn_dropout_prob=p_attn, out_dropout_prob=p_out, recompute_attention=True)
    m1.load_state_dict(g["state_dict"])
    m1.to(DEV).train()
    text, seg, img = g["text"].to(DEV), g["seg"].to(DEV), g["img"].to(DEV)
    torch.manual_seed(7)
    l0 = m0.loss(text, seg, img)
    l0.backward()
    n0 = len(seeds)
    torch.manual_seed(7)
    l1 = m1.loss(text, seg, img)
    l1.backward()
    assert torch.equal(l0.detach(), l1.detach())
    assert all(torch.equal(a, b) for a, b in zip(seeds[:n0], seeds[n0:]))
    g0, g1 = dict(m0.named_parameters()), dict(m1.named_parameters())
    for k in g0:
        assert rel_err(g1[k].grad, g0[k].grad) < 1e-3, (k, rel_err(g1[k].grad, g0[k].grad))
    cfg = g["cfg"]
    S = cfg["text_length"] + cfg["seg_tokens_per_dim"] ** 2 + cfg["image_tokens_per_dim"] ** 2
    B, H, heads = g["text"].shape[0], cfg["hidden_dim"], cfg["num_attn_heads"]
    shapes = [(B, heads, S, S), (B, S, H), (B, S, H)] * cfg["num_layers"]
    masks = [_mask(s, shp, p).double().cpu() for s, shp, p in zip(seeds[n0:], shapes, [p_attn, p_out, p_out] * cfg["num_layers"])]
    rl, rgrads = _reference_loss(g, masks, p_attn, p_out, monkeypatch)
    assert abs(float(l1) - float(rl)) < 1e-3 * max(1.0, float(rl))
    for k, gv in rgrads.items():
        assert rel_err(g1[k].grad, gv) < 5e-3, (k, rel_err(g1[k].grad, gv))
