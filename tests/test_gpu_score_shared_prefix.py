"""GPU: MakeAScene.score(num_samples=n) and its kernel, mas_attn_causal_prefix_forward (csrc/attn_causal.cu,
attn_causal_fwd<HD, false, false, true>): the kernel bit for bit against mas_attn_causal_forward on the concatenated rows and
within the causal-attention tests' 2e-5 of fp64; score(num_samples=n) bit for bit against the repeat_interleave call on
2-layer models of the bench's shape; the launches (prefix on the prompt rows only, num_samples=1 unchanged); the fallback
and the tiny fixture; agreement with generate's log-probabilities; the ValueError cases."""
import math
import os

import pytest
import torch

from conftest import GOLDEN, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BENCH = dict(image_vocab_size=8192, seg_vocab_size=1024, text_vocab_size=49408, image_tokens_per_dim=16, seg_tokens_per_dim=16,
             text_length=128)


def _kernel_inputs(P, n, Lp, L, heads, hd, where, seed):
    """Prefix [P,Lp,3H] and suffix [P*n,L,3H] activations; the largest |.| planted in the prefix or in the suffix."""
    g = torch.Generator().manual_seed(seed)
    H3 = 3 * heads * hd
    qp = torch.randn(P, Lp, H3, generator=g)
    qs = torch.randn(P * n, L, H3, generator=g)
    (qp if where == "prefix" else qs).view(-1)[int(torch.randint(0, (qp if where == "prefix" else qs).numel(), (1,), generator=g))] = -9.5
    return qp.to(DEV), qs.to(DEV)


def _concat_forward(qp, qs, n, heads, hd, am):
    """mas_attn_causal_forward over the concatenated [P*n, Lp+L, 3H] rows with the given amax -> ctx."""
    from mas_b200 import ops
    cat = torch.cat([qp.repeat_interleave(n, 0), qs], 1).contiguous()
    R, S, H3 = cat.shape
    P_ = torch.empty((R, heads, S, S), dtype=torch.float32, device=DEV)
    ctx = torch.empty((R, S, H3 // 3), dtype=torch.float32, device=DEV)
    ops.L.call("mas_attn_causal_forward", cat, am, P_, ctx, R, S, heads, hd, 1.0 / float(hd) ** 0.5)
    return ctx, cat


@pytest.mark.parametrize("where", ["prefix", "suffix"])
@pytest.mark.parametrize("P", [1, 4])
@pytest.mark.parametrize("n", [1, 2, 3, 8])
@pytest.mark.parametrize("L", [128, 256])
@pytest.mark.parametrize("Lp", [128, 384])
@pytest.mark.parametrize("hd", [64, 128])
def test_kernel_equals_the_causal_forward_on_the_concatenation(hd, Lp, L, n, P, where):
    from mas_b200 import _lib, ops
    heads = 2
    qp, qs = _kernel_inputs(P, n, Lp, L, heads, hd, where, seed=hd + Lp + L + 10 * n + P)
    am = ops.amax_joint(qp, qs)
    assert float(am) == 9.5
    with _lib.launch_trace() as names:
        got = ops.attn_causal_prefix(qp, qs, am, heads)
    assert names == ["attn_causal_prefix_fwd" + ("<128>" if hd == 128 else "")], names
    ref, _ = _concat_forward(qp, qs, n, heads, hd, am)
    assert torch.equal(got, ref[:, Lp:])


@pytest.mark.parametrize("heads,hd", [(16, 64), (8, 128)])
def test_kernel_against_fp64_at_the_bench_shape(heads, hd):
    """Prefix 384 (text 128 + segmentation 256), image 256, 2 prompts x 4 candidates, against fp64 attention over the
    concatenated rows: within the 2e-5 norm-wise bound of the causal-attention tests."""
    from mas_b200 import ops
    P, n, Lp, L = 2, 4, 384, 256
    qp, qs = _kernel_inputs(P, n, Lp, L, heads, hd, "suffix", seed=5)
    qp, qs = qp * 0.3, qs * 0.3
    got = ops.attn_causal_prefix(qp, qs, ops.amax_joint(qp, qs), heads)
    cat = torch.cat([qp.repeat_interleave(n, 0), qs], 1).double()
    R, S, H = P * n, Lp + L, heads * hd
    q, k, v = [t.reshape(R, S, heads, hd).permute(0, 2, 1, 3) for t in cat.split(H, dim=-1)]
    s = (q @ k.transpose(-1, -2)) / hd ** 0.5
    s = s.masked_fill(~torch.tril(torch.ones(S, S, dtype=torch.bool, device=DEV)), float("-inf"))
    ref = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(R, S, H)[:, Lp:]
    err = rel_err(got, ref)
    print("prefix attention hd %d vs fp64: %.2e" % (hd, err))
    assert err < 2e-5


def test_kernel_refuses_unsupported_shapes():
    from mas_b200 import ops
    for Lp, L, hd in ((100, 128, 64), (128, 200, 64), (128, 128, 96)):
        qp = torch.zeros(1, Lp, 3 * 2 * hd, device=DEV)
        qs = torch.zeros(2, L, 3 * 2 * hd, device=DEV)
        with pytest.raises(RuntimeError, match="attn_causal_prefix_forward"):
            ops.attn_causal_prefix(qp, qs, ops.amax_joint(qp, qs), 2)


_models = {}


def _model(heads, sandwich=True):
    """2 layers of the bench's model (hidden 1024), 16 heads of 64 or 8 of 128, with or without the sandwich LayerNorm."""
    key = (heads, sandwich)
    if key not in _models:
        from models.transformer import MakeAScene
        torch.manual_seed(heads)
        m = MakeAScene(2, 1024, heads, **BENCH)
        with torch.no_grad():
            for name, p in m.named_parameters():
                if name.endswith("weight") and ("ln" in name or "sandwich" in name):
                    p.uniform_(0.5, 1.5)
        for layer in m.transformer.layers:
            layer.cogview_sandwich_layernorm = sandwich
        _models[key] = m.to(DEV).eval()
    return _models[key]


def _inputs(m, B, n, seed=1):
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(1, m.text_vocab_size, (B, m.text_length), generator=g)
    text[:, 100:] = 0
    seg = torch.randint(0, 1024, (B, m.seg_length), generator=g)
    img = torch.randint(0, 8192, (B * n, m.image_length), generator=g)
    return text.to(DEV), seg.to(DEV), img.to(DEV)


def _guidance(kind, m, B, n):
    if kind == "none":
        return {}
    if kind == "scalar":
        return dict(guidance_scale=3.0)
    if kind == "rows":
        return dict(guidance_scale=torch.linspace(0.5, 5.0, B * n, device=DEV))
    unc = torch.randint(1, m.text_vocab_size, (B, m.text_length), generator=torch.Generator().manual_seed(7)).to(DEV)
    return dict(guidance_scale=2.0, uncond_text_tokens=unc)


def _repeated(m, text, seg, img, n, kw):
    kw = dict(kw)
    if kw.get("uncond_text_tokens") is not None:
        kw["uncond_text_tokens"] = kw["uncond_text_tokens"].repeat_interleave(n, 0)
    return m.score(text.repeat_interleave(n, 0), seg.repeat_interleave(n, 0), img, **kw)


@pytest.mark.parametrize("guidance", ["none", "scalar", "rows", "given_uncond"])
@pytest.mark.parametrize("n", [1, 4, 8])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("sandwich", [True, False])
@pytest.mark.parametrize("heads", [16, 8])
def test_score_equals_the_repeated_call(heads, sandwich, B, n, guidance, monkeypatch):
    from mas_b200 import _lib
    from models import transformer
    monkeypatch.setattr(transformer, "SCORE_SHARED_MIN_ROWS", 1)     # the shared form at every row count tested here
    m = _model(heads, sandwich)
    assert m._score_shares_prefix()
    text, seg, img = _inputs(m, B, n, seed=B * 10 + n)
    kw = _guidance(guidance, m, B, n)
    with _lib.launch_trace() as names:
        got = m.score(text, seg, img, num_samples=n, **kw)
    want = _repeated(m, text, seg, img, n, kw)
    assert got.shape == (B * n, m.image_length) and got.dtype == torch.float32
    assert torch.equal(got, want)
    assert bool(torch.isfinite(got).all()) and bool((got <= 0).all())
    suffix = "<128>" if heads == 8 else ""
    assert (names.count("attn_causal_prefix_fwd" + suffix) == (2 if n > 1 else 0)), set(names)
    assert names.count("attn_causal_fwd_stats" + suffix) == 2


def _recorded(monkeypatch):
    """Every C-ABI call as (name, its int arguments), passed through to the library."""
    from mas_b200 import ops
    rec, orig = [], ops.L.call
    monkeypatch.setattr(ops.L, "call", lambda name, *a: (rec.append((name, [x for x in a if isinstance(x, int)])), orig(name, *a))[1])
    return rec


@pytest.mark.parametrize("guided", [False, True])
def test_launches_prefix_on_prompt_rows_and_num_samples_1_unchanged(guided, monkeypatch):
    from models import transformer
    monkeypatch.setattr(transformer, "SCORE_SHARED_MIN_ROWS", 1)
    m = _model(16)
    B, n = 3, 4
    P = 2 * B if guided else B
    text, seg, img = _inputs(m, B, n)
    kw = dict(guidance_scale=2.0) if guided else {}
    rec = _recorded(monkeypatch)
    m.score(text, seg, img, num_samples=n, **kw)
    Lp, L = m.text_length + m.seg_length, m.image_length
    stats = [a for nm, a in rec if nm == "mas_attn_causal_forward_stats"]
    pref = [a for nm, a in rec if nm == "mas_attn_causal_prefix_forward"]
    assert [a[:2] for a in stats] == [[P, Lp]] * 2                    # (B, S): the prefix pass on the prompt rows only
    assert [a[:4] for a in pref] == [[P, n, Lp, L]] * 2
    emb = [a for nm, a in rec if nm == "mas_embed3_forward"]
    assert sorted(a[0] for a in emb) == sorted([P * m.text_length, P * m.seg_length, P * n * L])
    gemms = [a for nm, a in rec if nm == "mas_gemm_rows_f16"]
    assert sorted({a[0] for a in gemms}) == sorted({P * Lp, P * n * L})
    # num_samples=1 issues the calls of the call without it
    img1 = img[::n].contiguous()
    rec.clear()
    a = m.score(text, seg, img1, **kw)
    before = list(rec)
    rec.clear()
    b = m.score(text, seg, img1, num_samples=1, **kw)
    assert rec == before and torch.equal(a, b)
    assert not [nm for nm, _ in rec if nm == "mas_attn_causal_prefix_forward"]


def _tiny():
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, "transformer_tiny.pt"), weights_only=False)
    m = MakeAScene(**g["cfg"])
    m.load_state_dict(g["state_dict"])
    return m.to(DEV).eval(), g


@pytest.mark.parametrize("n", [1, 3])
def test_fallback_and_tiny_fixture(n):
    """The tiny config is off the fused route: num_samples repeats the prompts (bit for bit the repeated call, no prefix
    kernel), and the reference's logits still give the result within test_gpu_sampling_logprobs' 4e-3 ||z||_F."""
    from mas_b200 import _lib
    m, g = _tiny()
    assert not m._score_shares_prefix()
    text, seg = g["text"].to(DEV), g["seg"].to(DEV)
    img = g["img"].to(DEV).repeat_interleave(n, 0)
    with _lib.launch_trace() as names:
        lp = m.score(text, seg, img, num_samples=n, guidance_scale=None)
    assert not [k for k in names if "prefix" in k]
    assert torch.equal(lp, _repeated(m, text, seg, img, n, {}))
    z = g["logits"].double().repeat_interleave(n, 0)
    ref = torch.log_softmax(z, -1).gather(-1, img.cpu().unsqueeze(-1)).squeeze(-1)
    err, bound = float((lp.double().cpu() - ref).norm()), 4e-3 * float(z.norm())
    assert err <= bound, (err, bound)


@pytest.mark.parametrize("B,n,scale", [(1, 4, 2.0), (2, 4, None), (2, 8, 2.0)])
def test_generate_and_score_agree(B, n, scale, monkeypatch):
    """generate(num_samples=n, temperature=1) without filters, then score(num_samples=n) on the drawn tokens: up to 8 decode
    rows (fp32 decoding) within test_gpu_sampling_logprobs' bound on the mixed logits, above it the gap is printed."""
    from models import transformer
    monkeypatch.setattr(transformer, "SCORE_SHARED_MIN_ROWS", 1)
    m = _model(16)
    text, seg, _ = _inputs(m, B, n, seed=3)
    toks, lp = m.generate(text, seg, guidance_scale=scale, temperature=1.0, num_samples=n,
                          generator=torch.Generator(device=DEV).manual_seed(5), return_logprobs=True)
    sc = m.score(text, seg, toks, guidance_scale=scale, num_samples=n)
    assert torch.equal(sc, _repeated(m, text, seg, toks, n, dict(guidance_scale=scale)))
    tr, sr = text.repeat_interleave(n, 0), seg.repeat_interleave(n, 0)
    with torch.no_grad():
        c = m(tr, sr, toks).double().cpu()
        u = m(torch.zeros_like(tr), sr, toks).double().cpu() if scale else c
    s = scale or 1.0
    bound = 4e-3 * (abs(1 - s) * float(u.norm()) + s * float(c.norm()))
    gap = float((lp.double() - sc.double()).norm())
    rows = B * n * (2 if scale else 1)
    print("generate vs score(num_samples) B=%d n=%d scale=%s rows=%d: ||gap|| %.3e (bound %.3e)" % (B, n, scale, rows, gap, bound))
    assert math.isfinite(gap)
    if rows <= 8:
        assert gap <= bound, (gap, bound)


@pytest.mark.parametrize("B,n,guided,shared", [(1, 8, False, False), (1, 8, True, False), (3, 8, False, True), (1, 12, True, True)])
def test_default_row_threshold(B, n, guided, shared):
    """At the default SCORE_SHARED_MIN_ROWS (24 candidate rows, both streams counted) smaller calls repeat the prompts,
    larger ones share the prefix; the same bits either way."""
    from mas_b200 import _lib
    m = _model(16)
    text, seg, img = _inputs(m, B, n)
    kw = dict(guidance_scale=2.0) if guided else {}
    with _lib.launch_trace() as names:
        got = m.score(text, seg, img, num_samples=n, **kw)
    assert ("attn_causal_prefix_fwd" in names) == shared
    assert torch.equal(got, _repeated(m, text, seg, img, n, kw))


def test_errors():
    m = _model(16)
    B, n = 2, 4
    text, seg, img = _inputs(m, B, n)
    bad = [dict(num_samples=0), dict(num_samples=True), dict(num_samples=2.5), dict(img_tokens=img[:B]),
           dict(img_tokens=img[:, :-1]), dict(guidance_scale=torch.ones(B, device=DEV)),
           dict(guidance_scale=[2.0] * (B * n - 1)), dict(uncond_text_tokens=text.repeat_interleave(n, 0))]
    for kw in bad:
        args = dict(text_tokens=text, seg_tokens=seg, img_tokens=img, guidance_scale=2.0, num_samples=n)
        args.update(kw)
        with pytest.raises(ValueError):
            m.score(**args)
