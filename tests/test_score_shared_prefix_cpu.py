"""MakeAScene.score(num_samples=n), checked WITHOUT a GPU: the emulated C-ABI of tests/test_sampling_rows_cpu.py (fp16 Linear
route with real operand rounding, embeddings, LayerNorm, guidance mixes, cross-entropy) plus two emulations of the fused
causal attention (include/mas_b200.h): mas_attn_causal_forward_stats in fp64 on the 2 x fp16 operand split of its amax, per
128-query tile over that tile's causal keys as the kernel visits them, and mas_attn_causal_prefix_forward as that emulation
on the concatenation of the repeated prefix rows and the suffix rows. What is under test is the host side: the lockstep
layer loop gives the repeated call's bits, the prefix runs on P rows, every operand scale is the repeated call's."""
import numpy as np
import pytest
import torch

from test_host_logic_cpu import _addr, _f32
from test_sampling_batched_cpu import _scale_of
from test_sampling_rows_cpu import RowsEmu

TILE = 128


def _split(x, s):
    """The kernel's operand split: x * s as fp16 hi + fp16 lo, back in fp64."""
    hi = (x * s).astype(np.float16).astype(np.float64)
    lo = (x * s - hi).astype(np.float16).astype(np.float64)
    return (hi + lo) / s


class ScoreEmu(RowsEmu):
    """RowsEmu + the fused causal forward with statistics and its shared-prefix form; records (entry, rows, S, amax
    pointer, amax value) of every attention call and the amax every fp16 Linear operand was converted under."""

    def __init__(self):
        super().__init__()
        self.attn = []
        self.halves = []

    def mas_to_half(self, x, y, n, amax):
        self.halves.append((n, _addr(amax), float(_f32(_addr(amax), 1)[0])))
        super().mas_to_half(x, y, n, amax)

    def _stats(self, X, amax, B, S, heads, hd, scale):
        H = heads * hd
        a = float(_f32(_addr(amax), 1)[0])
        assert np.abs(X).max() <= a, "the operand scale must cover the operand"
        X = _split(X.reshape(B, S, 3, heads, hd).astype(np.float64), _scale_of(amax))
        ctx, m_out, l_out = np.zeros((B, S, heads, hd)), np.zeros((B, heads, S)), np.zeros((B, heads, S))
        for b in range(B):
            for h in range(heads):
                q, k, v = (np.ascontiguousarray(X[b, :, c, h]) for c in range(3))
                for t in range(S // TILE):
                    q0, nk = t * TILE, (t + 1) * TILE          # the tile's causal keys, as the kernel visits them
                    s = np.dot(q[q0:nk], np.ascontiguousarray(k[:nk].T)) * scale
                    s = np.where(np.tril(np.ones((TILE, nk)), q0) > 0, s, -np.inf)
                    m = s.max(-1)
                    e = np.exp(s - m[:, None])
                    l = e.sum(-1)
                    ctx[b, q0:nk, h] = np.dot(e / l[:, None], v[:nk])
                    m_out[b, h, q0:nk], l_out[b, h, q0:nk] = m, l
        return ctx.reshape(B, S, H), m_out, l_out

    def mas_attn_causal_forward_stats(self, qkv, amax, stats, ctx, B, S, heads, hd, scale, p, seed):
        assert p == 0.0 and S % TILE == 0
        H = heads * hd
        self.attn.append(("stats", B, S, _addr(amax), float(_f32(_addr(amax), 1)[0])))
        c, m, l = self._stats(_f32(_addr(qkv), B * S * 3 * H), amax, B, S, heads, hd, scale)
        _f32(_addr(ctx), B * S * H).reshape(B, S, H)[...] = c
        st = _f32(_addr(stats), 2 * B * heads * S).reshape(2, B, heads, S)
        st[0], st[1] = m, l

    def mas_attn_causal_prefix_forward(self, qkv_prefix, qkv, amax, ctx, P, n, Lp, L, heads, hd, scale):
        assert Lp % TILE == 0 and L % TILE == 0
        H = heads * hd
        self.attn.append(("prefix", P * n, Lp, _addr(amax), float(_f32(_addr(amax), 1)[0])))
        Xp = _f32(_addr(qkv_prefix), P * Lp * 3 * H).reshape(P, Lp, 3 * H)
        Xs = _f32(_addr(qkv), P * n * L * 3 * H).reshape(P * n, L, 3 * H)
        cat = np.ascontiguousarray(np.concatenate([np.repeat(Xp, n, 0), Xs], 1))
        c, _, _ = self._stats(cat, amax, P * n, Lp + L, heads, hd, scale)
        _f32(_addr(ctx), P * n * L * H).reshape(P * n, L, H)[...] = c[:, Lp:]


@pytest.fixture
def emu(monkeypatch):
    from mas_b200 import ops
    from models import transformer
    e = ScoreEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: True)
    monkeypatch.setattr(ops, "f16_operands", lambda: True)
    monkeypatch.setenv("MAS_LINEAR_F16", "1")
    monkeypatch.delenv("MAS_ATTN_FUSED", raising=False)
    monkeypatch.setattr(ops.L, "query", lambda name, *a: 256)
    monkeypatch.setattr(transformer, "SCORE_SHARED_MIN_ROWS", 1)     # the shared form at the small row counts of these tests
    return e


def _model(sandwich=True):
    """hidden 128, 2 heads of 64, text 64 + seg 8^2 (a 128-position prefix), image 16^2: the fused route's smallest shape."""
    from models.transformer import MakeAScene
    torch.manual_seed(0)
    m = MakeAScene(2, 128, 2, 256, 32, 300, 16, 8, 64)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith(("ln_in.weight", "ln_out.weight", "sandwich.weight")):
                p.uniform_(0.5, 1.5)
    if not sandwich:
        for layer in m.transformer.layers:
            layer.cogview_sandwich_layernorm = False
    m.eval()
    return m


def _inputs(m, B, n, seed=1):
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(1, m.text_vocab_size, (B, m.text_length), generator=g)
    text[:, -9:] = 0                                                    # padding: the per-position pad ids
    seg = torch.randint(0, 32, (B, m.seg_length), generator=g)
    img = torch.randint(0, 256, (B * n, m.image_length), generator=g)
    return text, seg, img


def _rep(t, n):
    return None if t is None else t.repeat_interleave(n, 0)


GUIDANCE = [dict(), dict(guidance_scale=2.5), dict(guidance_scale="rows"), dict(guidance_scale=2.5, uncond_text_tokens=True)]


def _kw(kw, m, B, n):
    kw = dict(kw)
    if kw.get("guidance_scale") == "rows":
        kw["guidance_scale"] = torch.linspace(0.5, 4.0, B * n)
    if kw.get("uncond_text_tokens") is True:
        kw["uncond_text_tokens"] = torch.randint(1, m.text_vocab_size, (B, m.text_length), generator=torch.Generator().manual_seed(9))
    return kw


@pytest.mark.parametrize("sandwich", [True, False])
@pytest.mark.parametrize("B,n", [(1, 4), (2, 3)])
@pytest.mark.parametrize("kw", GUIDANCE)
def test_shared_prefix_equals_the_repeated_call(emu, sandwich, B, n, kw):
    """Bit for bit the repeat_interleave call, guided or not, one scale or one per row, padded or given unconditional text;
    the prefix entries see the P prompt rows, the image positions the P * n candidate rows, and every fp16 Linear operand
    and attention call gets the scale the repeated call derives, the same for both parts."""
    m = _model(sandwich)
    text, seg, img = _inputs(m, B, n)
    kw = _kw(kw, m, B, n)
    P = B * (2 if "guidance_scale" in kw else 1)
    emu.attn.clear()
    emu.halves.clear()
    got = m.score(text, seg, img, num_samples=n, **kw)
    shared_attn, shared_halves = list(emu.attn), list(emu.halves)
    emu.attn.clear()
    emu.halves.clear()
    ref = m.score(_rep(text, n), _rep(seg, n), img, **dict(kw, uncond_text_tokens=_rep(kw.get("uncond_text_tokens"), n)))
    assert got.shape == (B * n, m.image_length) and got.dtype == torch.float32
    assert torch.equal(got, ref)
    Lp = m.text_length + m.seg_length
    layers = len(m.transformer.layers)
    # attention: per layer the prefix on P rows and the candidates on P * n, one amax (that of the repeated call's qkv)
    assert [a[:3] for a in shared_attn] == [("stats", P, Lp), ("prefix", P * n, Lp)] * layers
    assert [a[:3] for a in emu.attn] == [("stats", P * n, Lp + m.image_length)] * layers
    for li in range(layers):
        s, p = shared_attn[2 * li], shared_attn[2 * li + 1]
        assert s[3] == p[3] and s[4] == p[4] == emu.attn[li][4]
    # Linears: the 4 per layer in two parts under one amax each, then to_logits once on the gathered rows
    assert len(shared_halves) == 2 * 4 * layers + 1 and len(emu.halves) == 4 * layers + 1
    for i in range(4 * layers):
        hp, hs = shared_halves[2 * i], shared_halves[2 * i + 1]
        assert hp[1] == hs[1] and hp[2] == hs[2] == emu.halves[i][2]
        assert hp[0] // Lp * n * (Lp + m.image_length) == hs[0] // m.image_length * (Lp + m.image_length) == emu.halves[i][0]
    assert shared_halves[-1][2] == emu.halves[-1][2]


def test_num_samples_1_issues_the_calls_of_before(emu):
    m = _model()
    text, seg, img = _inputs(m, 2, 1)
    m.score(text, seg, img)                                             # packs the fp16 weight images once
    for kw in GUIDANCE:
        kw = _kw(kw, m, 2, 1)
        emu.args.clear()
        a = m.score(text, seg, img, **kw)
        before = [(name, [x for x in args if isinstance(x, (int, float))]) for name, args in emu.args]
        emu.args.clear()
        b = m.score(text, seg, img, num_samples=1, **kw)
        assert [(name, [x for x in args if isinstance(x, (int, float))]) for name, args in emu.args] == before
        assert torch.equal(a, b)
        assert "mas_attn_causal_prefix_forward" not in [name for name, _ in emu.args]


def test_fallback_repeats_the_prompts_where_the_fused_route_is_off(emu, monkeypatch):
    """MAS_ATTN_FUSED=0 (and any shape off the fused route) scores through the repeated call: no prefix entry."""
    m = _model()
    text, seg, img = _inputs(m, 1, 3)
    monkeypatch.setenv("MAS_ATTN_FUSED", "0")
    assert not m._score_shares_prefix()
    emu.args.clear()
    got = m.score(text, seg, img, num_samples=3, guidance_scale=2.0)
    names = [name for name, _ in emu.args]
    assert "mas_attn_causal_prefix_forward" not in names and "mas_attn_causal_forward_stats" not in names
    assert torch.equal(got, m.score(_rep(text, 3), _rep(seg, 3), img, guidance_scale=2.0))


@pytest.mark.parametrize("B,n,guided,shared", [(1, 8, False, False), (1, 8, True, False), (3, 8, False, True), (1, 12, True, True)])
def test_default_row_threshold(emu, monkeypatch, B, n, guided, shared):
    """At the default SCORE_SHARED_MIN_ROWS (24 candidate rows, both streams counted) smaller calls repeat the prompts,
    larger ones share the prefix; the same bits either way."""
    from models import transformer
    monkeypatch.setattr(transformer, "SCORE_SHARED_MIN_ROWS", 24)
    m = _model()
    text, seg, img = _inputs(m, B, n)
    kw = dict(guidance_scale=2.0) if guided else {}
    emu.args.clear()
    got = m.score(text, seg, img, num_samples=n, **kw)
    assert ("mas_attn_causal_prefix_forward" in [name for name, _ in emu.args]) == shared
    assert torch.equal(got, m.score(_rep(text, n), _rep(seg, n), img, **kw))


def test_argument_validation(emu):
    m = _model()
    B, n = 2, 3
    text, seg, img = _inputs(m, B, n)
    cases = [dict(num_samples=0), dict(num_samples=-1), dict(num_samples=True), dict(num_samples=2.0), dict(num_samples="3"),
             dict(num_samples=None),
             dict(img_tokens=img[:B]), dict(img_tokens=img[:, :-1]), dict(img_tokens=img[:B * n - 1]),
             dict(guidance_scale=torch.ones(B)), dict(guidance_scale=[2.0] * (B * n + 1)),
             dict(guidance_scale=torch.full((B * n,), float("nan"))),
             dict(uncond_text_tokens=_rep(text, n)), dict(seg_tokens=_rep(seg, n)), dict(text_tokens=_rep(text, n))]
    for kw in cases:
        args = dict(text_tokens=text, seg_tokens=seg, img_tokens=img, guidance_scale=2.0, num_samples=n)
        args.update(kw)
        with pytest.raises(ValueError):
            m.score(**args)
    assert not [name for name, _ in emu.args if name in ("mas_ce_forward", "mas_embed3_forward")]


def test_prefix_emulation_equals_the_stats_emulation_on_the_concatenation(emu):
    """The emulated new entry against the emulated fused forward on the concatenated rows (what the GPU test checks of the
    kernel): a guard that the emulation above compares like with like."""
    g = torch.Generator().manual_seed(3)
    P, n, Lp, L, heads, hd = 2, 3, 256, 128, 2, 64
    qp = torch.randn(P, Lp, 3 * heads * hd, generator=g)
    qs = torch.randn(P * n, L, 3 * heads * hd, generator=g) * 2
    am = torch.tensor([float(max(qp.abs().max(), qs.abs().max()))])
    from mas_b200 import ops
    got = ops.attn_causal_prefix(qp, qs, am, heads)
    cat = torch.cat([qp.repeat_interleave(n, 0), qs], 1)
    full = torch.empty(P * n, Lp + L, heads * hd)
    emu.mas_attn_causal_forward_stats(cat, am, torch.empty(2, P * n, heads, Lp + L), full, P * n, Lp + L, heads, hd, hd ** -0.5,
                                      0.0, None)
    assert torch.equal(got, full[:, Lp:])
