"""Per-token log-probabilities of MakeAScene.generate(return_logprobs=True) and MakeAScene.score, checked WITHOUT a GPU: the
emulated C-ABI of tests/test_sampling_controls_cpu.py (and the shared-prefix entries of
tests/test_sampling_shared_prefix_cpu.py) plus an fp64 restatement of mas_sample_filtered_logp (include/mas_b200.h). What is
under test is the host side: which entries a call issues, the output column each draw writes, the zeros of forced and greedy
positions, the return order, num_samples, the call sequence of score and its argument checks."""
import ctypes

import numpy as np
import pytest
import torch

from test_host_logic_cpu import _addr, _i64, _mat
from test_sampling_batched_cpu import _model, _tile
from test_sampling_controls_cpu import filtered_draw, filtered_keep
from test_sampling_shared_prefix_cpu import SharedEmu

SAMPLERS = ("mas_sample_topk", "mas_sample_filtered", "mas_sample_filtered_logp")


def filtered_logp(x, temperature, top_k, top_p, tok):
    """fp64 log-probability of token tok of one row under the draw's distribution: softmax(z) over the kept set, z = x / T."""
    z = np.asarray(x, dtype=np.float64) / temperature
    keep, _ = filtered_keep(z, top_k, top_p)
    assert keep[tok]
    return float(z[tok] - z.max() - np.log(np.exp(z[keep] - z.max()).sum()))


class LogpEmu(SharedEmu):
    """SharedEmu (ControlsEmu + the shared-prefix attention) + mas_sample_filtered_logp: the tokens of mas_sample_filtered and
    the fp64 log-probability each was drawn with, 0 for prompt and greedy rows; records the column it wrote."""

    def __init__(self):
        super().__init__()
        self.logp_cols = []

    def mas_sample_filtered_logp(self, logits, ld, R, V, temperature, top_k, top_p, u, ptok, pmask, pld, tokens, logp, logp_ld):
        self.mas_sample_filtered(logits, ld, R, V, temperature, top_k, top_p, u, ptok, pmask, pld, tokens)
        X = _mat(_addr(logits), R, V, ld, False).astype(np.float64)
        tok = _i64(_addr(tokens), R)
        forced = self.draws[-1]["forced"]
        for r in range(R):
            v = 0.0 if (r in forced or temperature == 0) else filtered_logp(X[r], temperature, top_k, top_p, int(tok[r]))
            ctypes.c_float.from_address(_addr(logp) + 4 * r * logp_ld).value = v
        self.logp_cols.append((_addr(logp), logp_ld))


@pytest.fixture
def emu(monkeypatch):
    from mas_b200 import ops
    e = LogpEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: False)
    monkeypatch.setattr(ops.L, "query", lambda name, *a: 256)
    monkeypatch.setattr(torch.cuda, "graph_pool_handle", lambda: None)
    return e


def _inputs(B):
    m, g = _model("tiny")
    return m, _tile(g["text"], B), _tile(g["seg"], B), _tile(g["img"], B)


def _gen(seed=17):
    return torch.Generator().manual_seed(seed)


def _mask(B, L, frac, seed):
    return torch.rand(B, L, generator=torch.Generator().manual_seed(seed)) < frac


CONFIGS = [dict(temperature=0.9, top_k=20), dict(temperature=0.8, top_k=0, top_p=0.7), dict(temperature=1.0, img_mask=0.5),
           dict(temperature=0, img_mask=0.5), dict(temperature=0), dict(img_tokens=True)]


def _kw(kw, m, B, img):
    kw = dict(kw)
    if "img_mask" in kw:
        kw.update(img_mask=_mask(B, m.image_length, kw["img_mask"], 1), img_tokens=img)
    elif kw.get("img_tokens") is True:
        kw["img_tokens"] = img
    return kw


@pytest.mark.parametrize("kw", CONFIGS)
def test_without_the_flag_the_same_entries_and_with_it_only_the_sampler_changes(emu, kw):
    """return_logprobs=False (or absent) issues exactly the entries of before, never the new one; True issues the same
    sequence with every sampler entry replaced by mas_sample_filtered_logp, and the same tokens."""
    m, text, seg, img = _inputs(2)
    kw = _kw(kw, m, 2, img)
    a = m.generate(text, seg, generator=_gen(), **kw)
    base = list(emu.names)
    assert "mas_sample_filtered_logp" not in base
    emu.names.clear()
    b = m.generate(text, seg, generator=_gen(), return_logprobs=False, **kw)
    assert emu.names == base and torch.equal(a, b)
    emu.names.clear()
    c, lp = m.generate(text, seg, generator=_gen(), return_logprobs=True, **kw)
    assert emu.names == ["mas_sample_filtered_logp" if n in SAMPLERS else n for n in base]
    assert torch.equal(a, c) and lp.dtype == torch.float32 and lp.shape == a.shape


@pytest.mark.parametrize("B,scale", [(2, None), (2, 2.5), (5, 2.5), (12, None)])
def test_drawn_positions_write_their_column_and_forced_ones_are_zero(emu, B, scale):
    """Every position with a draw calls mas_sample_filtered_logp once, on column t of the returned tensor (row stride
    image_length); drawn positions hold the fp64 log-probability of the returned (mixed) logits under the filters, forced
    positions exactly 0; tokens and logits are those of the call without the flag; guided and above 8 rows too."""
    m, text, seg, img = _inputs(B)
    L = m.image_length
    T = torch.randint(0, m.image_token_embedding.num_embeddings, (B, L), generator=torch.Generator().manual_seed(3))
    M = _mask(B, L, 0.4, B)
    kw = dict(guidance_scale=scale, temperature=0.8, top_k=40, top_p=0.7, img_tokens=T, img_mask=M, return_logits=True)
    toks0, lg0 = m.generate(text, seg, generator=_gen(5), **kw)
    emu.logp_cols.clear()
    emu.draws.clear()
    toks, lg, lp = m.generate(text, seg, generator=_gen(5), return_logprobs=True, **kw)
    assert torch.equal(toks, toks0) and torch.equal(lg, lg0)
    assert emu.logp_cols == [(lp.data_ptr() + 4 * t, L) for t in range(L)]
    assert bool((lp[M] == 0).all())
    for b in range(B):
        for t in range(L):
            if not M[b, t]:
                want = filtered_logp(lg[b, t].numpy(), 0.8, 40, 0.7, int(toks[b, t]))
                assert abs(float(lp[b, t]) - want) <= 1e-6 * (1 + abs(want)), (b, t)
                assert int(toks[b, t]) == filtered_draw(lg[b, t].numpy(), 0.8, 40, 0.7, float(emu.draws[t]["u"][b]))
    assert bool((lp <= 0).all()) and bool((lp[~M] < 0).any())


def test_greedy_and_teacher_forced_positions_are_zero(emu):
    m, text, seg, img = _inputs(3)
    L = m.image_length
    for kw in (dict(temperature=0), dict(img_tokens=img), dict(temperature=0, img_tokens=img, img_mask=_mask(3, L, 0.5, 2)),
               dict(temperature=0, guidance_scale=2.0)):
        toks, lp = m.generate(text, seg, return_logprobs=True, **kw)
        assert lp.shape == (3, L) and bool((lp == 0).all()) and torch.equal(toks, m.generate(text, seg, **kw)), kw


def test_return_order(emu):
    """tokens, then logits with return_logits, then logprobs; the plain call still returns the bare tensor."""
    m, text, seg, img = _inputs(2)
    kw = dict(guidance_scale=2.0, temperature=1.0, top_k=10)
    t0 = m.generate(text, seg, generator=_gen(), **kw)
    t1, lg1 = m.generate(text, seg, generator=_gen(), return_logits=True, **kw)
    t2, lp2 = m.generate(text, seg, generator=_gen(), return_logprobs=True, **kw)
    out = m.generate(text, seg, generator=_gen(), return_logits=True, return_logprobs=True, **kw)
    assert isinstance(t0, torch.Tensor) and len(out) == 3
    t3, lg3, lp3 = out
    assert torch.equal(t0, t1) and torch.equal(t0, t2) and torch.equal(t0, t3)
    assert torch.equal(lg1, lg3) and torch.equal(lp2, lp3) and lg3.dim() == 3 and lp3.shape == t0.shape


@pytest.mark.parametrize("B,n,scale", [(2, 3, 2.5), (3, 4, None)])
def test_num_samples_equals_repeat_interleave(emu, B, n, scale):
    m, text, seg, img = _inputs(B)
    L = m.image_length
    M = _mask(B * n, L, 0.3, 7)
    T = _tile(img, B * n)
    kw = dict(guidance_scale=scale, temperature=0.9, top_k=30, top_p=0.85, img_tokens=T, img_mask=M, return_logits=True,
              return_logprobs=True)
    a = m.generate(text, seg, generator=_gen(4), num_samples=n, **kw)
    if scale is not None:
        kw["uncond_text_tokens"] = torch.zeros_like(text).repeat_interleave(n, 0)
    b = m.generate(text.repeat_interleave(n, 0), seg.repeat_interleave(n, 0), generator=_gen(4), **kw)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def _score_ref(lg, img):
    """fp64 log_softmax of logits [B, L, V] gathered at img [B, L]."""
    return torch.log_softmax(lg.detach().double(), -1).gather(-1, img.unsqueeze(-1)).squeeze(-1)


@pytest.mark.parametrize("B", [2, 5])
def test_score_unguided_call_sequence_and_values(emu, B):
    """One causal pass (one embedding launch per segment: text, seg, image), to_logits, no mix, one mas_ce_forward over the
    B * image_length rows; the result is the fp64 log-softmax of forward()'s logits at the given tokens."""
    m, text, seg, img = _inputs(B)
    lp = m.score(text, seg, img)
    names = list(emu.names)
    assert names.count("mas_embed3_forward") == 3 and names.count("mas_ce_forward") == 1 and names[-1] == "mas_ce_forward"
    assert "mas_cfg_mix" not in names and not [n for n in names if n.startswith("mas_sample") or "decode" in n]
    ce = [a for n, a in emu.args if n == "mas_ce_forward"][0]
    assert ce[6:8] == (B * m.image_length, m.image_token_embedding.num_embeddings)
    assert lp.shape == (B, m.image_length) and lp.dtype == torch.float32
    ref = _score_ref(m(text, seg, img), img)
    assert float((lp.double() - ref).abs().max()) < 1e-5
    for s in (None, 1.0):                                            # guidance_scale 1 is the unguided distribution
        assert torch.equal(m.score(text, seg, img, guidance_scale=s), lp)


def test_score_guided_call_sequence_and_values(emu):
    """Both streams in one 2B-row pass, then mas_cfg_mix of the [B, L, V] halves and mas_ce_forward on the mix: the result is
    the log-softmax of uncond + s (cond - uncond) of two forward() calls (padded text by default, or the given one)."""
    B, s = 3, 2.5
    m, text, seg, img = _inputs(B)
    lp = m.score(text, seg, img, guidance_scale=s)
    names = list(emu.names)
    assert names.count("mas_embed3_forward") == 3 and names.count("mas_cfg_mix") == 1 and names.count("mas_ce_forward") == 1
    assert names.index("mas_cfg_mix") < names.index("mas_ce_forward")
    V, L = m.image_token_embedding.num_embeddings, m.image_length
    mix = [a for n, a in emu.args if n == "mas_cfg_mix"][0]
    assert mix[3:] == (B * L * V, s)
    emb = [a for n, a in emu.args if n == "mas_embed3_forward"]
    assert [a[7] for a in emb] == [2 * B * m.text_length, 2 * B * m.seg_length, 2 * B * L]
    for unc in (None, torch.randint(1, m.text_vocab_size, text.shape, generator=torch.Generator().manual_seed(2))):
        got = m.score(text, seg, img, guidance_scale=s, uncond_text_tokens=unc)
        cond = m(text, seg, img).detach().double()
        uncond = m(torch.zeros_like(text) if unc is None else unc, seg, img).detach().double()
        ref = _score_ref(uncond + s * (cond - uncond), img)
        assert float((got.double() - ref).abs().max()) < 1e-5
        if unc is None:
            assert torch.equal(got, lp)


def test_score_ignores_dropout_in_train_mode(emu):
    """A model built with dropout, in train mode, scores like its eval-mode self: no dropout entry is issued."""
    from models.transformer import MakeAScene
    m0, text, seg, img = _inputs(2)
    g = _model("tiny")[1]
    m = MakeAScene(**g["cfg"], attn_dropout_prob=0.3, out_dropout_prob=0.2)
    m.load_state_dict(g["state_dict"])
    m.train()
    emu.names.clear()
    a = m.score(text, seg, img, guidance_scale=2.0)
    assert not [n for n in emu.names if "dropout" in n]
    m.eval()
    assert torch.equal(a, m.score(text, seg, img, guidance_scale=2.0)) and m0.training is False


def test_argument_validation(emu):
    from mas_b200 import ops
    m, text, seg, img = _inputs(2)
    V = m.image_token_embedding.num_embeddings
    for bad in (1, 0, None, "yes", np.bool_(True), torch.tensor(True)):
        with pytest.raises(ValueError):
            m.generate(text, seg, return_logprobs=bad)
    bad_img_lo, bad_img_hi = img.clone(), img.clone()
    bad_img_lo[1, 3], bad_img_hi[0, -1] = -1, V
    cases = [dict(text_tokens=text[:, :-1]), dict(seg_tokens=seg[:1]), dict(img_tokens=img[:, :-1]),         # shapes
             dict(img_tokens=img[0]), dict(text_tokens=text[0]), dict(uncond_text_tokens=text[:1]),
             dict(img_tokens=img.tolist()),
             dict(text_tokens=text.int()), dict(seg_tokens=seg.int()), dict(img_tokens=img.int()),           # dtypes
             dict(uncond_text_tokens=text.float()),
             dict(img_tokens=torch.zeros(img.shape, dtype=torch.int64, device="meta")),                     # devices
             dict(seg_tokens=torch.zeros(seg.shape, dtype=torch.int64, device="meta")),
             dict(uncond_text_tokens=torch.zeros(text.shape, dtype=torch.int64, device="meta")),
             dict(img_tokens=bad_img_lo), dict(img_tokens=bad_img_hi)]                                       # range
    for kw in cases:
        args = dict(text_tokens=text, seg_tokens=seg, img_tokens=img, guidance_scale=2.0)
        args.update(kw)
        with pytest.raises(ValueError):
            m.score(**args)
    assert not [n for n in emu.names if n in ("mas_ce_forward", "mas_embed3_forward")]
    lg, u = torch.zeros(2, 8), torch.zeros(2)
    for logp in (torch.zeros(3), torch.zeros(2, dtype=torch.float64), torch.zeros(2, 1), torch.zeros(2, device="meta")):
        with pytest.raises(ValueError):
            ops.sample_topk(lg, 1.0, 0, u, logp=logp)
    with pytest.raises(ValueError):
        ops.token_logprobs(lg, torch.zeros(3, dtype=torch.int64))
    assert not [n for n in emu.names if n.startswith("mas_sample")]


def test_sample_topk_routes_every_logp_call_to_the_new_entry(emu):
    """With an output column the draw is always mas_sample_filtered_logp (plain, top-p, prompt, greedy); without one it is
    the entry of before. The column may be strided."""
    from mas_b200 import ops
    g = torch.Generator().manual_seed(1)
    lg, u = torch.randn(6, 40, generator=g) * 2, torch.rand(6, generator=g)
    prompt = (torch.arange(6, dtype=torch.int64), torch.tensor([1, 0, 0, 1, 0, 0], dtype=torch.bool))
    for kw, old in ((dict(), "mas_sample_topk"), (dict(top_p=0.6), "mas_sample_filtered"),
                    (dict(prompt=prompt), "mas_sample_filtered"), (dict(top_p=1.0), "mas_sample_topk")):
        emu.names.clear()
        a = ops.sample_topk(lg, 0.9, 5, u, **kw)
        out = torch.full((6, 3), 7.0)
        b = ops.sample_topk(lg, 0.9, 5, u, logp=out[:, 1], **kw)
        assert emu.names == [old, "mas_sample_filtered_logp"] and torch.equal(a, b), kw
        assert bool((out[:, [0, 2]] == 7.0).all())
        for r in range(6):
            forced = "prompt" in kw and bool(prompt[1][r])
            want = 0.0 if forced else filtered_logp(lg[r].numpy(), 0.9, 5, kw.get("top_p"), int(b[r]))
            assert abs(float(out[r, 1]) - want) <= 1e-6 * (1 + abs(want)), (kw, r)
    out = torch.full((6,), 7.0)
    ops.sample_topk(lg, 0.0, 0, None, logp=out)
    assert bool((out == 0).all())


def test_filtered_logp_restatement():
    """The fp64 restatement: log of the kept-set softmax; a single kept entry is certain."""
    z = np.log(np.array([0.5, 0.2, 0.2, 0.1]))
    assert abs(filtered_logp(z, 1.0, 0, None, 3) - np.log(0.1)) < 1e-12
    assert abs(filtered_logp(z, 1.0, 0, 0.6, 1) - np.log(0.2 / 0.9)) < 1e-12
    assert filtered_logp(z, 1.0, 1, None, 0) == 0.0
    assert abs(filtered_logp(2 * z, 2.0, 2, None, 2) - np.log(0.2 / 0.9)) < 1e-12
