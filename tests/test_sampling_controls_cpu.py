"""Nucleus (top-p) sampling and image-token prompts of MakeAScene.generate, checked WITHOUT a GPU: the emulated C-ABI of
tests/test_sampling_batched_cpu.py plus an fp64 restatement of mas_sample_filtered (include/mas_b200.h). What is under test is
the host side: which sampler entry a call issues, argument checks, the prompt columns and uniforms each position receives, and
that every position is conditioned on the tokens actually emitted."""
import ctypes

import numpy as np
import pytest
import torch

from test_host_logic_cpu import _addr, _f32, _i64, _mat
from test_sampling_batched_cpu import BatchedEmu, _model, _tile


def filtered_keep(z, top_k, top_p):
    """Kept set of one row z (fp64, already divided by the temperature) under top-k then top-p, ties decided by value
    (top_k_top_p_filtering's rule: an entry is kept when the mass of kept entries with a strictly larger z is <= top_p).
    Also returns every kept-by-top-k entry's mass above, relative to the kept total."""
    z = np.asarray(z, dtype=np.float64)
    V = z.shape[0]
    keep = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        keep = z >= np.sort(z)[-top_k]
    above = np.zeros(V)
    if top_p is not None and top_p < 1:
        p = np.where(keep, np.exp(z - z.max()), 0.0)
        total = p.sum()
        uniq, inv = np.unique(z, return_inverse=True)              # ascending values
        per_value = np.bincount(inv, weights=p, minlength=uniq.shape[0])
        above = (total - np.cumsum(per_value))[inv] / total         # mass of the strictly larger values
        keep = keep & (above <= top_p)
    return keep, above


def filtered_draw(x, temperature, top_k, top_p, u):
    """Token of one row: greedy at temperature 0, else the inverse CDF over the kept set at u, in index order."""
    x = np.asarray(x, dtype=np.float64)
    if temperature == 0:
        return int(np.argmax(x))
    z = x / temperature
    keep, _ = filtered_keep(z, top_k, top_p)
    c = np.cumsum(np.where(keep, np.exp(z - z.max()), 0.0))
    return min(int(np.searchsorted(c, u * c[-1], side="right")), x.shape[0] - 1)


class ControlsEmu(BatchedEmu):
    """BatchedEmu + mas_sample_filtered; records what every sampler call received."""

    def __init__(self):
        super().__init__()
        self.draws = []

    def mas_sample_filtered(self, logits, ld, R, V, temperature, top_k, top_p, u, ptok, pmask, pld, tokens):
        X = _mat(_addr(logits), R, V, ld, False).astype(np.float64)
        uu = _f32(_addr(u), R).copy() if u is not None else None
        out = _i64(_addr(tokens), R)
        forced = {}
        for r in range(R):
            if pmask is not None and ctypes.c_uint8.from_address(_addr(pmask) + r * pld).value:
                forced[r] = ctypes.c_int64.from_address(_addr(ptok) + 8 * r * pld).value
                out[r] = forced[r]
            else:
                out[r] = filtered_draw(X[r], temperature, top_k, top_p, None if uu is None else float(uu[r]))
        self.draws.append(dict(u=uu, forced=forced, top_p=top_p, temperature=temperature))


@pytest.fixture
def emu(monkeypatch):
    from mas_b200 import ops
    e = ControlsEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: False)
    monkeypatch.setattr(ops.L, "query", lambda name, *a: 256)
    monkeypatch.setattr(torch.cuda, "graph_pool_handle", lambda: None)
    return e


def _inputs(B):
    m, g = _model("tiny")
    return m, _tile(g["text"], B), _tile(g["seg"], B), _tile(g["img"], B)


def _mask(B, L, frac, seed):
    return torch.rand(B, L, generator=torch.Generator().manual_seed(seed)) < frac


def _gen(seed=17):
    return torch.Generator().manual_seed(seed)


def test_calls_without_new_arguments_issue_the_same_entries(emu):
    """No top_p, no img_mask: mas_sample_topk once per position, never the new entry; passing the defaults explicitly, or
    top_p >= 1, changes neither the entry sequence nor the tokens."""
    m, text, seg, img = _inputs(2)
    a = m.generate(text, seg, temperature=0.9, top_k=20, generator=_gen())
    base = list(emu.names)
    assert base.count("mas_sample_topk") == m.image_length and "mas_sample_filtered" not in base
    for kw in (dict(top_p=None, img_mask=None), dict(top_p=1.0), dict(top_p=1.5)):
        emu.names.clear()
        b = m.generate(text, seg, temperature=0.9, top_k=20, generator=_gen(), **kw)
        assert emu.names == base and torch.equal(a, b), kw
    for kw in (dict(img_tokens=img), dict(temperature=0)):          # teacher forcing and greedy: no sampler entry, as before
        emu.names.clear()
        m.generate(text, seg, **kw)
        assert not [n for n in emu.names if n.startswith("mas_sample")], kw


@pytest.mark.parametrize("kw", [dict(top_p=0.8), dict(img_mask="half"), dict(top_p=0.5, img_mask="half"), dict(temperature=0, img_mask="half")])
def test_top_p_and_prompts_route_to_the_filtered_entry(emu, kw):
    m, text, seg, img = _inputs(2)
    kw = dict(kw)
    if kw.get("img_mask") == "half":
        kw.update(img_mask=_mask(2, m.image_length, 0.5, 1), img_tokens=img)
    m.generate(text, seg, generator=_gen(), **{"temperature": 0.9, **kw})
    assert emu.names.count("mas_sample_filtered") == m.image_length and "mas_sample_topk" not in emu.names
    if kw.get("temperature", 0.9) == 0:
        assert all(d["u"] is None for d in emu.draws)                 # greedy draws no uniforms


def test_argument_validation(emu):
    from mas_b200 import ops
    m, text, seg, img = _inputs(2)
    L = m.image_length
    good = torch.zeros(2, L, dtype=torch.bool)
    for bad in (0, 0.0, -0.3, float("nan")):
        with pytest.raises(ValueError):
            m.generate(text, seg, top_p=bad)
        with pytest.raises(ValueError):
            ops.sample_topk(torch.zeros(2, 8), 1.0, 0, torch.zeros(2), top_p=bad)
    cases = [dict(img_mask=good),                                                          # no img_tokens
             dict(img_tokens=img, img_mask=torch.zeros(2, L - 1, dtype=torch.bool)),        # shape
             dict(img_tokens=img, img_mask=torch.zeros(3, L, dtype=torch.bool)),
             dict(img_tokens=img, img_mask=torch.zeros(2, L, dtype=torch.uint8)),           # dtype
             dict(img_tokens=img, img_mask=good.tolist()),
             dict(img_tokens=img.int(), img_mask=good),
             dict(img_tokens=img[:, :-1], img_mask=good),
             dict(img_tokens=img, img_mask=torch.zeros(2, L, dtype=torch.bool, device="meta"))]   # device
    for kw in cases:
        with pytest.raises(ValueError):
            m.generate(text, seg, **kw)
    assert not [n for n in emu.names if n.startswith("mas_sample")]
    with pytest.raises(ValueError):
        ops.sample_topk(torch.zeros(2, 8), 1.0, 0, torch.zeros(2), prompt=(torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.uint8)))
    with pytest.raises(ValueError):
        ops.sample_topk(torch.zeros(2, 8), 1.0, 0, torch.zeros(2), prompt=(torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.bool)))


@pytest.mark.parametrize("B,scale", [(2, None), (2, 2.5), (5, 2.5), (12, None)])
def test_forced_positions_and_drawn_ones_follow_the_rule(emu, B, scale):
    """Forced positions equal T; every drawn one equals the fp64 rule on the returned (mixed, unfiltered) logits at the
    generator's uniforms; the uniforms are drawn once per position whatever the mask; with guidance and at R > 8 too."""
    m, text, seg, img = _inputs(B)
    L = m.image_length
    T = torch.randint(0, m.image_token_embedding.num_embeddings, (B, L), generator=torch.Generator().manual_seed(3))
    M = _mask(B, L, 0.4, B)
    M[0, 0], M[-1, 1] = True, False
    temp, k, p = 0.8, 40, 0.7
    gen = _gen(5)
    toks, lg = m.generate(text, seg, guidance_scale=scale, temperature=temp, top_k=k, top_p=p, generator=gen, img_tokens=T,
                          img_mask=M, return_logits=True)
    assert len(emu.draws) == L
    ref_gen = _gen(5)
    for t in range(L):
        u = torch.rand(B, generator=ref_gen)
        assert np.array_equal(emu.draws[t]["u"], u.numpy())
        assert emu.draws[t]["forced"] == {b: int(T[b, t]) for b in range(B) if M[b, t]}
        for b in range(B):
            want = int(T[b, t]) if M[b, t] else filtered_draw(lg[b, t].numpy(), temp, k, p, float(u[b]))
            assert int(toks[b, t]) == want, (t, b)
    assert torch.equal(gen.get_state(), ref_gen.get_state())
    # every position was conditioned on the tokens emitted: feeding them back reproduces the logits bit for bit
    _, lg2 = m.generate(text, seg, guidance_scale=scale, img_tokens=toks, return_logits=True)
    assert torch.equal(lg2, lg)


@pytest.mark.parametrize("B,scale", [(2, 2.5), (10, None)])
def test_all_false_and_all_true_masks(emu, B, scale):
    """An all-false mask gives the unprompted call's tokens and logits with the same generator (and leaves the generator in
    the same state); an all-true mask gives teacher forcing by img_tokens."""
    m, text, seg, img = _inputs(B)
    L = m.image_length
    kw = dict(guidance_scale=scale, temperature=0.9, top_k=30, top_p=0.85, return_logits=True)
    g1, g2 = _gen(9), _gen(9)
    a, la = m.generate(text, seg, generator=g1, **kw)
    b, lb = m.generate(text, seg, generator=g2, img_tokens=img, img_mask=torch.zeros(B, L, dtype=torch.bool), **kw)
    assert torch.equal(a, b) and torch.equal(la, lb) and torch.equal(g1.get_state(), g2.get_state())
    c, lc = m.generate(text, seg, generator=_gen(9), img_tokens=img, img_mask=torch.ones(B, L, dtype=torch.bool), **kw)
    d, ld = m.generate(text, seg, guidance_scale=scale, img_tokens=img, return_logits=True)
    assert torch.equal(c, img) and torch.equal(d, img) and torch.equal(lc, ld)


def test_uniform_stream_does_not_depend_on_the_mask(emu):
    """Two different masks consume the same uniforms: the rows' draws at positions both masks leave open see the same u."""
    m, text, seg, img = _inputs(3)
    L = m.image_length
    us = []
    for seed in (1, 2):
        emu.draws.clear()
        g = _gen(4)
        m.generate(text, seg, temperature=1.0, generator=g, img_tokens=img, img_mask=_mask(3, L, 0.5, seed))
        us.append(np.stack([d["u"] for d in emu.draws]))
        assert torch.equal(g.get_state(), _advance(_gen(4), 3, L).get_state())
    assert us[0].shape == (L, 3) and np.array_equal(us[0], us[1])


def _advance(g, B, L):
    for _ in range(L):
        torch.rand(B, generator=g)
    return g


def test_filtered_keep_rule():
    """The fp64 restatement itself: ties at the boundary kept or dropped together, the top entry always kept."""
    z = np.log(np.array([0.5, 0.2, 0.2, 0.1]))
    keep, above = filtered_keep(z, 0, 0.6)
    assert keep.tolist() == [True, True, True, False] and np.allclose(above, [0, 0.5, 0.5, 0.9])
    keep, _ = filtered_keep(z, 0, 0.4)
    assert keep.tolist() == [True, False, False, False]
    keep, _ = filtered_keep(z, 2, 0.99)                         # top-k keeps the tie with the 2nd largest: 3 entries
    assert keep.tolist() == [True, True, True, False]
    assert filtered_keep(np.array([3.0, 0.0]), 0, 1e-9)[0].tolist() == [True, False]
