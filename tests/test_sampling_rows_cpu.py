"""Per-row sampling controls and seeds of MakeAScene.generate / score, checked WITHOUT a GPU: the emulated C-ABI of
tests/test_sampling_logprobs_cpu.py plus fp64 restatements of mas_sample_rows and mas_cfg_mix_rows (include/mas_b200.h), whose
seeded uniforms come from the numpy Philox4x32-10 of tests/test_dropout_cpu.py. What is under test is the host side: scalar
calls issue the entries they always did, per-row calls route every position to the new entries with one value per output
row, validation happens before any call, and the seeded uniform of a row depends on its seed and the position alone."""
import ctypes

import numpy as np
import pytest
import torch

from test_dropout_cpu import philox4x32_10
from test_host_logic_cpu import _addr, _f32, _i64, _mat
from test_sampling_batched_cpu import _model, _tile
from test_sampling_controls_cpu import filtered_draw
from test_sampling_logprobs_cpu import LogpEmu, filtered_logp

NEW = ("mas_sample_rows", "mas_cfg_mix_rows")
SAMPLERS = ("mas_sample_topk", "mas_sample_filtered", "mas_sample_filtered_logp", "mas_sample_rows")


def seeded_uniform(seed, position):
    """mas_sample_rows' uniform of a row with this int64 seed at this position: (word0 >> 8) * 2^-24 of Philox4x32-10 with
    counter (lo32(position), hi32(position), 0, 0) and key (lo32(seed), hi32(seed))."""
    s, p = int(seed) & 0xFFFFFFFFFFFFFFFF, int(position) & 0xFFFFFFFFFFFFFFFF
    w = philox4x32_10([p & 0xFFFFFFFF, p >> 32, 0, 0], [s & 0xFFFFFFFF, s >> 32])
    return float(np.float32(int(w[0]) >> 8) * np.float32(2.0 ** -24))


class RowsEmu(LogpEmu):
    """LogpEmu + mas_sample_rows (each row the fp64 rule at its own values; u or the seeded uniforms) and mas_cfg_mix_rows;
    records what every per-row call received."""

    def __init__(self):
        super().__init__()
        self.rows = []
        self.mixes = []

    def mas_sample_rows(self, logits, ld, R, V, temperature, top_k, top_p, u, seeds, position, ptok, pmask, pld, tokens, logp,
                        logp_ld):
        assert (u is None) != (seeds is None)
        X = _mat(_addr(logits), R, V, ld, False).astype(np.float64)
        T = _f32(_addr(temperature), R).astype(np.float64)
        K = np.ctypeslib.as_array((ctypes.c_int32 * R).from_address(_addr(top_k))).copy()
        P = _f32(_addr(top_p), R).astype(np.float64)
        sd = None if seeds is None else _i64(_addr(seeds), R).copy()
        uu = _f32(_addr(u), R).astype(np.float64) if u is not None else np.array([seeded_uniform(s, position) for s in sd])
        out = _i64(_addr(tokens), R)
        forced = {}
        for r in range(R):
            p = None if P[r] >= 1 else float(P[r])
            if pmask is not None and ctypes.c_uint8.from_address(_addr(pmask) + r * pld).value:
                forced[r] = out[r] = ctypes.c_int64.from_address(_addr(ptok) + 8 * r * pld).value
                v = 0.0
            else:
                out[r] = filtered_draw(X[r], float(T[r]), int(K[r]), p, float(uu[r]))
                v = 0.0 if T[r] == 0 else filtered_logp(X[r], float(T[r]), int(K[r]), p, int(out[r]))
            if logp is not None:
                ctypes.c_float.from_address(_addr(logp) + 4 * r * logp_ld).value = v
        self.rows.append(dict(temperature=T, top_k=K, top_p=P, u=uu, seeds=sd, position=position, forced=forced,
                              logp=None if logp is None else (_addr(logp), logp_ld)))

    def mas_cfg_mix_rows(self, cond, uncond, out, R, V, scale):
        s = _f32(_addr(scale), R).astype(np.float64)
        u = _f32(_addr(uncond), R * V).reshape(R, V).astype(np.float64)
        _f32(_addr(out), R * V).reshape(R, V)[...] = u + s[:, None] * (_f32(_addr(cond), R * V).reshape(R, V) - u)
        self.mixes.append(dict(R=R, V=V, scale=s))


@pytest.fixture
def emu(monkeypatch):
    from mas_b200 import ops
    e = RowsEmu()
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


def _mask(rows, L, frac, seed):
    return torch.rand(rows, L, generator=torch.Generator().manual_seed(seed)) < frac


def test_seeded_uniform_rule():
    """Random123's known answer (counter 0, key 0: word0 0x6627e8d5) gives the first uniform of seed 0; the uniforms lie in
    [0, 1), differ between seeds and positions, and a negative seed is its two's complement."""
    assert seeded_uniform(0, 0) == 0x6627E8 * 2.0 ** -24
    us = np.array([[seeded_uniform(s, t) for t in range(64)] for s in (0, 1, 2 ** 40 + 3, -5)])
    assert ((us >= 0) & (us < 1)).all() and len(np.unique(us)) == us.size
    assert seeded_uniform(-5, 3) == seeded_uniform(2 ** 64 - 5, 3) != seeded_uniform(5, 3)


SCALAR_CONFIGS = [dict(temperature=0.9, top_k=20), dict(temperature=0.8, top_p=0.7, guidance_scale=2.5),
                  dict(temperature=1.0, img_mask=0.5, guidance_scale=2.0, num_samples=2), dict(temperature=0, img_mask=0.5),
                  dict(temperature=0), dict(img_tokens=True, guidance_scale=3.0), dict(temperature=0.9, top_k=20, num_samples=3),
                  dict(temperature=0.9, guidance_scale=1.0)]


def _kw(kw, m, B, img):
    kw = dict(kw)
    rows = B * kw.get("num_samples", 1)
    if "img_mask" in kw:
        kw.update(img_mask=_mask(rows, m.image_length, kw["img_mask"], 1), img_tokens=_tile(img, rows))
    elif kw.get("img_tokens") is True:
        kw["img_tokens"] = _tile(img, rows)
    return kw


@pytest.mark.parametrize("logprobs", [False, True])
@pytest.mark.parametrize("kw", SCALAR_CONFIGS)
def test_scalar_calls_issue_the_entries_of_before(emu, kw, logprobs):
    """Scalars only, no seeds: never a new entry; one scalar sampler call per drawn position with the call's scalars (the
    routing of before: mas_sample_topk, _filtered or _filtered_logp, or none for greedy and teacher forcing), one mas_cfg_mix
    per position when guided; passing seeds=None changes nothing."""
    m, text, seg, img = _inputs(2)
    kw = _kw(kw, m, 2, img)
    a = m.generate(text, seg, generator=_gen(), return_logprobs=logprobs, **kw)
    base = list(emu.names)
    assert not [x for x in base if x in NEW]
    L = m.image_length
    guided = kw.get("guidance_scale") not in (None, 1.0)
    assert base.count("mas_cfg_mix") == (L if guided else 0)
    samplers = [x for x in base if x in SAMPLERS]
    if "img_mask" not in kw and ("img_tokens" in kw or not kw.get("temperature", 1.0)):
        assert samplers == []                                   # teacher forcing and greedy: no sampler entry
    else:
        want = ("mas_sample_filtered_logp" if logprobs else
                "mas_sample_filtered" if "top_p" in kw or "img_mask" in kw else "mas_sample_topk")
        assert samplers == [want] * L
    for name, args in emu.args:
        if name in SAMPLERS:
            assert isinstance(args[4], float) and abs(args[4] - float(kw.get("temperature", 1.0))) < 1e-12
    emu.names.clear()
    b = m.generate(text, seg, generator=_gen(), return_logprobs=logprobs, seeds=None, **kw)
    assert emu.names == base
    for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("B,n", [(2, 3), (3, 1)])
def test_per_row_calls_route_every_position(emu, B, n):
    """Per-row temperature, top_k, top_p and guidance: every position issues one mas_cfg_mix_rows over the B*n cond rows
    against their B*n uncond rows with each row's own scale, then one mas_sample_rows with the arrays laid out per output row;
    no scalar sampler or mix. Every drawn token is the fp64 rule on the returned (mixed) logits at that row's values and the
    generator's uniforms; forced positions keep their tokens; log p is that row's."""
    m, text, seg, img = _inputs(B)
    L, V, Bn = m.image_length, m.image_token_embedding.num_embeddings, B * n
    temps = [0.0, 0.7, 1.0, 1.3, 0.9, 1.1][:Bn]
    ks = [0, 1, 50, V, 7, 0][:Bn]
    ps = [1.0, 0.9, 0.5, 0.8, 2.0, 0.7][:Bn]
    scales = [2.5, 1.0, 3.0, 0.5, 2.0, 4.0][:Bn]
    T = _tile(img, Bn)
    M = _mask(Bn, L, 0.3, 5)
    toks, lg, lp = m.generate(text, seg, num_samples=n, temperature=torch.tensor(temps), top_k=ks, top_p=torch.tensor(ps),
                              guidance_scale=torch.tensor(scales, dtype=torch.float64), generator=_gen(3), img_tokens=T, img_mask=M,
                              return_logits=True, return_logprobs=True)
    assert not [x for x in emu.names if x in ("mas_cfg_mix", "mas_sample_topk", "mas_sample_filtered", "mas_sample_filtered_logp")]
    assert emu.names.count("mas_sample_rows") == L and emu.names.count("mas_cfg_mix_rows") == L
    assert all(d["R"] == Bn and d["V"] == V and np.array_equal(d["scale"], np.float32(scales)) for d in emu.mixes)
    ref_gen = _gen(3)
    for t, d in enumerate(emu.rows):
        assert d["position"] == t and d["seeds"] is None
        assert np.array_equal(d["temperature"], np.float32(temps)) and d["top_k"].tolist() == ks
        assert np.array_equal(d["top_p"], np.float32(ps))
        u = torch.rand(Bn, generator=ref_gen)
        assert np.array_equal(d["u"], u.double().numpy())
        assert d["logp"] == (lp.data_ptr() + 4 * t, L)
        for r in range(Bn):
            if M[r, t]:
                assert int(toks[r, t]) == int(T[r, t]) and float(lp[r, t]) == 0.0
                continue
            p = None if ps[r] >= 1 else ps[r]
            want = filtered_draw(lg[r, t].numpy(), float(np.float32(temps[r])), ks[r], p, float(u[r]))
            assert int(toks[r, t]) == want, (t, r)
            if temps[r] > 0:
                lw = filtered_logp(lg[r, t].numpy(), float(np.float32(temps[r])), ks[r], p, want)
                assert abs(float(lp[r, t]) - lw) <= 1e-6 * (1 + abs(lw))
    # the mix of each row is the scalar call's at that row's scale (teacher forcing: the same rows, only the mix differs). A
    # row at scale 1 is fmaf(1, c - u, u) of a guided call's 2 B n rows: the unguided call's logits to rounding while both
    # decode at the same precision (2 B n <= 8); above 8 rows the guided call decodes in fp16 and the unguided one may not.
    _, lg_rows = m.generate(text, seg, num_samples=n, img_tokens=T, guidance_scale=scales, return_logits=True)
    for r in range(Bn):
        _, lg_s = m.generate(text, seg, num_samples=n, img_tokens=T, guidance_scale=scales[r], return_logits=True)
        if scales[r] != 1.0:
            assert torch.equal(lg_rows[r], lg_s[r]), r
        elif 2 * Bn <= 8:
            assert float((lg_rows[r] - lg_s[r]).abs().max()) <= 1e-6 * float(lg_s[r].abs().max()), r


@pytest.mark.parametrize("scale", [None, 2.0])
@pytest.mark.parametrize("B,n", [(2, 1), (2, 3), (10, 1)])
def test_per_row_tensors_of_one_value_equal_the_scalar_call(emu, B, n, scale):
    """Tensors that hold the scalar's value in every row: the same tokens, logits, log p and generator state as the scalar
    call, at up to 8 and above 8 decode rows; a guidance tensor of ones is the unguided call."""
    m, text, seg, img = _inputs(B)
    Bn = B * n
    kw = dict(num_samples=n, return_logits=True, return_logprobs=True, img_tokens=_tile(img, Bn),
              img_mask=_mask(Bn, m.image_length, 0.3, 2))
    g1, g2 = _gen(8), _gen(8)
    # values exact in fp32: the emulated scalar entries compute with the Python float, the kernel with its fp32 rounding
    a = m.generate(text, seg, temperature=0.875, top_k=30, top_p=0.75, guidance_scale=scale, generator=g1, **kw)
    emu.names.clear()
    b = m.generate(text, seg, temperature=torch.full((Bn,), 0.875), top_k=torch.full((Bn,), 30, dtype=torch.int64),
                   top_p=[0.75] * Bn, guidance_scale=torch.full((Bn,), scale or 1.0), generator=g2, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and torch.equal(g1.get_state(), g2.get_state())
    assert ("mas_cfg_mix_rows" in emu.names) == (scale is not None) and "mas_cfg_mix" not in emu.names
    g3 = _gen(8)
    c = m.generate(text, seg, temperature=torch.zeros(Bn), guidance_scale=scale, generator=g3, **kw)
    d = m.generate(text, seg, temperature=0, guidance_scale=scale, **kw)
    assert all(torch.equal(x, y) for x, y in zip(c, d)) and torch.equal(g3.get_state(), _gen(8).get_state())   # greedy draws no u


def test_seeds_give_each_row_its_own_stream(emu):
    """With seeds every position's uniforms are seeded_uniform(seed, t) of each row (no generator is read); a row's tokens
    depend on its seed, not on its place in the batch or on the other rows: rows with equal seeds and settings are equal,
    and reordering the prompts' seeds reorders the rows."""
    m, text, seg, img = _inputs(2)
    L, n = m.image_length, 3
    seeds = torch.tensor([11, 11, -4, 11, 2 ** 40, 7], dtype=torch.int64)
    kw = dict(num_samples=n, temperature=1.0, top_k=0, return_logprobs=True)
    toks, lp = m.generate(text, seg, seeds=seeds, **kw)
    assert emu.names.count("mas_sample_rows") == L
    for t, d in enumerate(emu.rows):
        assert d["position"] == t and d["seeds"].tolist() == seeds.tolist()
        assert d["u"].tolist() == [seeded_uniform(s, t) for s in seeds.tolist()]
    assert torch.equal(toks[0], toks[1]) and torch.equal(lp[0], lp[1])
    same_prompt = text[:1].repeat(2, 1), seg[:1].repeat(2, 1)
    perm = torch.tensor([4, 5, 0, 1, 2, 3])
    t2, _ = m.generate(*same_prompt, seeds=seeds[perm], **kw)
    t1, _ = m.generate(*same_prompt, seeds=seeds, **kw)
    assert torch.equal(t2, t1[perm])
    t3, _ = m.generate(text[:1], seg[:1], seeds=seeds[:3], **kw)          # fewer rows: the same rows
    assert torch.equal(t3, toks[:3])


def test_validation_before_any_call(emu):
    m, text, seg, img = _inputs(2)
    n, Bn = 2, 4
    bad = [dict(temperature=torch.ones(Bn + 1)), dict(temperature=torch.ones(Bn, dtype=torch.int64)),
           dict(temperature=torch.ones(Bn, device="meta")), dict(temperature=torch.ones(2, 2)), dict(temperature=[1.0] * 3),
           dict(temperature=torch.tensor([1.0, -0.1, 1.0, 1.0])), dict(temperature=[1.0, float("inf"), 1.0, 1.0]),
           dict(temperature=[1.0, float("nan"), 1.0, 1.0]), dict(temperature=["a"] * Bn),
           dict(top_k=torch.tensor([1, 2, -1, 0])), dict(top_k=torch.ones(Bn)), dict(top_k=[1, 2, 3, 4.5]), dict(top_k=[True] * Bn),
           dict(top_p=torch.tensor([0.5, 0.0, 1.0, 1.0])), dict(top_p=[0.5, -0.2, 1.0, 1.0]), dict(top_p=[0.5, float("nan"), 1.0, 1.0]),
           dict(top_p=torch.ones(Bn, dtype=torch.int32)),
           dict(guidance_scale=torch.tensor([1.0, float("inf"), 2.0, 2.0])), dict(guidance_scale=[2.0, float("nan"), 2.0, 2.0]),
           dict(guidance_scale=torch.ones(Bn - 1)), dict(guidance_scale=torch.ones(Bn, dtype=torch.int64)),
           dict(seeds=torch.zeros(Bn, dtype=torch.int32)), dict(seeds=torch.zeros(Bn + 1, dtype=torch.int64)),
           dict(seeds=[1, 2, 3, 4]), dict(seeds=torch.zeros(Bn, dtype=torch.int64, device="meta")),
           dict(seeds=torch.zeros(Bn, dtype=torch.int64), generator=_gen()),
           dict(seeds=torch.zeros(Bn, dtype=torch.int64), temperature=-1.0), dict(top_k=[1] * Bn, top_p=0.0)]
    for kw in bad:
        with pytest.raises(ValueError):
            m.generate(text, seg, num_samples=n, **kw)
        assert emu.names == [], kw
    for s in (torch.ones(3), torch.tensor([2.0, float("nan")]), torch.ones(2, dtype=torch.int64), torch.ones(2, device="meta"), [2.0]):
        with pytest.raises(ValueError):
            m.score(text, seg, img, guidance_scale=s)
        assert emu.names == [], s
    from mas_b200 import ops
    lg = torch.zeros(2, 8)
    ctl = (torch.ones(2), torch.zeros(2, dtype=torch.int32), torch.ones(2))
    for kw in (dict(), dict(u=torch.zeros(2), seeds=torch.zeros(2, dtype=torch.int64)), dict(u=torch.zeros(3)),
               dict(seeds=torch.zeros(2, dtype=torch.int32))):
        with pytest.raises(ValueError):
            ops.sample_rows(lg, *ctl, **kw)
    with pytest.raises(ValueError):
        ops.sample_rows(lg, torch.ones(2), torch.zeros(2, dtype=torch.int64), torch.ones(2), u=torch.zeros(2))
    with pytest.raises(ValueError):
        ops.cfg_mix_rows(lg, lg, torch.ones(3))
    assert emu.names == []


def test_score_with_per_row_scales(emu):
    """One pass, one mas_cfg_mix_rows over the [B, L*V] halves with each row's scale; row b equals the scalar call at
    scale[b]; a tensor of ones is the unguided score."""
    B = 3
    m, text, seg, img = _inputs(B)
    L, V = m.image_length, m.image_token_embedding.num_embeddings
    scales = [2.5, 0.5, 4.0]
    lp = m.score(text, seg, img, guidance_scale=torch.tensor(scales))
    assert emu.names.count("mas_cfg_mix_rows") == 1 and "mas_cfg_mix" not in emu.names and emu.names[-1] == "mas_ce_forward"
    assert emu.mixes[-1]["R"] == B and emu.mixes[-1]["V"] == L * V
    for b, s in enumerate(scales):
        assert torch.equal(lp[b], m.score(text, seg, img, guidance_scale=s)[b]), b
    assert torch.equal(m.score(text, seg, img, guidance_scale=[1.0] * B), m.score(text, seg, img))
