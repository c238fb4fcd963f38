"""Per-row sampling controls and seeds on the GPU: mas_sample_rows against mas_sample_filtered_logp run row by row, the seeded
uniforms against the numpy Philox restatement, mas_cfg_mix_rows against mas_cfg_mix, and MakeAScene.generate / score with
per-row values against the scalar calls, bit for bit. Every per-row route is asserted from the library's launch trace."""
import numpy as np
import pytest
import torch

from test_gpu_sampling_logprobs import _gen, _load_model, _tile
from test_sampling_rows_cpu import seeded_uniform

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _bits(x):
    return x.contiguous().view(torch.int32)


def _row_logits(R, V, seed):
    """R rows of random logits, with rows of ties (a coarse grid, also at the maximum) and one dominant entry among them."""
    g = torch.Generator().manual_seed(seed)
    lg = torch.randn(R, V, generator=g) * 2.5
    lg[1::7] = torch.randint(0, 12, (len(range(1, R, 7)), V), generator=g).float() * 0.5
    lg[3::11, 5] = lg[3::11].max(1).values + 30.0
    return lg


def _controls(R, V, seed):
    """Per-row temperature {0, 0.7, 1, 1.3}, top_k {0, 1, 50, V}, top_p {off, 0.9, 0.5} in a mixed order, and a prompt mask."""
    g = torch.Generator().manual_seed(seed)
    T = torch.tensor([0.0, 0.7, 1.0, 1.3])[torch.randint(0, 4, (R,), generator=g)]
    K = torch.tensor([0, 1, 50, V], dtype=torch.int32)[torch.randint(0, 4, (R,), generator=g)]
    P = torch.tensor([1.0, 0.9, 0.5])[torch.randint(0, 3, (R,), generator=g)]
    ptok = torch.randint(0, V, (R,), generator=g)
    pmask = torch.rand(R, generator=g) < 0.15
    return T, K, P, ptok, pmask


@pytest.mark.parametrize("V", [8192, 5001])
@pytest.mark.parametrize("R", [1, 8, 256])
def test_sample_rows_is_the_scalar_entry_row_by_row(R, V):
    """Tokens equal and logp bitwise equal to mas_sample_filtered_logp called on each row alone with that row's values,
    greedy rows, prompt rows and rows of ties included; one launch, named sample_rows."""
    from mas_b200 import _lib, ops
    lg = _row_logits(R, V, R + V).to(DEV)
    T, K, P, ptok, pmask = (t.to(DEV) for t in _controls(R, V, 3 * R + V))
    u = torch.rand(R, generator=torch.Generator().manual_seed(V)).to(DEV)
    lp = torch.full((R, 3), float("nan"), device=DEV)
    with _lib.launch_trace() as names:
        tok = ops.sample_rows(lg, T, K, P, u=u, prompt=(ptok, pmask), logp=lp[:, 1])
        torch.cuda.synchronize()
    assert names == ["sample_rows"]
    assert bool(lp[:, [0, 2]].isnan().all())
    ref_tok = torch.empty(R, dtype=torch.int64, device=DEV)
    ref_lp = torch.empty(R, device=DEV)
    with _lib.launch_trace() as names:
        for r in range(R):
            ref_tok[r:r + 1] = ops.sample_topk(lg[r:r + 1], float(T[r]), int(K[r]), u[r:r + 1], top_p=float(P[r]),
                                               prompt=(ptok[r:r + 1], pmask[r:r + 1]), logp=ref_lp[r:r + 1])
        torch.cuda.synchronize()
    assert names == ["sample_filtered_logp"] * R
    assert torch.equal(tok, ref_tok) and torch.equal(_bits(lp[:, 1]), _bits(ref_lp))
    assert torch.equal(tok[pmask], ptok[pmask]) and bool((lp[pmask | (T == 0), 1] == 0).all())
    if R == 256:
        assert bool((lp[~pmask & (T > 0), 1] < 0).any())
    nolp = ops.sample_rows(lg, T, K, P, u=u, prompt=(ptok, pmask))
    assert torch.equal(nolp, tok)


@pytest.mark.parametrize("position", [0, 255, 2 ** 33 + 5])
def test_seeded_draw_equals_the_numpy_philox_uniforms(position):
    """With seeds at a position, the tokens and logp are those of the u entry fed the numpy restatement's uniforms for those
    seeds, bit for bit; equal seeds on equal rows give equal tokens wherever the rows sit."""
    from mas_b200 import _lib, ops
    R, V = 256, 8192
    lg = _row_logits(R, V, 5).to(DEV)
    lg[200:] = lg[0]                                      # rows 200.. repeat row 0 ...
    T, K, P, ptok, pmask = (t.to(DEV) for t in _controls(R, V, 9))
    T[200:], K[200:], P[200:], pmask[200:] = 1.0, 0, 1.0, False
    T[0], K[0], P[0], pmask[0] = 1.0, 0, 1.0, False
    g = torch.Generator().manual_seed(int(position) % 1000)
    seeds = torch.randint(-2 ** 62, 2 ** 62, (R,), generator=g, dtype=torch.int64)
    seeds[200:] = seeds[0]                                # ... with row 0's seed
    u = torch.tensor([seeded_uniform(int(s), position) for s in seeds], dtype=torch.float32)
    assert bool(((u >= 0) & (u < 1)).all())
    sd, u = seeds.to(DEV), u.to(DEV)
    lp_s, lp_u = torch.empty(R, device=DEV), torch.empty(R, device=DEV)
    with _lib.launch_trace() as names:
        tok_s = ops.sample_rows(lg, T, K, P, seeds=sd, position=position, prompt=(ptok, pmask), logp=lp_s)
        torch.cuda.synchronize()
    assert names == ["sample_rows"]
    tok_u = ops.sample_rows(lg, T, K, P, u=u, prompt=(ptok, pmask), logp=lp_u)
    assert torch.equal(tok_s, tok_u) and torch.equal(_bits(lp_s), _bits(lp_u))
    assert bool((tok_s[200:] == tok_s[0]).all())
    perm = torch.randperm(R, generator=g).to(DEV)       # the rows moved: each keeps its token
    tok_p = ops.sample_rows(lg[perm], T[perm], K[perm], P[perm], seeds=sd[perm], position=position, prompt=(ptok[perm], pmask[perm]))
    assert torch.equal(tok_p, tok_s[perm])


@pytest.mark.parametrize("V", [8192, 5001])
@pytest.mark.parametrize("R", [1, 8, 256])
def test_cfg_mix_rows_is_cfg_mix_per_row(R, V):
    from mas_b200 import _lib, ops
    g = torch.Generator().manual_seed(R * V)
    cond, uncond = (torch.randn(R, V, generator=g) * 3).to(DEV), (torch.randn(R, V, generator=g) * 3).to(DEV)
    scale = torch.cat([torch.tensor([1.0, 0.0, -1.5, 3.0]), torch.rand(max(R - 4, 0), generator=g) * 8 - 1])[:R].to(DEV)
    with _lib.launch_trace() as names:
        out = ops.cfg_mix_rows(cond, uncond, scale)
        torch.cuda.synchronize()
    assert names == ["cfg_mix_rows"]
    for r in range(R):
        assert torch.equal(_bits(out[r]), _bits(ops.cfg_mix(cond[r], uncond[r], float(scale[r])))), r


def _prompt(m, rows, seed):
    g = torch.Generator().manual_seed(seed)
    V = m.image_token_embedding.num_embeddings
    return (torch.randint(0, V, (rows, m.image_length), generator=g).to(DEV),
            (torch.rand(rows, m.image_length, generator=g) < 0.25).to(DEV))


# (B, n, scale): 8 decode rows (fp32) and 64 (fp16), guided (2 B n rows) and not, num_samples 1 and 4
SAME_VALUE = [(1, 4, 2.0), (2, 4, None), (4, 1, 2.0), (8, 1, None), (8, 4, 2.0), (16, 4, None), (32, 1, 2.0), (64, 1, None)]


@pytest.mark.parametrize("B,n,scale", SAME_VALUE)
def test_generate_with_per_row_tensors_of_one_value_is_the_scalar_call(B, n, scale):
    """Tokens, logits and log p bit for bit equal to the scalar call, eager and with use_graphs (capture and replay); the
    per-row call draws with sample_rows and mixes with cfg_mix_rows, the scalar call with the entries of before."""
    from mas_b200 import _lib
    m, g = _load_model()
    Bn = B * n
    text, seg = _tile(g["text"], B), _tile(g["seg"], B)
    T, M = _prompt(m, Bn, Bn)
    kw = dict(num_samples=n, img_tokens=T, img_mask=M, return_logits=True, return_logprobs=True)
    scalar = dict(temperature=0.9, top_k=40, top_p=0.9, guidance_scale=scale)
    rows = dict(temperature=torch.full((Bn,), 0.9, device=DEV), top_k=torch.full((Bn,), 40, device=DEV, dtype=torch.int64),
                top_p=[0.9] * Bn, guidance_scale=torch.full((Bn,), scale or 1.0, device=DEV))
    with _lib.launch_trace() as names_s:
        want = m.generate(text, seg, generator=_gen(), **scalar, **kw)
        torch.cuda.synchronize()
    with _lib.launch_trace() as names_r:
        got = m.generate(text, seg, generator=_gen(), **rows, **kw)
        torch.cuda.synchronize()
    L = m.image_length
    assert names_r.count("sample_rows") == L and "sample_filtered_logp" not in names_r and "cfg_mix" not in names_r
    assert names_r.count("cfg_mix_rows") == (L if scale else 0)
    assert names_s.count("sample_filtered_logp") == L and "sample_rows" not in names_s and "cfg_mix_rows" not in names_s
    for a, b in zip(want, got):
        assert torch.equal(_bits(a.float()) if a.is_floating_point() else a, _bits(b.float()) if b.is_floating_point() else b)
    for _ in range(2):
        gr = m.generate(text, seg, generator=_gen(), use_graphs=True, **rows, **kw)
        assert all(torch.equal(a, b) for a, b in zip(gr, want))
    m.reset_sampler()
    greedy_s = m.generate(text, seg, temperature=0, guidance_scale=scale, **kw)
    greedy_r = m.generate(text, seg, temperature=torch.zeros(Bn, device=DEV), guidance_scale=scale, **kw)
    assert all(torch.equal(a, b) for a, b in zip(greedy_s, greedy_r))


def test_seeded_sweep_rows_equal_the_scalar_calls():
    """B = 1, num_samples = 4, guided (8 fp32 decode rows): each sample its own guidance scale and temperature, all four the
    same seed. Sample j is bit for bit sample j of the scalar call at its settings with the same seeds: the prefix is shared
    and fp32 decoding computes every row on its own."""
    from mas_b200 import _lib
    m, g = _load_model()
    text, seg = g["text"][:1].to(DEV), g["seg"][:1].to(DEV)
    scales, temps = [1.5, 2.0, 3.0, 5.0], [0.7, 1.0, 1.3, 1.0]
    seeds = torch.full((4,), 1234, dtype=torch.int64, device=DEV)
    kw = dict(num_samples=4, top_k=40, top_p=0.9, seeds=seeds, return_logits=True, return_logprobs=True)
    with _lib.launch_trace() as names:
        toks, lg, lp = m.generate(text, seg, guidance_scale=torch.tensor(scales, device=DEV), temperature=temps, **kw)
        torch.cuda.synchronize()
    assert names.count("sample_rows") == m.image_length and names.count("cfg_mix_rows") == m.image_length
    for j in range(4):
        t_s, lg_s, lp_s = m.generate(text, seg, guidance_scale=scales[j], temperature=temps[j], **kw)
        assert all(torch.equal(t_s[i], t_s[0]) for i in range(4))          # one seed, one setting: four equal samples
        assert torch.equal(toks[j], t_s[j]) and torch.equal(_bits(lp[j]), _bits(lp_s[j])) and torch.equal(lg[j], lg_s[j]), j
    assert len({tuple(toks[j].tolist()) for j in range(4)}) > 1
    again = m.generate(text, seg, guidance_scale=torch.tensor(scales, device=DEV), temperature=temps, **kw)
    assert all(torch.equal(a, b) for a, b in zip(again, (toks, lg, lp)))


@pytest.mark.parametrize("B,n", [(2, 2), (8, 2)])
def test_teacher_forced_generate_with_per_row_guidance(B, n):
    """img_tokens given (nothing drawn): the returned logits of each row are those of the scalar-guidance call at its scale,
    bit for bit, at 8 (fp32) and 32 (fp16) decode rows. A row at scale 1 in a guided call is within rounding of the
    unguided call where both decode in fp32."""
    from mas_b200 import _lib
    m, g = _load_model()
    Bn = B * n
    text, seg = _tile(g["text"], B), _tile(g["seg"], B)
    img = _prompt(m, Bn, 7)[0]
    scales = [1.5, 2.5, 0.5, 4.0] * (Bn // 4)
    with _lib.launch_trace() as names:
        _, lg = m.generate(text, seg, num_samples=n, img_tokens=img, guidance_scale=torch.tensor(scales, device=DEV), return_logits=True)
        torch.cuda.synchronize()
    assert names.count("cfg_mix_rows") == m.image_length and "cfg_mix" not in names and "sample_rows" not in names
    for s in sorted(set(scales)):
        _, lg_s = m.generate(text, seg, num_samples=n, img_tokens=img, guidance_scale=s, return_logits=True)
        for r in range(Bn):
            if scales[r] == s:
                assert torch.equal(_bits(lg[r]), _bits(lg_s[r])), (s, r)
    if 2 * Bn <= 8:
        one = [1.0] + scales[1:]
        _, lg1 = m.generate(text, seg, num_samples=n, img_tokens=img, guidance_scale=one, return_logits=True)
        _, lgu = m.generate(text, seg, num_samples=n, img_tokens=img, return_logits=True)
        err = float((lg1[0] - lgu[0]).abs().max())
        print("scale-1 row of a guided call vs the unguided call: max |d logit| %.3e (max |logit| %.3e)" % (err, float(lgu[0].abs().max())))
        assert err <= 1e-5 * float(lgu[0].abs().max())


def test_score_with_per_row_scales():
    """score with a [B] scale tensor: row b is bit for bit the row of the call at scale[b]; one cfg_mix_rows launch."""
    from mas_b200 import _lib
    m, g = _load_model()
    B = 6
    text, seg = _tile(g["text"], B), _tile(g["seg"], B)
    img = _prompt(m, B, 11)[0]
    scales = [1.5, 2.5, 0.5, 4.0, 1.5, -1.0]
    with _lib.launch_trace() as names:
        lp = m.score(text, seg, img, guidance_scale=torch.tensor(scales, device=DEV))
        torch.cuda.synchronize()
    assert names.count("cfg_mix_rows") == 1 and "cfg_mix" not in names
    for b, s in enumerate(scales):
        assert torch.equal(_bits(lp[b]), _bits(m.score(text, seg, img, guidance_scale=s)[b])), b
    assert torch.equal(m.score(text, seg, img, guidance_scale=torch.ones(B, device=DEV)), m.score(text, seg, img))
    assert np.isfinite(lp.cpu().numpy()).all()
