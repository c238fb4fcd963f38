"""Per-token log-probabilities on the GPU: mas_sample_filtered_logp against an fp64 restatement of the draw's distribution,
MakeAScene.generate(return_logprobs=True) at fp32 and fp16 decoding, MakeAScene.score against the real reference's logits,
and the two routes against each other.

Error bound of the kernel's log p (fp32, u = 2^-24), from z = logits / temperature as the kernel computes them (fp32
quotients, fed to the fp64 reference as they are) and D = the largest mx - z over the kept set: z_tok - mx is rounded once
(u D); each kept term exp(z - mx) carries the rounding of its exponent (u D, relative) and expf's 2 ulp; the kept-set sum
adds per + 256 terms in sequence (per = ceil(V / 256) in a thread, then the 256 partials), (per + 256) u relative; logf
and the last subtraction add u log V and u |log p|. Twice the first-order sum:
    |log p - ref| <= 2 u (2 D + 2 + per + 256 + log V + |ref|).
score and generate against the reference: |d log p_t| <= |d z_t[tok]| + |d logsumexp z_t| <= 2 ||d z_t||_2, so over a
tensor ||d log p|| <= 2 ||d z||_F; logits that agree to 2e-3 relative (test_generate_teacher_forced_matches_reference_logits)
give ||d log p|| <= 4e-3 ||z||_F, and for the guided mix u + s (c - u) 4e-3 (|1 - s| ||u||_F + |s| ||c||_F)."""
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from test_sampling_controls_cpu import filtered_keep

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
R = 64
U = 2.0 ** -24
AMBIGUOUS = 1e-6      # an entry whose mass above lies this close to top_p may be decided either way (2^-40 fixed point)


def _logits(V, temperature, seed):
    """R rows of random logits with the special rows of tests/test_gpu_sampling_controls.py: 0 - masses .3 / .2 / .2 / .2 /
    .1 straddling top-p boundaries; 1 - one dominant entry; 2 - a coarse grid with ties everywhere (also at the maximum)."""
    g = torch.Generator().manual_seed(seed)
    lg = torch.randn(R, V, generator=g) * 2.5
    idx = torch.randperm(V, generator=g)[:5]
    lg[0] = -60.0 * temperature
    lg[0, idx] = torch.log(torch.tensor([0.3, 0.2, 0.2, 0.2, 0.1])) * temperature
    lg[1, int(idx[0])] = float(lg[1].max()) + 30.0 * temperature
    lg[2] = torch.randint(0, 12, (V,), generator=g).float() * 0.5 * temperature
    return lg, torch.rand(R, generator=g)


def _z32(lg, temperature):
    """z = logits / temperature as the kernel computes it: the IEEE fp32 quotient (fp64 division, rounded once to fp32, is
    correctly rounded), as fp64 numpy."""
    t = torch.tensor(temperature, dtype=torch.float32).double()
    return (lg.detach().cpu().double() / t).float().double().numpy()


def _check_rows(z32, tok, logp, top_k, top_p, V):
    """Every row against the fp64 rule on the kernel's own z; returns (max error, max error / bound, rows checked)."""
    worst, ratio, n = 0.0, 0.0, 0
    per = (V + 255) // 256
    for r in range(z32.shape[0]):
        z = z32[r]
        keep, above = filtered_keep(z, top_k, top_p)
        if top_p is not None and top_p < 1:
            topk_keep, _ = filtered_keep(z, top_k, None)
            if (topk_keep & (np.abs(above - top_p) <= AMBIGUOUS)).any():
                continue
        t = int(tok[r])
        assert keep[t], (r, t)
        mx = z.max()
        ref = z[t] - mx - math.log(np.exp(z[keep] - mx).sum())
        D = float(mx - z[keep].min())
        bound = 2 * U * (2 * D + 2 + per + 256 + math.log(V) + abs(ref))
        err = abs(float(logp[r]) - ref)
        assert err <= bound, (r, t, float(logp[r]), ref, bound)
        worst, ratio, n = max(worst, err), max(ratio, err / bound), n + 1
    return worst, ratio, n


@pytest.mark.parametrize("V", [8192, 5001])
@pytest.mark.parametrize("top_p", [None, 0.9, 0.5])
@pytest.mark.parametrize("top_k", [0, 1, 50])
@pytest.mark.parametrize("temperature", [0.7, 1.0, 1.3])
def test_logp_kernel_vs_fp64(temperature, top_k, top_p, V):
    """Tokens bit-identical to mas_sample_filtered (and to ops.sample_topk without logp); log p within the fp32 bound of the
    fp64 log-softmax over the fp64 rule's kept set; only the given column of the output is written."""
    from mas_b200 import _lib as L
    from mas_b200 import ops
    lg, u = _logits(V, temperature, int(temperature * 10) + 7 * top_k + int(100 * (top_p or 1)) + V)
    lg, u = lg.to(DEV), u.to(DEV)
    p = 1.0 if top_p is None else top_p
    ref_tok = torch.empty(R, dtype=torch.int64, device=DEV)
    L.call("mas_sample_filtered", lg, V, R, V, temperature, top_k, p, u, None, None, 0, ref_tok)
    out = torch.full((R, 3), float("nan"), device=DEV)
    tok = torch.empty(R, dtype=torch.int64, device=DEV)
    L.call("mas_sample_filtered_logp", lg, V, R, V, temperature, top_k, p, u, None, None, 0, tok, out[:, 1], 3)
    assert torch.equal(tok, ref_tok)
    assert torch.equal(tok, ops.sample_topk(lg, temperature, top_k, u, top_p=top_p))
    col = torch.empty(R, device=DEV)
    assert torch.equal(ops.sample_topk(lg, temperature, top_k, u, top_p=top_p, logp=col), tok)
    assert torch.equal(col, out[:, 1]) and bool(out[:, [0, 2]].isnan().all())
    z32 = _z32(lg, temperature)
    worst, ratio, n = _check_rows(z32, tok.cpu(), out[:, 1].cpu(), top_k, top_p, V)
    assert n >= R - 3
    if top_k == 1:
        assert float(out[:, 1].max()) <= 0 and float(out[3:, 1].abs().max()) == 0.0   # no ties at the maximum: certain
    print("logp kernel T=%g top_k=%d top_p=%s V=%d: max |err| %.3e (%.3f of the bound), %d rows" % (temperature, top_k, top_p, V,
                                                                                                     worst, ratio, n))


def test_prompt_and_greedy_rows_are_exactly_zero():
    """Prompt rows (mask set) and every greedy row get 0; the others equal the unprompted draw's log p; the column is read
    and written with its row stride (one column of [R, L] tensors)."""
    from mas_b200 import ops
    V = 8192
    lg, u = _logits(V, 1.0, 31)
    lg, u = lg.to(DEV), u.to(DEV)
    g = torch.Generator().manual_seed(2)
    T = torch.randint(0, V, (R, 7), generator=g).to(DEV)
    M = (torch.rand(R, 7, generator=g) < 0.5).to(DEV)
    free = torch.empty(R, device=DEV)
    free_tok = ops.sample_topk(lg, 1.0, 0, u, top_p=0.9, logp=free)
    lp = torch.full((R, 7), float("nan"), device=DEV)
    tok = ops.sample_topk(lg, 1.0, 0, u, top_p=0.9, prompt=(T[:, 3], M[:, 3]), logp=lp[:, 3])
    m3 = M[:, 3]
    assert torch.equal(tok, torch.where(m3, T[:, 3], free_tok))
    assert bool((lp[m3, 3] == 0).all()) and torch.equal(lp[~m3, 3], free[~m3]) and bool((free < 0).any())
    assert bool(lp[:, [0, 1, 2, 4, 5, 6]].isnan().all())
    for prompt in (None, (T[:, 5], M[:, 5])):
        for k, p in ((0, None), (5, 0.9)):
            z = torch.full((R,), float("nan"), device=DEV)
            gt = ops.sample_topk(lg, 0.0, k, None, top_p=p, prompt=prompt, logp=z)
            want = lg.argmax(-1) if prompt is None else torch.where(prompt[1], prompt[0], lg.argmax(-1))
            assert bool((z == 0).all()) and torch.equal(gt, want)


def _load_model(tag="tiny", **kw):
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, f"transformer_{tag}.pt"), weights_only=False)
    m = MakeAScene(**g["cfg"], **kw)
    m.load_state_dict(g["state_dict"])
    m.to(DEV).eval()
    m.device = DEV
    return m, g


def _tile(t, B):
    return t.repeat((B + t.shape[0] - 1) // t.shape[0], *([1] * (t.dim() - 1)))[:B].contiguous().to(DEV)


def _gen(seed=11):
    return torch.Generator(device=DEV).manual_seed(seed)


@pytest.mark.parametrize("B,n,scale", [(2, 2, 2.0), (4, 1, None), (3, 4, 2.0), (12, 1, None)])
def test_generate_logprobs(B, n, scale):
    """R = 8 / 4 rows (fp32 decoding) and 24 / 12 rows (fp16): tokens and logits do not depend on the flag; drawn positions
    hold the kernel bound's log p of the returned (mixed) logits, forced ones 0; eager and graphed calls agree bit for bit;
    num_samples = n equals the repeat_interleave call bit for bit."""
    m, g = _load_model()
    L, Vm = m.image_length, g["cfg"]["image_vocab_size"]
    text, seg = _tile(g["text"], B), _tile(g["seg"], B)
    gg = torch.Generator().manual_seed(B * n)
    T = torch.randint(0, Vm, (B * n, L), generator=gg).to(DEV)
    M = (torch.rand(B * n, L, generator=gg) < 0.3).to(DEV)
    kw = dict(guidance_scale=scale, temperature=0.9, top_k=40, top_p=0.9, img_tokens=T, img_mask=M, num_samples=n,
              return_logits=True)
    t0, lg0 = m.generate(text, seg, generator=_gen(), **kw)
    toks, lg, lp = m.generate(text, seg, generator=_gen(), return_logprobs=True, **kw)
    assert torch.equal(toks, t0) and torch.equal(lg, lg0)
    assert lp.shape == (B * n, L) and lp.dtype == torch.float32
    assert bool((lp[M] == 0).all()) and bool((lp[~M] < 0).any()) and bool((lp <= 0).all())
    z32 = _z32(lg, 0.9)
    free = (~M).cpu().numpy()
    worst, ratio, cnt = _check_rows(z32[free], toks.cpu().numpy()[free], lp.cpu().numpy()[free], 40, 0.9, Vm)
    assert cnt >= int(free.sum()) - 3
    print("generate logprobs B=%d n=%d scale=%s: max |err| %.3e (%.3f of the bound), %d positions" % (B, n, scale, worst, ratio, cnt))
    for _ in range(2):                                                # capture, then replay
        got = m.generate(text, seg, generator=_gen(), use_graphs=True, return_logprobs=True, **kw)
        assert all(torch.equal(a, b) for a, b in zip(got, (toks, lg, lp)))
    m.reset_sampler()
    if n > 1:
        rep = dict(kw, num_samples=1)
        if scale is not None:
            rep["uncond_text_tokens"] = torch.zeros_like(text).repeat_interleave(n, 0)
        got = m.generate(text.repeat_interleave(n, 0), seg.repeat_interleave(n, 0), generator=_gen(), return_logprobs=True, **rep)
        assert all(torch.equal(a, b) for a, b in zip(got, (toks, lg, lp)))


def _gather_logp(z, tok):
    return torch.log_softmax(z.double().cpu(), -1).gather(-1, tok.cpu().unsqueeze(-1)).squeeze(-1)


@pytest.mark.parametrize("tag", ["tiny", "wide"])
def test_score_matches_reference(tag):
    """Against fp64 log_softmax of the REAL reference's logits at its tokens, within 4e-3 ||z||_F (module docstring); and
    the negated per-row cross-entropies of this model's own forward() bit for bit."""
    from mas_b200 import ops
    m, g = _load_model(tag)
    text, seg, img = g["text"].to(DEV), g["seg"].to(DEV), g["img"].to(DEV)
    lp = m.score(text, seg, img)
    assert lp.shape == img.shape and lp.dtype == torch.float32
    ref = _gather_logp(g["logits"], img)
    err, bound = float((lp.double().cpu() - ref).norm()), 4e-3 * float(g["logits"].double().norm())
    assert err <= bound, (err, bound)
    with torch.no_grad():
        own = m(text, seg, img)
    V = own.shape[-1]
    assert torch.equal(lp, ops.token_logprobs(own.reshape(-1, V), img.reshape(-1)).view_as(lp))
    print("score %s vs reference: ||d log p|| %.3e (bound %.3e), max |d log p| %.3e" % (
        tag, err, bound, float((lp.double().cpu() - ref).abs().max())))


def test_score_guided_matches_two_forwards():
    """Guided score against fp64 log_softmax(u + s (c - u)) of two forward() calls (padded text, then a given one), within
    4e-3 (|1 - s| ||u||_F + |s| ||c||_F)."""
    m, g = _load_model("tiny")
    text, seg, img = g["text"].to(DEV), g["seg"].to(DEV), g["img"].to(DEV)
    s = 2.5
    for unc in (None, torch.randint(1, m.text_vocab_size, text.shape, generator=torch.Generator().manual_seed(4)).to(DEV)):
        with torch.no_grad():
            c = m(text, seg, img).double().cpu()
            u = m(torch.zeros_like(text) if unc is None else unc, seg, img).double().cpu()
        lp = m.score(text, seg, img, guidance_scale=s, uncond_text_tokens=unc)
        ref = _gather_logp(u + s * (c - u), img)
        err, bound = float((lp.double().cpu() - ref).norm()), 4e-3 * (abs(1 - s) * float(u.norm()) + s * float(c.norm()))
        assert err <= bound, (err, bound)
        print("guided score vs two forwards: ||d log p|| %.3e (bound %.3e)" % (err, bound))


@pytest.mark.parametrize("B,n,scale", [(2, 2, None), (2, 2, 2.0), (3, 4, 2.0), (12, 1, None)])
def test_generate_and_score_agree(B, n, scale):
    """generate(temperature=1) without filters, then score on the drawn tokens: the same distribution from the two routes.
    Up to 8 decode rows (fp32) within the 2e-3-derived bound on the mixed logits; above (fp16 decoding) the gap is printed."""
    m, g = _load_model()
    text, seg = _tile(g["text"], B), _tile(g["seg"], B)
    toks, lg, lp = m.generate(text, seg, guidance_scale=scale, temperature=1.0, num_samples=n, generator=_gen(5),
                              return_logits=True, return_logprobs=True)
    tr, sr = text.repeat_interleave(n, 0), seg.repeat_interleave(n, 0)
    sc = m.score(tr, sr, toks, guidance_scale=scale)
    with torch.no_grad():
        c = m(tr, sr, toks).double().cpu()
        u = m(torch.zeros_like(tr), sr, toks).double().cpu() if scale else c
    s = scale or 1.0
    bound = 4e-3 * (abs(1 - s) * float(u.norm()) + s * float(c.norm()))
    gap = float((lp.double() - sc.double()).norm())
    rows = B * n * (2 if scale else 1)
    print("generate vs score B=%d n=%d scale=%s rows=%d: ||gap|| %.3e, max |gap| %.3e (bound %.3e)" % (
        B, n, scale, rows, gap, float((lp - sc).abs().max()), bound))
    assert math.isfinite(gap)
    if rows <= 8:
        assert gap <= bound, (gap, bound)


def test_score_ignores_dropout():
    """A model built with attention and residual dropout, in train mode, scores bit-identically to its eval-mode self and to
    the same weights built without dropout."""
    m0, g = _load_model("tiny")
    m, _ = _load_model("tiny", attn_dropout_prob=0.2, out_dropout_prob=0.1)
    text, seg, img = g["text"].to(DEV), g["seg"].to(DEV), g["img"].to(DEV)
    m.train()
    a = m.score(text, seg, img, guidance_scale=2.0)
    b = m.score(text, seg, img, guidance_scale=2.0)
    m.eval()
    c = m.score(text, seg, img, guidance_scale=2.0)
    assert torch.equal(a, b) and torch.equal(a, c) and torch.equal(a, m0.score(text, seg, img, guidance_scale=2.0))
