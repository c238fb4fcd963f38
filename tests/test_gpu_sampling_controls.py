"""Nucleus (top-p) sampling and image-token prompts on the GPU: mas_sample_filtered against an fp64 restatement of
top_k_top_p_filtering (tests/test_sampling_controls_cpu.py::filtered_keep), and MakeAScene.generate with both controls."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from test_sampling_controls_cpu import filtered_keep

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
R, V = 256, 8192
AMBIGUOUS = 1e-6      # an entry whose mass above lies this close to top_p may be decided either way


def _draw(lg, temperature, top_k, top_p, u, prompt=None):
    from mas_b200 import ops
    return ops.sample_topk(lg.to(DEV), temperature, top_k, None if u is None else u.to(DEV), top_p=top_p, prompt=prompt).cpu()


def _logits(temperature, seed):
    """R rows of random logits, with special rows: 0 - three equal values straddling the top-p boundary of a position-based
    rule (masses .3 / .2 / .2 / .2 / .1 at random indices, the rest negligible); 1 - a top entry whose own mass exceeds
    top_p; 2 - a coarse grid with many ties everywhere."""
    g = torch.Generator().manual_seed(seed)
    lg = torch.randn(R, V, generator=g) * 2.5
    t = temperature if temperature > 0 else 1.0
    idx = torch.randperm(V, generator=g)[:5]
    lg[0] = -60.0 * t
    lg[0, idx] = torch.log(torch.tensor([0.3, 0.2, 0.2, 0.2, 0.1])) * t
    lg[1, int(idx[0])] = float(lg[1].max()) + 30.0 * t
    lg[2] = torch.randint(0, 12, (V,), generator=g).float() * 0.5 * t
    return lg, torch.rand(R, generator=g)


@pytest.mark.parametrize("temperature,top_k,top_p", [(1.0, 0, 0.9), (0.7, 100, 0.95), (1.3, 0, 0.5), (1.0, 50, 1.0), (0.5, 0, 0.99),
                                                     (1.0, 3000, 0.3)])
def test_filtered_kernel_vs_fp64_rule(temperature, top_k, top_p):
    """Every token lies in the fp64 kept set (or is an entry within AMBIGUOUS of the boundary) and in the u interval of the
    kept-set CDF in index order; probing the midpoint of every kept entry's interval returns that entry, so the kernel's kept
    set is the fp64 one (extra or missing entries would shift or remove intervals)."""
    lg, u = _logits(temperature, int(temperature * 100) + top_k + int(top_p * 1000))
    tok = _draw(lg, temperature, top_k, top_p, u)
    z = lg.double().numpy() / temperature
    probes_u, probes_rows, probes_want = [], [], []
    for r in range(R):
        keep, above = filtered_keep(z[r], top_k, top_p)
        topk_keep, _ = filtered_keep(z[r], top_k, None)
        amb = topk_keep & (np.abs(above - top_p) <= AMBIGUOUS) if top_p < 1 else np.zeros(V, dtype=bool)
        t = int(tok[r])
        assert keep[t] or amb[t], (r, t)
        if amb.any():
            continue
        p = np.where(keep, np.exp(z[r] - z[r].max()), 0.0)
        c = np.cumsum(p) / p.sum()
        lo = c[t - 1] if t > 0 else 0.0
        assert lo - 1e-5 <= float(u[r]) <= c[t] + 1e-5, (r, t, lo, float(u[r]), c[t])
        if r < 12:
            kept = np.flatnonzero(keep)
            lo_all = np.concatenate([[0.0], c[kept][:-1]])
            for e, a, b in zip(kept, lo_all, c[kept]):
                if b - a > 1e-4:
                    probes_u.append((a + b) / 2)
                    probes_rows.append(r)
                    probes_want.append(int(e))
    if top_p < 1:                                                   # row 1: the top entry alone
        assert int(tok[1]) == int(np.argmax(z[1])) and filtered_keep(z[1], top_k, top_p)[0].sum() == 1
    got = _draw(lg[probes_rows], temperature, top_k, top_p, torch.tensor(probes_u, dtype=torch.float32))
    assert got.tolist() == probes_want


def test_tie_group_at_the_boundary_is_kept_or_dropped_together():
    """Masses .3 / .2 / .2 / .2 / .1: top_p = .5 keeps .3 and all three .2 (mass above them .3), top_p = .25 keeps .3 alone."""
    lg, _ = _logits(1.0, 3)
    row = lg[:1].expand(4096, V).contiguous()
    u = torch.rand(4096, generator=torch.Generator().manual_seed(1))
    z = row[0].double()
    top = z.topk(5).indices
    for top_p, n in ((0.5, 4), (0.25, 1)):
        seen = set(_draw(row, 1.0, 0, top_p, u).tolist())
        assert seen == set(top[:n].tolist()), (top_p, seen)


def test_distribution_20000_rows():
    g = torch.Generator().manual_seed(21)
    row = torch.randn(50, generator=g)
    n = 20000
    temperature, top_k, top_p = 1.1, 30, 0.8
    tok = _draw(row.expand(n, 50).contiguous(), temperature, top_k, top_p, torch.rand(n, generator=g))
    z = row.double().numpy() / temperature
    keep, _ = filtered_keep(z, top_k, top_p)
    p = np.where(keep, np.exp(z - z.max()), 0.0)
    p = torch.from_numpy(p / p.sum())
    assert 3 <= int(keep.sum()) < top_k
    freq = torch.bincount(tok, minlength=50).double() / n
    assert float(freq[torch.from_numpy(~keep)].sum()) == 0.0
    assert float((freq - p).abs().max()) < 5 * float((p * (1 - p) / n).sqrt().max())


def test_greedy_is_first_argmax_with_ties():
    g = torch.Generator().manual_seed(5)
    lg = torch.randint(-4, 3, (R, V), generator=g).float()        # many entries share the maximum
    lg[7] = -float("inf")
    lg[7, 100] = lg[7, 4000] = 1.0
    want = lg.argmax(-1)
    assert torch.equal(_draw(lg, 0.0, 0, 0.9, None), want)
    mask = torch.zeros(R, dtype=torch.bool)
    assert torch.equal(_draw(lg, 0.0, 5, None, None, prompt=(torch.zeros(R, dtype=torch.int64, device=DEV), mask.to(DEV))), want)
    assert torch.equal(want.to(DEV), lg.to(DEV).argmax(-1))


def test_determinism_and_top_p_one_equals_topk():
    from mas_b200 import ops
    from mas_b200 import _lib as L
    lg, u = _logits(0.9, 77)
    lg, u = lg.to(DEV), u.to(DEV)
    a = _draw(lg, 0.9, 0, 0.93, u)
    for _ in range(3):
        assert torch.equal(_draw(lg, 0.9, 0, 0.93, u), a)
    for k in (0, 40, 1):
        ref = ops.sample_topk(lg, 0.9, k, u)
        tok = torch.empty(R, dtype=torch.int64, device=DEV)
        L.call("mas_sample_filtered", lg, V, R, V, 0.9, k, 1.0, u, None, None, 0, tok)
        assert torch.equal(tok, ref), k
        none_forced = (torch.zeros(R, dtype=torch.int64, device=DEV), torch.zeros(R, dtype=torch.bool, device=DEV))
        assert torch.equal(ops.sample_topk(lg, 0.9, k, u, prompt=none_forced), ref), k


def test_prompt_select_in_the_kernel():
    """Forced rows return the given token, the others exactly what the unprompted draw returns; the prompt columns are read
    with their row stride (a column of an [R, L] tensor)."""
    lg, u = _logits(1.0, 8)
    g = torch.Generator().manual_seed(2)
    T = torch.randint(0, V, (R, 7), generator=g).to(DEV)
    M = (torch.rand(R, 7, generator=g) < 0.5).to(DEV)
    free = _draw(lg, 1.0, 0, 0.9, u)
    tok = _draw(lg, 1.0, 0, 0.9, u, prompt=(T[:, 3], M[:, 3]))
    assert torch.equal(tok, torch.where(M[:, 3].cpu(), T[:, 3].cpu(), free))


def _load_model():
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, "transformer_tiny.pt"), weights_only=False)
    m = MakeAScene(**g["cfg"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).eval()
    m.device = DEV
    return m, g


def _tile(t, B):
    return t.repeat((B + t.shape[0] - 1) // t.shape[0], *([1] * (t.dim() - 1)))[:B].contiguous().to(DEV)


@pytest.mark.parametrize("B", [4, 64])
def test_generate_with_top_p_and_partial_mask(B):
    """Guided, top-p and a partial mask at B = 4 (8 rows, fp32 decode) and 64 (128 rows, fp16 decode): forced positions equal
    T, drawn ones lie in the fp64 kept set of the returned logits, graphs and eager give the same tokens, and feeding the tokens
    back as img_tokens reproduces the returned logits bit for bit (every position saw the tokens actually emitted)."""
    m, g = _load_model()
    L, Vm = m.image_length, g["cfg"]["image_vocab_size"]
    text, seg = _tile(g["text"], B), _tile(g["seg"], B)
    gg = torch.Generator().manual_seed(B)
    T = torch.randint(0, Vm, (B, L), generator=gg).to(DEV)
    M = (torch.rand(B, L, generator=gg) < 0.4).to(DEV)
    kw = dict(guidance_scale=2.0, temperature=0.9, top_k=60, top_p=0.8, img_tokens=T, img_mask=M, return_logits=True)
    toks, lg = m.generate(text, seg, generator=torch.Generator(device=DEV).manual_seed(3), **kw)
    assert torch.equal(toks[M], T[M])
    z = lg.double().cpu().numpy() / 0.9
    Mc, tc = M.cpu(), toks.cpu()
    for b in range(B):
        for t in range(L):
            if not Mc[b, t]:
                keep, above = filtered_keep(z[b, t], 60, 0.8)
                assert keep[tc[b, t]] or abs(above[tc[b, t]] - 0.8) <= AMBIGUOUS, (b, t)
    for _ in range(2):                                              # capture, then replay
        tg, lgg = m.generate(text, seg, generator=torch.Generator(device=DEV).manual_seed(3), use_graphs=True, **kw)
        assert torch.equal(tg, toks) and torch.equal(lgg, lg)
    m.reset_sampler()
    _, lg2 = m.generate(text, seg, guidance_scale=2.0, img_tokens=toks, return_logits=True)
    assert torch.equal(lg2, lg)
