"""CPU: the recomputing causal-attention backward (csrc/attn_causal.cu, mas_attn_causal_backward) restated in fp64 numpy with
the kernels' tiling (128-row resident tiles, 64-row streamed blocks, causal block ranges, per-row m / l from the forward's
online pass, D pre-pass, dropout mask regenerated at ((b heads + h) S + q) S + k) against torch autograd; the dS bound the
kernel's operand scale rests on; the model flag's plumbing and the route's shape checks."""
import numpy as np
import pytest
import torch

from test_dropout_cpu import keep_mask, scale_of

BM, BN = 128, 64


def _forward_stats(q, k, scale):
    """Row maxima / sums of the scaled causal scores as the forward's pass 0 forms them: online over 128-key blocks."""
    S = q.shape[0]
    m = np.full(S, -np.inf)
    l = np.zeros(S)
    for kb in range(0, S, BM):
        s = (q @ k[kb:kb + BM].T) * scale
        s[np.arange(S)[:, None] < np.arange(kb, kb + BM)[None, :]] = -np.inf
        mn = np.maximum(m, s.max(1))
        ok = mn > -np.inf
        add = np.where(ok[:, None], np.exp(s - np.where(ok, mn, 0)[:, None]), 0).sum(1)
        l = np.where(ok, l * np.exp(np.where(ok, m - mn, 0)) + add, l)
        m = np.where(ok, mn, m)
    return m, l


def _tiled_backward(q, k, v, dO, ctx, m, l, keep, p, scale):
    """dq, dk, dv of one (sequence, head) by the two kernels' loops; keep [S, S] bool."""
    S, hd = q.shape
    s_ = scale_of(p)
    D = (dO * ctx).sum(1)
    dq, dk, dv = np.zeros_like(q), np.zeros_like(k), np.zeros_like(v)
    # DKV: rows = a 128-key tile, columns = the query blocks of 64 at or below the diagonal
    for r0 in range(0, S, BM):
        keys = np.arange(r0, r0 + BM)
        for cb in range(r0, S, BN):
            qs = np.arange(cb, cb + BN)
            vis = keys[:, None] <= qs[None, :]
            pt = np.where(vis, np.exp((k[keys] @ q[qs].T) * scale - m[qs][None, :]) / l[qs][None, :], 0.0)
            kt = keep[np.ix_(qs, keys)].T
            dpt = (v[keys] @ dO[qs].T) * np.where(kt, s_, 0.0)
            dst = pt * (dpt - D[qs][None, :])
            dv[keys] += (pt * kt) @ dO[qs] * s_
            dk[keys] += dst @ q[qs] * scale
    # DQ: rows = a 128-query tile, columns = its causal key blocks of 64
    for r0 in range(0, S, BM):
        qs = np.arange(r0, r0 + BM)
        for cb in range(0, r0 + BM, BN):
            keys = np.arange(cb, cb + BN)
            vis = keys[None, :] <= qs[:, None]
            pr = np.where(vis, np.exp((q[qs] @ k[keys].T) * scale - m[qs][:, None]) / l[qs][:, None], 0.0)
            dp = (dO[qs] @ v[keys].T) * np.where(keep[np.ix_(qs, keys)], s_, 0.0)
            dq[qs] += (pr * (dp - D[qs][:, None])) @ k[keys] * scale
    return dq, dk, dv


@pytest.mark.parametrize("B,S,heads,p", [(1, 128, 1, 0.0), (2, 256, 2, 0.0), (2, 256, 2, 0.3), (1, 384, 1, 0.2)])
def test_tiled_backward_matches_autograd(B, S, heads, p):
    hd = 64
    H = heads * hd
    scale = 1.0 / hd ** 0.5
    g = torch.Generator().manual_seed(S + heads)
    qkv = torch.randn(B, S, 3 * H, generator=g, dtype=torch.float64) * 1.5
    w = torch.randn(B, S, H, generator=g, dtype=torch.float64)
    seed = -1234567890123 + S
    keep = keep_mask(seed, B * heads * S * S, p).reshape(B, heads, S, S)
    x = qkv.clone().requires_grad_(True)
    q, k, v = [t.view(B, S, heads, hd).permute(0, 2, 1, 3) for t in x.split(H, dim=-1)]
    sc = (q @ k.transpose(-1, -2)) * scale
    sc = sc.masked_fill(~torch.tril(torch.ones(S, S, dtype=torch.bool)), float("-inf"))
    ref = ((torch.softmax(sc, -1) * torch.from_numpy(keep) * scale_of(p)) @ v).permute(0, 2, 1, 3).reshape(B, S, H)
    (ref * w).sum().backward()

    a = qkv.numpy()
    got = np.zeros_like(a)
    ctx_all = np.zeros((B, S, H))
    for b in range(B):
        for h in range(heads):
            cq, ck, cv = (a[b, :, t * H + h * hd:t * H + (h + 1) * hd] for t in range(3))
            m, l = _forward_stats(cq, ck, scale)
            pr = np.tril(np.exp((cq @ ck.T) * scale - m[:, None]) / l[:, None])
            c = (pr * keep[b, h] * scale_of(p)) @ cv
            ctx_all[b, :, h * hd:(h + 1) * hd] = c
            dO = w[b, :, h * hd:(h + 1) * hd].numpy()
            dq, dk, dv = _tiled_backward(cq, ck, cv, dO, c, m, l, keep[b, h], p, scale)
            for t, d in enumerate((dq, dk, dv)):
                got[b, :, t * H + h * hd:t * H + (h + 1) * hd] = d
            # the bound behind the dS operand scale: |dS| <= 2 hd max|dO| max|qkv| / (1 - p)
            D = (dO * c).sum(1)
            ds = pr * ((dO @ cv.T) * np.where(keep[b, h], scale_of(p), 0.0) - D[:, None])
            assert np.abs(ds).max() <= 2 * hd * np.abs(dO).max() * np.abs(a).max() * scale_of(p)
    np.testing.assert_allclose(ctx_all, ref.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(got, x.grad.numpy(), rtol=1e-10, atol=1e-10)


def test_flag_reaches_every_attention_and_keeps_the_state_dict():
    from models.transformer import MakeAScene, SelfAttention
    cfg = dict(num_layers=3, hidden_dim=128, num_attn_heads=2, image_vocab_size=64, seg_vocab_size=32, text_vocab_size=80,
               image_tokens_per_dim=8, seg_tokens_per_dim=4, text_length=48)
    torch.manual_seed(0)
    a = MakeAScene(**cfg)
    torch.manual_seed(0)
    b = MakeAScene(**cfg, recompute_attention=True)
    atts = [m for m in b.modules() if isinstance(m, SelfAttention)]
    assert len(atts) == 3 and all(m.recompute_attention for m in atts)
    assert not any(m.recompute_attention for m in a.modules() if isinstance(m, SelfAttention))
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa.keys()) == list(sb.keys())
    assert all(torch.equal(sa[k], sb[k]) for k in sa)


@pytest.mark.parametrize("S,hd,tc", [(200, 64, True), (256, 32, True), (128, 64, False)])
def test_recompute_raises_where_the_fused_kernels_cannot_run(S, hd, tc, monkeypatch):
    """No silent fall-back to storing P: an ineligible shape or the SIMT route raises before any launch."""
    from mas_b200 import ops
    calls = []
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: tc)
    monkeypatch.setattr(ops.L, "call", lambda *a: calls.append(a[0]))
    qkv = torch.zeros(1, S, 3 * 2 * hd)
    with pytest.raises(RuntimeError, match="head dim 64, S % 128 == 0"):
        ops.CausalAttentionFn.apply(qkv, 2, 0.0, True)
    assert not calls
