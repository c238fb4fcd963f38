"""MakeAScene.generate(num_samples=n) on the GPU: the shared-prefix decode attention (mas_attn_decode_shared(_append)(_f16)) is
bitwise the unshared entry on the concatenated cache, and n samples per prompt are bitwise the repeat_interleave call, tokens
and logits, eager and graphed, at fp32 and fp16 row counts, with the fused and the unfused decode step; teacher forcing still
reproduces the reference's logits."""
import os

import pytest
import torch

from conftest import GOLDEN, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.mark.parametrize("dt", [torch.float32, torch.float16])
@pytest.mark.parametrize("hd", [32, 64, 128])
@pytest.mark.parametrize("R,n", [(16, 8), (24, 6), (12, 3), (6, 1)])
@pytest.mark.parametrize("rows_per_block", [0, 1, 2, 4])
@pytest.mark.parametrize("at", ["first", "last"])
@pytest.mark.parametrize("append", [True, False])
def test_shared_kernel_is_the_unshared_kernel_on_the_concatenated_cache(dt, hd, R, n, rows_per_block, at, append):
    """ctx and the stored k / v are torch.equal to mas_attn_decode_append(_f16) (append) or, after mas_kv_append(_f16) into the
    suffix cache, to mas_attn_decode(_f16) (the two add the token's own term in different partial groups) over
    [prefix row r // n | suffix row r]; n = 6 with 4 rows per block leaves a 2-row slice, n = 3 with 2 a 1-row slice."""
    from mas_b200 import ops
    heads, P, Tsuf = 4, 384, 256
    pos = P if at == "first" else P + Tsuf - 1
    H = heads * hd
    gen = torch.Generator().manual_seed(hd * 100 + R + n)
    qkv = torch.randn(R, 3 * H, generator=gen).to(DEV)
    kp = torch.randn(R // n, heads, P, hd, generator=gen).to(DEV, dt)
    vp = torch.randn(R // n, heads, P, hd, generator=gen).to(DEV, dt)
    ks = torch.randn(R, heads, Tsuf, hd, generator=gen).to(DEV, dt)
    vs = torch.randn(R, heads, Tsuf, hd, generator=gen).to(DEV, dt)
    kc = torch.cat([kp.repeat_interleave(n, 0), ks], 2).contiguous()
    vc = torch.cat([vp.repeat_interleave(n, 0), vs], 2).contiguous()
    kp0, vp0 = kp.clone(), vp.clone()
    if append:
        ref = ops.attn_decode_append(qkv, kc, vc, pos)
        ctx = ops.attn_decode_shared_append(qkv, kp, vp, ks, vs, pos, rows_per_block)
    else:
        ops.kv_append(qkv.view(R, 1, -1), kc, vc, pos)
        ops.kv_append(qkv.view(R, 1, -1), ks, vs, pos - P)
        ref = ops.attn_decode(qkv, kc, vc, pos + 1)
        ctx = ops.attn_decode_shared(qkv, kp, vp, ks, vs, pos + 1, rows_per_block)
    torch.cuda.synchronize()
    assert torch.equal(ctx, ref)
    assert torch.equal(ks, kc[:, :, P:]) and torch.equal(vs, vc[:, :, P:])      # this token stored at slot pos - P, rest untouched
    assert torch.equal(kp, kp0) and torch.equal(vp, vp0)


def test_shared_kernel_rejects_bad_arguments():
    from mas_b200 import _lib as L
    heads, hd, P, Tsuf = 2, 64, 8, 4
    qkv = torch.zeros(4, 3 * heads * hd, device=DEV)
    kp = torch.zeros(2, heads, P, hd, device=DEV)
    ks = torch.zeros(4, heads, Tsuf, hd, device=DEV)
    ctx = torch.empty(4, heads * hd, device=DEV)
    for R, n, pos, rpb in [(4, 3, P, 0), (4, 2, P - 1, 0), (4, 2, P + Tsuf, 0), (4, 2, P, 3), (4, 2, P, 8)]:
        with pytest.raises(Exception):
            L.call("mas_attn_decode_shared_append", qkv, kp, kp, ks, ks, ctx, R, n, heads, hd, P, Tsuf, pos, rpb)


def test_shared_wrapper_checks_the_cache_extents():
    from mas_b200 import ops
    heads, hd, P, Tsuf, R = 2, 64, 8, 4, 4
    qkv = torch.zeros(R, 3 * heads * hd, device=DEV)
    kp, ks = torch.zeros(2, heads, P, hd, device=DEV), torch.zeros(R, heads, Tsuf, hd, device=DEV)
    bad = [(kp, kp[:1].clone(), ks, ks), (kp, kp, ks, ks[:, :, :2].clone()), (kp, kp, ks, ks.half()),
           (kp, kp, torch.zeros(R, heads, Tsuf, 32, device=DEV), ks), (kp, kp, ks.transpose(2, 3).contiguous().transpose(2, 3), ks),
           (kp, kp, torch.zeros(3, heads, Tsuf, hd, device=DEV), torch.zeros(3, heads, Tsuf, hd, device=DEV))]
    for caches in bad:
        with pytest.raises(RuntimeError):
            ops.attn_decode_shared_append(qkv, *caches, P)
        with pytest.raises(RuntimeError):
            ops.attn_decode_shared(qkv, *caches, P + 1)


def _bench_shaped_model(sandwich=True):
    """Two layers of the sampling benchmark's shape (the paper's token lengths, 64-wide heads): the prefix pass runs the fused
    causal attention core and the fp16 training GEMMs, as in the full model. Without the sandwich LayerNorm a decode step takes
    the unfused form (_decode_step_plain)."""
    from models.transformer import MakeAScene
    torch.manual_seed(0)
    m = MakeAScene(num_layers=2, hidden_dim=512, num_attn_heads=8, image_vocab_size=8192, seg_vocab_size=1024, text_vocab_size=49408,
                   image_tokens_per_dim=16, seg_tokens_per_dim=16, text_length=128).to(DEV).eval()
    for layer in m.transformer.layers:
        layer.cogview_sandwich_layernorm = sandwich
    m.device = DEV
    return m


def _rep(t, n):
    return t.repeat_interleave(n, 0)


@pytest.mark.parametrize("B,n", [(1, 4), (4, 8), (16, 8)])          # 8 rows (fp32), 64 and 256 rows (fp16), with guidance
@pytest.mark.parametrize("draw", ["top_k", "top_p_mask"])
@pytest.mark.parametrize("sandwich", [True, False])
def test_generate_is_the_repeat_interleave_call(B, n, draw, sandwich):
    m = _bench_shaped_model(sandwich)
    gen = torch.Generator().manual_seed(B)
    text = torch.randint(1, 40000, (B, 128), generator=gen).to(DEV)
    text[:, 100:] = 0                                                 # padding: the per-position pad ids
    seg = torch.randint(0, 1024, (B, 256), generator=gen).to(DEV)
    uncond = torch.zeros_like(text)
    uncond[:, :3] = torch.randint(1, 40000, (B, 3), generator=gen).to(DEV)
    kw = dict(guidance_scale=3.0, temperature=1.0, top_k=64, return_logits=True)
    if draw == "top_p_mask":
        kw.update(top_p=0.9, img_tokens=torch.randint(0, 8192, (B * n, 256), generator=gen).to(DEV),
                  img_mask=(torch.rand(B * n, 256, generator=gen) < 0.3).to(DEV))
    ref_t, ref_l = m.generate(_rep(text, n), _rep(seg, n), uncond_text_tokens=_rep(uncond, n),
                              generator=torch.Generator(device=DEV).manual_seed(7), **kw)
    for graphs in (False, True, True):                                 # eager, capture, replay
        t, lg = m.generate(text, seg, uncond_text_tokens=uncond, num_samples=n, use_graphs=graphs,
                           generator=torch.Generator(device=DEV).manual_seed(7), **kw)
        assert t.shape == (B * n, 256) and lg.shape == (B * n, 256, 8192)
        assert torch.equal(t, ref_t), graphs
        assert torch.equal(lg, ref_l), graphs
    dec = m._sampler
    assert dec.samples == n and dec.rows == 2 * B * n
    m.generate(_rep(text, n), _rep(seg, n), uncond_text_tokens=_rep(uncond, n), use_graphs=True, img_tokens=ref_t)
    assert m._sampler is not dec and m._sampler.samples == 1          # same rows, other grouping: a new decoder
    m.reset_sampler()


def _load_model(tag):
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, f"transformer_{tag}.pt"), weights_only=False)
    m = MakeAScene(**g["cfg"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).eval()
    m.device = DEV
    return m, g


@pytest.mark.parametrize("tag", ["tiny", "wide"])
@pytest.mark.parametrize("n", [3, 8, 64])
def test_teacher_forced_samples_match_reference(tag, n):
    """Each prompt's n teacher-forced samples reproduce the reference's logits to 2e-3 (the bar of the batched test)."""
    m, g = _load_model(tag)
    img = _rep(g["img"], n).to(DEV)
    toks, lg = m.generate(g["text"].to(DEV), g["seg"].to(DEV), img_tokens=img, num_samples=n, return_logits=True)
    assert torch.equal(toks, img)
    assert rel_err(lg, _rep(g["logits"], n).to(DEV)) < 2e-3
