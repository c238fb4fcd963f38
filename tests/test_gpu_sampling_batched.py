"""MakeAScene.generate above 8 rows on the GPU: the narrow-row fp16 Linear (mas_linear_rows_f16), the fp16 KV cache entries,
mas_layernorm2_forward at any row count, and the whole batched decoder against the REAL reference's fixtures."""
import math
import os

import pytest
import torch

from conftest import GOLDEN, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SHAPES = [(3072, 1024, 0), (1024, 1024, 0), (4096, 1024, 1), (1024, 4096, 0), (8192, 1024, 0), (192, 64, 0)]


def _gelu(v):
    return 0.5 * v * (1.0 + torch.tanh(0.7978845608028654 * v * (1.0 + 0.044715 * v * v)))


def _operands(R, N, K, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(R, K, generator=gen)
    w = torch.randn(N, K, generator=gen) / K ** 0.5
    b = torch.randn(N, generator=gen)
    return x.to(DEV), w.to(DEV), b.to(DEV)


def _rounded_x(x16, am):
    """The fp16 copy as fp64 values of x (the power-of-two operand scale undone)."""
    scale = 2.0 ** (14 - math.floor(math.log2(float(am))))
    return x16.double() / scale


def _linear_rows(x16, am, w, b, act):
    """mas_linear_rows_f16 on a given fp16 copy (the weight image padded and packed like ops.linear_small does)."""
    from mas_b200 import ops
    from mas_b200 import _lib as L
    R, K = x16.shape
    N = w.shape[0]
    wpk = ops._packed_linear_weight(ops._padded(w, (-(-N // 128) * 128, K)), False, DEV)
    ws = torch.empty(max(int(L.query("mas_linear_rows_f16_ws_bytes", R, N, K)), 16), dtype=torch.uint8, device=DEV)
    y = torch.empty(R, N, device=DEV)
    L.call("mas_linear_rows_f16", x16, R, K, wpk, y, N, N, b, am, act, ws, ws.numel())
    return y


@pytest.mark.parametrize("N,K,act", SHAPES)
@pytest.mark.parametrize("R", [9, 16, 100, 256, 300])
def test_narrow_gemm_vs_fp64(R, N, K, act):
    """mas_linear_rows_f16, and ops.linear_small (whichever form it selects) above 8 rows, against fp64 products of the same
    fp16-rounded operands: only fp32 accumulation error remains (an indexing or split-K bug shows as O(1))."""
    from mas_b200 import ops
    x, w, b = _operands(R, N, K, R * 7 + N + K)
    y = ops.linear_small(x, w, b, act=act)
    x16, am = ops.rows_to_half(x)
    ref = _rounded_x(x16, am) @ w.half().double().T + b.double()
    if act:
        ref = _gelu(ref)
    assert y.shape == (R, N)
    assert rel_err(y, ref) < 1e-4
    assert rel_err(_linear_rows(x16, am, w, b, act), ref) < 1e-4


def test_narrow_gemm_determinism_and_row_independence():
    """Two launches are bitwise equal; rows shared by a 16-row and a 256-row call are bitwise equal when the operand scale is
    the same (the split depends on (N, K) only); both agree with the training kernel on the same fp16 copy."""
    from mas_b200 import ops
    N, K = 3072, 1024
    x, w, b = _operands(256, N, K, 11)
    x[3, 5] = 40.0                     # the max lies in a row both calls share: both fp16 copies have the same scale
    x16, am = ops.rows_to_half(x)
    y1 = _linear_rows(x16, am, w, b, 0)
    assert torch.equal(y1, _linear_rows(x16, am, w, b, 0))
    assert rel_err(y1, ops.gemm_rows_f16(x16, am, w, False, b)) < 1e-4
    x16s, ams = ops.rows_to_half(x[:16].contiguous())
    assert float(ams) == float(am)
    assert torch.equal(_linear_rows(x16s, ams, w, b, 0), y1[:16])


@pytest.mark.parametrize("hd", [16, 32, 64, 128])
@pytest.mark.parametrize("length", [1, 130, 257, 640])
def test_fp16_cache_decode_vs_fp64(hd, length):
    from mas_b200 import ops
    R, heads, tmax = 5, 3, 640
    H = heads * hd
    gen = torch.Generator().manual_seed(hd * 1000 + length)
    qkv_all = torch.randn(R, length, 3 * H, generator=gen).to(DEV)
    kc = torch.zeros(R, heads, tmax, hd, dtype=torch.float16, device=DEV)
    vc = torch.zeros_like(kc)
    if length > 1:
        ops.kv_append(qkv_all[:, :length - 1], kc, vc, 0)
    ops.kv_append(qkv_all[:, length - 1:], kc, vc, length - 1)
    k = qkv_all[..., H:2 * H].reshape(R, length, heads, hd).permute(0, 2, 1, 3)
    v = qkv_all[..., 2 * H:].reshape(R, length, heads, hd).permute(0, 2, 1, 3)
    assert torch.equal(kc[:, :, :length], k.half()) and torch.equal(vc[:, :, :length], v.half())
    q = qkv_all[:, -1, :H].reshape(R, heads, 1, hd).double()
    p = torch.softmax((q @ k.half().double().transpose(-1, -2)) / hd ** 0.5, -1)
    ref = (p @ v.half().double()).reshape(R, H)
    ctx = ops.attn_decode(qkv_all[:, -1].contiguous(), kc, vc, length)
    assert rel_err(ctx, ref) < 1e-5
    kc2, vc2 = torch.zeros_like(kc), torch.zeros_like(vc)
    if length > 1:
        ops.kv_append(qkv_all[:, :length - 1], kc2, vc2, 0)
    ctx2 = ops.attn_decode_append(qkv_all[:, -1].contiguous(), kc2, vc2, length - 1)
    assert torch.equal(kc2, kc) and torch.equal(vc2, vc)      # the append stores exactly fp16(k), fp16(v)
    assert rel_err(ctx2, ref) < 1e-5


@pytest.mark.parametrize("R", [65, 256])
def test_layernorm_pair_any_rows(R):
    from mas_b200 import ops
    H = 1024
    gen = torch.Generator().manual_seed(R)
    x = torch.randn(R, H, generator=gen) * 3 + 0.5
    r = torch.randn(R, H, generator=gen)
    ln1, ln2 = torch.nn.LayerNorm(H, eps=1e-5), torch.nn.LayerNorm(H, eps=1e-5)
    with torch.no_grad():
        for ln in (ln1, ln2):
            ln.weight.copy_(torch.randn(H, generator=gen))
            ln.bias.copy_(torch.randn(H, generator=gen))
        ref1 = ln1.double()(x.double()) + r.double()
        ref2 = ln2.double()(ref1)
    ln1.float().to(DEV)
    ln2.float().to(DEV)
    y1, y2 = ops.layernorm2(x.to(DEV), ln1, r.to(DEV), ln2)
    assert rel_err(y1, ref1) < 1e-5 and rel_err(y2, ref2) < 1e-5


def _load_model(tag):
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, f"transformer_{tag}.pt"), weights_only=False)
    m = MakeAScene(**g["cfg"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).eval()
    m.device = DEV
    return m, g


def _tile(t, B):
    return t.repeat((B + t.shape[0] - 1) // t.shape[0], *([1] * (t.dim() - 1)))[:B].contiguous().to(DEV)


@pytest.mark.parametrize("tag", ["tiny", "wide"])
@pytest.mark.parametrize("R", [10, 128, 256])
def test_generate_batched_teacher_forced_matches_reference(tag, R):
    """The fixture's rows tiled to R rows: the reference's logits to 2e-3 (the bar of the 8-row test), and every copy of a
    fixture row bitwise equal to the first."""
    m, g = _load_model(tag)
    n = g["text"].shape[0]
    img = _tile(g["img"], R)
    toks, lg = m.generate(_tile(g["text"], R), _tile(g["seg"], R), img_tokens=img, return_logits=True)
    assert torch.equal(toks, img)
    assert rel_err(lg, _tile(g["logits"], R)) < 2e-3
    for r in range(n, R):
        assert torch.equal(lg[r], lg[r % n]), r


def test_generate_batched_guidance_greedy_seeded_and_graphs():
    m, g = _load_model("tiny")
    B, s = 6, 2.5                                   # 12 rows with guidance
    text, seg, img = _tile(g["text"], B), _tile(g["seg"], B), _tile(g["img"], B)
    with torch.no_grad():
        cond = m(text, seg, img)
        uncond = m(torch.zeros_like(text), seg, img)
    _, lg = m.generate(text, seg, guidance_scale=s, img_tokens=img, return_logits=True)
    assert rel_err(lg, uncond + s * (cond - uncond)) < 2e-3
    toks, lg = m.generate(text, seg, guidance_scale=s, temperature=0, return_logits=True)
    assert torch.equal(toks, lg.argmax(-1))
    V = g["cfg"]["image_vocab_size"]
    a = m.generate(text, seg, guidance_scale=s, temperature=0.9, top_k=5, generator=torch.Generator(device=DEV).manual_seed(7))
    b, lgb = m.generate(text, seg, guidance_scale=s, temperature=0.9, top_k=5, generator=torch.Generator(device=DEV).manual_seed(7),
                        return_logits=True)
    assert torch.equal(a, b) and int(a.min()) >= 0 and int(a.max()) < V
    kth = lgb.topk(5, dim=-1).values[..., -1]
    assert bool((lgb.gather(-1, b.unsqueeze(-1)).squeeze(-1) >= kth).all())
    for _ in range(2):                               # capture, then replay
        _, lg_g = m.generate(text, seg, guidance_scale=s, img_tokens=img, return_logits=True, use_graphs=True)
        _, lg_e = m.generate(text, seg, guidance_scale=s, img_tokens=img, return_logits=True)
        assert torch.equal(lg_g, lg_e)
    c = m.generate(text, seg, guidance_scale=s, temperature=0.9, top_k=5, generator=torch.Generator(device=DEV).manual_seed(7),
                   use_graphs=True)
    assert torch.equal(c, a)
    m.reset_sampler()


def test_graphed_decoder_follows_in_place_weight_updates():
    """Above 8 rows the graphs read fp16 weight images. After an in-place update of every parameter (an optimizer step), the
    next generate(use_graphs=True) must use the new weights: bitwise equal to eager decoding of the updated model."""
    m, g = _load_model("wide")
    text, seg, img = _tile(g["text"], 10), _tile(g["seg"], 10), _tile(g["img"], 10)
    for _ in range(2):
        _, lg_g = m.generate(text, seg, img_tokens=img, return_logits=True, use_graphs=True)
    _, lg_e = m.generate(text, seg, img_tokens=img, return_logits=True)
    assert torch.equal(lg_g, lg_e)
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(0.97)
    torch.cuda.empty_cache()
    _, lg_g2 = m.generate(text, seg, img_tokens=img, return_logits=True, use_graphs=True)
    _, lg_e2 = m.generate(text, seg, img_tokens=img, return_logits=True)
    assert not torch.equal(lg_e2, lg_e)
    assert torch.equal(lg_g2, lg_e2)
    m.reset_sampler()
