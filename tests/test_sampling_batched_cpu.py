"""MakeAScene.generate above 8 rows, checked WITHOUT a GPU: the emulated C-ABI of tests/test_host_logic_cpu.py plus the entries
of the batched decode path with their real fp16 rounding (the narrow-row Linear on fp16-rounded operands with fp64 products,
fp16 KV caches rounded to nearest). What is under test is the host side: which entry serves which row count, the cache
dtype, and that the batched decode still reproduces the reference's logits."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_err
from test_host_logic_cpu import Emu, _addr, _f32, _mat


def _f16(p, n):
    return np.ctypeslib.as_array((ctypes.c_uint16 * n).from_address(_addr(p))).view(np.float16)


def _scale_of(amax):
    if amax is None:
        return 1.0
    a = float(_f32(_addr(amax), 1)[0])
    return 1.0 if not np.isfinite(a) or a <= 0 else 2.0 ** (14 - int(np.floor(np.log2(a))))


def _gelu(v):
    return 0.5 * v * (1.0 + np.tanh(0.7978845608028654 * v * (1.0 + 0.044715 * v * v)))


class BatchedEmu(Emu):
    """Emu + the fp16 decode entries (include/mas_b200.h)."""

    def __init__(self):
        super().__init__()
        self.packs = {}
        self.args = []

    def __call__(self, name, *a):
        self.args.append((name, a))
        super().__call__(name, *a)

    def mas_pack_gemm_tc16(self, w, out, N, K, transpose):
        W = _f32(_addr(w), N * K).reshape(N, K).astype(np.float16).astype(np.float64)
        self.packs[_addr(out)] = W.T.copy() if transpose else W

    def mas_linear_rows_f16(self, x16, R, K, wpk, y, ldy, N, bias, x_amax, act, ws, ws_bytes):
        X = _f16(x16, R * K).reshape(R, K).astype(np.float64) / _scale_of(x_amax)
        Wp = self.packs[_addr(wpk)]
        assert Wp.shape[1] == K and Wp.shape[0] % 128 == 0 and Wp.shape[0] - N < 128, (Wp.shape, N, K)
        assert not Wp[N:].any(), "the padded weight rows must be zero"
        o = X @ Wp[:N].T
        if bias is not None:
            o = o + _f32(_addr(bias), N)[None, :]
        _mat(_addr(y), R, N, ldy, False)[...] = _gelu(o) if act == 1 else o

    def mas_gemm_rows_f16(self, x16, M, K, wpk, y, ldy, N, bias, residual, x_amax, alpha):
        X = _f16(x16, M * K).reshape(M, K).astype(np.float64) / _scale_of(x_amax)
        Wp = self.packs[_addr(wpk)]
        assert Wp.shape[1] == K and Wp.shape[0] % 128 == 0 and Wp.shape[0] - N < 128 and residual is None
        o = alpha * (X @ Wp[:N].T)
        if bias is not None:
            o = o + _f32(_addr(bias), N)[None, :]
        _mat(_addr(y), M, N, ldy, False)[...] = o

    def mas_kv_append_f16(self, qkv, R, T, heads, hd, kc, vc, Tmax, pos0):
        H = heads * hd
        Q = _f32(_addr(qkv), R * T * 3 * H).reshape(R, T, 3, heads, hd)
        K_ = _f16(kc, R * heads * Tmax * hd).reshape(R, heads, Tmax, hd)
        V_ = _f16(vc, R * heads * Tmax * hd).reshape(R, heads, Tmax, hd)
        K_[:, :, pos0:pos0 + T] = Q[:, :, 1].transpose(0, 2, 1, 3).astype(np.float16)
        V_[:, :, pos0:pos0 + T] = Q[:, :, 2].transpose(0, 2, 1, 3).astype(np.float16)

    def mas_attn_decode_f16(self, qkv, kc, vc, ctx, R, heads, hd, Tmax, length):
        H = heads * hd
        q = _f32(_addr(qkv), R * 3 * H).reshape(R, 3, heads, hd)[:, 0].astype(np.float64)
        K_ = _f16(kc, R * heads * Tmax * hd).reshape(R, heads, Tmax, hd)[:, :, :length].astype(np.float64)
        V_ = _f16(vc, R * heads * Tmax * hd).reshape(R, heads, Tmax, hd)[:, :, :length].astype(np.float64)
        s = np.einsum("rhd,rhtd->rht", q, K_) / np.sqrt(hd)
        p = np.exp(s - s.max(-1, keepdims=True))
        p = p / p.sum(-1, keepdims=True)
        _f32(_addr(ctx), R * H).reshape(R, heads, hd)[...] = np.einsum("rht,rhtd->rhd", p, V_)

    def mas_attn_decode_append_f16(self, qkv, kc, vc, ctx, R, heads, hd, Tmax, pos):
        self.mas_kv_append_f16(qkv, R, 1, heads, hd, kc, vc, Tmax, pos)
        self.mas_attn_decode_f16(qkv, kc, vc, ctx, R, heads, hd, Tmax, pos + 1)


@pytest.fixture
def emu(monkeypatch):
    from mas_b200 import ops
    e = BatchedEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: False)
    monkeypatch.setattr(ops.L, "query", lambda name, *a: 256)
    monkeypatch.setattr(torch.cuda, "graph_pool_handle", lambda: None)
    return e


def _model(tag):
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, f"transformer_{tag}.pt"), weights_only=False)
    m = MakeAScene(**g["cfg"])
    m.load_state_dict(g["state_dict"])
    m.device = torch.device("cpu")
    m.eval()
    return m, g


def _tile(t, B):
    return t.repeat((B + t.shape[0] - 1) // t.shape[0], *([1] * (t.dim() - 1)))[:B].contiguous()


@pytest.mark.parametrize("tag", ["tiny", "wide"])
@pytest.mark.parametrize("B", [9, 40])
def test_generate_batched_teacher_forced_matches_reference(emu, tag, B):
    """The fixture's two rows tiled to B rows (R = B > 8): every copy reproduces the REAL reference's logits to 2e-3."""
    m, g = _model(tag)
    toks, lg = m.generate(_tile(g["text"], B), _tile(g["seg"], B), img_tokens=_tile(g["img"], B), return_logits=True)
    assert torch.equal(toks, _tile(g["img"], B))
    ref = _tile(g["logits"], B)
    for r in range(B):
        assert rel_err(lg[r], ref[r]) < 2e-3, r


def test_generate_batched_guidance_mix(emu):
    """B = 5 with guidance (R = 10): the mix equals uncond + s (cond - uncond) from the module's own forward."""
    m, g = _model("tiny")
    text, seg, img = _tile(g["text"], 5), _tile(g["seg"], 5), _tile(g["img"], 5)
    with torch.no_grad():
        cond = m(text, seg, img)
        uncond = m(torch.zeros_like(text), seg, img)
    _, lg = m.generate(text, seg, guidance_scale=2.5, img_tokens=img, return_logits=True)
    assert rel_err(lg, uncond + 2.5 * (cond - uncond)) < 2e-3
    assert "mas_linear_rows_f16" in emu.names and "mas_linear_small" not in emu.names


def test_entry_routing_by_row_count(emu):
    """R > 8: no mas_linear_small, one mas_attn_decode_append_f16 per layer and step, the prefix appended to the fp16 caches.
    R <= 8: exactly the fp32 entries and counts of the strict-fp32 decoder."""
    m, g = _model("tiny")
    layers, steps = len(m.transformer.layers), m.image_length - 1
    m.generate(_tile(g["text"], 12), _tile(g["seg"], 12), img_tokens=_tile(g["img"], 12))
    n = emu.names
    assert n.count("mas_linear_small") == 0
    assert n.count("mas_attn_decode_append_f16") == layers * steps and n.count("mas_attn_decode_append") == 0
    assert n.count("mas_kv_append_f16") == layers and n.count("mas_kv_append") == 0
    linears = 4 * layers * steps + steps + 1            # decode steps + to_logits after the prefix and after every step
    assert n.count("mas_linear_rows_f16") == linears
    emu.names.clear()
    m.generate(g["text"], g["seg"], img_tokens=g["img"])
    n = emu.names
    assert n.count("mas_linear_small") == linears
    assert n.count("mas_attn_decode_append") == layers * steps and n.count("mas_kv_append") == layers
    assert not [x for x in n if x.endswith("_f16") or x == "mas_to_half"]


def test_linear_small_falls_back_to_8_row_chunks(emu):
    """K % 64 != 0 above 8 rows: the fp32 kernel over chunks of at most 8 rows, nothing else."""
    from mas_b200 import ops
    gen = torch.Generator().manual_seed(3)
    x, w, b = torch.randn(19, 36, generator=gen), torch.randn(10, 36, generator=gen), torch.randn(10, generator=gen)
    y = ops.linear_small(x, w, b, act=1)
    ref = torch.nn.functional.gelu(torch.nn.functional.linear(x.double(), w.double(), b.double()), approximate="tanh")
    assert rel_err(y, ref) < 1e-6
    rows = [a[6] for name, a in emu.args if name == "mas_linear_small"]
    assert rows == [8, 8, 3]


def test_fp16_cache_and_layernorm_pair_at_40_rows(emu):
    from models.transformer import _GraphedDecoder
    m, g = _model("tiny")
    assert _GraphedDecoder(m, 40, torch.device("cpu")).kc[0].dtype == torch.float16
    assert _GraphedDecoder(m, 8, torch.device("cpu")).kc[0].dtype == torch.float32
    m.generate(_tile(g["text"], 40), _tile(g["seg"], 40), img_tokens=_tile(g["img"], 40))
    rows = {a[8] for name, a in emu.args if name == "mas_layernorm2_forward"}
    assert rows == {40}
    assert emu.names.count("mas_layernorm2_forward") == 2 * len(m.transformer.layers) * (m.image_length - 1)


def test_linear_above_8_rows_routes_by_shape_and_rows(emu):
    """The narrow split form up to the shape's row limit, beyond it the training GEMM (+ the GELU kernel for act=1); both from
    the same cached weight image, padded to 128 output features."""
    from mas_b200 import ops
    gen = torch.Generator().manual_seed(5)
    for R, N, K, act, entries in [(64, 96, 64, 1, ["mas_linear_rows_f16"]), (65, 96, 64, 1, ["mas_gemm_rows_f16", "mas_gelu_forward"]),
                                  (128, 1024, 1024, 0, ["mas_linear_rows_f16"]), (129, 1024, 1024, 0, ["mas_gemm_rows_f16"])]:
        x, w, b = torch.randn(R, K, generator=gen), torch.randn(N, K, generator=gen) / K ** 0.5, torch.randn(N, generator=gen)
        emu.names.clear()
        y = ops.linear_small(x, w, b, act=act)
        ref = torch.nn.functional.linear(x.double(), w.half().double(), b.double())
        if act:
            ref = torch.nn.functional.gelu(ref, approximate="tanh")
        assert rel_err(y, ref) < 2e-3
        assert [n for n in emu.names if n not in ("mas_amax", "mas_to_half", "mas_pack_gemm_tc16")] == entries, (R, N, emu.names)


def test_decoder_holds_weight_images_and_tracks_parameter_versions(emu):
    from models.transformer import _GraphedDecoder, _param_version
    m, g = _model("tiny")
    dec = _GraphedDecoder(m, 12, torch.device("cpu"))
    assert len(dec.images) == 4 * len(m.transformer.layers) + 1 and emu.names.count("mas_pack_gemm_tc16") == len(dec.images)
    assert _GraphedDecoder(m, 8, torch.device("cpu")).images == []
    assert dec.version == _param_version(m)
    with torch.no_grad():
        m.transformer.layers[0].mlp.lin2.weight.mul_(1.0)
    assert dec.version != _param_version(m)
