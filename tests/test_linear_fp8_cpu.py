"""The FP8 Linear route (csrc/gemm_f8.cu, ops.linear / LinearFn(fp8=True), MakeAScene(fp8_linear=True)) without a GPU:
  * the scale rule and the e4m3 / e5m2 conversion restated in numpy, bit for bit against torch's float8 casts;
  * the transposed, zero-padded layout of the cast pass;
  * the new entries' size queries and refusals on the real library (no launch), and their header declarations;
  * LinearFn's FP8 branch and the MakeAScene flag plumbing above an emulated C-ABI, against an fp64 restatement of the quantised
    computation (the pattern of test_host_logic_cpu.py);
  * the flag leaves the state_dict alone and refuses anything but a bool."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from test_host_logic_cpu import Emu, _addr, _f32

FORMATS = {"e4m3": (7, 3, 448.0, 7, torch.float8_e4m3fn), "e5m2": (15, 2, 57344.0, 14, torch.float8_e5m2)}   # bias, mantissa, max, top


def scale_of(amax, fmt):
    """The power of two that puts amax in [2^top, 2^(top+1)) (tc::operand_scale<top>): 1 for a zero, subnormal or non-finite
    amax; its biased exponent is clamped to [1, 254]."""
    a = np.float32(amax)
    e = int((a.view(np.uint32) >> 23) & 0xFF)
    if e == 0 or e == 255:
        return 1.0
    se = min(max(127 + FORMATS[fmt][3] - (e - 127), 1), 254)
    return 2.0 ** (se - 127)


def fp8_bits(v, fmt):
    """uint8 codes of round-to-nearest-even, saturate-to-finite conversions of the fp32 values v (NaN -> 0x7F | sign)."""
    bias, mant, vmax = FORMATS[fmt][:3]
    v = np.asarray(v, np.float32).astype(np.float64)
    sign = np.signbit(v).astype(np.int64) << 7
    nan = np.isnan(v)
    a = np.minimum(np.abs(np.where(nan, 0.0, v)), vmax)
    emin = 1 - bias
    e = np.maximum(np.floor(np.log2(np.where(a > 0, a, 1.0))), emin)
    r = np.round(a / 2.0 ** (e - mant)) * 2.0 ** (e - mant)                # numpy rounds halves to even
    e2 = np.floor(np.log2(np.where(r > 0, r, 1.0)))
    normal = r >= 2.0 ** emin
    code = np.where(normal, (e2 + bias) * 2 ** mant + (r / 2.0 ** e2 - 1.0) * 2 ** mant, r / 2.0 ** (emin - mant))
    bits = code.astype(np.int64) | sign
    nan_code = 0x7F if fmt == "e4m3" else 0x7E
    return np.where(nan, nan_code | sign, bits).astype(np.uint8)


def decode(bits, fmt):
    return torch.from_numpy(np.ascontiguousarray(bits)).view(FORMATS[fmt][4]).double().numpy()


def quantise(x, fmt, amax=None):
    """(fp8 codes of x * s, s) with s from max|x| (or amax)."""
    x = np.asarray(x, np.float32)
    s = scale_of(np.abs(x).max() if amax is None else amax, fmt)
    return fp8_bits((x.astype(np.float64) * s).astype(np.float32), fmt), s


# ------------------------------------------------------------------------------------------------ scale rule and conversion
@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_scale_rule_puts_the_maximum_in_the_top_binade(fmt):
    top = FORMATS[fmt][3]
    rng = np.random.default_rng(1)
    for a in np.concatenate([10.0 ** rng.uniform(-30, 30, 500), [1.0, 2.0, 0.75, 448.0, 3e38, 2.0 ** -110]]).astype(np.float32):
        s = scale_of(a, fmt)
        assert 2.0 ** top <= float(a) * s < 2.0 ** (top + 1), (a, s)
    for a in (0.0, np.inf, -np.inf, np.nan, 1e-40):
        assert scale_of(a, fmt) == 1.0
    assert scale_of(2.0 ** -125, fmt) == 2.0 ** 127      # clamped: 2^(top + 125) is not an fp32 number


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_conversion_matches_torch_float8_casts_bit_for_bit(fmt):
    bias, mant, vmax, top, dt = FORMATS[fmt]
    rng = np.random.default_rng(2)
    x = np.concatenate([rng.standard_normal(20000) * 10.0 ** rng.uniform(-6, 3, 20000),
                        np.arange(-2 ** (top + 1), 2 ** (top + 1), 0.0625),          # every rounding tie of the top binades
                        [0.0, -0.0, vmax, -vmax, vmax * 1.2, 2.0 ** (1 - bias - mant), 2.0 ** (-bias - mant), 3e38, -np.inf,
                         np.inf, np.nan]]).astype(np.float32)
    mine = fp8_bits(x, fmt)
    ref = torch.from_numpy(x).clamp(-vmax, vmax).to(dt).view(torch.uint8).numpy()      # torch's cast gives NaN / Inf out of range
    finite = ~np.isnan(x)
    assert np.array_equal(mine[finite], ref[finite])
    assert np.isnan(decode(mine[~finite], fmt)).all()
    # a scaled tensor never saturates: its largest element is below the format's maximum
    q, s = quantise(x[np.isfinite(x)], fmt)
    assert np.abs(decode(q, fmt)).max() < 2.0 ** (top + 1) and np.abs(decode(q, fmt)).max() <= vmax


def transposed(codes, M):
    """The [K, M'] layout of mas_to_fp8's y_cols: the transpose of [M, K] codes, M' = M rounded up to 16, zero columns."""
    K = codes.shape[1]
    out = np.zeros((K, (M + 15) // 16 * 16), np.uint8)
    out[:, :M] = codes.T
    return out


@pytest.mark.parametrize("M", [1, 16, 37, 640])
def test_transposed_layout_is_zero_padded_to_16_rows(M):
    rng = np.random.default_rng(M)
    x = rng.standard_normal((M, 48)).astype(np.float32)
    q, _ = quantise(x, "e4m3")
    t = transposed(q, M)
    assert t.shape == (48, (M + 15) // 16 * 16) and t.shape[1] % 16 == 0
    assert np.array_equal(t[:, :M], q.T) and not t[:, M:].any()
    # the padding contributes nothing to a contraction over the rows
    assert np.array_equal(decode(t, "e4m3") @ decode(t, "e4m3").T, decode(q, "e4m3").T @ decode(q, "e4m3"))


# ------------------------------------------------------------------------------------------------ the C entries on this host
def test_header_declares_the_fp8_entries():
    from conftest import ROOT
    from mas_b200 import _lib, ops
    src = open(os.path.join(ROOT, "include", "mas_b200.h")).read()
    for name in ("mas_to_fp8_ws_bytes", "mas_to_fp8", "mas_pack_gemm_f8", "mas_gemm_rows_f8", "mas_wgrad_rows_f8_ws_bytes",
                 "mas_wgrad_rows_f8"):
        assert re.search(r"\b%s\(" % name, src) and name in _lib.exported_symbols(), name
    assert "#define MAS_FP8_E4M3 0" in src and "#define MAS_FP8_E5M2 1" in src
    assert (ops.FP8_E4M3, ops.FP8_E5M2) == (0, 1)


def test_size_queries_and_refusals_need_no_launch():
    """The workspace queries and every refusal of the new entries run on the host before any CUDA call."""
    from mas_b200 import _lib
    lib = _lib.load()
    assert lib.mas_to_fp8_ws_bytes(5120, 1024) == 80 * 1024 * 4           # one fp32 partial per 64-row tile and column
    assert lib.mas_to_fp8_ws_bytes(65, 16) == 2 * 16 * 4 and lib.mas_to_fp8_ws_bytes(0, 16) == 0
    assert lib.mas_wgrad_rows_f8_ws_bytes(0, 128, 128) == 0
    # 1024 x 1024 is 64 tiles of 128 x 128: split-K fills the SMs, its partials need a workspace; 3072 x 1024 needs none
    assert lib.mas_wgrad_rows_f8_ws_bytes(5120, 1024, 1024) % (1024 * 1024 * 4) == 0
    assert lib.mas_wgrad_rows_f8_ws_bytes(5120, 1024, 1024) >= 2 * 1024 * 1024 * 4
    fake, fake2 = ctypes.c_void_p(4096), ctypes.c_void_p(8192)
    odd = ctypes.c_void_p(4100)
    n0 = _lib.launch_count()
    refusals = [
        ("mas_to_fp8", (None, 64, 64, 0, fake, fake, None, None, None, 0), -1),
        ("mas_to_fp8", (fake, 64, 64, 0, fake, None, None, None, None, 0), -1),       # nothing to write
        ("mas_to_fp8", (fake, 64, 40, 0, fake, fake, None, None, None, 0), -2),       # K % 16
        ("mas_to_fp8", (fake, 0, 64, 0, fake, fake, None, None, None, 0), -2),
        ("mas_to_fp8", (fake, 64, 64, 2, fake, fake, None, None, None, 0), -1),       # format
        ("mas_to_fp8", (fake, 64, 64, 0, fake, odd, None, None, None, 0), -1),        # alignment
        ("mas_to_fp8", (fake, 64, 64, 0, fake, fake, None, fake2, fake2, 255), -4),   # column sums without workspace
        ("mas_pack_gemm_f8", (fake, 128, 128, fake, None, fake), -1),
        ("mas_pack_gemm_f8", (fake, 120, 128, fake, fake2, fake), -2),
        ("mas_gemm_rows_f8", (fake, 64, 128, 0, fake, fake2, 128, None, None, fake, 128), -1),   # no weight scale
        ("mas_gemm_rows_f8", (fake, 64, 120, 0, fake, fake2, 128, fake, None, fake, 128), -2),
        ("mas_gemm_rows_f8", (fake, 64, 128, 3, fake, fake2, 128, fake, None, fake, 128), -1),
        ("mas_gemm_rows_f8", (fake, 64, 128, 0, fake, fake2, 128, fake, None, fake, 100), -1),   # ldy < N
        ("mas_gemm_rows_f8", (odd, 64, 128, 0, fake, fake2, 128, fake, None, fake, 128), -1),
        ("mas_wgrad_rows_f8", (fake, fake2, 64, 128, 128, None, fake, fake, fake, 1 << 30), -1),
        ("mas_wgrad_rows_f8", (fake, fake2, 0, 128, 128, fake, fake, fake, fake, 1 << 30), -2),
        ("mas_wgrad_rows_f8", (fake, fake2, 5120, 1024, 1024, fake, fake, fake, fake, 16), -4),
        ("mas_wgrad_rows_f8", (fake, odd, 64, 128, 128, fake, fake, fake, fake, 1 << 30), -1),
    ]
    for name, args, code in refusals:
        assert getattr(lib, name)(*args, None) == code, (name, args)
        assert name[4:].encode() in lib.mas_last_error(), lib.mas_last_error()
    assert _lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------ host logic over the C-ABI
class Fp8Emu(Emu):
    """The entries of the FP8 route by their header semantics (numpy conversion above), on the memory the pointers name."""

    def __init__(self):
        super().__init__()
        self.fmt = {}

    @staticmethod
    def _u8(p, n):
        return np.ctypeslib.as_array((ctypes.c_uint8 * n).from_address(_addr(p)))

    def mas_to_fp8(self, x, M, K, fmt, amax, rows, cols, colsum, ws, ws_bytes):
        f = ("e4m3", "e5m2")[fmt]
        X = _f32(_addr(x), M * K).reshape(M, K)
        q, _ = quantise(X, f, amax=_f32(_addr(amax), 1)[0])
        if rows is not None:
            self._u8(rows, M * K)[...] = q.reshape(-1)
        if cols is not None:
            t = transposed(q, M)
            self._u8(cols, t.size)[...] = t.reshape(-1)
        if colsum is not None:
            assert ws is not None and ws_bytes >= (M + 63) // 64 * K * 4
            _f32(_addr(colsum), K)[...] = X.astype(np.float64).sum(0)

    def mas_pack_gemm_f8(self, w, N, K, w8, w8t, amax):
        self.mas_amax(w, N * K, amax)
        self.mas_to_fp8(w, N, K, 0, amax, w8, w8t, None, None, 0)

    def mas_gemm_rows_f8(self, x8, M, K, fmt, x_amax, w8, N, w_amax, bias, y, ldy):
        f = ("e4m3", "e5m2")[fmt]
        X = decode(self._u8(x8, M * K).reshape(M, K), f) / scale_of(_f32(_addr(x_amax), 1)[0], f)
        W = decode(self._u8(w8, N * K).reshape(N, K), "e4m3") / scale_of(_f32(_addr(w_amax), 1)[0], "e4m3")
        o = X @ W.T
        if bias is not None:
            o = o + _f32(_addr(bias), N)[None, :]
        _f32(_addr(y), M * ldy).reshape(M, ldy)[:, :N] = o

    def mas_wgrad_rows_f8(self, x8t, dy8t, M, N, K, x_amax, dy_amax, dw, ws, ws_bytes):
        Mp = (M + 15) // 16 * 16
        Xt = decode(self._u8(x8t, K * Mp).reshape(K, Mp), "e4m3") / scale_of(_f32(_addr(x_amax), 1)[0], "e4m3")
        Dt = decode(self._u8(dy8t, N * Mp).reshape(N, Mp), "e5m2") / scale_of(_f32(_addr(dy_amax), 1)[0], "e5m2")
        _f32(_addr(dw), N * K).reshape(N, K)[...] = Dt @ Xt.T


@pytest.fixture
def emu8(monkeypatch):
    from mas_b200 import ops
    e = Fp8Emu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: False)
    monkeypatch.setattr(ops.L, "query", lambda name, *a: 1 << 20)
    monkeypatch.setattr(ops, "f16_operands", lambda: True)
    monkeypatch.setenv("MAS_LINEAR_F16", "1")
    return e


def dq(t, fmt):
    """fp64 values of the quantised tensor under its own scale, by torch's casts: dequantised operand."""
    vmax, dt = FORMATS[fmt][2], FORMATS[fmt][4]
    s = scale_of(float(t.abs().max()), fmt)
    return (t.float() * s).clamp(-vmax, vmax).to(dt).double() / s


@pytest.mark.parametrize("shape,bias", [((3, 37, 128), True), ((130, 256), False)])
def test_linear_fn_fp8_branch_against_the_quantised_computation(emu8, shape, bias):
    from mas_b200 import ops
    g = torch.Generator().manual_seed(shape[-1])
    N, K = 384, shape[-1]
    x = torch.randn(shape, generator=g).requires_grad_(True)
    W = (torch.randn(N, K, generator=g) * 0.05).requires_grad_(True)
    b = torch.randn(N, generator=g).requires_grad_(True) if bias else None
    dy = torch.randn(shape[:-1] + (N,), generator=g) * 1e-3
    y = ops.linear(x, W, b, True)
    y.backward(dy)
    assert "mas_gemm_rows_f8" in emu8.names and "mas_gemm_rows_f16" not in emu8.names
    xq, wq, dyq = dq(x.detach().reshape(-1, K), "e4m3"), dq(W.detach(), "e4m3"), dq(dy.reshape(-1, N), "e5m2")
    ref_y = xq @ wq.T + (b.detach().double() if bias else 0)
    assert torch.allclose(y.detach().reshape(-1, N).double(), ref_y, rtol=1e-6, atol=1e-6)
    assert torch.allclose(x.grad.reshape(-1, K).double(), dyq @ wq, rtol=1e-6, atol=1e-9)
    assert torch.allclose(W.grad.double(), dyq.T @ xq, rtol=1e-6, atol=1e-9)
    if bias:
        assert torch.allclose(b.grad.double(), dy.reshape(-1, N).double().sum(0), rtol=1e-6, atol=1e-9)
    # only x^T (1 byte per element, rows padded to 16) and the scale source are saved for the backward
    assert emu8.names.count("mas_to_fp8") == 2 and emu8.names.count("mas_pack_gemm_f8") == 1


def test_linear_fp8_route_rule(emu8, monkeypatch):
    """The FP8 route is taken only when the call records a graph and linear_fp8_on holds; otherwise the fp16 route runs."""
    from mas_b200 import ops
    x = torch.randn(4, 128)
    W = torch.randn(256, 128).requires_grad_(True)

    def route(*a, **k):
        emu8.names.clear()
        ops.linear(*a, **k)
        return "fp8" if "mas_gemm_rows_f8" in emu8.names else "f16" if "mas_gemm_rows_f16" in emu8.names else "other"
    assert route(x, W, None, True) == "fp8"
    assert route(x, W.detach(), None, True) == "f16"                       # nothing requires a gradient
    with torch.no_grad():
        assert route(x, W, None, True) == "f16"
    assert route(x, W, None, False) == "f16"
    monkeypatch.setenv("MAS_LINEAR_F16", "0")
    assert route(x, W, None, True) == "other"
    monkeypatch.setenv("MAS_LINEAR_F16", "1")
    monkeypatch.setattr(ops, "f16_operands", lambda: False)
    assert route(x, W, None, True) == "other"
    assert not ops.linear_fp8_on(256, 128)


def _wide_model(fp8):
    from conftest import GOLDEN
    from models.transformer import MakeAScene
    g = torch.load(os.path.join(GOLDEN, "transformer_wide.pt"), weights_only=False)
    m = MakeAScene(**g["cfg"], fp8_linear=fp8)
    m.load_state_dict(g["state_dict"])
    m.device = torch.device("cpu")
    return m, g


def test_make_a_scene_flag_plumbing(emu8):
    """fp8_linear=True puts the four Linear layers of every TransformerLayer on the FP8 route in training and leaves to_logits and
    every no-grad call on the fp16 one; the loss and gradients stay near the reference's (tests/golden/transformer_wide.pt)."""
    from conftest import rel_err
    m, g = _wide_model(True)
    L = g["cfg"]["num_layers"]
    lins = [l for layer in m.transformer.layers for l in (layer.attn.qkv, layer.attn.out_proj, layer.mlp.lin1, layer.mlp.lin2)]
    assert all(l.fp8 for l in lins) and not m.to_logits[1].fp8
    loss = m.loss(g["text"], g["seg"], g["img"])
    loss.backward()
    assert emu8.names.count("mas_gemm_rows_f8") == 2 * 4 * L                       # forward + data gradient
    assert emu8.names.count("mas_wgrad_rows_f8") == 4 * L
    assert emu8.names.count("mas_gemm_rows_f16") == 2 and emu8.names.count("mas_wgrad_rows_f16") == 1   # to_logits
    assert abs(float(loss.detach()) - float(g["loss"])) < 1e-2 * float(g["loss"])
    named = dict(m.named_parameters())
    errs = {k: rel_err(named[k].grad, gv) for k, gv in g["grads"].items()}
    assert max(errs.values()) < 0.2, errs          # e4m3 keeps 3 mantissa bits: 0.104 at most here (the loss: 9e-4)
    emu8.names.clear()
    with torch.no_grad():
        m(g["text"], g["seg"], g["img"])
    assert not any("f8" in n for n in emu8.names)
    lins[0].fp8 = False                                                              # one layer by hand
    emu8.names.clear()
    m.loss(g["text"], g["seg"], g["img"]).backward()
    assert emu8.names.count("mas_gemm_rows_f8") == 2 * (4 * L - 1)


def test_flag_leaves_the_state_dict_alone():
    from models.transformer import MakeAScene, Transformer
    cfg = dict(num_layers=2, hidden_dim=128, num_attn_heads=2, image_vocab_size=16, seg_vocab_size=8, text_vocab_size=8,
               image_tokens_per_dim=2, seg_tokens_per_dim=2, text_length=4)
    torch.manual_seed(0)
    a = MakeAScene(**cfg).state_dict()
    torch.manual_seed(0)
    b = MakeAScene(**cfg, fp8_linear=True).state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    t = Transformer(2, 128, 2, 2, 2, 4, fp8_linear=True)
    assert all(layer.mlp.lin1.fp8 for layer in t.layers)


@pytest.mark.parametrize("bad", [1, 0, "yes", None, 1.0, torch.tensor(True)])
def test_bad_flag_raises_value_error(bad):
    from models.transformer import MakeAScene, Transformer
    with pytest.raises(ValueError):
        MakeAScene(1, 128, 2, 16, 8, 8, 2, 2, 4, fp8_linear=bad)
    with pytest.raises(ValueError):
        Transformer(1, 128, 2, 2, 2, 4, fp8_linear=bad)
