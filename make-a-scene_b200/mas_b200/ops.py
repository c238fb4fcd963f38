"""torch.autograd.Function wrappers over the C-ABI kernels (one Function per fused unit of the hot path).

Activations are fp32 tensors of logical shape [N,C,H,W] in channels-last (NHWC) memory; any other layout
arriving at a module boundary is converted once with mas_copy_strided. All arithmetic happens in
libmas_b200.so; torch is used for allocation, autograd bookkeeping and (for SyncBatchNorm) the NCCL
all-reduce of 2*C statistics.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import _lib as L

GN_GROUPS = 32
GN_EPS = 1e-6

import os

# "f16": fp16 operands on the 3x3 tensor-core kernels (same 11-bit significand as TF32, twice the MMA rate; operand scales
# from a device-side amax); "tf32": TF32 operands. MAS_CONV_OPERANDS overrides the default for A/B measurements.
_cfg = {"impl": L.IMPL_AUTO, "operands": os.environ.get("MAS_CONV_OPERANDS", "f16")}


def set_operand_format(fmt: str):
    """Operand format of the 3x3 convolution tensor-core kernels: "f16" (default) or "tf32"."""
    if fmt not in ("f16", "tf32"):
        raise ValueError(fmt)
    _cfg["operands"] = fmt


def get_operand_format() -> str:
    return _cfg["operands"]


def amax(x):
    """max|x| as a device scalar (stays on the device: the kernels derive their power-of-two operand scale from it)."""
    out = torch.empty(1, dtype=torch.float32, device=x.device)
    L.call("mas_amax", x, x.numel(), out)
    return out


def set_impl(impl: int):
    """Select the contraction implementation globally (IMPL_AUTO / IMPL_SIMT / IMPL_TC)."""
    _cfg["impl"] = int(impl)


def get_impl() -> int:
    return _cfg["impl"]


def _need_cuda(x):
    if not x.is_cuda:
        raise RuntimeError("make-a-scene_b200 kernels run on CUDA (sm_90a) only; got a %s tensor — there is no CPU path"
                           % x.device.type)
    if x.dtype != torch.float32:
        raise RuntimeError("make-a-scene_b200 kernels take float32 tensors, got %s" % x.dtype)


def nhwc(x: torch.Tensor) -> torch.Tensor:
    """Return x in dense channels-last memory (no copy if it already is)."""
    _need_cuda(x)
    if x.dim() != 4:
        raise RuntimeError("expected a 4-D [N,C,H,W] tensor")
    if x.is_contiguous(memory_format=torch.channels_last) and x.stride(1) == 1:
        return x
    y = torch.empty_like(x, memory_format=torch.channels_last)
    L.call("mas_copy_strided", x, L.t4(x), y, L.t4(y))
    return y


def empty_nhwc(n, c, h, w, like):
    return torch.empty((n, c, h, w), dtype=torch.float32, device=like.device, memory_format=torch.channels_last)


# ------------------------------------------------------------------------------------------------ raw (no-autograd) helpers
def gn_stats(x):
    n, c, h, w = x.shape
    mean = torch.empty(n * GN_GROUPS, dtype=torch.float32, device=x.device)
    rstd = torch.empty_like(mean)
    nb = L.query("mas_gn_ws_bytes", n, h * w, c, GN_GROUPS)
    ws = L.workspace(nb, x.device)
    L.call("mas_gn_stats", x, n, h * w, c, GN_GROUPS, GN_EPS, mean, rstd, ws, ws.numel())
    return mean, rstd


def gn_apply(x, mean, rstd, gamma, beta, silu, rtf32=False):
    n, c, h, w = x.shape
    y = torch.empty_like(x)
    L.call("mas_gn_apply", x, mean, rstd, gamma, beta, y, n, h * w, c, GN_GROUPS, int(silu), int(rtf32))
    return y


def gn_backward(dy, x, mean, rstd, gamma, beta, silu, dx_add=None, want_act=False, act_f16=False, shadow=False, add_amax=None,
                shadow_only=False):
    """want_act: also return act(GN(x)) (re-materialised as a by-product of the first backward pass). With fp16 operands
    selected, max|dx| is produced by the same pass and attached to dx (attach_amax) for the tensor-core kernels that
    consume it. shadow: dx is also written as an fp16 channels-last tensor scaled by a power of two from a rigorous bound on
    max|dx| (attached: shadow_of) - the operand the TMA-fed data-gradient convolution reads; add_amax = max|dx_add|.
    shadow_only: the fp32 dx is not written at all; the first return value is then the (shadow, scale source) pair."""
    n, c, h, w = x.shape
    shadow = shadow or shadow_only
    dx = None if shadow_only else torch.empty_like(x)
    dg = torch.empty_like(gamma)
    db = torch.empty_like(beta)
    # act_f16: the re-materialised activation only feeds the fp16-operand weight gradient -> written as fp16 (half the bytes)
    act = torch.empty_like(x, dtype=torch.float16 if act_f16 else torch.float32) if want_act else None
    am = torch.empty(1, dtype=torch.float32, device=x.device) if (f16_operands() and not shadow_only) else None
    dx16 = bound = None
    if shadow:
        dx16 = torch.empty_like(x, dtype=torch.float16)
        bound = torch.empty(1, dtype=torch.float32, device=x.device)
        if dx_add is not None and add_amax is None:
            add_amax = amax_of(dx_add)
    nb = L.query("mas_gn_ws_bytes", n, h * w, c, GN_GROUPS)
    ws = L.workspace(nb, x.device)
    L.call("mas_gn_backward", dy, x, mean, rstd, gamma, beta, dx_add, dx, dg, db, act, int(act_f16 and want_act), am,
           add_amax if shadow else None, dx16, bound, n, h * w, c, GN_GROUPS, int(silu), ws, ws.numel())
    if shadow_only:
        dx = (dx16, bound)
    else:
        attach_amax(dx, am)
        if shadow:
            dx._mas_shadow = (dx16, bound, dx._version, dx.data_ptr())
    if want_act:
        return dx, dg, db, act
    return dx, dg, db


def shadow_of(t):
    """(fp16 shadow, scale source) attached by the kernel that wrote t, if t is unchanged since; else None."""
    st = getattr(t, "_mas_shadow", None)
    if st is not None and st[2] == t._version and st[3] == t.data_ptr() and st[0].device == t.device and st[0].shape == t.shape:
        return st[0], st[1]
    return None


def attach_amax(t, am):
    """Carry max|t| (device scalar produced by the kernel that wrote t) with the tensor object; autograd hands the same
    object to the consuming Function's backward."""
    if am is not None:
        t._mas_amax = (am, t._version, t.data_ptr())
    return t


def amax_of(t):
    """max|t| as a device scalar: the value attached by the producing kernel if t is unchanged since, else one pass."""
    st = getattr(t, "_mas_amax", None)
    if st is not None and st[1] == t._version and st[2] == t.data_ptr() and st[0].device == t.device:
        return st[0]
    return amax(t)


def _conv_out_hw(h, w, mode):
    if mode == L.CONV_S1:
        return h, w
    if mode == L.CONV_S2:
        return h // 2, w // 2
    return 2 * h, 2 * w


def _tc_on():
    return _cfg["impl"] != L.IMPL_SIMT


def _nhwc4(n, h, w, c):
    """mas_tensor4 of a dense channels-last [n, c, h, w] tensor."""
    return L.Tensor4(n, h, w, c, h * w * c, w * c, c, 1)


def conv_tc_eligible(x, cout, mode):
    """True when conv3x3 of dense-NHWC x with `cout` output channels runs on the tensor-core kernel."""
    if not _tc_on() or not _is_dense_nhwc(x):
        return False
    n, _, h, w = x.shape
    ho, wo = _conv_out_hw(h, w, mode)
    return bool(L.query("mas_conv3x3_tc_eligible", L.t4(x), _nhwc4(n, ho, wo, cout), mode))


def gn_table(mean, rstd, gamma, beta, n, c):
    """(scale, shift) per (image, channel): act(GroupNorm(x)) = act(x*sc + sh) — consumed by the conv producers."""
    t = torch.empty((n, c, 2), dtype=torch.float32, device=mean.device)
    L.call("mas_gn_table", mean, rstd, gamma, beta, n, c, GN_GROUPS, t)
    return t


def _stats_part(y, want):
    """Partial sums for the GroupNorm-statistics epilogue of the tensor-core kernel writing y: a (sum, sum of squares) pair per
    channel and 128-pixel tile. None when no statistics are wanted or the channels do not split into 4-channel quads per group."""
    n, c, h, w = y.shape
    if not want or c % (4 * GN_GROUPS):
        return None
    return torch.empty(n * (h * w // 128) * c * 2, dtype=torch.float32, device=y.device)


def _finalize_stats(part, n, c, hw):
    """(mean, rstd) per (image, group) from the per-128-pixel-tile partials of a statistics epilogue (None without partials)."""
    if part is None:
        return None
    mean = torch.empty(n * GN_GROUPS, dtype=torch.float32, device=part.device)
    rstd = torch.empty_like(mean)
    L.call("mas_gn_finalize_partials", part, hw // 128, n, c, GN_GROUPS, hw, GN_EPS, mean, rstd)
    return mean, rstd


def conv3x3_raw(x, weight, bias, residual, mode, out_nchw=False, transpose=False, table=None, silu=True, want_stats=False,
                prepack=False, x_amax=None, pad_out=False):
    """y = conv3x3(x; weight) (+bias, +residual). transpose=True applies the data-gradient operand
    (taps flipped, Cin<->Cout). Dense NHWC shapes with Cin%8==0, Cout%128==0, Hout%16==0, Wout%8==0 run on the
    tensor-core kernel; everything else (edge layers, NCHW views, small images) on the fp32 SIMT kernel.
    table: fused GroupNorm(+SiLU) prologue (tensor path only); want_stats: also return the output's GroupNorm
    (mean, rstd) from the fused epilogue (None when the tensor path does not apply).
    pad_out: the fp16 tensor-core kernel also takes an output width off the 128-wide tile. The weight and bias are zero-padded to
    the tile, the kernel stores round_up(Cout, 4) channels and the Cout real ones come back as a channels-last view. Without
    fp16 operands, or where even the padded shape does not fit, such a call runs on the fp32 SIMT kernel, never the TF32 one."""
    n, _, h, w = x.shape
    cout = weight.shape[1] if transpose else weight.shape[0]
    cin = weight.shape[0] if transpose else weight.shape[1]
    ho, wo = _conv_out_hw(h, w, mode)
    xs = L.t4(x)
    f16 = _cfg["operands"] == "f16" and cin % 16 == 0
    ck = _round_up(cout, 128) if pad_out else cout          # output channels the tensor-core kernel computes
    if (_tc_on() and not out_nchw and (f16 or not pad_out)
            and L.query("mas_conv3x3_tc_eligible", xs, _nhwc4(n, ho, wo, ck), mode)):
        y = empty_nhwc(n, _round_up(cout, 4), ho, wo, x)
        ys = L.t4(y)
        wt = _packed_conv_weight(weight.contiguous(), weight, ck, cin, transpose, x.device, prepack, f16)
        bias = None if bias is None else _padded(bias, (ck,))
        part = _stats_part(y, want_stats)
        if f16:
            # post-GroupNorm activations (prologue) are O(1) by construction; anything else (gradients above all) gets a
            # power-of-two scale from its largest magnitude
            xa = (x_amax if x_amax is not None else amax_of(x)) if table is None else None
            L.call("mas_conv3x3_fprop_tc16", x, xs, wt, bias, residual, y, ys, mode, table, int(silu), part, xa)
        else:
            L.call("mas_conv3x3_fprop_tc", x, xs, wt, bias, residual, y, ys, mode, table, int(silu), part)
        stats = _finalize_stats(part, n, cout, ho * wo)
        if y.shape[1] != cout:
            y = y[:, :cout]
    else:
        if table is not None:
            raise RuntimeError("fused GroupNorm prologue requested for a shape that is not tensor-path eligible")
        if _cfg["impl"] == L.IMPL_TC:
            raise RuntimeError("IMPL_TC requested but the conv shape is not eligible for the tensor-core kernel")
        if out_nchw:
            y = torch.empty((n, cout, ho, wo), dtype=torch.float32, device=x.device)
        else:
            y = empty_nhwc(n, cout, ho, wo, x)
        wp = torch.empty(9 * cout * cin, dtype=torch.float32, device=x.device)
        L.call("mas_pack_conv3x3", weight.contiguous(), wp, weight.shape[0], weight.shape[1], int(transpose), 0)
        L.call("mas_conv3x3_fprop", x, xs, wp, bias, residual, y, L.t4(y), mode, L.IMPL_SIMT)
        stats = None
    if want_stats:
        return y, stats
    return y


def conv_tma_on():
    """TMA-fed fp16 convolution kernel (csrc/conv_tma.cu) for stride-1 3x3 layers whose input has an fp16 shadow."""
    return f16_operands() and os.environ.get("MAS_CONV_TMA", "1") != "0"


def conv_h_eligible(n, cin, h, w, cout):
    return conv_tma_on() and cin % 64 == 0 and cout % 128 == 0 and h % 16 == 0 and w % 8 == 0


def to_half(x, x_amax=None):
    """fp16 channels-last shadow of x (scaled by the power-of-two operand scale of *x_amax when given)."""
    if not _is_dense_nhwc(x):
        raise RuntimeError("to_half expects a dense channels-last tensor")
    y = torch.empty_like(x, dtype=torch.float16)
    L.call("mas_to_half", x, y, x.numel(), x_amax)
    return y


def gn_apply_f16(x, mean, rstd, gamma, beta, silu):
    """act(GroupNorm(x)) written as the fp16 channels-last shadow the TMA-fed convolution reads (values are O(1): unscaled)."""
    n, c, h, w = x.shape
    y = torch.empty_like(x, dtype=torch.float16)
    L.call("mas_gn_apply", x, mean, rstd, gamma, beta, y, n, h * w, c, GN_GROUPS, int(silu), 2)
    return y


def conv3x3_h_raw(x16, weight, bias, residual, transpose=False, want_stats=False, prepack=False, x_amax=None):
    """Stride-1 conv3x3 of an fp16 channels-last shadow on the TMA-fed tensor-core kernel (fp32 output, same epilogues as
    conv3x3_raw). x_amax: the device scalar the shadow was scaled with (None: unscaled)."""
    n, _, h, w = x16.shape
    cout = weight.shape[1] if transpose else weight.shape[0]
    cin = weight.shape[0] if transpose else weight.shape[1]
    y = empty_nhwc(n, cout, h, w, x16)
    wt = _packed_conv_weight(weight.contiguous(), weight, cout, cin, transpose, x16.device, prepack, True)
    part = _stats_part(y, want_stats)
    L.call("mas_conv3x3_fprop_tc16h", x16, L.t4(x16), wt, bias, residual, y, L.t4(y), part, x_amax)
    if want_stats:
        return y, _finalize_stats(part, n, cout, h * w)
    return y


# Packed operand images of the convolution weights, cached per parameter: a packing stays valid until the weight's version
# counter moves (optimizer step / load_state_dict), so a training step packs every weight once (forward and data-gradient
# images in one pass) and evaluation / gradient accumulation / the benchmark's optimizer-free steps pack nothing at all.
# The entry holds a weak reference to the weight (identity, not storage address: the allocator reuses addresses).
_packs = {}


def _pack_entry(weight):
    k = id(weight)
    ent = _packs.get(k)
    if ent is not None and ent[0]() is weight and ent[1] == weight._version and ent[2] == weight.data_ptr():
        return ent[3]
    import weakref
    d = {}
    _packs[k] = (weakref.ref(weight, lambda _r, k=k: _packs.pop(k, None)), weight._version, weight.data_ptr(), d)
    return d


def _cached(t, key, make):
    """The tensor stored under `key` for t's current version, built by make() when absent or not on t's device."""
    ent = _pack_entry(t)
    hit = ent.get(key)
    if hit is None or hit.device != t.device:
        hit = ent[key] = make()
    return hit


def _padded(t, shape):
    """t zero-padded at the end of each dimension to `shape`, cached per version of t (t itself when it has that shape)."""
    if tuple(t.shape) == tuple(shape):
        return t

    def make():
        p = torch.zeros(shape, dtype=t.dtype, device=t.device)
        p[tuple(slice(0, s) for s in t.shape)] = t.detach()
        return p
    return _cached(t, ("pad",) + tuple(shape), make)


def _packed_conv_weight(wc, weight, cout, cin, transpose, dev, prepack=False, f16=False):
    """Tensor-core operand image of a 3x3 weight (wc: its contiguous form) for a convolution with `cout` output and `cin`
    input channels (transpose: the data gradient). Extents larger than the weight's zero-pad it first: the output side to the
    128-wide tile, the input side to the K step or to the data-gradient image's tile."""
    rows, cols = (cin, cout) if transpose else (cout, cin)       # in the weight's [Cout, Cin] order
    dt = torch.float16 if f16 else torch.float32

    def make():
        w = wc if (rows, cols) == tuple(weight.shape[:2]) else _padded(weight, (rows, cols, 3, 3))
        wt = torch.empty(9 * rows * cols, dtype=dt, device=dev)
        if prepack and not transpose and rows % 128 == 0 and cols % 128 == 0:
            # forward of a training step whose backward will run the data gradient: it wants the transposed packing
            wd = torch.empty_like(wt)
            if f16:
                L.call("mas_pack_conv3x3_tc16", w, wt, wd, rows, cols, 0)
            else:
                L.call("mas_pack_conv3x3_tc_pair", w, wt, wd, rows, cols)
            _pack_entry(weight)[("d", f16, rows, cols)] = wd
        elif f16:
            L.call("mas_pack_conv3x3_tc16", w, wt, None, rows, cols, int(transpose))
        else:
            L.call("mas_pack_conv3x3_tc", w, wt, rows, cols, int(transpose))
        return wt
    return _cached(weight, ("d" if transpose else "f", f16, rows, cols), make)


def phase_mode(x, cout, mode):
    """CONV_UP_PHASE / CONV_S2_PHASE when the Upsample / Downsample convolution of dense-NHWC x runs phase-decomposed on the
    TMA-fed kernels (forward, data and weight gradient), else None. MAS_CONV_PHASE=0 keeps the register-staged route for A/B runs."""
    if mode not in (L.CONV_UP, L.CONV_S2) or not conv_tma_on() or os.environ.get("MAS_CONV_PHASE", "1") == "0":
        return None
    if not _is_dense_nhwc(x):
        return None
    n, _, h, w = x.shape
    ho, wo = _conv_out_hw(h, w, mode)
    pm = L.CONV_UP_PHASE if mode == L.CONV_UP else L.CONV_S2_PHASE
    return pm if L.query("mas_conv3x3_tc_eligible", L.t4(x), _nhwc4(n, ho, wo, cout), pm) else None


def conv3x3_phase_raw(x16, weight, bias, pmode, transpose=False, x_amax=None):
    """Phase-decomposed Upsample / Downsample convolution (forward, or its data gradient with transpose=True) of an fp16
    channels-last shadow x16, scaled by the power-of-two operand scale of *x_amax."""
    n, c, h, w = x16.shape
    cout = weight.shape[1] if transpose else weight.shape[0]
    up_side = (pmode == L.CONV_UP_PHASE) != transpose   # the destination is the 2x side
    y = empty_nhwc(n, cout, 2 * h if up_side else h // 2, 2 * w if up_side else w // 2, x16)

    def make():
        wt = torch.empty(16 * weight.shape[0] * weight.shape[1], dtype=torch.float16, device=x16.device)
        L.call("mas_pack_conv3x3_phase16", weight.contiguous(), wt, weight.shape[0], weight.shape[1], pmode, int(transpose))
        return wt
    wt = _cached(weight, ("phase", pmode, transpose), make)
    L.call("mas_conv3x3_phase_tc16h", x16, L.t4(x16), wt, bias, y, L.t4(y), pmode, int(transpose), x_amax)
    return y


def conv3x3_phase_wgrad_raw(x16, x_amax, dy16, dy_amax, pmode, want_bias=True):
    """Weight (and bias) gradient of a phase-decomposed Upsample / Downsample convolution from the fp16 shadows of its input
    and output gradient, each scaled by the power-of-two operand scale of its device scalar (None: unscaled)."""
    cout, cin = dy16.shape[1], x16.shape[1]
    dw = torch.empty((cout, cin, 3, 3), dtype=torch.float32, device=x16.device)
    db = torch.empty(cout, dtype=torch.float32, device=x16.device) if want_bias else None
    ws = L.workspace(L.query("mas_conv3x3_phase_wgrad_tc16_ws_bytes", L.t4(x16), L.t4(dy16), pmode), x16.device)
    L.call("mas_conv3x3_phase_wgrad_tc16", x16, L.t4(x16), x_amax, dy16, L.t4(dy16), dy_amax, dw, db, pmode, ws, ws.numel())
    return dw, db


def conv3x3_wgrad_raw(x, dy, cout, cin, mode, want_bias=True, table=None, silu=True, dy_amax=None):
    """table: x is the PRE-normalisation tensor and act(GroupNorm(x)) is recomputed while staging (tensor path only)."""
    dw = torch.empty((cout, cin, 3, 3), dtype=torch.float32, device=x.device)
    db = torch.empty(cout, dtype=torch.float32, device=x.device) if want_bias else None
    nb = L.query("mas_conv3x3_wgrad_ws_bytes", L.t4(x), L.t4(dy), mode)
    ws = L.workspace(nb, x.device)
    padded = cout != dy.shape[1]      # dw sized for round_up(channels of dy, 128): the explicit padded path of Conv3x3Fn
    if (_tc_on() and _cfg["operands"] == "f16" and wgrad_f16_on() and _is_dense_nhwc(x) and _is_dense_nhwc(dy)
            and (padded or L.query("mas_conv3x3_wgrad_tc_eligible", L.t4(x), L.t4(dy), mode))):
        flags = int(x.dtype == torch.float16) | (2 if dy.dtype == torch.float16 else 0)   # bit 1: dy is a scaled fp16 shadow
        if dy.dtype == torch.float16 and dy_amax is None:
            raise RuntimeError("an fp16 output-gradient shadow needs the device scalar its scale was derived from")
        L.call("mas_conv3x3_wgrad_tc16", x, flags, L.t4(x), dy, L.t4(dy), dw, db, mode, table, int(silu),
               dy_amax if dy_amax is not None else amax_of(dy), cout, ws, ws.numel())
        return dw, db
    if x.dtype == torch.float16 or dy.dtype == torch.float16:
        raise RuntimeError("fp16 operands can only feed the fp16-operand tensor-core weight gradient")
    if padded:
        raise RuntimeError("padded weight gradient needs the fp16 tensor-core kernel")
    L.call("mas_conv3x3_wgrad", x, L.t4(x), dy, L.t4(dy), dw, db, mode, _cfg["impl"], table, int(silu), ws, ws.numel())
    return dw, db


def wgrad_f16_eligible(x, dout, c1w):
    """Both convolutions of a ResnetBlock (Cin -> Cout on x's extent, Cout -> Cout) take the fp16 tensor-core weight gradient."""
    if not (f16_operands() and wgrad_f16_on() and _is_dense_nhwc(x) and _is_dense_nhwc(dout)):
        return False
    n, cin, h, w = x.shape
    cout = c1w.shape[0]
    return cin % 32 == 0 and cout % 128 == 0 and h % 8 == 0 and w % 8 == 0


def wgrad_f16_on():
    return os.environ.get("MAS_WGRAD_F16", "1") != "0"


def f16_operands():
    return _tc_on() and _cfg["operands"] == "f16"


def conv3x3_dgrad_raw(dy, weight, mode, dy_amax=None):
    """Data gradient of the 3x3 family: the same kernel with flipped/transposed weights (+ zero-stuffed input map for the
    stride-2 conv, or a 2x2 sum-pool after it for the upsampling conv). dy_amax: max|dy| if the caller already has it."""
    if mode == L.CONV_S1:
        return conv3x3_raw(dy, weight, None, None, L.CONV_S1, transpose=True, x_amax=dy_amax)
    if mode == L.CONV_S2:
        return conv3x3_raw(dy, weight, None, None, L.CONV_ZS, transpose=True, x_amax=dy_amax)
    du = conv3x3_raw(dy, weight, None, None, L.CONV_S1, transpose=True, x_amax=dy_amax)
    n, cin, h2, w2 = du.shape
    dx = empty_nhwc(n, cin, h2 // 2, w2 // 2, du)
    L.call("mas_sumpool2x2", du, dx, n, h2 // 2, w2 // 2, cin)
    return dx


def gemm(A, B, C, M, N, K, batch=1, lda=None, ldb=None, ldc=None, sa=0, sb=0, sc=0, ta=False, tb=False, alpha=1.0,
         bias=None, residual=None, impl=None):
    """Pointers may be tensors or (tensor, element_offset) pairs. impl: override of the global selection (L.IMPL_TC3 = the
    fp32-accurate 3xTF32 tensor-core GEMM)."""
    def p(v):
        if isinstance(v, tuple):
            import ctypes
            t, off = v
            return ctypes.c_void_p(t.data_ptr() + 4 * off)
        return v
    L.call("mas_gemm", p(A), p(B), p(C), M, N, K, batch, lda, ldb, ldc, sa, sb, sc, int(ta), int(tb), float(alpha), p(bias),
           p(residual), _cfg["impl"] if impl is None else impl)


def gemm_w(A, lda, weight, C, ldc, M, transpose=False, alpha=1.0, bias=None, residual=None, stats_part=None):
    """C[M,N] = alpha * A[M,K] . W^T (+bias +residual) for a 1x1-convolution weight W [Nout, Kin] (transpose=True: A . W,
    the data gradient). A / C may be (tensor, element_offset) pairs with row pitches lda / ldc."""
    nout, kin = weight.shape[0], weight.shape[1]
    N, K = (kin, nout) if transpose else (nout, kin)
    w2 = weight.contiguous()
    if _tc_on() and N % 128 == 0 and K % 32 == 0 and lda % 4 == 0 and ldc % 4 == 0:
        import ctypes

        def p(v):
            return ctypes.c_void_p(v[0].data_ptr() + 4 * v[1]) if isinstance(v, tuple) else v
        dev = (A[0] if isinstance(A, tuple) else A).device
        wt = torch.empty(N * K, dtype=torch.float32, device=dev)
        L.call("mas_pack_gemm_tc", w2, wt, nout, kin, int(transpose))
        L.call("mas_gemm_rows_packed", p(A), lda, wt, p(C), ldc, M, N, K, float(alpha), bias, p(residual), stats_part)
        return True
    else:
        # W stored [Nout,Kin]: forward needs B^T (tb), the data gradient takes it as stored [K=Nout, N=Kin]
        gemm(A, w2, C, M, N, K, lda=lda, ldb=kin, ldc=ldc, tb=not transpose, alpha=alpha, bias=bias, residual=residual)
        return False


def conv1x1_raw(x, weight, bias, residual=None):
    """x NHWC [N,Cin,H,W] -> NHWC [N,Cout,H,W]; rows GEMM with W stored [Cout,Cin]."""
    n, cin, h, w = x.shape
    cout = weight.shape[0]
    y = empty_nhwc(n, cout, h, w, x)
    gemm_w(x, cin, weight, y, cout, n * h * w, bias=bias, residual=residual)
    return y


def conv1x1_dgrad_raw(dy, weight, residual=None):
    n, cout, h, w = dy.shape
    cin = weight.shape[1]
    dx = empty_nhwc(n, cin, h, w, dy)
    gemm_w(dy, cout, weight, dx, cin, n * h * w, transpose=True, residual=residual)
    return dx


def conv1x1_wgrad_raw(x_rows, dy_rows, M, cin, cout, want_bias=True, ldx=None, ldy=None, dy_off=0):
    import ctypes
    dev = x_rows.device
    dy_ptr = ctypes.c_void_p(dy_rows.data_ptr() + 4 * dy_off)
    dw = torch.empty((cout, cin, 1, 1), dtype=torch.float32, device=dev)
    db = torch.empty(cout, dtype=torch.float32, device=dev) if want_bias else None
    nb = L.query("mas_conv1x1_wgrad_ws_bytes", M, cin, cout)
    ws = L.workspace(nb, dev)
    L.call("mas_conv1x1_wgrad", x_rows, ldx or cin, dy_ptr, ldy or cout, M, cin, cout, dw, db, _cfg["impl"], ws, ws.numel())
    return dw, db


def attach_stats(t, mean, rstd):
    """Carry the GroupNorm statistics a kernel epilogue computed for `t` to the next module (same tensor object)."""
    if mean is not None:
        t._mas_gn = (mean, rstd, t._version)
    return t


def take_stats(t):
    st = getattr(t, "_mas_gn", None)
    if st is not None and st[2] == t._version and st[0].device == t.device:
        return st[0], st[1]
    return None, None


# ------------------------------------------------------------------------------------------------ autograd Functions
class GroupNormFn(torch.autograd.Function):
    """Normalize (+ optional fused Swish) — modules.py:35-41,194-196."""

    @staticmethod
    def forward(ctx, x, weight, bias, silu):
        x = nhwc(x)
        mean, rstd = gn_stats(x)
        y = gn_apply(x, mean, rstd, weight, bias, silu)
        ctx.save_for_backward(x, weight, bias, mean, rstd)
        ctx.silu = silu
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, bias, mean, rstd = ctx.saved_tensors
        dx, dg, db = gn_backward(nhwc(dy), x, mean, rstd, weight, bias, ctx.silu)
        return dx, dg, db, None


class SiLUFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        _need_cuda(x)
        x = x.contiguous() if not (x.is_contiguous() or x.is_contiguous(memory_format=torch.channels_last)) else x
        y = torch.empty_like(x)
        L.call("mas_silu_forward", x, y, x.numel())
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        if dy.stride() != x.stride():
            d2 = torch.empty_like(x)
            if x.dim() == 4:
                L.call("mas_copy_strided", dy, L.t4(dy), d2, L.t4(d2))
            else:
                d2.copy_(dy)
            dy = d2
        dx = torch.empty_like(x)
        L.call("mas_silu_backward", dy, x, dx, x.numel())
        return dx


def _is_dense_nhwc(t):
    return t.dim() == 4 and t.stride(1) == 1 and t.is_contiguous(memory_format=torch.channels_last)


class Conv3x3Fn(torch.autograd.Function):
    """nn.Conv2d 3x3 / Downsample / Upsample (modules.py:44-81,93-104) with optional fused residual add.
    3-channel edge layers (conv_in reading the NCHW image, conv_out writing the NCHW reconstruction) use the
    direct fp32 edge kernels; everything else goes through conv3x3_raw (wgmma or SIMT)."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, mode, out_nchw):
        _need_cuda(x)
        cout, cin = weight.shape[0], weight.shape[1]
        n, _, h, w = x.shape
        edge = 0
        tc_pad_in = (mode == L.CONV_S1 and f16_operands() and residual is None and cout % 128 == 0 and h % 16 == 0 and w % 8 == 0
                     and (cin % 16 != 0) and (cin > 64 or cin <= 4))
        if mode == L.CONV_S1 and residual is None and cin == 3 and cout > 4 and not tc_pad_in:
            edge = 1
            y = empty_nhwc(n, cout, h, w, x)
            L.call("mas_edge_small_cin_fprop", x, L.t4(x), weight.contiguous(), bias, y, L.t4(y), 0)
        elif mode == L.CONV_S1 and residual is None and cout == 3 and cin > 4 and cin % 4 == 0 and cin <= 1024:
            edge = 2
            x = nhwc(x)
            y = (torch.empty((n, cout, h, w), dtype=torch.float32, device=x.device) if out_nchw else empty_nhwc(n, cout, h, w, x))
            L.call("mas_edge_small_cout_fprop", x, L.t4(x), weight.contiguous(), bias, y, L.t4(y))
        elif tc_pad_in:
            # channel count off the 16-wide K step of the tensor kernels (the 159-channel VQ-SEG maps; the 3-channel image of
            # conv_in, where 10x padded FLOPs on the tensor cores still beat the FFMA edge kernel 4x): zero-pad the input channels
            # (one tiled transposing copy from the caller's NCHW tensor) and the weight (cached per version), run the
            # tensor-core kernels
            edge = 4
            cp = _round_up(cin, 32)          # 32: the weight-gradient kernel's input-channel tile
            x = pad_nhwc(x, cp)
            y = conv3x3_raw(x, _padded(weight, (cout, cp, 3, 3)), bias, None, L.CONV_S1)
        elif (mode == L.CONV_S1 and f16_operands() and residual is None and cout % 128 != 0 and cout > 128 and cin % 16 == 0
              and h % 16 == 0 and w % 8 == 0):
            # output width off the 128-wide tile (the 159-channel VQ-SEG decoder head): the result is RETURNED AS A
            # CHANNELS-LAST VIEW [N, cout, H, W] of the round_up(cout, 4)-channel buffer the padded kernel writes (the
            # weighted-BCE kernels take it as it is; `out_nchw` is not honoured here: a contiguous NCHW copy of a 1.3 GB
            # logits tensor would cost more than the convolution)
            edge = 5
            x = nhwc(x)
            y = conv3x3_raw(x, weight, bias, None, L.CONV_S1, pad_out=True)
        elif residual is None and not out_nchw and phase_mode(x, cout, mode) is not None:
            # Upsample / Downsample as four small convolutions over phase planes read straight from an fp16 shadow of x
            edge = 6
            ctx.pmode = phase_mode(x, cout, mode)
            am = amax_of(x)
            x16 = to_half(x, am)
            y = conv3x3_phase_raw(x16, weight, bias, ctx.pmode, x_amax=am)
            if mode == L.CONV_UP:
                # a following ResnetBlock without shortcut writes its input gradient's fp16 shadow: the data gradient here reads it
                y._mas_res_out = True
            # the weight gradient reads the shadow and nothing else in the backward reads x: keep half the bytes, or none
            want_w = ctx.needs_input_grad[1] or (bias is not None and ctx.needs_input_grad[2])
            x, ctx.x_amax = (x16, am) if want_w else (None, None)
        elif (mode == L.CONV_S2 and _tc_on() and residual is None and not out_nchw and _is_dense_nhwc(x) and cin % 8 == 0
              and cout % 128 == 0 and h % 32 == 0 and w % 16 == 0):
            edge = 3  # stride-2 conv on the stride-1 tensor kernels through space-to-depth
            x4 = empty_nhwc(n, 4 * cin, h // 2, w // 2, x)
            L.call("mas_space_to_depth", x, x4, n, h, w, cin)
            w9 = torch.empty((cout, 4 * cin, 3, 3), dtype=torch.float32, device=x.device)
            L.call("mas_s2d_pack_weights", weight.contiguous(), w9, cout, cin)
            y = conv3x3_raw(x4, w9, bias, None, L.CONV_S1)
            x = x4   # saved for the weight gradient (the 4C-channel view carries the same data)
        else:
            y = conv3x3_raw(x, weight, bias, residual, mode, out_nchw, prepack=ctx.needs_input_grad[0])
        ctx.save_for_backward(x, weight)
        ctx.mode, ctx.has_bias, ctx.has_res, ctx.edge = mode, bias is not None, residual is not None, edge
        return y



    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        cout, cin = weight.shape[0], weight.shape[1]
        dx = dw = db = dres = None
        want_w = ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2])
        if ctx.edge == 1:
            if ctx.needs_input_grad[0]:
                dx = conv3x3_dgrad_raw(dy, weight, ctx.mode)
            if want_w:
                dyd = nhwc(dy)
                dw = torch.empty_like(weight)
                db = torch.empty(cout, dtype=torch.float32, device=x.device)
                ws = L.workspace(L.query("mas_edge_wgrad_ws_bytes", cout), x.device)
                L.call("mas_edge_small_cin_wgrad", x, L.t4(x), dyd, L.t4(dyd), dw, db, ws, ws.numel())
        elif ctx.edge == 2:
            n, _, h, w = x.shape
            if ctx.needs_input_grad[0]:
                dx = empty_nhwc(n, cin, h, w, x)
                L.call("mas_edge_small_cin_fprop", dy, L.t4(dy), weight.contiguous(), None, dx, L.t4(dx), 1)
            if want_w:
                dw = torch.empty_like(weight)
                db = torch.empty(cout, dtype=torch.float32, device=x.device)
                ws = L.workspace(L.query("mas_edge_wgrad_ws_bytes", cin), x.device)
                L.call("mas_edge_small_cout_wgrad", x, L.t4(x), dy, L.t4(dy), dw, db, ws, ws.numel())
        elif ctx.edge == 4:
            cp = x.shape[1]                                              # x is the zero-padded channels-last copy
            dy = nhwc(dy)
            am = amax_of(dy)
            if want_w:
                dwp, db = conv3x3_wgrad_raw(x, dy, cout, cp, L.CONV_S1, ctx.has_bias, dy_amax=am)
                dw = dwp[:, :cin].contiguous()
            if ctx.needs_input_grad[0]:
                dx = conv3x3_dgrad_raw(dy, _padded(weight, (cout, cp, 3, 3)), L.CONV_S1, am)[:, :cin]
        elif ctx.edge == 5:
            cpo = _round_up(cout, 4)
            full = getattr(dy, "_mas_pad_base", None)                    # the loss kernel wrote the gradient padded already
            if full is None or full.shape[1] != cpo or full.data_ptr() != dy.data_ptr() or not _is_dense_nhwc(full):
                full = pad_nhwc(dy.contiguous() if not dy.is_contiguous() and _cl_pitch(dy) is None else dy, cpo)
            am = amax_of(full)
            if ctx.needs_input_grad[0]:
                dx = conv3x3_raw(full, _padded(weight, (cpo, cin, 3, 3)), None, None, L.CONV_S1, transpose=True, x_amax=am)
            if want_w:
                dwk, dbk = conv3x3_wgrad_raw(x, full, _round_up(cout, 128), cin, L.CONV_S1, True, dy_amax=am)
                dw, db = dwk[:cout].contiguous(), dbk[:cout].contiguous()
        elif ctx.edge == 6:
            # x is the input's fp16 shadow here (None when no weight gradient was asked for); both gradients read one dy shadow
            dy = nhwc(dy)
            sh = shadow_of(dy)
            if sh is None:
                am = amax_of(dy)
                sh = (to_half(dy, am), am)
            if ctx.needs_input_grad[0]:
                dx = conv3x3_phase_raw(sh[0], weight, None, ctx.pmode, transpose=True, x_amax=sh[1])
            if want_w:
                dw, db = conv3x3_phase_wgrad_raw(x, ctx.x_amax, sh[0], sh[1], ctx.pmode, ctx.has_bias)
        elif ctx.edge == 3:
            if ctx.needs_input_grad[0]:
                dx = conv3x3_dgrad_raw(nhwc(dy), weight, ctx.mode)       # zero-stuffed map on the tensor kernel
            if want_w:
                dw9, db = conv3x3_wgrad_raw(x, nhwc(dy), cout, 4 * cin, L.CONV_S1, ctx.has_bias)
                dw = torch.empty_like(weight)
                L.call("mas_s2d_unpack_wgrad", dw9, dw, cout, cin)
        else:
            dy = nhwc(dy)
            am = amax_of(dy) if f16_operands() else None
            if ctx.needs_input_grad[0]:
                dx = conv3x3_dgrad_raw(dy, weight, ctx.mode, am)
            if want_w:
                dw, db = conv3x3_wgrad_raw(x, dy, cout, cin, ctx.mode, ctx.has_bias, dy_amax=am)
        if not ctx.has_bias:
            db = None
        if ctx.has_res and ctx.needs_input_grad[3]:
            dres = dy
        return dx, dw, db, dres, None, None


class Conv1x1Fn(torch.autograd.Function):
    """nn.Conv2d 1x1 (nin_shortcut, quant_conv[0], post_quant_conv — modules.py:113-117, vqvae.py:15,18)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        x = nhwc(x)
        y = conv1x1_raw(x, weight, bias)
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = nhwc(dy)
        n, cin, h, w = x.shape
        cout = weight.shape[0]
        dx = conv1x1_dgrad_raw(dy, weight) if ctx.needs_input_grad[0] else None
        dw, db = conv1x1_wgrad_raw(x, dy, n * h * w, cin, cout, ctx.has_bias)
        return dx, dw, db


class ResnetBlockFn(torch.autograd.Function):
    """ResnetBlock.forward as one unit (modules.py:119-136): GN+SiLU -> conv3x3 -> GN+SiLU -> conv3x3 (+1x1 shortcut) + x.
    Tensor path (all img_config blocks): GroupNorm+SiLU is applied inside the convolutions' operand producers (the
    activated tensors are never written), each convolution's epilogue emits the statistics of the NEXT GroupNorm, the
    residual add lives in conv2's epilogue; in backward the weight-gradient kernel re-activates its input on the fly and
    the shortcut gradient is folded into the GroupNorm-backward apply (identity) or the shortcut GEMM's epilogue (nin).
    Returns (out, mean, rstd): the statistics of `out` for the following block's first GroupNorm (or None)."""

    @staticmethod
    def forward(ctx, x, mean_in, rstd_in, n1w, n1b, c1w, c1b, n2w, n2b, c2w, c2b, sw, sb, dx_shadow=False):
        x = nhwc(x)
        n, cin, h, w = x.shape
        cout = c1w.shape[0]
        if mean_in is None:
            mean_in, rstd_in = gn_stats(x)
        m1, r1 = mean_in, rstd_in
        fused = conv_tc_eligible(x, cout, L.CONV_S1) and cin % 8 == 0 and cout % (4 * GN_GROUPS) == 0
        # shadow mode: act(GN(.)) is written ONCE as an fp16 channels-last tensor (half the bytes of the fp32 activation the
        # unfused path stores), the convolutions read it through the copy engine (conv_tma.cu) and the backward pass feeds the
        # same tensor to the weight-gradient kernel instead of re-materialising it
        hmode = (fused and conv_h_eligible(n, cin, h, w, cout) and conv_h_eligible(n, cout, h, w, cout)
                 and wgrad_f16_on() and cin % 32 == 0)
        sc = x if sw is None else conv1x1_raw(x, sw, sb)
        if hmode:
            a1 = gn_apply_f16(x, m1, r1, n1w, n1b, True)
            h1, st2 = conv3x3_h_raw(a1, c1w, c1b, None, want_stats=True, prepack=ctx.needs_input_grad[0])
            m2, r2 = st2
            a2 = gn_apply_f16(h1, m2, r2, n2w, n2b, True)
            out, st_out = conv3x3_h_raw(a2, c2w, c2b, sc, want_stats=True, prepack=any(ctx.needs_input_grad))
            if not any(ctx.needs_input_grad):
                a1 = a2 = None
        elif fused:
            t1 = gn_table(m1, r1, n1w, n1b, n, cin)
            h1, st2 = conv3x3_raw(x, c1w, c1b, None, L.CONV_S1, table=t1, want_stats=True, prepack=ctx.needs_input_grad[0])
            m2, r2 = st2
            t2 = gn_table(m2, r2, n2w, n2b, n, cout)
            out, st_out = conv3x3_raw(h1, c2w, c2b, sc, L.CONV_S1, table=t2, want_stats=True, prepack=any(ctx.needs_input_grad))
            a1 = a2 = None
        else:
            a1 = gn_apply(x, m1, r1, n1w, n1b, True)
            h1 = conv3x3_raw(a1, c1w, c1b, None, L.CONV_S1, prepack=ctx.needs_input_grad[0])
            m2, r2 = gn_stats(h1)
            a2 = gn_apply(h1, m2, r2, n2w, n2b, True)
            out = conv3x3_raw(a2, c2w, c2b, sc, L.CONV_S1, prepack=any(ctx.needs_input_grad))
            st_out = None
        ctx.save_for_backward(x, h1, a1, a2, m1, r1, m2, r2, n1w, n1b, c1w, n2w, n2b, c2w, sw)
        ctx.has_sc, ctx.fused = sw is not None, fused and not hmode   # shadow mode keeps a1 / a2 like the unfused path
        ctx.hmode, ctx.dx_shadow = hmode, bool(dx_shadow) and hmode and sw is None
        if st_out is None:
            mo = ro = None
        else:
            mo, ro = st_out
            ctx.mark_non_differentiable(mo, ro)
        ctx.set_materialize_grads(False)   # no zero-fill launches for the (non-differentiable) statistics outputs
        return out, mo, ro

    @staticmethod
    def backward(ctx, dout, _gm, _gr):
        if dout is None:
            return (None,) * 14
        x, h1, a1, a2, m1, r1, m2, r2, n1w, n1b, c1w, n2w, n2b, c2w, sw = ctx.saved_tensors
        dout = nhwc(dout)
        cout, cin = c1w.shape[0], c1w.shape[1]
        n, _, h, w = x.shape
        am_out = amax_of(dout) if f16_operands() else None   # from the producing kernel, else one pass; serves dgrad and wgrad
        hmode = ctx.hmode and conv_tma_on()
        sh_out = shadow_of(dout) if hmode else None
        if hmode and sh_out is None and am_out is not None:
            # dout comes from a kernel that does not write shadows (head of a chain of blocks): one conversion pass feeds both
            # the data gradient and the weight gradient of conv2 (cheaper than their register-staged forms)
            sh_out = (to_half(dout, am_out), am_out)
        if sh_out is not None:
            # dout was written by a GroupNorm backward together with its fp16 shadow: pure TMA + MMA data gradient
            d_a2 = conv3x3_h_raw(sh_out[0], c2w, None, None, transpose=True, x_amax=sh_out[1])
        else:
            d_a2 = conv3x3_dgrad_raw(dout, c2w, L.CONV_S1, am_out)
        # fused forward never stored act(GN(.)): the GroupNorm backward re-materialises it as a by-product of its first pass
        # (cheaper than re-activating inside the weight-gradient kernel's producers: measured +0.8 ms per full-res call)
        # the activation re-materialised for the weight gradient goes straight into an fp16 operand: write it as fp16
        a16 = ctx.fused and wgrad_f16_eligible(x, dout, c1w)
        sh_h1 = None
        if ctx.fused:
            d_h1, dn2w, dn2b, a2 = gn_backward(d_a2, h1, m2, r2, n2w, n2b, True, want_act=True, act_f16=a16)
        elif hmode:
            # the gradient of conv1's output only feeds conv1's data and weight gradients: it exists as an fp16 shadow only
            sh_h1, dn2w, dn2b = gn_backward(d_a2, h1, m2, r2, n2w, n2b, True, shadow_only=True)
        else:
            d_h1, dn2w, dn2b = gn_backward(d_a2, h1, m2, r2, n2w, n2b, True)
        del d_a2
        if sh_out is not None and a2.dtype == torch.float16:
            dc2w, dc2b = conv3x3_wgrad_raw(a2, sh_out[0], cout, cout, L.CONV_S1, dy_amax=sh_out[1])   # both operands as fp16 shadows
        else:
            dc2w, dc2b = conv3x3_wgrad_raw(a2, dout, cout, cout, L.CONV_S1, dy_amax=am_out)
        del a2, sh_out
        if sh_h1 is not None:
            d_h1, am_h1 = sh_h1
            d_a1 = conv3x3_h_raw(d_h1, c1w, None, None, transpose=True, x_amax=am_h1)
        else:
            am_h1 = amax_of(d_h1) if f16_operands() else None
            d_a1 = conv3x3_dgrad_raw(d_h1, c1w, L.CONV_S1, am_h1)
        del sh_h1
        if ctx.has_sc:
            r_ = gn_backward(d_a1, x, m1, r1, n1w, n1b, True, want_act=ctx.fused, act_f16=a16)
            dxm, dn1w, dn1b = r_[0], r_[1], r_[2]
            if ctx.fused:
                a1 = r_[3]
            dx = conv1x1_dgrad_raw(dout, sw, residual=dxm)   # dout.Wn + dx_main
            dsw, dsb = conv1x1_wgrad_raw(x, dout, n * h * w, cin, cout)
        else:
            r_ = gn_backward(d_a1, x, m1, r1, n1w, n1b, True, dx_add=dout, want_act=ctx.fused, act_f16=a16,
                             shadow=ctx.dx_shadow and hmode, add_amax=am_out)
            dx, dn1w, dn1b = r_[0], r_[1], r_[2]
            if ctx.fused:
                a1 = r_[3]
            dsw = dsb = None
        del d_a1
        dc1w, dc1b = conv3x3_wgrad_raw(a1, d_h1, cout, cin, L.CONV_S1, dy_amax=am_h1)
        del a1, d_h1
        return dx, None, None, dn1w, dn1b, dc1w, dc1b, dn2w, dn2b, dc2w, dc2b, dsw, dsb, None


class AttnBlockFn(torch.autograd.Function):
    """AttnBlock.forward as one unit (modules.py:167-191): GN -> q,k,v 1x1 -> softmax(q^T k / sqrt(c)) over keys
    -> v.P^T -> proj_out 1x1 -> + x."""

    @staticmethod
    def forward(ctx, x, mean_in, rstd_in, nw, nb, qw, qb, kw, kb, vw, vb, pw, pb):
        x = nhwc(x)
        n, c, h, w = x.shape
        hw, M = h * w, n * h * w
        if mean_in is None:
            mean_in, rstd_in = gn_stats(x)
        mean, rstd = mean_in, rstd_in
        dev = x.device
        hn = empty_nhwc(n, c, h, w, x)
        qkv = torch.empty((M, 3 * c), dtype=torch.float32, device=dev)
        P = torch.empty((n, hw, hw), dtype=torch.float32, device=dev)
        O = empty_nhwc(n, c, h, w, x)
        out = empty_nhwc(n, c, h, w, x)
        # proj_out's epilogue emits the statistics of the following GroupNorm when it runs on the tensor path
        part = None
        if _tc_on() and hw % 128 == 0 and c % 128 == 0:
            part = torch.empty((M // 128) * c * 2, dtype=torch.float32, device=dev)
        ws = L.workspace(L.query("mas_attnblock_ws_bytes", n, hw, c, GN_GROUPS), dev)
        L.call("mas_attnblock_forward", x, n, hw, c, GN_GROUPS, mean, rstd, nw, nb, qw.contiguous(), qb, kw.contiguous(), kb,
               vw.contiguous(), vb, pw.contiguous(), pb, hn, qkv, P, O, out, part, _cfg["impl"], ws, ws.numel())
        ctx.save_for_backward(x, mean, rstd, hn, qkv, P, O, nw, nb, qw, kw, vw, pw)
        ctx.set_materialize_grads(False)   # no zero-fill launches for the (non-differentiable) statistics outputs
        if part is not None:
            mo, ro = _finalize_stats(part, n, c, hw)
            ctx.mark_non_differentiable(mo, ro)
            return out, mo, ro
        return out, None, None

    @staticmethod
    def backward(ctx, dout, _gm, _gr):
        if dout is None:
            return (None,) * 13
        x, mean, rstd, hn, qkv, P, O, nw, nb, qw, kw, vw, pw = ctx.saved_tensors
        dout = nhwc(dout)
        n, c, h, w = x.shape
        hw = h * w
        dev = x.device
        dx = torch.empty_like(x)
        dnw, dnb = torch.empty_like(nw), torch.empty_like(nb)
        dqkv_w = torch.empty((3 * c,) + tuple(qw.shape[1:]), dtype=torch.float32, device=dev)
        dqkv_b = torch.empty(3 * c, dtype=torch.float32, device=dev)
        dpw = torch.empty_like(pw, memory_format=torch.contiguous_format)
        dpb = torch.empty(c, dtype=torch.float32, device=dev)
        ws = L.workspace(L.query("mas_attnblock_ws_bytes", n, hw, c, GN_GROUPS), dev)
        am = torch.empty(1, dtype=torch.float32, device=dev) if f16_operands() else None
        L.call("mas_attnblock_backward", dout, x, n, hw, c, GN_GROUPS, mean, rstd, nw, nb, qw.contiguous(), kw.contiguous(),
               vw.contiguous(), pw.contiguous(), hn, qkv, P, O, dx, dnw, dnb, dqkv_w, dqkv_b, dpw, dpb, am, _cfg["impl"], ws,
               ws.numel())
        attach_amax(dx, am)
        return (dx, None, None, dnw, dnb, dqkv_w[:c], dqkv_b[:c], dqkv_w[c:2 * c], dqkv_b[c:2 * c], dqkv_w[2 * c:], dqkv_b[2 * c:],
                dpw, dpb)


class BatchNormFn(torch.autograd.Function):
    """nn.SyncBatchNorm(embed_dim) training forward/backward (vqvae.py:16): local sums by kernel, the 2*C
    statistics are all-reduced over NCCL when a process group is active (the one cross-rank step of the forward)."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, momentum, eps, sync):
        x = nhwc(x)
        n, c, h, w = x.shape
        R = n * h * w
        # [sum(x) | sum(x^2) | row count] as fp64: ranks may hold different numbers of rows (uneven last batch), so the
        # count is reduced with the sums like nn.SyncBatchNorm's per-rank counts (vqvae.py:16) and read on the device
        buf = torch.empty(2 * c + 1, dtype=torch.float64, device=x.device)
        L.call("mas_bn_stats", x, R, c, buf)
        world = 1
        if sync and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            world = dist.get_world_size()
            dist.all_reduce(buf)
        mean = torch.empty(c, dtype=torch.float32, device=x.device)
        invstd = torch.empty_like(mean)
        L.call("mas_bn_finalize", buf, 0.0, c, float(eps), float(momentum), mean, invstd, running_mean, running_var)
        y = torch.empty_like(x)
        L.call("mas_bn_apply", x, mean, invstd, weight, bias, y, R, c)
        ctx.save_for_backward(x, weight, mean, invstd)
        ctx.world = world
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, invstd = ctx.saved_tensors
        dy = nhwc(dy)
        n, c, h, w = x.shape
        R = n * h * w
        local = torch.empty(2 * c + 1, dtype=torch.float64, device=x.device)
        L.call("mas_bn_backward_reduce", dy, x, mean, invstd, R, c, local)
        glob = local
        if ctx.world > 1:
            glob = local.clone()
            dist.all_reduce(glob)
        dx = torch.empty_like(x)
        dg = torch.empty_like(weight)
        db = torch.empty_like(weight)
        L.call("mas_bn_backward_apply", dy, x, mean, invstd, weight, glob, local, 0.0, dx, dg, db, R, c)
        return dx, dg, db, None, None, None, None, None


def batchnorm_eval(x, weight, bias, running_mean, running_var, eps):
    x = nhwc(x)
    n, c, h, w = x.shape
    invstd = torch.empty_like(running_var)
    L.call("mas_bn_invstd", running_var, float(eps), invstd, c)
    y = torch.empty_like(x)
    L.call("mas_bn_apply", x, running_mean, invstd, weight, bias, y, n * h * w, c)
    return y


# ------------------------------------------------------------------------------------------------ PatchGAN discriminator
def _packed_conv4x4_weight(weight, transpose):
    """mas_pack_conv4x4 image of a [Cout,Cin,4,4] weight, cached per parameter version (D's weights change only at its
    optimizer step, so the three forwards and the backward passes of one training step share one packing)."""
    def make():
        cout, cin = weight.shape[:2]
        wp = torch.empty(16 * cout * cin, dtype=torch.float32, device=weight.device)
        L.call("mas_pack_conv4x4", weight.detach().contiguous(), wp, cout, cin, int(transpose))
        return wp
    return _cached(weight, ("c4", bool(transpose)), make)


def conv4x4_out_hw(h, w, stride):
    return (h - 2) // stride + 1, (w - 2) // stride + 1


def conv4x4_tc_route(x, cout, stride):
    """True when the 4x4 convolution of dense-NHWC x runs as the 3x3 convolution of its shift map on the fp16 tensor-core
    kernels (include/mas_b200.h, mas_conv4x4_shift_map): model.2 / 5 / 8 of the discriminator at 256^2."""
    if not f16_operands() or not _is_dense_nhwc(x):
        return False
    n, cin, h, w = x.shape
    if stride == 2 and (h % 2 or w % 2):
        return False
    hs, ws = h // stride, w // stride
    return cin % 4 == 0 and bool(L.query("mas_conv3x3_tc_eligible", _nhwc4(n, hs, ws, 4 * cin), _nhwc4(n, hs, ws, cout), L.CONV_S1))


def _conv4x4_as_3x3(weight, stride):
    """[Cout, 4*Cin, 3, 3] weight of the shift-map route, cached per parameter version (its own packings then stay cached)."""
    def make():
        cout, cin = weight.shape[:2]
        w3 = torch.empty((cout, 4 * cin, 3, 3), dtype=torch.float32, device=weight.device)
        L.call("mas_conv4x4_remap_weight", weight.detach().contiguous(), w3, cout, cin, stride, 1)
        return w3
    return _cached(weight, ("c4to3", stride), make)


class Conv4x4Fn(torch.autograd.Function):
    """nn.Conv2d(cin, cout, 4, stride, 1) (losses/discriminator.py:21,27-28,34), optionally followed by LeakyReLU(slope)
    (discriminator.py:21). x may have any strides (the first layer reads the caller's NCHW image); the output is dense NHWC.
    The backward computes only what autograd asks for: no weight gradient while D is frozen (the generator step), no data
    gradient for a leaf image (the discriminator step)."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, slope):
        _need_cuda(x)
        n, cin, h, w = x.shape
        cout = weight.shape[0]
        if tuple(weight.shape) != (cout, cin, 4, 4):
            raise RuntimeError("Conv4x4Fn: weight %s does not match a 4x4 kernel over %d channels" % (tuple(weight.shape), cin))
        ho, wo = conv4x4_out_hw(h, w, stride)
        act = slope is not None
        ctx.stride, ctx.slope, ctx.has_bias = int(stride), slope, bias is not None
        ctx.tc = not act and conv4x4_tc_route(x, cout, stride)
        if ctx.tc:
            xm = empty_nhwc(n, 4 * cin, h // stride, w // stride, x)
            L.call("mas_conv4x4_shift_map", x, L.t4(x), xm, int(stride))
            y = conv3x3_raw(xm, _conv4x4_as_3x3(weight, stride), bias, None, L.CONV_S1)
            if stride == 1:
                y = y[:, :, :ho, :wo]          # the 3x3 output has one extra row and column
            ctx.in_shape = x.shape
            ctx.save_for_backward(xm, weight, None)
            return y
        y = empty_nhwc(n, cout, ho, wo, x)
        L.call("mas_conv4x4", x, L.t4(x), _packed_conv4x4_weight(weight, False), bias, y, L.t4(y), int(stride),
               float(slope) if act else 0.0, int(act))
        ctx.save_for_backward(x, weight, y if act else None)
        return y

    @staticmethod
    def _backward_tc(ctx, dy):
        xm, weight, _ = ctx.saved_tensors
        n, cin, h, w = ctx.in_shape
        cout, s = weight.shape[0], ctx.stride
        if s == 1:
            # the dropped last row / column of the 3x3 output must carry a zero gradient
            dyp = empty_nhwc(n, cout, h, w, dy).zero_()
            inner = dyp[:, :, :h - 1, :w - 1]
            L.call("mas_copy_strided", dy, L.t4(dy), inner, L.t4(inner))
        else:
            dyp = nhwc(dy)
        w3 = _conv4x4_as_3x3(weight, s)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dxm = conv3x3_raw(dyp, w3, None, None, L.CONV_S1, transpose=True)
            dx = empty_nhwc(n, cin, h, w, dyp)
            L.call("mas_conv4x4_shift_map_adjoint", dxm, dx, L.t4(dx), s)
        if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
            dw3, db = conv3x3_wgrad_raw(xm, dyp, cout, 4 * cin, L.CONV_S1, want_bias=ctx.has_bias and ctx.needs_input_grad[2])
            if ctx.needs_input_grad[1]:
                dw = torch.empty_like(weight, memory_format=torch.contiguous_format)
                L.call("mas_conv4x4_remap_weight", dw3, dw, cout, cin, s, 0)
        return dx, dw, db, None, None

    @staticmethod
    def backward(ctx, dy):
        _need_cuda(dy)
        if ctx.tc:
            return Conv4x4Fn._backward_tc(ctx, dy)
        x, weight, y = ctx.saved_tensors
        if ctx.slope is not None:
            dy = nhwc(dy)
            dz = torch.empty_like(y)
            L.call("mas_lrelu_backward", dy, y, float(ctx.slope), dz, dz.numel())
            dy = dz
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = empty_nhwc(*x.shape, like=x)
            L.call("mas_conv4x4_dgrad", dy, L.t4(dy), _packed_conv4x4_weight(weight, True), dx, L.t4(dx), ctx.stride)
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(weight, memory_format=torch.contiguous_format)
            nb = L.query("mas_conv4x4_wgrad_ws_bytes", L.t4(x), L.t4(dy))
            ws = L.workspace(nb, x.device)
            L.call("mas_conv4x4_wgrad", x, L.t4(x), dy, L.t4(dy), dw, ctx.stride, ws, ws.numel())
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = torch.empty(weight.shape[0], dtype=torch.float32, device=x.device)
            ws = L.workspace(L.query("mas_colsum_ws_bytes", L.t4(dy)), x.device)
            L.call("mas_colsum", dy, L.t4(dy), db, ws, ws.numel())
        return dx, dw, db, None, None


class BatchNormLReLUFn(torch.autograd.Function):
    """nn.BatchNorm2d (training mode: statistics of this call's batch, running statistics updated) followed by
    LeakyReLU(slope) (losses/discriminator.py:29-30); slope = 1 is the plain BatchNorm2d."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, momentum, eps, slope):
        x = nhwc(x)
        n, c, h, w = x.shape
        R = n * h * w
        buf = torch.empty(2 * c + 1, dtype=torch.float64, device=x.device)
        L.call("mas_bn_stats", x, R, c, buf)
        mean = torch.empty(c, dtype=torch.float32, device=x.device)
        invstd = torch.empty_like(mean)
        L.call("mas_bn_finalize", buf, 0.0, c, float(eps), float(momentum), mean, invstd, running_mean, running_var)
        y = torch.empty_like(x)
        L.call("mas_bn_apply_lrelu", x, mean, invstd, weight, bias, float(slope), y, R, c)
        ctx.slope = float(slope)
        ctx.save_for_backward(x, weight, mean, invstd, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, invstd, y = ctx.saved_tensors
        dy = nhwc(dy)
        n, c, h, w = x.shape
        R = n * h * w
        sums = torch.empty(2 * c + 1, dtype=torch.float64, device=x.device)
        ws = L.workspace(L.query("mas_bn_backward_reduce_lrelu_ws_bytes", R, c), x.device)
        L.call("mas_bn_backward_reduce_lrelu", dy, y, ctx.slope, x, mean, invstd, R, c, sums, ws, ws.numel())
        dx = torch.empty_like(x)
        dg = db = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            dg, db = torch.empty_like(weight), torch.empty_like(weight)
        L.call("mas_bn_backward_apply_lrelu", dy, y, ctx.slope, x, mean, invstd, weight, sums, dx, dg, db, R, c)
        return dx, dg, db, None, None, None, None, None


def batchnorm_lrelu_eval(x, weight, bias, running_mean, running_var, eps, slope):
    x = nhwc(x)
    n, c, h, w = x.shape
    invstd = torch.empty_like(running_var)
    L.call("mas_bn_invstd", running_var, float(eps), invstd, c)
    y = torch.empty_like(x)
    L.call("mas_bn_apply_lrelu", x, running_mean, invstd, weight, bias, float(slope), y, n * h * w, c)
    return y


class VQFn(torch.autograd.Function):
    """Codebook distance+argmin+gather+loss+straight-through (modules.py:501-515) in one kernel."""

    @staticmethod
    def forward(ctx, z, E, beta):
        z = nhwc(z)
        n, d, h, w = z.shape
        R, K = n * h * w, E.shape[0]
        E = E.contiguous()
        idx = torch.empty(R, dtype=torch.int64, device=z.device)
        zq = torch.empty_like(z)
        loss = torch.empty((), dtype=torch.float32, device=z.device)
        nb = L.query("mas_vq_ws_bytes", R, K, d)
        ws = L.workspace(nb, z.device)
        L.call("mas_vq_forward", z, E, R, K, d, float(beta), idx, zq, loss, ws, ws.numel())
        ctx.save_for_backward(z, E, idx)
        ctx.beta = float(beta)
        ctx.mark_non_differentiable(idx)
        return zq, loss, idx

    @staticmethod
    def backward(ctx, g_zq, g_loss, _g_idx):
        z, E, idx = ctx.saved_tensors
        n, d, h, w = z.shape
        R, K = n * h * w, E.shape[0]
        g_zq = nhwc(g_zq) if g_zq is not None else None
        if g_loss is not None:
            g_loss = g_loss.contiguous()
        grad_z = torch.empty_like(z) if ctx.needs_input_grad[0] else None
        grad_E = torch.zeros_like(E) if ctx.needs_input_grad[1] else None
        L.call("mas_vq_backward", g_zq, g_loss, z, E, idx, R, K, d, ctx.beta, grad_z, grad_E)
        return grad_z, grad_E, None


def vq_select_path(tensor_core_filter: bool):
    """Codebook arg-min implementation: tensor-core filter + exact re-evaluation (default) or the all-pairs FFMA kernel."""
    rc = L.load().mas_vq_select_path(1 if tensor_core_filter else 0)
    if rc != 0:
        raise RuntimeError("mas_vq_select_path failed")


class VQGivenFn(torch.autograd.Function):
    """Codebook gather + loss + straight-through for caller-supplied indices (no argmin): modules.py:506-515 with
    `min_encoding_indices` given. Same backward kernel as VQFn."""

    @staticmethod
    def forward(ctx, z, E, beta, idx):
        z = nhwc(z)
        n, d, h, w = z.shape
        R, K = n * h * w, E.shape[0]
        E = E.contiguous()
        idx = idx.contiguous().view(-1)
        if idx.numel() != R or idx.dtype != torch.int64:
            raise RuntimeError("VQGivenFn: need %d int64 indices" % R)
        zq = torch.empty_like(z)
        loss = torch.empty((), dtype=torch.float32, device=z.device)
        ws = L.workspace(L.query("mas_vq_ws_bytes", R, K, d), z.device)
        L.call("mas_vq_forward_given", z, E, idx, R, K, d, float(beta), zq, loss, ws, ws.numel())
        ctx.save_for_backward(z, E, idx)
        ctx.beta = float(beta)
        return zq, loss

    @staticmethod
    def backward(ctx, g_zq, g_loss):
        z, E, idx = ctx.saved_tensors
        n, d, h, w = z.shape
        R, K = n * h * w, E.shape[0]
        g_zq = nhwc(g_zq) if g_zq is not None else None
        if g_loss is not None:
            g_loss = g_loss.contiguous()
        grad_z = torch.empty_like(z) if ctx.needs_input_grad[0] else None
        grad_E = torch.zeros_like(E) if ctx.needs_input_grad[1] else None
        L.call("mas_vq_backward", g_zq, g_loss, z, E, idx, R, K, d, ctx.beta, grad_z, grad_E)
        return grad_z, grad_E, None, None


def vq_gather(E, idx):
    R, (K, D) = idx.numel(), E.shape
    out = torch.empty((R, D), dtype=torch.float32, device=E.device)
    L.call("mas_vq_gather", E.contiguous(), idx.contiguous().view(-1), R, K, D, out)
    return out


def _round_up(v, m):
    return (v + m - 1) // m * m


def pad_nhwc(x, cp):
    """x [N,C,H,W] -> logical [N,cp,H,W] in dense channels-last memory with channels >= C zero (cp >= C)."""
    _need_cuda(x)
    n, c, h, w = x.shape
    base = torch.empty((n, h, w, cp), dtype=torch.float32, device=x.device)
    if x.is_contiguous() and c * 33 * 4 <= 48 * 1024:
        L.call("mas_nchw_to_nhwc_pad", x, base, n, c, cp, h, w)
    else:
        if cp > c:
            base[..., c:].zero_()
        view = base.permute(0, 3, 1, 2)[:, :c]
        L.call("mas_copy_strided", x, L.t4(x), view, L.t4(view))
    return base.permute(0, 3, 1, 2)


def _cl_pitch(t):
    """Channel pitch if t [N,C,H,W] is a channels-last view whose pixels are `pitch` floats apart (pitch >= C), else None."""
    if t.dim() != 4 or t.stride(1) != 1:
        return None
    n, c, h, w = t.shape
    pitch = t.stride(3)
    if pitch < c or t.stride(2) != w * pitch or (n > 1 and t.stride(0) != h * w * pitch):
        return None
    return pitch


class BCELogitsFn(torch.autograd.Function):
    """binary_cross_entropy_with_logits(pos_weight) mean (losses/loss_seg.py:15-19). With the VQ-SEG step's own layouts
    (channels-last logits - the padded view the decoder's last convolution returns - and an NCHW target) loss and
    gradient are two tiled kernels and the gradient is produced directly in the padded channels-last buffer the convolution's
    backward consumes; other layouts take the generic strided kernel. Nothing of the backward runs in torch."""

    @staticmethod
    def forward(ctx, logits, target, pos_weight):
        _need_cuda(logits)
        n, c, h, w = logits.shape
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        cp = _cl_pitch(logits)
        if cp is not None and target.is_contiguous() and w % 32 == 0 and c * 33 * 4 <= 48 * 1024:
            ws = L.workspace(L.query("mas_bce_cl_ws_bytes", n, h, w), logits.device)
            L.call("mas_bce_cl_forward", logits, target, pos_weight, n, c, cp, h, w, loss, ws, ws.numel())
            ctx.save_for_backward(logits, target, pos_weight)
            ctx.cp = cp
            return loss
        grad = torch.empty_like(logits)
        nb = L.query("mas_bce_ws_bytes", L.t4(logits))
        ws = L.workspace(nb, logits.device)
        L.call("mas_bce_logits", logits, L.t4(logits), target, L.t4(target), pos_weight, loss, grad, L.t4(grad),
               1.0 / logits.numel(), ws, ws.numel())
        ctx.save_for_backward(grad)
        ctx.cp = None
        return loss

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        if ctx.cp is None:
            (grad,) = ctx.saved_tensors
            out = torch.empty_like(grad)
            src = grad if grad.is_contiguous() or grad.is_contiguous(memory_format=torch.channels_last) else grad.contiguous()
            out = torch.empty_like(src)
            L.call("mas_scale_by", src, g, out, src.numel())
            return out, None, None
        logits, target, pw = ctx.saved_tensors
        n, c, h, w = logits.shape
        base = torch.empty((n, h, w, ctx.cp), dtype=torch.float32, device=logits.device)
        L.call("mas_bce_cl_backward", logits, target, pw, g, n, c, ctx.cp, h, w, base)
        full = base.permute(0, 3, 1, 2)
        grad = full[:, :c]
        grad._mas_pad_base = full          # the padded tensor this view lives in (picked up by the convolution's backward)
        return grad, None, None


# ------------------------------------------------------------------------------------------------ tier 2: token transformer
class LayerNormFn(torch.autograd.Function):
    """nn.LayerNorm(hidden, eps) over the last dim, optionally fused with a residual add: LN(x) + residual."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, eps):
        _need_cuda(x)
        x = x.contiguous()
        H = x.shape[-1]
        R = x.numel() // H
        y = torch.empty_like(x)
        mean = torch.empty(R, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        res = residual.contiguous() if residual is not None else None
        L.call("mas_layernorm_forward", x, weight, bias, res, y, mean, rstd, R, H, float(eps))
        ctx.save_for_backward(x, weight, mean, rstd)
        ctx.has_res = residual is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, rstd = ctx.saved_tensors
        dy = dy.contiguous()
        H = x.shape[-1]
        R = x.numel() // H
        dx = torch.empty_like(x)
        dg = torch.empty_like(weight)
        db = torch.empty_like(weight)
        ws = L.workspace(L.query("mas_layernorm_ws_bytes", R, H), x.device)
        L.call("mas_layernorm_backward", dy, x, mean, rstd, weight, dx, dg, db, R, H, ws, ws.numel())
        return dx, dg, db, (dy if ctx.has_res else None), None


class GeluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        _need_cuda(x)
        x = x.contiguous()
        y = torch.empty_like(x)
        L.call("mas_gelu_forward", x, y, x.numel())
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dx = torch.empty_like(x)
        L.call("mas_gelu_backward", dy.contiguous(), x, dx, x.numel())
        return dx


def linear_f16_on(nout, kin):
    """Linear layers on the TMA-fed fp16 kernels (csrc/gemm_tma.cu: forward, data gradient and weight gradient): both widths
    multiples of 128, fp16 operand format selected. MAS_LINEAR_F16=0 keeps the register-staged TF32 kernels."""
    return f16_operands() and nout % 128 == 0 and kin % 128 == 0 and os.environ.get("MAS_LINEAR_F16", "1") != "0"


def _packed_linear_weight(weight, transpose, dev):
    """fp16 operand image of an nn.Linear weight [N,K] (transpose: of W^T, the data-gradient operand), cached per parameter
    version like the convolution packings."""
    def make():
        n, k = weight.shape
        wt = torch.empty(n * k, dtype=torch.float16, device=dev)
        L.call("mas_pack_gemm_tc16", weight.contiguous(), wt, n, k, int(transpose))
        return wt
    return _cached(weight, ("lin16", bool(transpose)), make)


def rows_to_half(x2d):
    """(fp16 copy of a dense [M,K] matrix under the power-of-two scale of its max|.|, that maximum as a device scalar)."""
    am = amax(x2d)
    x16 = torch.empty(x2d.shape, dtype=torch.float16, device=x2d.device)
    L.call("mas_to_half", x2d, x16, x2d.numel(), am)
    return x16, am


def gemm_rows_f16(x16, am, weight, transpose=False, bias=None):
    """y[M, N] = x[M, K] . W^T (+bias) (transpose: x[M, N] . W, the data gradient) on mas_gemm_rows_f16 from the fp16 copy."""
    M, kc = x16.shape
    nout = weight.shape[1] if transpose else weight.shape[0]
    y = torch.empty((M, nout), dtype=torch.float32, device=x16.device)
    L.call("mas_gemm_rows_f16", x16, M, kc, _packed_linear_weight(weight, transpose, x16.device), y, nout, nout, bias, None, am, 1.0)
    return y


def wgrad_rows_f16(x16, am_x, dy16, am_dy, want_bias=True):
    """dW [N,K] = dy^T . x and the bias gradient from the two fp16 copies (mas_wgrad_rows_f16)."""
    M, K = x16.shape
    N = dy16.shape[1]
    dw = torch.empty((N, K), dtype=torch.float32, device=x16.device)
    db = torch.empty(N, dtype=torch.float32, device=x16.device) if want_bias else None
    ws = L.workspace(L.query("mas_wgrad_rows_f16_ws_bytes", M, N, K), x16.device)
    L.call("mas_wgrad_rows_f16", x16, dy16, M, N, K, dw, db, am_x, am_dy, ws, ws.numel())
    return dw, db


class LinearFn(torch.autograd.Function):
    """nn.Linear on the last dim. Both widths % 128 == 0: the TMA-fed fp16 kernels - the input is converted ONCE to fp16 (kept
    for the weight gradient instead of the fp32 tensor), the output gradient once for both the data and the weight gradient.
    Else the register-staged TF32 row GEMM (out % 128 == 0, in % 32 == 0), else fp32 SIMT."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        _need_cuda(x)
        x = x.contiguous()
        K, N = x.shape[-1], weight.shape[0]
        R = x.numel() // K
        ctx.f16 = linear_f16_on(N, K)
        ctx.has_bias = bias is not None
        ctx.xshape = x.shape
        if ctx.f16:
            x16, am = rows_to_half(x.view(R, K))
            y = gemm_rows_f16(x16, am, weight, False, bias).view(x.shape[:-1] + (N,))
            ctx.save_for_backward(x16, am, weight)
            return y
        y = torch.empty(x.shape[:-1] + (N,), dtype=torch.float32, device=x.device)
        gemm_w(x, K, weight, y, N, R, bias=bias)
        ctx.save_for_backward(x, weight)
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        if ctx.f16:
            x16, am_x, weight = ctx.saved_tensors
            N, K = weight.shape
            R = x16.shape[0]
            dy16, am_dy = rows_to_half(dy.view(R, N))
            dx = gemm_rows_f16(dy16, am_dy, weight, True).view(ctx.xshape) if ctx.needs_input_grad[0] else None
            dw, db = wgrad_rows_f16(x16, am_x, dy16, am_dy, ctx.has_bias)
            return dx, dw, db
        x, weight = ctx.saved_tensors
        K, N = x.shape[-1], weight.shape[0]
        R = x.numel() // K
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            gemm_w(dy, N, weight, dx, K, R, transpose=True)
        dw, db = conv1x1_wgrad_raw(x, dy, R, K, N, ctx.has_bias)
        return dx, dw.view(N, K), db


def _attn_impl(S_, hd):
    """Token-attention contractions (transformer.py:77-103): the 3xTF32 tensor-core GEMM (fp32-level accuracy, like the
    reference's torch.matmul with TF32 off) when the extents fit its tiles (the 640-token / 64-wide heads of the paper's
    configuration do), else the global selection."""
    if _tc_on() and S_ % 64 == 0 and hd % 64 == 0:
        return L.IMPL_TC3
    return None


def gemm2(A, B, C, M, N, K, outer, batch, lda, ldb, ldc, osa, osb, osc, sa, sb, sc, ta=False, tb=False, alpha=1.0, impl=None, causal=0):
    """outer x batch matrices in one call (mas_gemm_batched2): matrix (o, i) at o * os? + i * s?. Pointers as in gemm().
    causal: the header's structure hint for the causal attention matrices (zero blocks are skipped by the 3xTF32 kernel)."""
    import ctypes

    def at(v, o):
        t, off = v if isinstance(v, tuple) else (v, 0)
        return ctypes.c_void_p(t.data_ptr() + 4 * (off + o))
    step = max(1, 65535 // batch)        # grid.z limit of the single-launch kernel
    for o0 in range(0, outer, step):
        n = min(step, outer - o0)
        L.call("mas_gemm_batched2", at(A, o0 * osa), at(B, o0 * osb), at(C, o0 * osc), M, N, K, n, batch, lda, ldb, ldc, osa, osb, osc,
               sa, sb, sc, int(ta), int(tb), float(alpha), _cfg["impl"] if impl is None else impl, int(causal))


def attn_causal_fused_on(S_, hd):
    """The fused wgmma forward core (csrc/attn_causal.cu): head dim 64, S % 128 == 0, tensor path enabled.
    MAS_ATTN_FUSED=0 selects the GEMM / softmax / GEMM sequence instead."""
    return _tc_on() and hd == 64 and S_ % 128 == 0 and S_ >= 128 and os.environ.get("MAS_ATTN_FUSED", "1") != "0"


class CausalAttentionFn(torch.autograd.Function):
    """softmax_causal((q / sqrt(hd)) k^T) v per (batch, head) from the fused qkv activation [B,S,3H]
    (transformer.py:77-103; head h owns columns h*hd..(h+1)*hd of each third). Every contraction is ONE launch over all
    (batch element, head) pairs (two-level batch strides: the heads are column slices of the fused activation)."""

    @staticmethod
    def forward(ctx, qkv, heads):
        _need_cuda(qkv)
        qkv = qkv.contiguous()
        B, S_, H3 = qkv.shape
        H = H3 // 3
        hd = H // heads
        alpha = 1.0 / float(hd) ** 0.5
        impl = _attn_impl(S_, hd)
        P = torch.empty((B, heads, S_, S_), dtype=torch.float32, device=qkv.device)
        ctxv = torch.empty((B, S_, H), dtype=torch.float32, device=qkv.device)
        SS = S_ * S_
        if attn_causal_fused_on(S_, hd):
            # scores, causal softmax and P v in one kernel per (sequence, head, 128-query tile); P is written once for the backward
            L.call("mas_attn_causal_forward", qkv, amax(qkv), P, ctxv, B, S_, heads, hd, alpha)
        else:
            # S = alpha q k^T
            gemm2(qkv, (qkv, H), P, S_, S_, hd, B, heads, H3, H3, S_, S_ * H3, S_ * H3, heads * SS, hd, hd, SS, tb=True, alpha=alpha,
                  impl=impl, causal=3)
            L.call("mas_softmax_causal_forward", P, P, B * heads, S_, S_)
            # ctx = P v
            gemm2(P, (qkv, 2 * H), ctxv, S_, hd, S_, B, heads, S_, H3, H, heads * SS, S_ * H3, S_ * H, SS, hd, hd, impl=impl, causal=1)
        ctx.save_for_backward(qkv, P)
        ctx.heads = heads
        return ctxv

    @staticmethod
    def backward(ctx, dctx):
        qkv, P = ctx.saved_tensors
        dctx = dctx.contiguous()
        heads = ctx.heads
        B, S_, H3 = qkv.shape
        H = H3 // 3
        hd = H // heads
        alpha = 1.0 / float(hd) ** 0.5
        impl = _attn_impl(S_, hd)
        dqkv = torch.empty_like(qkv)
        dP = torch.empty_like(P)
        SS = S_ * S_
        oq, op_, oc = S_ * H3, heads * SS, S_ * H
        # P and dS are lower-triangular (key <= query): the contractions skip the zero blocks (causal hints of mas_gemm_batched2)
        # dV = P^T dO ; dP = dO V^T (only the entries the softmax backward reads)
        gemm2(P, dctx, (dqkv, 2 * H), S_, hd, S_, B, heads, S_, H, H3, op_, oc, oq, SS, hd, hd, ta=True, impl=impl, causal=2)
        gemm2(dctx, (qkv, 2 * H), dP, S_, S_, hd, B, heads, H, H3, S_, oc, oq, op_, hd, hd, SS, tb=True, impl=impl, causal=3)
        L.call("mas_softmax_causal_backward", P, dP, dP, B * heads, S_, S_, alpha)     # dS (already times 1/sqrt(hd)), zeros above the diagonal
        # dQ = dS K ; dK = dS^T Q
        gemm2(dP, (qkv, H), dqkv, S_, hd, S_, B, heads, S_, H3, H3, op_, oq, oq, SS, hd, hd, impl=impl, causal=1)
        gemm2(dP, qkv, (dqkv, H), S_, hd, S_, B, heads, S_, H3, H3, op_, oq, oq, SS, hd, hd, ta=True, impl=impl, causal=2)
        return dqkv, None


class CrossEntropyFn(torch.autograd.Function):
    """F.cross_entropy(logits.view(-1, V), target.view(-1)) (mean; train.py:150-153) on mas_ce_forward / mas_ce_backward.
    logits [..., V] fp32 (last dim contiguous), target int64 [...]; targets outside [0, V) are ignored rows."""

    @staticmethod
    def forward(ctx, logits, target):
        _need_cuda(logits)
        V = logits.shape[-1]
        lg = logits.reshape(-1, V)
        if lg.stride(-1) != 1:
            lg = lg.contiguous()
        tg = target.reshape(-1).to(torch.int64).contiguous()
        R = lg.shape[0]
        if tg.numel() != R:
            raise ValueError("cross_entropy: %d logit rows vs %d targets" % (R, tg.numel()))
        rows = torch.empty(R, dtype=torch.float32, device=lg.device)
        lse = torch.empty(R, dtype=torch.float32, device=lg.device)
        out = torch.empty(2, dtype=torch.float32, device=lg.device)
        L.call("mas_ce_forward", lg, lg.stride(0), tg, rows, lse, out, R, V)
        ctx.save_for_backward(lg, tg, lse, out)
        ctx.shape = logits.shape
        return out[0]

    @staticmethod
    def backward(ctx, dloss):
        lg, tg, lse, out = ctx.saved_tensors
        R, V = lg.shape
        d = torch.empty((R, V), dtype=torch.float32, device=lg.device)
        L.call("mas_ce_backward", lg, lg.stride(0), tg, lse, out, dloss.contiguous().to(torch.float32), d, V, R, V)
        return d.view(ctx.shape), None


def cross_entropy(logits, target):
    return CrossEntropyFn.apply(logits, target)


def sample_topk(logits, temperature, top_k, u):
    """One token per row of logits [R,V]: softmax(logits / temperature) restricted to the top_k entries, drawn by inverse CDF
    at the caller's uniforms u [R] (device fp32 in [0,1))."""
    _need_cuda(logits)
    logits = logits.contiguous()
    R, V = logits.shape
    tok = torch.empty(R, dtype=torch.int64, device=logits.device)
    L.call("mas_sample_topk", logits, V, R, V, float(temperature), int(top_k) if top_k else 0, u.contiguous(), tok)
    return tok


# ---- autoregressive sampling (inference only; SURVEY.md 8f-3) --------------------------------------------------
def linear_small(x, weight, bias, act=0):
    """nn.Linear for a handful of rows ([R<=8, K] -> [R, N]): the weight-streaming decode kernel, strict fp32.
    act=1 fuses the tanh-GELU of MLP.lin1 (transformer.py:11-14)."""
    _need_cuda(x)
    x = x.contiguous()
    R, K = x.shape
    N = weight.shape[0]
    y = torch.empty((R, N), dtype=torch.float32, device=x.device)
    L.call("mas_linear_small", x, K, weight.contiguous(), bias, y, N, R, N, K, int(act))
    return y


def kv_append(qkv, kcache, vcache, pos0):
    """qkv [R,T,3H] (fused q|k|v activation) -> caches [R,heads,Tmax,hd] at positions pos0..pos0+T-1."""
    R, heads, Tmax, hd = kcache.shape
    T = qkv.shape[1]
    L.call("mas_kv_append", qkv.contiguous(), R, T, heads, hd, kcache, vcache, Tmax, int(pos0))


def attn_decode(qkv, kcache, vcache, length):
    """One query per (row, head) (qkv [R,3H]) against the first `length` cached positions -> ctx [R,H]."""
    R, heads, Tmax, hd = kcache.shape
    ctx = torch.empty((R, heads * hd), dtype=torch.float32, device=qkv.device)
    L.call("mas_attn_decode", qkv.contiguous(), kcache, vcache, ctx, R, heads, hd, Tmax, int(length))
    return ctx


def attn_decode_append(qkv, kcache, vcache, pos):
    """attn_decode with the cache append folded in: stores this token's k / v (qkv [R,3H]) at position pos, attends over
    positions 0..pos -> ctx [R,H]."""
    R, heads, Tmax, hd = kcache.shape
    ctx = torch.empty((R, heads * hd), dtype=torch.float32, device=qkv.device)
    L.call("mas_attn_decode_append", qkv.contiguous(), kcache, vcache, ctx, R, heads, hd, Tmax, int(pos))
    return ctx


def layernorm2(x, ln1, residual, ln2):
    """(y1, y2) = (residual + ln1(x), ln2(y1)) for a few rows [R,H] in one launch (inference; nn.LayerNorm modules)."""
    _need_cuda(x)
    x = x.contiguous()
    R, H = x.shape
    y1, y2 = torch.empty_like(x), torch.empty_like(x)
    L.call("mas_layernorm2_forward", x, ln1.weight, ln1.bias, None if residual is None else residual.contiguous(), y1, ln2.weight,
           ln2.bias, y2, R, H, float(ln1.eps), float(ln2.eps))
    return y1, y2


def cfg_mix(cond, uncond, scale):
    """Classifier-free guidance on logits: uncond + scale * (cond - uncond)."""
    out = torch.empty_like(cond)
    L.call("mas_cfg_mix", cond.contiguous(), uncond.contiguous(), out, cond.numel(), float(scale))
    return out


class EmbedFn(torch.autograd.Function):
    """Token + (row, column | position) embedding sums for the text / segmentation / image segments, written straight
    into the concatenated [B, total, H] sequence (transformer.py:350-364)."""

    @staticmethod
    def forward(ctx, segs, total, H, *tables):
        # segs: list of (token_ids [B,L] int64, pos_ids_a [L] int64, pos_ids_b [L] int64 or None, offset); tables: 3 per segment
        dev = tables[0].device
        B = segs[0][0].shape[0]
        out = torch.empty((B, total, H), dtype=torch.float32, device=dev)
        for i, (ids, pa, pb, off) in enumerate(segs):
            t0, t1, t2 = tables[3 * i:3 * i + 3]
            Lg = ids.shape[1]
            L.call("mas_embed3_forward", t0, ids.contiguous(), t1, pa, t2 if pb is not None else None, pb, out, B * Lg, H, Lg, total, off)
        ctx.segs, ctx.total, ctx.H = segs, total, H
        ctx.shapes = [t.shape for t in tables]
        return out

    @staticmethod
    def backward(ctx, dout):
        dout = dout.contiguous()
        grads = []
        for i, (ids, pa, pb, off) in enumerate(ctx.segs):
            d0 = torch.zeros(ctx.shapes[3 * i], dtype=torch.float32, device=dout.device)
            d1 = torch.zeros(ctx.shapes[3 * i + 1], dtype=torch.float32, device=dout.device)
            d2 = torch.zeros(ctx.shapes[3 * i + 2], dtype=torch.float32, device=dout.device) if pb is not None else None
            Lg = ids.shape[1]
            L.call("mas_embed3_backward", dout, ids.contiguous(), d0, pa, d1, pb, d2, ids.shape[0] * Lg, ctx.H, Lg, ctx.total, off)
            grads += [d0, d1, d2]
        return (None, None, None) + tuple(grads)


# ---- LPIPS perceptual loss (losses/lpips.py) -------------------------------------------------------------------------
LPIPS_BLOCKS = (2, 2, 3, 3, 3)   # 3x3 convolutions per VGG16 block; each block ends in a tap, blocks 1-4 in a 2x2 max-pool


def _lpips_first_dgrad_weight(weight):
    """conv1_1's data-gradient weight (3 output channels: taps flipped, Cin <-> Cout) for mas_edge_small_cout_fprop."""
    return _cached(weight, "lpips_dgrad", lambda: weight.detach().flip(2, 3).transpose(0, 1).contiguous())


class LPIPSFn(torch.autograd.Function):
    """LPIPS.forward (losses/lpips.py:66-73) as one unit: ScalingLayer, VGG16 up to relu5_3 and the five heads over ONE
    batch of 2B images [real; fake] -> p [B, 1, 1, 1].

    p_b depends on image b alone, so d p / d fake = g.view(B, 1, 1, 1) * J with J_b = d p_b / d fake_b. The first backward
    runs the VGG data gradient once from a unit seed, keeps J and drops the activations; every later traversal of a
    retained graph (loss_img.py's autograd.grad(retain_graph=True), then backward()) is one scaling kernel.
    convs: the 13 (weight, bias) pairs in layer order; lins: the five [1, C, 1, 1] head weights."""

    @staticmethod
    def forward(ctx, real, fake, shift, scale, convs, lins, keep):
        _need_cuda(real)
        _need_cuda(fake)
        if real.dim() != 4 or real.shape != fake.shape or real.shape[1] != 3:
            raise RuntimeError("LPIPS expects real and fake images of equal shape [B, 3, H, W], got %s and %s"
                               % (tuple(real.shape), tuple(fake.shape)))
        B, _, H, W = real.shape
        if H < 16 or W < 16:
            raise RuntimeError("LPIPS needs images of at least 16 x 16 pixels (four 2x2 max-pools), got %d x %d" % (H, W))
        real, fake = real.contiguous(), fake.contiguous()
        dev = real.device
        x = empty_nhwc(2 * B, 3, H, W, real)
        L.call("mas_lpips_prep", real, fake, shift, scale, x, B, H, W)
        nblk = int(L.load().mas_lpips_head_blocks())
        part = torch.empty((5, B, nblk), dtype=torch.float64, device=dev)
        acts, hws = [], []
        cur, am, ci = x, None, 0
        for blk, nconv in enumerate(LPIPS_BLOCKS):
            for _ in range(nconv):
                wgt, bias = convs[ci]
                if ci == 0:
                    h = empty_nhwc(2 * B, wgt.shape[0], H, W, x)
                    L.call("mas_edge_small_cin_fprop", x, L.t4(x), wgt.contiguous(), bias, h, L.t4(h), 0)
                else:
                    h = conv3x3_raw(cur, wgt, bias, None, L.CONV_S1, x_amax=am, pad_out=True)
                am = torch.empty(1, dtype=torch.float32, device=dev)
                L.call("mas_lpips_relu", h, h.numel(), am)
                if keep:
                    acts.append(h)
                cur, ci = h, ci + 1
            _, c, hh, ww = cur.shape
            L.call("mas_lpips_head_forward", cur, lins[blk].contiguous(), B, hh, ww, c, part[blk])
            hws.append(hh * ww)
            if blk < len(LPIPS_BLOCKS) - 1:
                p = empty_nhwc(2 * B, c, hh // 2, ww // 2, cur)
                am = torch.empty(1, dtype=torch.float32, device=dev)
                L.call("mas_lpips_maxpool", cur, p, 2 * B, hh, ww, c, am)
                cur = p
        out = torch.empty((B, 1, 1, 1), dtype=torch.float32, device=dev)
        L.call("mas_lpips_head_finalize", part, B, *hws, out)
        ctx.acts = acts if keep else None
        ctx.convs, ctx.lins, ctx.scale, ctx.shape = convs, lins, scale, (B, H, W)
        ctx.J = None
        return out

    @staticmethod
    def backward(ctx, g):
        if torch.is_grad_enabled():
            raise RuntimeError("LPIPS does not support create_graph (double backward)")
        want_r, want_f = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        B, H, W = ctx.shape
        if ctx.J is None:
            if ctx.acts is None:
                raise RuntimeError("LPIPS: the forward ran without gradient tracking; nothing was saved for a backward")
            g0, G = (0 if want_r else B), (2 * B if want_r and want_f else B)
            acts, convs, lins = ctx.acts, ctx.convs, ctx.lins
            dev = acts[0].device
            dpool, ci = None, len(convs)
            for blk in reversed(range(len(LPIPS_BLOCKS))):
                tap = acts[ci - 1]
                _, c, hh, ww = tap.shape
                dz = empty_nhwc(G, c, hh, ww, tap)
                am = torch.empty(1, dtype=torch.float32, device=dev)
                L.call("mas_lpips_tap_backward", tap, lins[blk].contiguous(), B, hh, ww, c, g0, G, dpool, dz, am)
                first = ci - LPIPS_BLOCKS[blk]
                for k in reversed(range(first, ci)):
                    wgt = convs[k][0]
                    if k == 0:
                        dx = empty_nhwc(G, 3, H, W, dz)
                        L.call("mas_edge_small_cout_fprop", dz, L.t4(dz), _lpips_first_dgrad_weight(wgt), None, dx, L.t4(dx))
                    else:
                        dx = conv3x3_raw(dz, wgt, None, None, L.CONV_S1, transpose=True, x_amax=am, pad_out=True)
                    if k > first:   # the input of conv k is the ReLU output of conv k - 1: its mask, as a select
                        am = torch.empty(1, dtype=torch.float32, device=dev)
                        L.call("mas_lpips_relu_backward", dx, acts[k - 1][g0:g0 + G], dx, dx.numel(), am)
                    dz = dx
                dpool, ci = dz, first   # gradient of the block's input: the previous max-pool's output (block 0: the prep)
            J = torch.empty((G, 3, H, W), dtype=torch.float32, device=dev)
            L.call("mas_lpips_prep_backward", dpool, ctx.scale, J, G, H, W)
            ctx.J, ctx.acts = J, None
        J = ctx.J
        if g.dtype != torch.float32 or g.dim() != 4 or g.shape[0] != B:
            raise RuntimeError("LPIPS backward: expected a float32 [B, 1, 1, 1] gradient")
        per = 3 * H * W
        grads = []
        off = 0
        for want in (want_r, want_f):
            if not want:
                grads.append(None)
                continue
            d = torch.empty((B, 3, H, W), dtype=torch.float32, device=J.device)
            L.call("mas_lpips_scale_jacobian", J[off:off + B], g, g.stride(0), d, B, per)
            grads.append(d)
            off += B
        return grads[0], grads[1], None, None, None, None, None
