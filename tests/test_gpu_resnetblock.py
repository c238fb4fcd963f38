"""The VQGAN ResnetBlock (ops.ResnetBlockFn over csrc/conv_tma.cu, csrc/contract_tc.cu and the GroupNorm kernels of
csrc/norm.cu) against fp64, on every route the unit selects inside one call:

    route         selected by                                        3x3 convolutions               act(GN(.)) for the convolutions
    shadow        Cin % 128, Cout % 128, H % 16, W % 8 (default)      TMA-fed fp16 (conv_tma.cu)     written once as fp16 (a1, a2 saved)
    fused         Cin % 128 != 0, or MAS_CONV_TMA=0, MAS_WGRAD_F16=0  register-staged fp16 or TF32   table prologue; re-materialised in
                  or TF32 operands                                                                  the GroupNorm backward for wgrad
    unfused       Cout % 128 != 0, H % 16 != 0                       fp32 FFMA (wgrad fp16 if it    written as fp32 (a1, a2 saved)
                                                                     fits the wgrad tiles)
    simt          IMPL_SIMT                                          fp32 FFMA everywhere           written as fp32

Accuracy is judged against the error torch itself makes on the same inputs (the yardstick): torch float32 with TF32 on for
the tensor-core stages and for whole-block quantities of a tensor-core route (the fp16 operands carry TF32's 11 significant
bits), torch float32 with TF32 off for the GroupNorm stages and the SIMT route. The kernel's error must stay within a factor
of the yardstick's, plus a floor for quantities torch gets (almost) exactly, norm-wise and on the worst slice: the worst
image for the activations, out and dx, the worst output channel for the convolution weight gradients, so that one bad
image, 64-channel item or split-K partial cannot hide in a norm. The intermediates saved for the backward pass (h1, a1, a2
and the statistics m1, r1, m2, r2) and the statistics of out that conv2's epilogue emits (mo, ro) are each checked against
fp64 of the kernel's own input to that stage, so the ~1e-3 error of the TF32-level convolutions cannot mask a 1e-5 slip in
a GroupNorm stage. Relative errors here have no absolute floor: the `grad` condition scales the upstream gradient to 1e-7.

The epilogue statistics (m2, r2, mo, ro) are sums and sums of squares over 128 fp32 elements, added up in fp64 by
mas_gn_finalize_partials as var = E[x^2] - E[x]^2. With |mean| / std = k per group the fp32 partials lose about
2^-24 k^2 of the variance to cancellation per partial, about 2^-24 k^2 / sqrt(P) over the P partials of a group; torch's
Welford does not. mas_gn_stats (m1, r1) has the same kind of error from its 4-pixel fp32 sums, about ten times smaller. In
the `offset` condition (k ~ 32 for x, h1 and out) rstd is therefore held to RSTD_CANCEL * 2^-24 * (1 + k^2) / sqrt(P) per
(image, group) instead of the yardstick factor; every other condition holds it to the yardstick.

The factors are set from the ratios kernel error / yardstick error measured on an H100 SXM (80 GB, 700 W), largest over
all shapes and conditions here, at about twice the largest ratio:
  GroupNorm stages, FFMA, statistics      largest 2.03 (dx of the unfused route at 24x24; mostly 0.5-1.3)
  fp16 / TF32 tensor-core stages, block   largest 2.96 (the chain's AttnBlock weights; the ResnetBlock's 2.88, dsw). Bias
                                          gradients, column sums torch takes in fp32 either way, reach 11.9 at 1.2e-6: under
                                          FLOOR_TF32 + 6x
  epilogue statistics, `offset`           err / (2^-24 (1 + k^2) / sqrt(P)) largest 2.61 (mo / ro, MAS_CONV_TMA=0)
The shadow route's bias gradients of conv1 and conv2 sum the fp16 shadow of dy (the weight-gradient kernel's operand):
11-bit terms, so about 2e-4 relative for a gradient of random sign, 2000x torch's fp32 column sum but the same error as
every other TF32-class gradient of the block. They are held to FLOOR_F16_SUM (measured largest 2.3e-4).
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

GROUPS, EPS = 32, 1e-6
FACTOR_FP32, FACTOR_TF32 = 4.0, 6.0
FLOOR32 = 5e-7      # ~4 fp32 ulps
FLOOR_TF32 = 1e-6   # bias gradients are column sums, which torch computes in fp32 with or without TF32
RSTD_CANCEL = 6.0   # rstd at |mean| / std = k: |error| <= RSTD_CANCEL * 2^-24 * (1 + k^2) / sqrt(P) + FLOOR32 (`offset`)
FLOOR_F16_SUM = 5e-4   # a bias gradient summed from an fp16 dy shadow: 2^-12 relative rounding per term
ORDER = ("n1w", "n1b", "c1w", "c1b", "n2w", "n2b", "c2w", "c2b", "sw", "sb")

# every ResnetBlock of the 256-px img_config model and the half-empty tile pair (W = 24: three 8-wide tiles) on the shadow
# route; Cin = 64 runs conv1's weight gradient on the 64-channel wgrad_t16 variant, on the fused route (conv1's data gradient
# would have 64 output channels, which the TMA-fed kernel does not take); the rest pin the other routes
CASES = [((2, 128, 128, 256, 256), "shadow"), ((4, 128, 128, 128, 128), "shadow"), ((2, 128, 256, 64, 64), "shadow"),
         ((12, 256, 256, 64, 64), "shadow"), ((2, 256, 512, 32, 32), "shadow"), ((2, 512, 512, 32, 32), "shadow"),
         ((32, 512, 512, 16, 16), "shadow"), ((2, 512, 256, 64, 64), "shadow"), ((2, 256, 128, 128, 128), "shadow"),
         ((3, 128, 128, 16, 24), "shadow"),
         ((2, 32, 128, 32, 32), "fused"), ((1, 64, 128, 32, 16), "fused"),
         ((2, 128, 128, 64, 64), "fused_tma0"), ((12, 256, 512, 32, 32), "fused_tma0"),
         ((2, 128, 128, 64, 64), "fused_f32act"), ((12, 256, 512, 32, 32), "fused_f32act"),
         ((2, 128, 128, 64, 64), "fused_tf32"), ((12, 256, 512, 32, 32), "fused_tf32"),
         ((2, 64, 64, 32, 32), "unfused"), ((2, 128, 128, 24, 24), "unfused"),
         ((2, 128, 128, 64, 64), "simt")]


def _ids(cases):
    return [f"{r}-{'x'.join(map(str, s))}" for s, r in cases]


@pytest.fixture
def state(monkeypatch):
    """TF32 off, and the implementation / operand format restored after the test; `state(route)` selects a route's switches."""
    from mas_b200 import _lib as L, ops
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, ops.get_impl(), ops.get_operand_format())
    _set_tf32(False)
    monkeypatch.setenv("MAS_CONV_TMA", "1")
    monkeypatch.setenv("MAS_WGRAD_F16", "1")
    ops.set_impl(L.IMPL_AUTO)
    ops.set_operand_format("f16")

    def select(route):
        if route == "fused_tma0":
            monkeypatch.setenv("MAS_CONV_TMA", "0")
        elif route == "fused_f32act":
            monkeypatch.setenv("MAS_WGRAD_F16", "0")
        elif route == "fused_tf32":
            ops.set_operand_format("tf32")
        elif route == "simt":
            ops.set_impl(L.IMPL_SIMT)
    yield select
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved[:2]
    ops.set_impl(saved[2])
    ops.set_operand_format(saved[3])


def _set_tf32(on):
    torch.backends.cuda.matmul.allow_tf32 = on
    torch.backends.cudnn.allow_tf32 = on


# ------------------------------------------------------------------------------------------------ error measures
def _rel(a, b):
    """||a - b|| / ||b|| in fp64 (no absolute floor: the comparisons must stay meaningful at any gradient scale)."""
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _worst(a, b, nrows):
    """Largest relative error over the rows of a and b viewed as [nrows, -1]."""
    a = a.detach().double().reshape(nrows, -1)
    b = b.detach().double().reshape(nrows, -1)
    return float(((a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-300)).max())


def _check(tag, name, kern, yard, ref, nrows=None, factor=FACTOR_FP32, floor=FLOOR32):
    """kernel error <= factor * yardstick error + floor, norm-wise and (nrows) on the worst row."""
    ek, ey = _rel(kern, ref), _rel(yard, ref)
    line = f"{tag} {name}: norm {ek:.3e} / {ey:.3e} = {ek / max(ey, 1e-300):.2f}"
    ok = ek <= factor * ey + floor
    if nrows is not None:
        rk, ry = _worst(kern, ref, nrows), _worst(yard, ref, nrows)
        line += f"; worst row {rk:.3e} / {ry:.3e} = {rk / max(ry, 1e-300):.2f}"
        ok = ok and rk <= factor * ry + floor
    print("ratio", line)
    assert ok, line


# ------------------------------------------------------------------------------------------------ the block in torch
def _act(x, mean, rstd, w, b):
    """silu(GroupNorm(x)) with the given statistics [N * GROUPS]."""
    n, c = x.shape[:2]
    xg = x.reshape(n, GROUPS, -1)
    xh = ((xg - mean.view(n, GROUPS, 1).to(x.dtype)) * rstd.view(n, GROUPS, 1).to(x.dtype)).view_as(x)
    return F.silu(xh * w.view(1, c, 1, 1) + b.view(1, c, 1, 1))


def _stats(t):
    """(mean, rstd) per (image, group) in t's dtype (torch's var_mean: Welford, no cancellation)."""
    var, mean = torch.var_mean(t.reshape(t.shape[0], GROUPS, -1), dim=2, unbiased=False)
    return mean.reshape(-1), (var + EPS).rsqrt().reshape(-1)


def _shortcut(x, prm):
    return F.conv2d(x, prm["sw"], prm["sb"]) if "sw" in prm else x


def _block(x, prm):
    """GN+SiLU -> conv3x3 -> GN+SiLU -> conv3x3 + shortcut(x), modules.py's ResnetBlock.forward in the dtype of x."""
    h = F.conv2d(F.silu(F.group_norm(x, GROUPS, prm["n1w"], prm["n1b"], eps=EPS)), prm["c1w"], prm["c1b"], padding=1)
    h = F.silu(F.group_norm(h, GROUPS, prm["n2w"], prm["n2b"], eps=EPS))
    return _shortcut(x, prm) + F.conv2d(h, prm["c2w"], prm["c2b"], padding=1)


def _torch_block(x, prm, g, dt, tf32):
    """out, dx and the parameter gradients of _block in dtype dt (convolutions on TF32 when tf32)."""
    _set_tf32(tf32)
    try:
        xl = x.detach().to(dt).contiguous().requires_grad_()
        pl = {k: v.detach().to(dt).requires_grad_() for k, v in prm.items()}
        out = _block(xl, pl)
        out.backward(g.to(dt).contiguous())
    finally:
        _set_tf32(False)
    return out.detach(), xl.grad, {k: v.grad for k, v in pl.items()}


# ------------------------------------------------------------------------------------------------ inputs
def _inputs(shape, seed, dev="cuda:0"):
    """x with images of very different scale (x1 ... x100) and per-channel offsets; a non-uniform upstream gradient."""
    n, cin, cout, h, w = shape
    gen = torch.Generator().manual_seed(seed)
    scale = torch.logspace(0, 2, n).view(n, 1, 1, 1)
    x = (torch.randn(n, cin, h, w, generator=gen) + 0.5 * torch.randn(1, cin, 1, 1, generator=gen)) * scale

    def b(c, s):
        return torch.randn(c, generator=gen) * s
    prm = dict(n1w=1 + b(cin, 0.2), n1b=b(cin, 0.2), c1w=torch.randn(cout, cin, 3, 3, generator=gen) / (9 * cin) ** 0.5,
               c1b=b(cout, 0.1), n2w=1 + b(cout, 0.2), n2b=b(cout, 0.2),
               c2w=torch.randn(cout, cout, 3, 3, generator=gen) / (9 * cout) ** 0.5, c2b=b(cout, 0.1))
    if cin != cout:
        prm.update(sw=torch.randn(cout, cin, 1, 1, generator=gen) / cin ** 0.5, sb=b(cout, 0.1))
    g = torch.randn(n, cout, h, w, generator=gen) * (1 + torch.arange(n).view(n, 1, 1, 1)) * (0.5 + torch.rand(1, cout, 1, 1, generator=gen))
    return x.to(dev), {k: v.to(dev) for k, v in prm.items()}, g.to(dev)


def _cond_grad(x, prm, g):
    """upstream gradient at the benchmark's magnitude: every power-of-two operand scale and the gradient shadows far from 1."""
    return x, prm, g * 1e-7


def _cond_outlier(x, prm, g):
    """one x element at ~40 sigma of its (image, group): the dx-shadow bound and the fp16 operand scales see it."""
    x = x.clone()
    n, c = x.shape[:2]
    x[n // 2, c // 3, x.shape[2] // 2, x.shape[3] // 3] += 40 * float(x[n // 2].std())
    return x, prm, g


def _cond_offset(x, prm, g):
    """conv biases and x such that x, h1 and out have |mean| / std ~ 32 in every (image, group)."""
    n, c = x.shape[:2]
    x = torch.randn(x.shape, generator=torch.Generator().manual_seed(5)).to(x.device) + 32.0
    p = {k: v.double() for k, v in prm.items()}
    x64 = x.double()
    h = F.conv2d(F.silu(F.group_norm(x64, GROUPS, p["n1w"], p["n1b"], eps=EPS)), p["c1w"], None, padding=1)
    prm = dict(prm, c1b=torch.full_like(prm["c1b"], 32.0 * float(h.std())))
    p["c1b"] = prm["c1b"].double()
    r = _block(x64, dict(p, c2b=torch.zeros_like(p["c2b"])))
    bias = 32.0 * float(r.std()) - r.mean(dim=(0, 2, 3))
    return x, dict(prm, c2b=bias.float()), g


CONDITIONS = {"grad": _cond_grad, "outlier": _cond_outlier, "offset": _cond_offset}
COND_CASES = [((2, 128, 128, 64, 64), "shadow"), ((12, 256, 256, 64, 64), "shadow"), ((2, 128, 128, 64, 64), "fused_tma0"),
              ((2, 128, 128, 24, 24), "unfused")]


# ------------------------------------------------------------------------------------------------ the kernel run
def _run_kernel(x, prm, g, dx_shadow):
    from mas_b200 import _lib as L, ops
    xk = x.detach().contiguous(memory_format=torch.channels_last).requires_grad_()
    pk = {k: v.detach().clone().requires_grad_() for k, v in prm.items()}
    seen = {}
    xk.register_hook(lambda d: seen.__setitem__("dx", d))
    args = [pk.get(k) for k in ORDER]
    t0 = L.tc_launch_count()
    L.profile_start()
    try:
        out, mo, ro = ops.ResnetBlockFn.apply(xk, None, None, *args, dx_shadow)
        fn = out.grad_fn
        saved = fn.saved_tensors[:8]   # (x, h1, a1, a2, m1, r1, m2, r2): read before backward frees them
        route = dict(hmode=fn.hmode, fused=fn.fused, dx_shadow=fn.dx_shadow, has_sc=fn.has_sc)
        out.backward(g.contiguous(memory_format=torch.channels_last))
    finally:
        calls = L.profile_report(lambda k: k.split("|")[0])
    torch.cuda.synchronize()
    return dict(out=out.detach(), mo=mo, ro=ro, dx=seen["dx"], grads={k: v.grad for k, v in pk.items()}, saved=saved,
                route=route, calls={k: c for k, (c, _) in calls.items()}, tc=L.tc_launch_count() - t0)


def _assert_route(tag, route, k, shape):
    """The route the call took: ctx attributes, C-ABI call counts over forward + backward, tensor-core launches."""
    n, cin, cout, h, w = shape
    r, c = k["route"], k["calls"]
    cnt = lambda name: c.get(name, 0)   # noqa: E731
    print(f"route {tag}: {r} tc={k['tc']} " + " ".join(f"{a}={b}" for a, b in sorted(c.items())))
    assert r["has_sc"] == (cin != cout), tag
    assert cnt("mas_conv1x1_wgrad") == (1 if cin != cout else 0), tag
    if route == "shadow":
        assert r["hmode"] and not r["fused"], tag
        # both convolutions and both data gradients read fp16 shadows through TMA; act(GN(.)) written once per norm; the
        # statistics of the second norm and of out from the convolution epilogues; one conversion of the caller's dout
        assert cnt("mas_conv3x3_fprop_tc16h") == 4 and cnt("mas_conv3x3_wgrad_tc16") == 2, tag
        assert cnt("mas_gn_apply") == 2 and cnt("mas_gn_stats") == 1 and cnt("mas_gn_finalize_partials") == 2, tag
        assert cnt("mas_gn_backward") == 2 and cnt("mas_to_half") == 1 and cnt("mas_gn_table") == 0, tag
        assert cnt("mas_conv3x3_fprop_tc16") == 0 and cnt("mas_conv3x3_fprop") == 0, tag
        assert r["dx_shadow"] == (cin == cout), tag
    elif route.startswith("fused"):
        assert r["fused"] and not r["hmode"] and not r["dx_shadow"], tag
        # GroupNorm + SiLU in the convolutions' table prologue, statistics of the second norm from conv1's epilogue
        assert cnt("mas_gn_table") == 2 and cnt("mas_gn_apply") == 0 and cnt("mas_gn_finalize_partials") == 2, tag
        assert cnt("mas_gn_stats") == 1 and cnt("mas_conv3x3_fprop_tc16h") == 0 and cnt("mas_to_half") == 0, tag
        fprop = "mas_conv3x3_fprop_tc" if route == "fused_tf32" else "mas_conv3x3_fprop_tc16"
        other = "mas_conv3x3_fprop_tc16" if route == "fused_tf32" else "mas_conv3x3_fprop_tc"
        assert cnt(fprop) >= 3 and cnt(other) == 0, tag   # both forwards and conv2's data gradient (conv1's: Cin permitting)
        if route in ("fused_f32act", "fused_tf32"):
            assert cnt("mas_conv3x3_wgrad") == 2 and cnt("mas_conv3x3_wgrad_tc16") == 0, tag
        else:
            assert cnt("mas_conv3x3_wgrad_tc16") == 2 and cnt("mas_conv3x3_wgrad") == 0, tag
    else:
        assert not r["fused"] and not r["hmode"] and not r["dx_shadow"], tag
        # act(GN(.)) written in fp32 and both statistics from mas_gn_stats; the 3x3 convolutions on the fp32 SIMT kernel
        assert cnt("mas_gn_apply") == 2 and cnt("mas_gn_stats") == 2 and cnt("mas_gn_finalize_partials") == 0, tag
        assert cnt("mas_gn_table") == 0 and cnt("mas_conv3x3_fprop") == 4, tag
        assert cnt("mas_conv3x3_fprop_tc16h") == 0 and cnt("mas_conv3x3_fprop_tc16") == 0 and cnt("mas_conv3x3_fprop_tc") == 0, tag
        if route == "simt":
            assert k["tc"] == 0 and cnt("mas_conv3x3_wgrad") == 2, tag
    if route == "shadow" or route.startswith("fused"):
        assert k["tc"] > 0, f"{tag}: no tensor-core launch"


def _check_dx_shadow(tag, dx):
    """dx's fp16 shadow is (dx * s).half() bit for bit, s = 2^(14 - floor(log2 bound)), with bound >= max|dx|."""
    from mas_b200 import ops
    sh = ops.shadow_of(dx)
    assert sh is not None, f"{tag}: dx carries no fp16 shadow"
    dx16, bound = sh
    b, mx = float(bound), float(dx.abs().max())
    print(f"ratio {tag} dx shadow: bound / max|dx| = {b / mx:.3f}")
    assert b >= mx, f"{tag}: shadow bound {b} below max|dx| {mx}"
    s = 2.0 ** (14 - (math.frexp(b)[1] - 1))
    assert torch.equal(dx16, (dx * s).half()), f"{tag}: the dx shadow is not (dx * {s}).half()"


def _verify(tag, shape, route, x, prm, g, offset=False):
    """Runs the block on the kernels twice (bit-identical), checks the route, every intermediate against fp64 of its own
    input, and out, dx and every parameter gradient against fp64 autograd from x."""
    n, cin, cout, h, w = shape
    dx_shadow = cin == cout
    k = _run_kernel(x, prm, g, dx_shadow)
    k2 = _run_kernel(x, prm, g, dx_shadow)
    _assert_route(tag, route, k, shape)
    for name in ("out", "mo", "ro", "dx"):
        assert (k[name] is None) == (k2[name] is None), f"{tag}: {name}"
        assert k[name] is None or torch.equal(k[name], k2[name]), f"{tag}: two runs differ in {name}"
    for name, v in k["grads"].items():
        assert torch.equal(v, k2["grads"][name]), f"{tag}: two runs differ in d{name}"
    del k2
    if k["route"]["dx_shadow"]:
        _check_dx_shadow(tag, k["dx"])

    # TF32 yardstick for the stages on tensor cores: the 3x3 convolutions and their data gradients (not on the unfused and
    # SIMT routes), and the weight gradients wherever a tensor-core kernel ran
    conv_tc = route not in ("unfused", "simt")
    wgrad_tc = conv_tc or k["tc"] > 0
    cnv = dict(factor=FACTOR_TF32, floor=FLOOR_TF32) if conv_tc else {}
    wgr = dict(factor=FACTOR_TF32, floor=FLOOR_TF32) if wgrad_tc else {}
    p64 = {kk: v.double() for kk, v in prm.items()}
    xk, h1, a1, a2, m1, r1, m2, r2 = k["saved"]
    x64 = x.double()

    def stats(tag2, mk, rk, t, bound=False):
        ref_m, ref_r = _stats(t.double())
        yard_m, yard_r = _stats(t)
        # the mean's error in units of its group's std (a group mean near zero has no meaningful relative error): RMS over
        # the (image, group) pairs and the worst one
        ek, ey = (mk.double() - ref_m) * ref_r, (yard_m.double() - ref_m) * ref_r
        rms = lambda e: float(e.norm()) / e.numel() ** 0.5   # noqa: E731
        line = (f"{tag} {tag2} mean (/ std): rms {rms(ek):.3e} / {rms(ey):.3e} = {rms(ek) / max(rms(ey), 1e-300):.2f}; worst "
                f"{float(ek.abs().max()):.3e} / {float(ey.abs().max()):.3e} = {float(ek.abs().max() / ey.abs().max().clamp_min(1e-300)):.2f}")
        print("ratio", line)
        assert rms(ek) <= FACTOR_FP32 * rms(ey) + FLOOR32 and float(ek.abs().max()) <= FACTOR_FP32 * float(ey.abs().max()) + FLOOR32, line
        if not bound:
            _check(tag, tag2 + " rstd", rk, yard_r, ref_r, nrows=n * GROUPS)
            return
        # fp32 partial sums of squares: the cancellation in E[x^2] - E[x]^2 grows as (mean / std)^2; the rounding errors of
        # the P = (elements per group) / 128 partials add up like a random walk
        var, mean = torch.var_mean(t.double().reshape(n, GROUPS, -1), dim=2, unbiased=False)
        k2_ = (mean * mean / var).reshape(-1)
        unit = 2.0 ** -24 * (1 + k2_) / (t[0].numel() / GROUPS / 128) ** 0.5
        err = (rk.double() - ref_r).abs() / ref_r
        lim = RSTD_CANCEL * unit + FLOOR32
        ey = float(((yard_r.double() - ref_r).abs() / ref_r).max())
        print(f"ratio {tag} {tag2} rstd (offset): max err {float(err.max()):.3e} at (mean/std)^2 up to {float(k2_.max()):.0f};"
              f" err / (2^-24 (1 + k^2) / sqrt(P)) = {float((err / unit).max()):.2f}; torch {ey:.3e}")
        assert bool((err <= lim).all()), f"{tag}: {tag2} rstd beyond the cancellation bound"

    # ---- intermediates, each against fp64 of the kernel's own input to that stage
    stats("m1 r1", m1, r1, x, bound=offset)
    fp16_act = a1 is not None and a1.dtype == torch.float16
    if a1 is not None:
        ref = _act(x64, *_stats(x64), p64["n1w"], p64["n1b"])
        yard = _act(x, *_stats(x), prm["n1w"], prm["n1b"])
        _check(tag, "a1", a1, yard.half() if fp16_act else yard, ref, nrows=n)
    a1in = a1 if a1 is not None else _act(x, m1, r1, prm["n1w"], prm["n1b"])   # fused: the table prologue's activation
    ref = F.conv2d(a1in.double(), p64["c1w"], p64["c1b"], padding=1)
    _set_tf32(conv_tc)
    yard = F.conv2d(a1in.float(), prm["c1w"], prm["c1b"], padding=1)
    _set_tf32(False)
    _check(tag, "h1", h1, yard, ref, nrows=n, **cnv)
    stats("m2 r2", m2, r2, h1, bound=offset)
    if a2 is not None:
        ref = _act(h1.double(), *_stats(h1.double()), p64["n2w"], p64["n2b"])
        yard = _act(h1, *_stats(h1), prm["n2w"], prm["n2b"])
        _check(tag, "a2", a2, yard.half() if fp16_act else yard, ref, nrows=n)
    a2in = a2 if a2 is not None else _act(h1, m2, r2, prm["n2w"], prm["n2b"])
    ref = _shortcut(x64, p64) + F.conv2d(a2in.double(), p64["c2w"], p64["c2b"], padding=1)
    _set_tf32(conv_tc)
    yard = _shortcut(x, prm) + F.conv2d(a2in.float(), prm["c2w"], prm["c2b"], padding=1)
    _set_tf32(False)
    _check(tag, "out (from a2)", k["out"], yard, ref, nrows=n, **cnv)
    if route in ("unfused", "simt"):
        assert k["mo"] is None and k["ro"] is None, f"{tag}: statistics emitted off the tensor path"
    else:
        stats("mo ro", k["mo"], k["ro"], k["out"], bound=offset)

    # ---- the whole block, forward and backward, against fp64 autograd from x
    out_ref, dx_ref, gr_ref = _torch_block(x, prm, g, torch.float64, False)
    out_yard, dx_yard, gr_yard = _torch_block(x, prm, g, torch.float32, conv_tc)
    # the unfused route's weight gradients may run on the fp16 kernel while its convolutions do not: their own TF32 yardstick
    gr_yard_w = _torch_block(x, prm, g, torch.float32, True)[2] if wgrad_tc and not conv_tc else gr_yard
    _check(tag, "out", k["out"], out_yard, out_ref, nrows=n, **cnv)
    _check(tag, "dx", k["dx"], dx_yard, dx_ref, nrows=n, **cnv)
    for name in prm:
        wname = name in ("c1w", "c1b", "c2w", "c2b", "sw", "sb")
        tol = wgr if wname else cnv
        if route == "shadow" and name in ("c1b", "c2b"):
            # the shadow route's weight gradients read dy only as an fp16 shadow: the bias gradient sums 11-bit terms
            tol = dict(tol, floor=FLOOR_F16_SUM)
        rows = cout if name in ("c1w", "c2w", "sw") else None   # worst output channel of the weight gradients
        _check(tag, "d" + name, k["grads"][name], (gr_yard_w if wname else gr_yard)[name], gr_ref[name], nrows=rows, **tol)
    return k


@pytest.mark.parametrize("shape,route", CASES, ids=_ids(CASES))
def test_resnetblock_vs_fp64(shape, route, state):
    state(route)
    x, prm, g = _inputs(shape, seed=sum(shape))
    _verify(f"{route}-{shape}", shape, route, x, prm, g)


@pytest.mark.parametrize("cond", list(CONDITIONS))
@pytest.mark.parametrize("shape,route", COND_CASES, ids=_ids(COND_CASES))
def test_resnetblock_conditioned(shape, route, cond, state):
    state(route)
    x, prm, g = CONDITIONS[cond](*_inputs(shape, seed=7 * sum(shape)))
    _verify(f"{route}-{cond}-{shape}", shape, route, x, prm, g, offset=cond == "offset")


# ------------------------------------------------------------------------------------------------ chains of blocks
def _module_params(mod):
    """{(module index, name): parameter} of an nn.Sequential of ResnetBlock / AttnBlock."""
    return {(i, name): p for i, m in enumerate(mod) for name, p in m.named_parameters()}


def _torch_chain(mod, x, g, dt, tf32):
    from models import modules as M
    from test_gpu_attnblock import _block as attn_block, _scale32
    _set_tf32(tf32)
    try:
        xl = x.detach().to(dt).contiguous().requires_grad_()
        pl = {key: p.detach().to(dt).requires_grad_() for key, p in _module_params(mod).items()}
        h = xl
        for i, m in enumerate(mod):
            q = {name: pl[(i, name)] for (j, name) in pl if j == i}
            if isinstance(m, M.ResnetBlock):
                prm = {"n1w": q["norm1.weight"], "n1b": q["norm1.bias"], "c1w": q["conv1.weight"], "c1b": q["conv1.bias"],
                       "n2w": q["norm2.weight"], "n2b": q["norm2.bias"], "c2w": q["conv2.weight"], "c2b": q["conv2.bias"]}
                h = _block(h, prm)
            else:
                prm = {"nw": q["norm.weight"], "nb": q["norm.bias"]}
                for a in ("q", "k", "v"):
                    prm[a + "w"], prm[a + "b"] = q[a + ".weight"], q[a + ".bias"]
                prm["pw"], prm["pb"] = q["proj_out.weight"], q["proj_out.bias"]
                h = attn_block(h, prm, _scale32(h.shape[1]))
        h.backward(g.to(dt).contiguous())
    finally:
        _set_tf32(False)
    return h.detach(), xl.grad, {key: p.grad for key, p in pl.items()}


CHAINS = [((2, 128, 64, 64), ("res", "res")), ((12, 512, 16, 16), ("res", "res", "attn"))]


@pytest.mark.parametrize("shape,kinds", CHAINS, ids=["-".join(k) + "-" + "x".join(map(str, s)) for s, k in CHAINS])
def test_resnetblock_chain_vs_fp64(shape, kinds, state):
    """nn.Sequential of ResnetBlocks (and an AttnBlock) through models.modules: the second unit takes its GroupNorm statistics
    from the first one's epilogue, writes its dx as an fp16 shadow, and the first unit's backward reads that shadow."""
    from mas_b200 import _lib as L, ops
    from models import modules as M
    dev = torch.device("cuda:0")
    n, c, h, w = shape
    torch.manual_seed(sum(shape))
    mod = torch.nn.Sequential(*[M.ResnetBlock(in_channels=c, out_channels=c, dropout=0.0) if k == "res" else M.AttnBlock(c)
                                for k in kinds])
    with torch.no_grad():
        for name, p in mod.named_parameters():
            if "norm" in name:
                p.add_(0.2 * torch.randn_like(p))
    mod.to(dev)
    gen = torch.Generator().manual_seed(3)
    x = (torch.randn(n, c, h, w, generator=gen) * torch.logspace(0, 2, n).view(n, 1, 1, 1)).to(dev)
    g = (torch.randn(n, c, h, w, generator=gen) * (1 + torch.arange(n).view(n, 1, 1, 1))).to(dev)
    tag = "chain-" + "-".join(kinds) + f"-{shape}"

    def run():
        for p in mod.parameters():
            p.grad = None
        xk = x.contiguous(memory_format=torch.channels_last).requires_grad_()
        seen = {}
        y1 = mod[0](xk)
        y1.register_hook(lambda d: seen.__setitem__("d1", ops.shadow_of(d)))
        h1 = y1
        fns = [y1.grad_fn]
        for m in list(mod)[1:]:
            h1 = m(h1)
            fns.append(h1.grad_fn)
        route = [(getattr(f, "hmode", None), getattr(f, "dx_shadow", None)) for f in fns]
        h1.backward(g.contiguous(memory_format=torch.channels_last))
        torch.cuda.synchronize()
        return h1.detach(), xk.grad, {key: p.grad.clone() for key, p in _module_params(mod).items()}, seen, route

    L.profile_start()
    try:
        out, dx, grads, seen, route = run()
    finally:
        calls = {k: cc for k, (cc, _) in L.profile_report(lambda k: k.split("|")[0]).items()}
    out2, dx2, grads2, _, _ = run()
    print(f"route {tag}: {route} " + " ".join(f"{a}={b}" for a, b in sorted(calls.items())))
    assert torch.equal(out, out2) and torch.equal(dx, dx2) and all(torch.equal(grads[k], grads2[k]) for k in grads), tag
    # (hmode, dx_shadow): the first unit's input is the caller's tensor, the second's the first unit's output
    assert route[0] == (True, False) and route[1] == (True, True), f"{tag}: {route}"
    assert calls.get("mas_gn_stats", 0) == 1, f"{tag}: GroupNorm statistics recomputed inside the chain"
    assert seen["d1"] is not None, f"{tag}: the second unit's dx carries no fp16 shadow"
    assert calls.get("mas_to_half", 0) == 1, f"{tag}: the first unit converted its dout instead of reading the shadow"

    out_ref, dx_ref, gr_ref = _torch_chain(mod, x, g, torch.float64, False)
    out_yard, dx_yard, gr_yard = _torch_chain(mod, x, g, torch.float32, True)
    tol = dict(factor=FACTOR_TF32, floor=FLOOR_TF32)
    _check(tag, "out", out, out_yard, out_ref, nrows=n, **tol)
    _check(tag, "dx", dx, dx_yard, dx_ref, nrows=n, **tol)
    for key in grads:
        name = f"{key[0]}.{key[1]}"
        if name.endswith("k.bias"):
            continue      # zero in exact arithmetic (softmax over keys is invariant to a per-query constant)
        rows = grads[key].shape[0] if grads[key].dim() == 4 else None
        f16_sum = name.endswith(("conv1.bias", "conv2.bias"))   # summed from an fp16 dy shadow, as in the shadow-route cases
        _check(tag, "d" + name, grads[key], gr_yard[key], gr_ref[key], nrows=rows, **dict(tol, floor=FLOOR_F16_SUM) if f16_sum else tol)


# ------------------------------------------------------------------------------------------------ GroupNorm + Swish alone
@pytest.mark.parametrize("shape", [(32, 512, 16, 16), (2, 128, 256, 256), (12, 256, 64, 64)])
def test_groupnorm_swish_vs_fp64(shape, state):
    """Normalize + Swish as one GroupNormFn (the encoder's and decoder's last norms), forward and backward, at the batch
    sizes that run the eight-image loops of the backward reductions whole (32) and with a remainder (12)."""
    from models import modules as M
    dev = torch.device("cuda:0")
    n, c, h, w = shape
    gen = torch.Generator().manual_seed(sum(shape))
    x = ((torch.randn(n, c, h, w, generator=gen) + torch.randn(1, c, 1, 1, generator=gen)) * torch.logspace(0, 2, n).view(n, 1, 1, 1)).to(dev)
    g = (torch.randn(n, c, h, w, generator=gen) * (1 + torch.arange(n).view(n, 1, 1, 1))).to(dev)
    norm = M.Normalize(c)
    with torch.no_grad():
        norm.weight.add_(0.2 * torch.randn(c, generator=gen))
        norm.bias.add_(0.2 * torch.randn(c, generator=gen))
    norm.to(dev)
    xk = x.contiguous(memory_format=torch.channels_last).requires_grad_()
    y = norm(xk, silu=True)
    y.backward(g.contiguous(memory_format=torch.channels_last))

    def ref(dt):
        xl = x.to(dt).requires_grad_()
        wl, bl = norm.weight.detach().to(dt).requires_grad_(), norm.bias.detach().to(dt).requires_grad_()
        yl = F.silu(F.group_norm(xl, GROUPS, wl, bl, eps=EPS))
        yl.backward(g.to(dt))
        return yl.detach(), xl.grad, wl.grad, bl.grad
    r64, r32 = ref(torch.float64), ref(torch.float32)
    tag = f"gn-swish-{shape}"
    for i, (name, kern) in enumerate((("y", y), ("dx", xk.grad), ("dgamma", norm.weight.grad), ("dbeta", norm.bias.grad))):
        _check(tag, name, kern, r32[i], r64[i], nrows=n if i < 2 else None)
