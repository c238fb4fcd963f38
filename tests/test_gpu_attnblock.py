"""The VQGAN AttnBlock (ops.AttnBlockFn over csrc/attn.cu and csrc/attn_fused.cu) against fp64, on every route the shape
selects inside the forward call:

    route     shape                                      q/k/v and proj_out 1x1     QK^T -> softmax -> PV
    fused256  HW == 256, C % 256 == 0                    TF32 row GEMM              attn_core_fwd<256> (2 x fp16 operand split)
    fused128  HW == 128, C % 256 == 0                    TF32 row GEMM              attn_core_fwd<128>
    tc3       C % 128 == 0, HW % 128 == 0, not fused     TF32 row GEMM              3xTF32 GEMM + softmax
    rows      C % 128 == 0, HW % 128 != 0                TF32 row GEMM              FFMA GEMM + softmax
    simt      C % 128 != 0, or IMPL_SIMT                 FFMA                       FFMA GEMM + softmax

Accuracy is judged against the error torch itself makes on the same inputs (the yardstick), not against fixed tolerances:
a stage that claims fp32-level accuracy (the fused core, 3xTF32, FFMA, softmax, GroupNorm) against torch's float32 with
TF32 off, a TF32 stage (the row GEMMs, and every whole-block quantity of a shape whose row GEMMs run on the tensor cores)
against torch's float32 with TF32 on. The kernel's error must stay within a factor of the yardstick's, plus a small floor
for quantities torch gets (almost) exactly. Errors are compared norm-wise and on the worst query row (P, O) or image (out,
dx), so one bad 128-query tile cannot hide in a norm. The intermediates are checked against fp64 of the kernel's own inputs,
which keeps the fused core's ~1e-6 error visible under the ~5e-4 of the TF32 projections around it: a core that lost one of
the correction MMAs of its operand split, or scaled its logits by (1 + 2^-12), is off by 1e-4 or more in P or O and fails
here by a factor of 100 or more, while the block output and the fixture tests do not show it.

The factors are set from the ratios kernel error / yardstick error measured on an H100 SXM (80 GB, 700 W), largest over
all shapes and conditions here, at about twice the largest ratio:
  FFMA, softmax, GroupNorm          largest 4.6 (worst row of P on the FFMA GEMM at HW=128, C=512; mostly 1.0-1.3)
  TF32 row GEMMs, whole block       largest 3.2, typically ~2 (the proj_out bias gradient, a column sum that neither side
                                    runs on TF32, reaches 5.3 at batch 32, at 5.6e-7: under FLOOR_TF32)
  operand-split tensor cores        largest 13.4 (the 3xTF32 contractions, at C=512 or HW=1024; the fused core: 10.3)
The split operands carry 22 significant bits rather than 24, and their error grows about linearly with the contraction
length where strict fp32's grows as its square root: 3xTF32 S = Q K^T is 4.7x torch's error at C=128 and 9x at C=512.
"""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu

GROUPS, EPS = 32, 1e-6
FACTOR_FP32, FACTOR_TF32, FACTOR_SPLIT = 8.0, 6.0, 24.0
FLOOR32 = 5e-7      # ~4 fp32 ulps
FLOOR_TF32 = 1e-6   # bias gradients are column sums, which torch computes in fp32 with or without TF32
ORDER = ("nw", "nb", "qw", "qb", "kw", "kb", "vw", "vb", "pw", "pb")

# (N, C, H, W) -> route. (2, 1024, 16, 16) runs the fused core over four 256-channel halves of O (C = 768 would give three,
# but the GroupNorm kernels take power-of-two channel counts only and refuse it).
SHAPES = [((2, 512, 16, 16), "fused256"), ((32, 512, 16, 16), "fused256"), ((2, 1024, 16, 16), "fused256"),
          ((3, 256, 16, 8), "fused128"), ((1, 512, 8, 16), "fused128"),
          ((2, 512, 32, 32), "tc3"), ((2, 256, 32, 16), "tc3"), ((2, 128, 16, 16), "tc3"),
          ((2, 512, 8, 8), "rows"), ((2, 512, 12, 12), "rows"), ((2, 128, 7, 9), "rows"),
          ((2, 64, 16, 16), "simt")]
# tensor-core launches of one forward call (attn.cu): QKV row GEMM, then the fused core or two 3xTF32 GEMMs, proj_out row GEMM
TC_LAUNCHES = {"fused256": 3, "fused128": 3, "tc3": 4, "rows": 2, "simt": 0}


@pytest.fixture
def tf32_state():
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    _set_tf32(False)
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _set_tf32(on):
    torch.backends.cuda.matmul.allow_tf32 = on
    torch.backends.cudnn.allow_tf32 = on


def _scale32(c):
    """c ** -0.5 rounded to fp32, the scale the kernels and the module's float32 multiply both use."""
    return float(torch.tensor(c ** -0.5, dtype=torch.float32))


def _rows(t):
    """[N, C, H, W] -> [N, HW, C]"""
    n, c, h, w = t.shape
    return t.permute(0, 2, 3, 1).reshape(n, h * w, c)


def _core(q, k, v, scale):
    P = torch.softmax((q @ k.transpose(1, 2)) * scale, dim=-1)
    return P, P @ v


def _block(x, prm, scale):
    """GroupNorm(32) -> q, k, v 1x1 -> softmax(q k^T * scale) over keys -> P v -> proj_out 1x1 -> + x, in the dtype of x."""
    n, c, h, w = x.shape
    hn = F.group_norm(x, GROUPS, prm["nw"], prm["nb"], eps=EPS)
    H = _rows(hn)
    q, k, v = (H @ prm[a + "w"].view(c, c).T + prm[a + "b"] for a in "qkv")
    _, O = _core(q, k, v, scale)
    y = O @ prm["pw"].view(c, c).T + prm["pb"]
    return x + y.view(n, h, w, c).permute(0, 3, 1, 2)


def _torch_block(x, prm, g, dt, tf32):
    """out, dx and the parameter gradients of _block in dtype dt (matmuls on TF32 when tf32)."""
    _set_tf32(tf32)
    xl = x.detach().to(dt).requires_grad_()
    pl = {k: v.detach().to(dt).requires_grad_() for k, v in prm.items()}
    out = _block(xl, pl, _scale32(x.shape[1]))
    out.backward(g.to(dt))
    _set_tf32(False)
    return out.detach(), xl.grad, {k: v.grad for k, v in pl.items()}


def _worst(a, b, nrows):
    """Largest relative error over the rows of a and b viewed as [nrows, -1] (fp64, on the device)."""
    a = a.detach().double().reshape(nrows, -1)
    b = b.detach().double().reshape(nrows, -1)
    return float(((a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-30)).max())


def _check(tag, name, kern, yard, ref, nrows=None, factor=FACTOR_FP32, floor=FLOOR32):
    """kernel error <= factor * yardstick error + floor, norm-wise and (nrows) on the worst row."""
    ek, ey = rel_err(kern, ref), rel_err(yard, ref)
    line = f"{tag} {name}: norm {ek:.3e} / {ey:.3e} = {ek / max(ey, 1e-30):.2f}"
    ok = ek <= factor * ey + floor
    if nrows is not None:
        rk, ry = _worst(kern, ref, nrows), _worst(yard, ref, nrows)
        line += f"; worst row {rk:.3e} / {ry:.3e} = {rk / max(ry, 1e-30):.2f}"
        ok = ok and rk <= factor * ry + floor
    print("ratio", line)
    assert ok, line


def _params(c, gen):
    def w(s):
        return torch.randn(c, c, 1, 1, generator=gen) * (s / c ** 0.5)

    def b(s):
        return torch.randn(c, generator=gen) * s
    return dict(nw=1 + b(0.2), nb=b(0.2), qw=w(1.5), qb=b(0.1), kw=w(1.5), kb=b(0.1), vw=w(1.0), vb=b(0.1), pw=w(1.0), pb=b(0.1))


def _inputs(shape, seed):
    n, c, h, w = shape
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(n, c, h, w, generator=gen) + 0.5 * torch.randn(1, c, 1, 1, generator=gen)
    prm = _params(c, gen)
    # upstream gradient: neither uniform over images nor over channels
    g = torch.randn(n, c, h, w, generator=gen) * (1 + torch.arange(n).view(n, 1, 1, 1)) * (0.5 + torch.rand(1, c, 1, 1, generator=gen))
    return x, prm, g


def _run_kernel(x, prm, g):
    from mas_b200 import _lib as L, ops
    xk = x.detach().contiguous(memory_format=torch.channels_last).requires_grad_()
    pk = {k: v.detach().clone().requires_grad_() for k, v in prm.items()}
    args = [pk[k] for k in ORDER]
    t0 = L.tc_launch_count()
    out, mo, ro = ops.AttnBlockFn.apply(xk, None, None, *args)
    tc = L.tc_launch_count() - t0
    hn, qkv, P, O = out.grad_fn.saved_tensors[3:7]
    again = ops.AttnBlockFn.apply(xk, None, None, *args)[0]
    hn2, qkv2, P2, O2 = again.grad_fn.saved_tensors[3:7]
    same = all(torch.equal(a, b) for a, b in ((out, again), (hn, hn2), (qkv, qkv2), (P, P2), (O, O2)))
    del again, hn2, qkv2, P2, O2
    out.backward(g.contiguous(memory_format=torch.channels_last))
    torch.cuda.synchronize()
    return dict(out=out.detach(), mo=mo, ro=ro, tc=tc, same=same, hn=hn, qkv=qkv, P=P, O=O, dx=xk.grad,
                grads={k: v.grad for k, v in pk.items()})


def _verify(tag, shape, route, impl, x, prm, g, whole_block=True):
    """Runs the block on the kernels and checks everything against fp64; returns the kernel results. whole_block=False
    skips the comparison of out and the gradients with fp64 computed from x (see the "huge" condition)."""
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    n, c, h, w = shape
    hw = h * w
    x, g = x.to(dev), g.to(dev)
    prm = {k: v.to(dev) for k, v in prm.items()}
    ops.set_impl(impl)
    try:
        k = _run_kernel(x, prm, g)
    finally:
        ops.set_impl(L.IMPL_AUTO)
    simt = impl == L.IMPL_SIMT
    rows_tc = not simt and c % 128 == 0
    rows_tol = dict(factor=FACTOR_TF32, floor=FLOOR_TF32) if rows_tc else {}
    core_tol = dict(factor=FACTOR_SPLIT) if not simt and route in ("fused256", "fused128", "tc3") else {}

    assert k["tc"] == (0 if simt else TC_LAUNCHES[route]), f"{tag}: {k['tc']} tensor-core launches, not the {route} route"
    assert k["same"], f"{tag}: two forward calls differ"

    # ---- intermediates, each against fp64 of the kernel's own input to that stage
    x64 = x.double()
    hn_ref = F.group_norm(x64, GROUPS, prm["nw"].double(), prm["nb"].double(), eps=EPS)
    hn_yard = F.group_norm(x, GROUPS, prm["nw"], prm["nb"], eps=EPS)
    _check(tag, "hn", k["hn"], hn_yard, hn_ref, nrows=n)

    H = _rows(k["hn"])
    wcat = torch.cat([prm[a + "w"].view(c, c) for a in "qkv"])
    bcat = torch.cat([prm[a + "b"] for a in "qkv"])
    qkv_ref = H.double() @ wcat.double().T + bcat.double()
    _set_tf32(rows_tc)
    qkv_yard = H @ wcat.T + bcat
    _set_tf32(False)
    qkv = k["qkv"].view(n, hw, 3 * c)
    _check(tag, "qkv", qkv, qkv_yard, qkv_ref, nrows=n * hw, **rows_tol)

    scale = _scale32(c)
    q, kk, v = qkv[..., :c], qkv[..., c:2 * c], qkv[..., 2 * c:]
    P_ref, O_ref = _core(q.double(), kk.double(), v.double(), scale)
    P_yard, O_yard = _core(q, kk, v, scale)
    O = _rows(k["O"])
    _check(tag, "P", k["P"], P_yard, P_ref, nrows=n * hw, **core_tol)
    _check(tag, "O", O, O_yard, O_ref, nrows=n * hw, **core_tol)
    P64 = k["P"].double()
    assert float(P64.min()) >= 0.0, f"{tag}: negative probability"
    assert float((P64.sum(-1) - 1).abs().max()) <= 1e-6, f"{tag}: rows of P do not sum to 1"

    # ---- the whole block, forward and backward, against fp64 autograd from x
    if whole_block:
        out_ref, dx_ref, gr_ref = _torch_block(x, prm, g, torch.float64, False)
        out_yard, dx_yard, gr_yard = _torch_block(x, prm, g, torch.float32, rows_tc)
        _check(tag, "out", k["out"], out_yard, out_ref, nrows=n, **rows_tol)
        _check(tag, "dx", k["dx"], dx_yard, dx_ref, nrows=n, **rows_tol)
        for name in ORDER:   # rel_err compares the (mathematically zero) k.bias gradient on an absolute scale
            _check(tag, "d" + name, k["grads"][name], gr_yard[name], gr_ref[name], **rows_tol)

    # ---- statistics of the next GroupNorm, emitted by proj_out's epilogue on the tensor path with HW % 128 == 0
    if rows_tc and hw % 128 == 0:
        o64 = k["out"].double().reshape(n, GROUPS, -1)
        var, mean = torch.var_mean(o64, dim=2, unbiased=False)
        var32, mean32 = torch.var_mean(k["out"].reshape(n, GROUPS, -1), dim=2, unbiased=False)
        _check(tag, "stats mean", k["mo"], mean32.reshape(-1), mean.reshape(-1))
        _check(tag, "stats rstd", k["ro"], (var32 + EPS).rsqrt().reshape(-1), (var + EPS).rsqrt().reshape(-1))
    else:
        assert k["mo"] is None and k["ro"] is None, f"{tag}: statistics emitted off the tensor path"
    return k, x, prm


@pytest.mark.parametrize("impl_name", ["auto", "simt"])
@pytest.mark.parametrize("shape,route", SHAPES, ids=[f"{r}-{'x'.join(map(str, s))}" for s, r in SHAPES])
def test_attnblock_vs_fp64(shape, route, impl_name, tf32_state):
    from mas_b200 import _lib as L
    impl = L.IMPL_SIMT if impl_name == "simt" else L.IMPL_AUTO
    x, prm, g = _inputs(shape, seed=sum(shape))
    _verify(f"{route}-{impl_name}-{shape}", shape, route, impl, x, prm, g)


# ------------------------------------------------------------------------------------------------ conditioned inputs
def _peaked(prm, x):
    """q and k weights scaled so the logits span about +-40: P is nearly one-hot."""
    c = x.shape[1]
    p64 = {k: v.double() for k, v in prm.items()}
    H = _rows(F.group_norm(x.double(), GROUPS, p64["nw"], p64["nb"], eps=EPS))
    q, k = (H @ p64[a + "w"].view(c, c).T + p64[a + "b"] for a in "qk")
    f = (40.0 / float(((q @ k.transpose(1, 2)) * c ** -0.5).abs().max())) ** 0.5
    for a in ("qw", "qb", "kw", "kb"):
        prm[a] = prm[a] * f


def _flat(prm, x):
    prm["qw"] = torch.zeros_like(prm["qw"])
    prm["qb"] = torch.zeros_like(prm["qb"])


def _zero(prm, x):
    for a in ("qw", "qb", "kw", "kb", "vw", "vb"):
        prm[a] = torch.zeros_like(prm[a])


def _magnitude(f):
    def cond(prm, x):
        for a in ("qw", "qb", "kw", "kb", "vw", "vb"):
            prm[a] = prm[a] * f
    return cond


def _small_v(prm, x):
    prm["vw"] = prm["vw"] * 2.0 ** -12
    prm["vb"] = prm["vb"] * 2.0 ** -12


CONDITIONS = {"peaked": _peaked, "flat": _flat, "zero": _zero, "tiny": _magnitude(1e-4), "huge": _magnitude(1e4),
              "small_v": _small_v}
COND_SHAPES = [((2, 512, 16, 16), "fused256"), ((3, 256, 16, 8), "fused128"), ((2, 128, 16, 16), "tc3")]


@pytest.mark.parametrize("cond", list(CONDITIONS))
@pytest.mark.parametrize("shape,route", COND_SHAPES, ids=[f"{r}-{'x'.join(map(str, s))}" for s, r in COND_SHAPES])
def test_attnblock_conditioned(shape, route, cond, tf32_state):
    from mas_b200 import _lib as L
    x, prm, g = _inputs(shape, seed=7 * sum(shape))
    CONDITIONS[cond](prm, x)
    # at |qkv| ~ 1e4 the logits are ~1e8 and P is one-hot: a row whose two largest logits lie closer than the TF32 rounding
    # of q and k (~5e4 there) may pick another key in any float32 computation, torch's included, so out and the gradients
    # are not compared with fp64 from x; P and O are, from the kernel's own qkv
    k, x, prm = _verify(f"{route}-{cond}-{shape}", shape, route, L.IMPL_AUTO, x, prm, g, whole_block=cond != "huge")
    n, c, h, w = shape
    hw = h * w
    if cond in ("flat", "zero"):
        # S == 0 exactly: every probability is fp32(1 / HW), and O is the key mean of v
        assert torch.equal(k["P"], torch.full_like(k["P"], 1.0 / hw))
        assert torch.all(k["grads"]["kb"] == 0) and torch.all(k["grads"]["kw"] == 0)   # dK = dS^T Q with Q == 0
    if cond == "flat":
        v = k["qkv"].view(n, hw, 3 * c)[..., 2 * c:]
        O_ref = v.double().mean(dim=1, keepdim=True).expand(n, hw, c)
        O_yard = v.mean(dim=1, keepdim=True).expand(n, hw, c)
        _check(f"{route}-flat-{shape}", "O = key mean of v", _rows(k["O"]), O_yard, O_ref, nrows=n * hw, factor=FACTOR_SPLIT)
    if cond == "zero":
        # max|qkv| == 0: the operand split takes scale 1; O is exactly zero and proj_out adds its bias to x alone
        assert torch.equal(k["qkv"], torch.zeros_like(k["qkv"]))
        assert torch.equal(k["O"], torch.zeros_like(k["O"]))
        assert torch.equal(k["out"], x + prm["pb"].view(1, c, 1, 1))


# ------------------------------------------------------------------------------------------------ the building blocks
@pytest.mark.parametrize("impl_name", ["tc3", "simt"])
@pytest.mark.parametrize("hw,c", [(256, 128), (256, 512), (1024, 128), (1024, 512)])
def test_token_contractions_as_attn_calls_them(hw, c, impl_name, tf32_state):
    """The six token contractions of the block (S, O, dV, dP, dQ, dK) through mas_gemm with exactly the operands of
    attn.cu: column slices of the [N*HW, 3C] qkv activation (pitch 3C at offsets 0, C, 2C), batch strides, ta / tb."""
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    impl = L.IMPL_TC3 if impl_name == "tc3" else L.IMPL_SIMT
    n = 2
    gen = torch.Generator().manual_seed(hw + c)
    qkv = torch.randn(n * hw, 3 * c, generator=gen).to(dev)
    P = torch.softmax(3 * torch.randn(n, hw, hw, generator=gen), -1).to(dev)
    dO = torch.randn(n * hw, c, generator=gen).to(dev)
    dS = (torch.randn(n, hw, hw, generator=gen) / hw).to(dev)
    sP, sQ, sO = hw * hw, hw * 3 * c, hw * c
    scale = _scale32(c)
    q, k, v = (qkv.view(n, hw, 3 * c)[..., i * c:(i + 1) * c] for i in range(3))
    dO3 = dO.view(n, hw, c)
    tag = f"gemm-{impl_name}-hw{hw}-c{c}"

    def run(fn_ref, call, out_shape, slot=None):
        """call writes its result into a fresh buffer (the slot-th C-column slice of a [N*HW, 3C] buffer when slot is set;
        the other columns must keep their sentinel)."""
        if slot is None:
            out = torch.full(out_shape, 7.0, device=dev)
            call(out)
            got = out
        else:
            buf = torch.full((n * hw, 3 * c), 7.0, device=dev)
            call(buf, slot * c)
            got = buf.view(n, hw, 3 * c)[..., slot * c:(slot + 1) * c]
            rest = torch.cat([buf[:, :slot * c], buf[:, (slot + 1) * c:]], 1)
            assert torch.all(rest == 7.0), f"{tag}: wrote outside its column slice"
        ref = fn_ref(torch.float64)
        yard = fn_ref(torch.float32)
        _check(tag, call.__name__, got, yard, ref, nrows=got.numel() // got.shape[-1],
               factor=FACTOR_SPLIT if impl == L.IMPL_TC3 else FACTOR_FP32)

    def S(out):
        ops.gemm(qkv, (qkv, c), out, hw, hw, c, n, 3 * c, 3 * c, hw, sQ, sQ, sP, False, True, scale, impl=impl)

    def O(out):
        ops.gemm(P, (qkv, 2 * c), out, hw, c, hw, n, hw, 3 * c, c, sP, sQ, sO, False, False, 1.0, impl=impl)

    def dV(buf, off):
        ops.gemm(P, dO, (buf, off), hw, c, hw, n, hw, c, 3 * c, sP, sO, sQ, True, False, 1.0, impl=impl)

    def dP(out):
        ops.gemm(dO, (qkv, 2 * c), out, hw, hw, c, n, c, 3 * c, hw, sO, sQ, sP, False, True, 1.0, impl=impl)

    def dQ(buf, off):
        ops.gemm(dS, (qkv, c), (buf, off), hw, c, hw, n, hw, 3 * c, 3 * c, sP, sQ, sQ, False, False, 1.0, impl=impl)

    def dK(buf, off):
        ops.gemm(dS, qkv, (buf, off), hw, c, hw, n, hw, 3 * c, 3 * c, sP, sQ, sQ, True, False, 1.0, impl=impl)

    run(lambda dt: (q.to(dt) @ k.to(dt).transpose(1, 2)) * scale, S, (n, hw, hw))
    run(lambda dt: P.to(dt) @ v.to(dt), O, (n, hw, c))
    run(lambda dt: P.to(dt).transpose(1, 2) @ dO3.to(dt), dV, None, slot=2)
    run(lambda dt: dO3.to(dt) @ v.to(dt).transpose(1, 2), dP, (n, hw, hw))
    run(lambda dt: dS.to(dt) @ k.to(dt), dQ, None, slot=0)
    run(lambda dt: dS.to(dt).transpose(1, 2) @ q.to(dt), dK, None, slot=1)


def _logits(rows, cols, gen):
    s = 3 * torch.randn(rows, cols, generator=gen)
    s[::5] *= 80.0 / s[::5].abs().amax(1, keepdim=True)   # every fifth row reaches +-80
    return s


@pytest.mark.parametrize("cols", [16, 63, 144, 256, 1024])
def test_softmax_forward_vs_fp64(cols, tf32_state):
    """mas_softmax_forward in place, as attn.cu calls it; 45 rows leave the last 8-row block partial."""
    from mas_b200 import _lib as L
    dev = torch.device("cuda:0")
    rows = 45
    s = _logits(rows, cols, torch.Generator().manual_seed(cols)).to(dev)
    p = s.clone()
    L.call("mas_softmax_forward", p, p, rows, cols)
    _check(f"softmax-fwd-{cols}", "P", p, torch.softmax(s, -1), torch.softmax(s.double(), -1), nrows=rows)
    assert float(p.min()) >= 0.0


@pytest.mark.parametrize("cols", [16, 63, 144, 256, 1024])
def test_softmax_backward_vs_fp64(cols, tf32_state):
    """mas_softmax_backward with the attention scale, dP overwritten by dS as attn.cu calls it."""
    from mas_b200 import _lib as L
    dev = torch.device("cuda:0")
    rows = 45
    gen = torch.Generator().manual_seed(100 + cols)
    p = torch.softmax(_logits(rows, cols, gen), -1).to(dev)
    dp = torch.randn(rows, cols, generator=gen).to(dev)
    scale = _scale32(512)

    def ref(dt):
        pp, dd = p.to(dt), dp.to(dt)
        return pp * (dd - (pp * dd).sum(-1, keepdim=True)) * scale
    ds = dp.clone()
    L.call("mas_softmax_backward", p, ds, ds, rows, cols, scale)
    _check(f"softmax-bwd-{cols}", "dS", ds, ref(torch.float32), ref(torch.float64), nrows=rows)
