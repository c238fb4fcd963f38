"""PatchGAN discriminator drop-in (losses/discriminator.py) without a GPU: parameter layout and seeded initialisation
against the real reference (tests/golden/discriminator.pt), resolution of the `losses` package next to a reference
checkout, the index geometry of the 4x4 kernels, and the host logic of ops.Conv4x4Fn / ops.BatchNormLReLUFn over an
emulation of the C-ABI entries' documented semantics (include/mas_b200.h) that reads and writes the CPU tensors' memory
through the pointers and mas_tensor4 strides the units pass.  The kernels themselves are tested on the GPU
(tests/test_gpu_discriminator.py)."""
import ctypes
import hashlib
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, PKG, rel_err


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "discriminator.pt"), weights_only=False)


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


def _images(case):
    gen = torch.Generator().manual_seed(case["seed"] + 1000)
    shape = (case["batch"], 3, case["size"], case["size"])
    return torch.rand(shape, generator=gen), torch.rand(shape, generator=gen)


# ------------------------------------------------------------------------------------------------ parameters
@pytest.mark.parametrize("name", ["256", "72"])
def test_state_dict_and_seeded_init_match_reference(golden, name):
    from losses.discriminator import Discriminator, weights_init
    case = golden[name]
    torch.manual_seed(case["seed"])
    m = Discriminator()
    m.apply(weights_init)
    sd = m.state_dict()
    assert list(sd) == list(case["init"]) and len(sd) == 22
    for k, v in sd.items():
        ref = case["init"][k]
        assert tuple(v.shape) == ref["shape"] and str(v.dtype) == ref["dtype"], k
        assert _sha(v) == ref["sha256"], k          # bit for bit
    real, fake = _images(case)
    assert _sha(torch.cat([real, fake])) == case["images_sha256"]


# ------------------------------------------------------------------------------------------------ package resolution
def test_losses_package_resolves_next_to_reference(tmp_path):
    ref = tmp_path / "ref" / "losses"
    ref.mkdir(parents=True)
    (ref / "__init__.py").write_text("from .loss_seg import BCELossWithQuant, VQVAEWithBCELoss\n"
                                     "from .loss_img import VQLPIPSWithDiscriminator\n")
    (ref / "loss_img.py").write_text("from .discriminator import Discriminator, weights_init\n"
                                     "class VQLPIPSWithDiscriminator:\n    pass\n")
    (ref / "loss_seg.py").write_text("class BCELossWithQuant:\n    pass\nclass VQVAEWithBCELoss:\n    pass\n")
    (ref / "discriminator.py").write_text("raise ImportError('the reference discriminator must not be picked up')\n")
    prog = textwrap.dedent("""
        import sys
        sys.path[:0] = [%r, %r]
        import losses.discriminator as d
        assert "losses.loss_img" not in sys.modules and "losses.lpips" not in sys.modules
        import losses.loss_img as li
        assert li.Discriminator is d.Discriminator and li.weights_init is d.weights_init
        assert d.__file__.startswith(%r)
        import losses
        assert losses.VQLPIPSWithDiscriminator is li.VQLPIPSWithDiscriminator
        assert losses.BCELossWithQuant.__module__ == "losses.loss_seg"
        assert sys.modules["losses.loss_seg"].__file__.startswith(%r)
        print("ok")
    """) % (PKG, str(tmp_path / "ref"), PKG, str(tmp_path / "ref"))
    r = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr


# ------------------------------------------------------------------------------------------------ kernel geometry
def _gather_fwd(x, stride):
    """conv4x4_kernel<false> A operand: A[m=(n,oh,ow)][k=(t,ci)] = x(n, s*oh-1+kh, s*ow-1+kw, ci), 0 outside."""
    n, h, w, c = x.shape
    ho, wo = (h - 2) // stride + 1, (w - 2) // stride + 1
    A = np.zeros((n, ho, wo, 16, c))
    for oh in range(ho):
        for ow in range(wo):
            for t in range(16):
                ih, iw = stride * oh - 1 + (t >> 2), stride * ow - 1 + (t & 3)
                if 0 <= ih < h and 0 <= iw < w:
                    A[:, oh, ow, t] = x[:, ih, iw]
    return A.reshape(n * ho * wo, 16 * c), (n, ho, wo)


def _gather_dgrad(dy, h, w, stride):
    """conv4x4_kernel<true> A operand: A[m=(n,ih,iw)][k=(t,co)] = dy(n, (ih+1-kh)/s, (iw+1-kw)/s, co) when both quotients are
    exact and inside dy, else 0."""
    n, ho, wo, c = dy.shape
    A = np.zeros((n, h, w, 16, c))
    for ih in range(h):
        for iw in range(w):
            for t in range(16):
                u, v = ih + 1 - (t >> 2), iw + 1 - (t & 3)
                if u % stride or v % stride:
                    continue
                oh, ow = u // stride, v // stride
                if 0 <= oh < ho and 0 <= ow < wo:
                    A[:, ih, iw, t] = dy[:, oh, ow]
    return A.reshape(n * h * w, 16 * c)


def _pack(w, transpose):
    """mas_pack_conv4x4: [(t*Cin + ci)][co], transposed [(t*Cout + co)][ci]."""
    cout, cin = w.shape[:2]
    wt = w.reshape(cout, cin, 16)
    return (wt.transpose(2, 0, 1).reshape(16 * cout, cin) if transpose else wt.transpose(2, 1, 0).reshape(16 * cin, cout))


@pytest.mark.parametrize("stride,h,w", [(2, 10, 9), (2, 8, 8), (1, 7, 6), (1, 9, 9)])
def test_tap_geometry_fp64(stride, h, w):
    rng = np.random.default_rng(stride * 100 + h)
    cin, cout, n = 5, 6, 2
    x = rng.standard_normal((n, h, w, cin))
    wt = rng.standard_normal((cout, cin, 4, 4))
    A, (n_, ho, wo) = _gather_fwd(x, stride)
    y = (A @ _pack(wt, False)).reshape(n, ho, wo, cout)
    xt, wtt = torch.from_numpy(x).permute(0, 3, 1, 2), torch.from_numpy(wt)
    y_ref = F.conv2d(xt, wtt, stride=stride, padding=1).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(y, y_ref, rtol=1e-12, atol=1e-12)
    dy = rng.standard_normal((n, ho, wo, cout))
    dx = (_gather_dgrad(dy, h, w, stride) @ _pack(wt, True)).reshape(n, h, w, cin)
    dx_ref = F.conv_transpose2d(torch.from_numpy(dy).permute(0, 3, 1, 2), wtt, stride=stride, padding=1,
                                output_padding=((h - 2) % stride, (w - 2) % stride))
    np.testing.assert_allclose(dx, dx_ref.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)
    # weight gradient: dw[co][(t,ci)] = dy^T . A
    dw = (dy.reshape(-1, cout).T @ A).reshape(cout, 16, cin).transpose(0, 2, 1).reshape(cout, cin, 4, 4)
    xr = xt.clone().requires_grad_(True)
    wr = wtt.clone().requires_grad_(True)
    F.conv2d(xr, wr, stride=stride, padding=1).backward(torch.from_numpy(dy).permute(0, 3, 1, 2))
    np.testing.assert_allclose(dw, wr.grad.numpy(), rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ shift-map (tensor-core) route
def _tap4(a, p, stride):
    """csrc/conv4x4.cu tap4_of: the 4x4 tap that 3x3 tap a of plane p stands for (-1: none)."""
    if stride == 2:
        kh = 2 * a - 1 + p
        return kh if 0 <= kh < 4 else -1
    return a if p == 0 else (3 if a == 2 else -1)


def _shift_map(x, stride):
    """mas_conv4x4_shift_map: X'(i, j, (2p+q)*C + c) = x(s*i + p, s*j + q, c), 0 outside; x [n, h, w, c]."""
    n, h, w, c = x.shape
    hs, ws = h // stride, w // stride
    out = np.zeros((n, hs, ws, 4 * c))
    for pq in range(4):
        p, q = pq >> 1, pq & 1
        for i in range(hs):
            for j in range(ws):
                if stride * i + p < h and stride * j + q < w:
                    out[:, i, j, pq * c:(pq + 1) * c] = x[:, stride * i + p, stride * j + q]
    return out


def _shift_map_adjoint(dm, h, w, stride):
    n, hs, ws, c4 = dm.shape
    c = c4 // 4
    dx = np.zeros((n, h, w, c))
    for pq in range(4):
        p, q = pq >> 1, pq & 1
        for i in range(hs):
            for j in range(ws):
                if stride * i + p < h and stride * j + q < w:
                    dx[:, stride * i + p, stride * j + q] += dm[:, i, j, pq * c:(pq + 1) * c]
    return dx


def _remap(w4, stride):
    cout, cin = w4.shape[:2]
    w3 = np.zeros((cout, 4 * cin, 3, 3))
    for pq in range(4):
        for a in range(3):
            for b in range(3):
                kh, kw = _tap4(a, pq >> 1, stride), _tap4(b, pq & 1, stride)
                if kh >= 0 and kw >= 0:
                    w3[:, pq * cin:(pq + 1) * cin, a, b] = w4[:, :, kh, kw]
    return w3


def _unmap(dw3, cin, stride):
    dw = np.zeros((dw3.shape[0], cin, 4, 4))
    for pq in range(4):
        for a in range(3):
            for b in range(3):
                kh, kw = _tap4(a, pq >> 1, stride), _tap4(b, pq & 1, stride)
                if kh >= 0 and kw >= 0:
                    dw[:, :, kh, kw] = dw3[:, pq * cin:(pq + 1) * cin, a, b]
    return dw


@pytest.mark.parametrize("stride,h,w", [(2, 8, 10), (2, 6, 6), (1, 8, 8), (1, 7, 9)])
def test_shift_map_route_fp64(stride, h, w):
    """The 4x4 convolution as the 3x3 stride-1 pad-1 convolution of the shift map (forward, data gradient through the
    adjoint map, weight gradient through the inverse weight remap) equals F.conv2d in fp64; each 4x4 tap has exactly one
    representative.  At stride 1 the 3x3 output has an extra last row and column: the output gradient there must be zero,
    and a poisoned padding row / column changes dx and dw."""
    rng = np.random.default_rng(stride * 1000 + h * 10 + w)
    n, cin, cout = 2, 3, 5
    x = rng.standard_normal((n, h, w, cin))
    w4 = rng.standard_normal((cout, cin, 4, 4))
    assert sum(_tap4(a, p, stride) >= 0 for a in range(3) for p in range(2)) == 4
    xt = torch.from_numpy(x).permute(0, 3, 1, 2).requires_grad_(True)
    wt = torch.from_numpy(w4).requires_grad_(True)
    y_ref = F.conv2d(xt, wt, stride=stride, padding=1)
    ho, wo = y_ref.shape[2:]
    dy = torch.from_numpy(rng.standard_normal(y_ref.shape))
    y_ref.backward(dy)

    xm = torch.from_numpy(_shift_map(x, stride)).permute(0, 3, 1, 2).requires_grad_(True)
    w3 = torch.from_numpy(_remap(w4, stride)).requires_grad_(True)
    y3 = F.conv2d(xm, w3, padding=1)
    assert y3.shape[2:] == ((ho, wo) if stride == 2 else (ho + 1, wo + 1))
    np.testing.assert_allclose(y3[:, :, :ho, :wo].detach().numpy(), y_ref.detach().numpy(), rtol=1e-12, atol=1e-12)

    def grads(pad_value):
        dyp = torch.full(y3.shape, pad_value, dtype=torch.float64)
        dyp[:, :, :ho, :wo] = dy
        gx, gw = torch.autograd.grad(y3, (xm, w3), dyp, retain_graph=True)
        dx = _shift_map_adjoint(gx.permute(0, 2, 3, 1).numpy(), h, w, stride)
        return dx.transpose(0, 3, 1, 2), _unmap(gw.numpy(), cin, stride)

    dx, dw = grads(0.0)
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dw, wt.grad.numpy(), rtol=1e-12, atol=1e-12)
    if stride == 1:
        dx_bad, dw_bad = grads(7.0)
        assert np.abs(dx_bad - xt.grad.numpy()).max() > 1e-3 and np.abs(dw_bad - wt.grad.numpy()).max() > 1e-3


# ------------------------------------------------------------------------------------------------ emulated C-ABI
def _addr(v):
    if v is None:
        return 0
    if isinstance(v, torch.Tensor):
        return v.data_ptr()
    if isinstance(v, ctypes.c_void_p):
        return v.value or 0
    raise TypeError(type(v))


def _f32(p, n):
    return np.ctypeslib.as_array((ctypes.c_float * int(n)).from_address(_addr(p)))


def _f64(p, n):
    return np.ctypeslib.as_array((ctypes.c_double * int(n)).from_address(_addr(p)))


def _view4(p, t4):
    dims, strides = (t4.n, t4.h, t4.w, t4.c), (t4.sn, t4.sh, t4.sw, t4.sc)
    extent = 1 + sum((d - 1) * s for d, s in zip(dims, strides))
    return np.lib.stride_tricks.as_strided(_f32(p, extent), dims, tuple(4 * s for s in strides))


class DiscEmu:
    """The discriminator's C-ABI entries on CPU memory; the 4x4 convolutions accumulate in fp64 tap by tap."""

    def __init__(self):
        self.names = []

    def __call__(self, name, *a):
        self.names.append(name)
        getattr(self, name)(*a)

    @staticmethod
    def _taps(h, w, stride, ho, wo):
        for t in range(16):
            kh, kw = t >> 2, t & 3
            yield t, slice(kh, kh + stride * (ho - 1) + 1, stride), slice(kw, kw + stride * (wo - 1) + 1, stride)

    def mas_pack_conv4x4(self, w, wp, cout, cin, transpose):
        src = _f32(w, cout * cin * 16).reshape(cout, cin, 4, 4).astype(np.float64)
        _f32(wp, cout * cin * 16)[:] = _pack(src, transpose).reshape(-1)

    def mas_conv4x4(self, x, xs, wp, bias, y, ys, stride, slope, act):
        xv = np.pad(_view4(x, xs).astype(np.float64), ((0, 0), (1, 1), (1, 1), (0, 0)))
        cin, cout = xs.c, ys.c
        W = _f32(wp, 16 * cin * cout).reshape(16, cin, cout).astype(np.float64)
        acc = np.zeros((ys.n, ys.h, ys.w, cout))
        for t, sh, sw in self._taps(xs.h, xs.w, stride, ys.h, ys.w):
            acc += xv[:, sh, sw] @ W[t]
        if bias is not None:
            acc += _f32(bias, cout)
        acc = acc.astype(np.float32)
        if act:
            acc = np.where(acc > 0, acc, acc * np.float32(slope))
        _view4(y, ys)[...] = acc

    def mas_conv4x4_dgrad(self, dy, dys, wp, dx, dxs, stride):
        dyv = _view4(dy, dys).astype(np.float64)
        cout, cin = dys.c, dxs.c
        W = _f32(wp, 16 * cin * cout).reshape(16, cout, cin).astype(np.float64)
        acc = np.zeros((dxs.n, dxs.h + 4, dxs.w + 4, cin))
        for t, sh, sw in self._taps(dxs.h, dxs.w, stride, dys.h, dys.w):
            acc[:, sh, sw] += dyv @ W[t]
        _view4(dx, dxs)[...] = acc[:, 1:1 + dxs.h, 1:1 + dxs.w].astype(np.float32)

    def mas_conv4x4_wgrad(self, x, xs, dy, dys, dw, stride, ws, nbytes):
        xv = np.pad(_view4(x, xs).astype(np.float64), ((0, 0), (1, 1), (1, 1), (0, 0)))
        dyv = _view4(dy, dys).astype(np.float64).reshape(-1, dys.c)
        out = np.zeros((dys.c, xs.c, 16))
        for t, sh, sw in self._taps(xs.h, xs.w, stride, dys.h, dys.w):
            out[:, :, t] = dyv.T @ xv[:, sh, sw].reshape(-1, xs.c)
        _f32(dw, out.size)[:] = out.reshape(-1).astype(np.float32)

    def mas_colsum(self, x, t, out, ws, nbytes):
        _f32(out, t.c)[:] = _view4(x, t).astype(np.float64).sum(axis=(0, 1, 2)).astype(np.float32)

    def mas_lrelu_backward(self, dy, y, slope, dx, n):
        d, yy = _f32(dy, n), _f32(y, n)
        _f32(dx, n)[:] = np.where(yy > 0, d, d * np.float32(slope))

    def mas_copy_strided(self, x, xs, y, ys):
        _view4(y, ys)[...] = _view4(x, xs)

    def mas_bn_stats(self, x, R, C, out):
        xv = _f32(x, R * C).reshape(R, C).astype(np.float64)
        o = _f64(out, 2 * C + 1)
        o[:C], o[C:2 * C], o[2 * C] = xv.sum(0), (xv * xv).sum(0), R

    def mas_bn_finalize(self, stats, count, C, eps, mom, mean, invstd, rm, rv):
        s = _f64(stats, 2 * C + 1)
        cnt = count if count > 0 else s[2 * C]
        m = s[:C] / cnt
        var = np.maximum(s[C:2 * C] / cnt - m * m, 0)
        _f32(mean, C)[:] = m
        _f32(invstd, C)[:] = 1.0 / np.sqrt(var + eps)
        if rm is not None:
            r_m, r_v = _f32(rm, C), _f32(rv, C)
            r_m[:] = (1 - mom) * r_m.astype(np.float64) + mom * m
            r_v[:] = (1 - mom) * r_v.astype(np.float64) + mom * var * cnt / (cnt - 1)

    def mas_bn_invstd(self, rv, eps, invstd, C):
        _f32(invstd, C)[:] = 1.0 / np.sqrt(_f32(rv, C).astype(np.float64) + eps)

    def mas_bn_apply_lrelu(self, x, mean, invstd, g, b, slope, y, R, C):
        v = ((_f32(x, R * C).reshape(R, C) - _f32(mean, C)) * _f32(invstd, C) * _f32(g, C) + _f32(b, C)).astype(np.float32)
        _f32(y, R * C)[:] = np.where(v > 0, v, v * np.float32(slope)).reshape(-1)

    def _dz(self, dy, y, slope, R, C):
        d, yy = _f32(dy, R * C).reshape(R, C), _f32(y, R * C).reshape(R, C)
        return np.where(yy > 0, d, d * np.float32(slope)).astype(np.float64)

    def mas_bn_backward_reduce_lrelu(self, dy, y, slope, x, mean, invstd, R, C, out, ws, nbytes):
        dz = self._dz(dy, y, slope, R, C)
        xh = (_f32(x, R * C).reshape(R, C) - _f32(mean, C)) * _f32(invstd, C)
        o = _f64(out, 2 * C + 1)
        o[:C], o[C:2 * C], o[2 * C] = dz.sum(0), (dz * xh).sum(0), R

    def mas_bn_backward_apply_lrelu(self, dy, y, slope, x, mean, invstd, g, sums, dx, dg, db, R, C):
        dz = self._dz(dy, y, slope, R, C)
        s = _f64(sums, 2 * C + 1)
        xh = (_f32(x, R * C).reshape(R, C) - _f32(mean, C)) * _f32(invstd, C)
        _f32(dx, R * C)[:] = (_f32(g, C) * _f32(invstd, C) * (dz - s[:C] / R - xh * s[C:2 * C] / R)).reshape(-1)
        if dg is not None:
            _f32(db, C)[:] = s[:C]
            _f32(dg, C)[:] = s[C:2 * C]


@pytest.fixture()
def emu(monkeypatch):
    from mas_b200 import ops
    e = DiscEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops.L, "query", lambda name, *a: 64)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: False)     # the 4x4 SIMT route; the shift-map route is pinned below
    return e


def _check(rec, t, tol):
    t = t.detach().double()
    assert abs(float(t.norm()) - rec["norm"]) <= tol * rec["norm"]
    if "full" in rec:
        assert rel_err(t, rec["full"]) < tol
    else:
        assert rel_err(t.reshape(-1)[rec["idx"]], rec["val"]) < tol


def _stats(m, ref):
    sd = m.state_dict()
    for k, v in ref.items():
        if "num_batches" in k:
            assert int(sd[k]) == int(v), k
        else:
            assert rel_err(sd[k], v) < 1e-5, k


@pytest.mark.parametrize("name", ["72", "256"])
def test_host_logic_train_step_against_golden(emu, golden, name):
    """train.py:84-98 on the emulated entries: discriminator step, then the generator step with D frozen (autograd.grad with
    retain_graph=True, then backward on the same graph)."""
    from losses.discriminator import Discriminator, weights_init
    case = golden[name]
    torch.manual_seed(case["seed"])
    m = Discriminator()
    m.apply(weights_init)
    m.train()
    real, fake = _images(case)
    lr, lf = m(real), m(fake)
    assert lr.shape == case["logits_real"].shape and lr.is_contiguous()
    assert rel_err(lr, case["logits_real"]) < 1e-3 and rel_err(lf, case["logits_fake"]) < 1e-3
    del emu.names[:]
    (0.5 * (torch.relu(1.0 - lr).mean() + torch.relu(1.0 + lf).mean())).backward()
    d_names = list(emu.names)
    for k, p in m.named_parameters():
        _check(case["grads"][k], p.grad, 3e-3)
    _stats(m, case["stats_d"])
    # per forward graph: the images are leaves (no model.0 data gradient); every layer has a weight gradient
    assert d_names.count("mas_conv4x4_dgrad") == 2 * 4 and d_names.count("mas_conv4x4_wgrad") == 2 * 5
    assert d_names.count("mas_pack_conv4x4") == 4          # transposed packings of model.2/5/8/11, once each

    for p in m.parameters():
        p.requires_grad_(False)
    rec = fake.clone().requires_grad_(True)
    lg = m(rec)
    g = -torch.mean(lg)
    del emu.names[:]
    (d1,) = torch.autograd.grad(g, rec, retain_graph=True)
    g.backward()
    g_names = list(emu.names)
    assert "mas_conv4x4_wgrad" not in g_names and "mas_colsum" not in g_names
    assert g_names.count("mas_pack_conv4x4") == 1          # model.0's transposed packing: first needed here
    assert g_names.count("mas_conv4x4_dgrad") == 2 * 5
    assert rel_err(lg, case["logits_g"]) < 1e-3
    _check(case["drec_grad"], d1, 3e-3)
    _check(case["drec_backward"], rec.grad, 3e-3)
    _stats(m, case["stats_g"])
