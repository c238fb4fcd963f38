"""Host logic of the face loss (ops.FacePlan, ops.FaceLossFn, losses.face_loss) WITHOUT a GPU: ops.L.call is replaced by an
emulation of the C-ABI entries' documented semantics (include/mas_b200.h) that reads and writes the CPU tensors' memory
through the pointers, mas_tensor4 strides and scalars the unit passes, in fp64 with REAL fp16 rounding of every fp16 operand.
The drop-in then runs end to end on the CPU against the real reference's golden (tests/golden/face_loss.pt) and the fp64
restatement: the 14-int face table as the kernels read it, the crop span kept for the backward, the seed placement at the
layer ends and the stride-2 hand-over, the unit-seed input gradient and its reuse on a retained graph. The kernels
themselves are tested on the GPU (tests/test_gpu_face_loss.py)."""
import copy
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from face_common import case_inputs, load_golden, restated_loss, seeded_face_loss
from test_host_logic_vq_cpu import VqEmu, _addr, _f16, _f32, _scale, _t, _view4

CROP = 254


def _i8(p, n):
    return np.ctypeslib.as_array((ctypes.c_int8 * int(n)).from_address(_addr(p)))


def _u8(p, n):
    return np.ctypeslib.as_array((ctypes.c_uint8 * int(n)).from_address(_addr(p)))


def _f64(p, n):
    return np.ctypeslib.as_array((ctypes.c_double * int(n)).from_address(_addr(p)))


def _nhwc(p, n, h, w, c):
    return _f32(p, n * h * w * c).reshape(n, h, w, c)


class FaceEmu(VqEmu):
    """VqEmu (to_half, the 3x3 family) plus the fp16 row GEMM, the ReLU helpers and the mas_face_* entries."""

    def __init__(self, tab_len=None):
        super().__init__()
        self.gemm_packs = {}

    # ---- reused entries ------------------------------------------------------------------------------------------------
    def mas_pack_gemm_tc16(self, w, out, N, K, transpose):
        W = _f32(w, N * K).reshape(N, K).astype(np.float16).astype(np.float64)
        self.gemm_packs[_addr(out)] = W.T.copy() if transpose else W      # rows: output features of the product

    def mas_gemm_rows_f16(self, x16, M, K, wpk, y, ldy, N, bias, residual, x_amax, alpha):
        X = _f16(x16, M * K).reshape(M, K).astype(np.float64) / _scale(x_amax)
        Wp = self.gemm_packs[_addr(wpk)]
        assert Wp.shape[1] == K and Wp.shape[0] % 128 == 0 and Wp.shape[0] >= N, (Wp.shape, N, K)
        o = alpha * (X @ Wp[:N].T)
        if bias is not None:
            o = o + _f32(bias, N).astype(np.float64)
        Y = _f32(y, M * ldy).reshape(M, ldy)
        if residual is not None:
            o = o + _f32(residual, M * ldy).reshape(M, ldy)[:, :N]
        Y[:, :N] = o

    def mas_lpips_relu(self, y, n, amax):
        v = _f32(y, n)
        v[...] = np.maximum(v, 0)
        _f32(amax, 1)[0] = v.max()

    def mas_lpips_relu_backward(self, dy, y, dx, n, amax):
        o = np.where(_f32(y, n) > 0, _f32(dy, n), np.float32(0))
        _f32(dx, n)[...] = o
        _f32(amax, 1)[0] = np.abs(o).max()

    def mas_lpips_scale_jacobian(self, J, g, g_stride, out, B, per):
        gv = _f32(g, 1 + (B - 1) * g_stride)[::max(g_stride, 1)][:B] if g_stride else np.repeat(_f32(g, 1), B)
        _f32(out, B * per).reshape(B, per)[...] = gv[:, None] * _f32(J, B * per).reshape(B, per)

    # ---- face entries ----------------------------------------------------------------------------------------------------
    @staticmethod
    def _axes(tab, wts, f, H, W):
        """Per axis the [254, extent of the image] gather matrix of face f, as mas_face_prepare reads the table."""
        m = [int(v) for v in tab[14 * f:14 * f + 14]]
        src, side, top, left, ch, cw, ky, kx, o_sy, o_sx, o_ay, o_ax, o_wy, o_wx = m
        mats = []
        for o_s, o_w, k, ext, org, lim in ((o_sy, o_wy, ky, ch, top, H), (o_sx, o_wx, kx, cw, left, W)):
            M = np.zeros((CROP, lim))
            for o in range(CROP):
                for i in range(k):
                    c = int(tab[o_s + o]) + i
                    if c < ext and 0 <= org + c < lim:
                        M[o, org + c] += wts[o_w + o * k + i]
            mats.append(M)
        return src, side, top, left, ch, cw, (o_ay, o_ax, o_sy, o_sx, ky, kx), mats

    def _tab(self, tab, F_):
        meta = _view_i32(tab, 14 * F_)
        n = int(max(meta[14 * f + 10] + 2 * meta[14 * f + 4] for f in range(F_)))
        n = max(n, int(max(meta[14 * f + 11] + 2 * meta[14 * f + 5] for f in range(F_))))
        t = _view_i32(tab, n)
        nw = int(max(meta[14 * f + 13] + CROP * meta[14 * f + 7] for f in range(F_)))
        return t, nw

    def mas_face_prepare(self, tab, wts, F_, img, is_, rec, rs, out):
        t, nw = self._tab(tab, F_)
        w = _f32(wts, nw).astype(np.float32).astype(np.float64)
        o = _nhwc(out, F_, CROP, CROP, 3)
        for f in range(F_):
            side = int(t[14 * f + 1])
            ts = rs if side else is_
            im = _view4(rec if side else img, ts).astype(np.float64)          # [n, h, w, 3]
            src, *_, mats = self._axes(t, w, f, ts.h, ts.w)
            o[f] = np.einsum("yh,hwc,xw->yxc", mats[0], im[src], mats[1], optimize=True)

    def mas_face_prepare_backward(self, tab, wts, f0, G, side, d, J, B, H, W):
        meta = _view_i32(tab, 14 * (f0 + G))
        t, nw = self._tab(tab, f0 + G)
        w = _f32(wts, nw).astype(np.float64)
        out = np.zeros((B, 3, H, W))
        D = _nhwc(d, G, CROP, CROP, 3).astype(np.float64)
        for g in range(G):
            f = f0 + g
            if int(meta[14 * f + 1]) != side:
                continue
            src, *_, mats = self._axes(t, w, f, H, W)
            out[src] += np.einsum("yh,yxc,xw->chw", mats[0], D[g], mats[1], optimize=True)
        _f32(J, B * 3 * H * W)[...] = out.reshape(-1)

    def mas_face_stem_forward(self, x, w, y, N, H, W):
        X = _t(_nhwc(x, N, H, W, 3)).permute(0, 3, 1, 2)
        Wt = _t(_f32(w, 64 * 3 * 49).reshape(64, 3, 7, 7))
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        _nhwc(y, N, Ho, Wo, 64)[...] = F.conv2d(X, Wt, stride=2, padding=3).permute(0, 2, 3, 1).numpy()

    def mas_face_stem_backward(self, dy, w, dx, N, H, W):
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        D = _t(_nhwc(dy, N, Ho, Wo, 64)).permute(0, 3, 1, 2)
        Wt = _t(_f32(w, 64 * 3 * 49).reshape(64, 3, 7, 7))
        g = torch.nn.grad.conv2d_input((N, 3, H, W), Wt, D, stride=2, padding=3)
        _nhwc(dx, N, H, W, 3)[...] = g.permute(0, 2, 3, 1).numpy()

    @staticmethod
    def _z(x, bn, N, H, W, C):
        b = _f32(bn, 2 * C).reshape(2, C)
        return _nhwc(x, N, H, W, C) * b[0] + b[1], b[0]                     # fp32, as the kernel

    def mas_face_pool_forward(self, x, bn, y, arg, N, H, W, C, amax):
        z, _ = self._z(x, bn, N, H, W, C)
        r = torch.from_numpy(np.maximum(z, 0).astype(np.float32)).permute(0, 3, 1, 2)
        Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
        win = F.unfold(r, 3, stride=2).reshape(N, C, 9, Ho, Wo)
        idx = win.argmax(dim=2)                                               # the first maximum, row-major
        best = win.gather(2, idx[:, :, None]).squeeze(2)
        _nhwc(y, N, Ho, Wo, C)[...] = best.permute(0, 2, 3, 1).numpy()
        _u8(arg, N * Ho * Wo * C)[...] = idx.permute(0, 2, 3, 1).numpy().reshape(-1)
        if amax is not None:
            _f32(amax, 1)[0] = float(best.max())

    @staticmethod
    def _seed(sgn, coef, f0, P, G, per):
        S = _i8(sgn, P * per).reshape(P, per).astype(np.float64) * coef
        return np.stack([S[f] if f < P else -S[f - P] for f in range(f0, f0 + G)])

    def mas_face_pool_backward(self, x, bn, arg, dp, sgn, coef, f0, P, G, H, W, C, dx):
        out = np.zeros((G, H, W, C))
        if dp is not None:
            Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
            idx = torch.from_numpy(_u8(arg, G * Ho * Wo * C).reshape(G, Ho, Wo, C).astype(np.int64)).permute(0, 3, 1, 2)
            D = _t(_nhwc(dp, G, Ho, Wo, C)).permute(0, 3, 1, 2)
            onehot = F.one_hot(idx, 9).permute(0, 1, 4, 2, 3).double() * D[:, :, None]
            routed = F.fold(onehot.reshape(G, C * 9, Ho * Wo), (H, W), 3, stride=2).permute(0, 2, 3, 1).numpy()
            z, s = self._z(x, bn, G, H, W, C)
            out = np.where(z > 0, routed * s, 0.0)
        if sgn is not None:
            out = out + self._seed(sgn, coef, f0, P, G, H * W * C).reshape(G, H, W, C)
        _nhwc(dx, G, H, W, C)[...] = out

    def mas_face_l1_forward(self, f, n, sgn, part):
        v = _f32(f, 2 * n).astype(np.float64)
        d = v[:n] - v[n:]
        p = _f64(part, 128)
        p[...] = 0
        p[0] = np.abs(d).sum()
        if sgn is not None:
            _i8(sgn, n)[...] = np.sign(d).astype(np.int8)

    def mas_face_l1_finalize(self, part, c0, c1, c2, c3, c4, terms, loss):
        p = _f64(part, 5 * 128).reshape(5, 128)
        t = np.array([c * p[l].sum() for l, c in enumerate((c0, c1, c2, c3, c4))], dtype=np.float32)
        _f32(terms, 5)[...] = t
        _f32(loss, 1)[0] = np.float32(sum(float(v) for v in t))

    def mas_face_subsample_half(self, x, y16, N, H, W, C, amax):
        sub = _nhwc(x, N, H, W, C)[:, ::2, ::2].astype(np.float64) * _scale(amax)
        _f16(y16, sub.size)[...] = sub.astype(np.float16).reshape(-1)

    def mas_face_relu_seed_backward(self, out, dout, half, sgn, coef, f0, P, G, H, W, C, dz, amax):
        g = np.zeros((G, H, W, C))
        if dout is not None:
            if half:
                g[:, ::2, ::2] = _nhwc(dout, G, (H + 1) // 2, (W + 1) // 2, C)
            else:
                g = _nhwc(dout, G, H, W, C).astype(np.float64)
        if sgn is not None:
            g = g + self._seed(sgn, coef, f0, P, G, H * W * C).reshape(G, H, W, C)
        o = np.where(_nhwc(out, G, H, W, C) > 0, g, 0.0)
        _nhwc(dz, G, H, W, C)[...] = o
        _f32(amax, 1)[0] = np.abs(o).max()


def _view_i32(p, n):
    return np.ctypeslib.as_array((ctypes.c_int32 * int(n)).from_address(_addr(p)))


def _dense(t):
    return t.sc == 1 and t.sw == t.c and t.sh == t.w * t.c and t.sn == t.h * t.w * t.c


@pytest.fixture
def face_emu(monkeypatch):
    from mas_b200 import ops
    e = FaceEmu()
    monkeypatch.setattr(ops.L, "call", e)

    def query(name, *a):
        if name == "mas_conv3x3_tc_eligible":        # dense NHWC, Cin % 8, Cout % 128, Hout % 16, Wout % 8, S1 / UP / ZS
            xs, ys, mode = a
            return int(_dense(xs) and _dense(ys) and xs.c % 8 == 0 and ys.c % 128 == 0 and ys.h % 16 == 0 and ys.w % 8 == 0
                       and mode in (0, 2, 3))
        if name == "mas_face_l1_blocks":
            return 128
        raise AssertionError(name)
    monkeypatch.setattr(ops.L, "query", query)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: True)
    return e


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def _pinned_reference(m, img, rec, boxes, feats, want_img):
    """fp64 restatement's loss under OUR sign pattern, and its gradients."""
    signs = [torch.sign(a - b) for a, b in (f.double().chunk(2) for f in feats)]
    i = img.double().requires_grad_(want_img)
    r = rec.double().requires_grad_(True)
    _, _, _, loss = restated_loss(m, i, r, boxes, signs=signs)
    loss.backward()
    return i.grad, r.grad


@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_face_loss_host_logic_against_golden(face_emu, golden, name):
    case = golden[name]
    m, _ = seeded_face_loss(case)
    ref = copy.deepcopy(m)
    img, rec = case_inputs(case)
    boxes = case["boxes"]
    crops, feats, terms, loss = m.features(img, rec, boxes)
    c = case["crops"]
    assert tuple(crops.shape) == case["crops_shape"]
    assert rel_err(crops.reshape(-1)[c["idx"]], c["val"]) < 1e-5
    for f, halves in zip(feats, case["features"]):
        for h, r in zip(f.chunk(2), halves):
            assert rel_err(h.reshape(-1)[r["idx"]], r["val"]) < 1.5e-3
    assert rel_err(terms, torch.tensor(case["terms"])) < 1e-3 and float(loss) == pytest.approx(case["loss"], rel=1e-3)
    # the module's route: prepare once, 16 blocks, the five taps
    n = face_emu.names
    assert n.count("mas_face_prepare") == 1 and n.count("mas_face_stem_forward") == 1 and n.count("mas_face_l1_forward") == 5
    assert n.count("mas_face_subsample_half") == 3 and n.count("mas_gemm_rows_f16") == 16 * 2 + 4

    del face_emu.names[:]
    r = rec.clone().requires_grad_(True)
    out = m(img, r, boxes)
    if case["n"] >= 6:                             # only gt crops run: nothing depends on rec (the reference's d rec is 0)
        assert not out.requires_grad and float(out) == float(loss) and case["drec"]["norm"] == 0
        return
    (d1,) = torch.autograd.grad(out, r, retain_graph=True)
    names_first = list(face_emu.names)
    out.backward()
    assert torch.equal(r.grad, d1)                                           # second traversal: same gradient
    assert face_emu.names[len(names_first):] == ["mas_lpips_scale_jacobian"]  # ... from the kept unit-seed gradient
    assert names_first.count("mas_face_relu_seed_backward") == 16 and names_first.count("mas_face_pool_backward") == 1
    # only the rec-side crops ran backward: the span starts after the gt crops of the pairing
    assert names_first.count("mas_face_prepare_backward") == 1
    _, g_ref = _pinned_reference(ref, img, rec, boxes, feats, False)
    assert rel_err(d1, g_ref) < 3e-3
    d = case["drec"]
    assert abs(float(d1.norm()) - d["norm"]) <= 2e-2 * d["norm"]


def test_both_inputs_and_span_against_restatement(face_emu, golden):
    """case b with img and rec both wanted: every crop runs backward and both gradients match the pinned restatement; the
    rec gradient equals the one of the rec-only span."""
    case = golden["b"]
    m, _ = seeded_face_loss(case)
    ref = copy.deepcopy(m)
    img, rec = case_inputs(case)
    boxes = case["boxes"]
    _, feats, _, _ = m.features(img, rec, boxes)
    i, r = img.clone().requires_grad_(True), rec.clone().requires_grad_(True)
    m(i, r, boxes).backward()
    gi, gr = _pinned_reference(ref, img, rec, boxes, feats, True)
    assert rel_err(i.grad, gi) < 3e-3 and rel_err(r.grad, gr) < 3e-3
    r2 = rec.clone().requires_grad_(True)
    m(img, r2, boxes).backward()
    assert rel_err(r2.grad, r.grad) < 1e-6


def test_prepare_faces_returns_all_stacked_crops(face_emu, golden):
    from face_common import prepare
    case = golden["c"]
    m, _ = seeded_face_loss(case)
    img, rec = case_inputs(case)
    x = m.prepare_faces(img, rec, case["boxes"])
    assert tuple(x.shape) == (14, 3, 254, 254)
    crops = [[], []]
    for side, src in enumerate((img, rec)):
        for b, bb in enumerate(case["boxes"]):
            for box in bb:
                crops[side].append(prepare(src[b:b + 1].double(), src[b:b + 1].double(), [[box]])[0])
    assert rel_err(x, torch.stack(crops[0] + crops[1])) < 1e-6
    assert m.prepare_faces(img, rec, [[], []]) is None
