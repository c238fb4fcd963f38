"""Object-aware loss (losses/object_loss.py) WITHOUT a GPU: the host plan (size classes, extents, weights, the 16-pixel drop
rule, refusals), and the module end to end above an emulation of the C-ABI entries' documented semantics (include/mas_b200.h)
that reads and writes the CPU tensors' memory, with the 3x3 convolutions of tests/test_host_logic_vq_cpu.py (real fp16
operand rounding), against the per-box loop of the real reference (tests/golden/object_loss.pt). The kernels are tested on
the GPU (tests/test_gpu_object_loss.py)."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import rel_err
from object_common import case_images, case_module, load_golden, restated_loop
from test_face_loss_host_logic_cpu import FaceEmu, _dense, _f64
from test_host_logic_vq_cpu import _addr, _f32

ROW = 6


def _i32(p, n):
    return np.ctypeslib.as_array((ctypes.c_int32 * int(n)).from_address(_addr(p)))


def _rows(tab, K):
    return _i32(tab, ROW * K).reshape(K, ROW).astype(np.int64)


# ------------------------------------------------------------------------------------------------ plan
def test_plan_classes_extents_weights_and_drop_rule():
    from mas_b200 import ops
    boxes = [[[0, 0, 16, 16], [10, 20, 110, 90], [5, 5, 15, 100], [3, 4, 20, 19.9]],
             torch.tensor([[-10, 30, 50, 100, 7.0], [0, 0, 256, 256, 1.0], [60, 50, 160, 170, 0.0]])]
    plan = ops.ObjectPlan((2, 3, 256, 256), (2, 3, 256, 256), boxes)
    # [5, 5, 15, 100] is 10 wide; [3, 4, 20, 19.9] reads y1 = int(19.9) = 19, 15 high: both dropped, not counted in n_b
    assert plan.dropped == [(0, [5, 5, 15, 100]), (0, [3, 4, 20, 19])]
    assert plan.n_img == [2, 3] and plan.K == 5
    assert plan.boxes == [(0, 0, 0, 16, 16), (0, 20, 10, 70, 100), (1, 30, -10, 70, 60), (1, 0, 0, 256, 256), (1, 50, 60, 120, 100)]
    assert plan.w == pytest.approx([1 / 3, 1 / 3, 1 / 4, 1 / 4, 1 / 4])
    # per side the next power of two, at least 16; classes in (Hc, Wc) order, crops in box order within a class
    assert [(hc, wc, rows) for hc, wc, rows, _ in plan.classes] == [(16, 16, [0]), (128, 64, [2]), (128, 128, [1, 4]),
                                                                     (256, 256, [3])]
    assert [ops.object_class_side(n) for n in (1, 15, 16, 17, 32, 33, 255, 256, 257)] == [16, 16, 16, 32, 32, 64, 256, 256, 512]
    tab = plan.tab.numpy()
    for hc, wc, rows, off in plan.classes:
        K = len(rows)
        t = tab[off:off + ROW * K].reshape(K, ROW)
        assert [list(r) for r in t] == [list(plan.boxes[k]) + [k] for k in rows]
        offs = tab[off + ROW * K:off + ROW * K + 3]                    # per-image row ranges, B + 1 entries
        imgs = [plan.boxes[k][0] for k in rows]
        assert list(offs) == [0, imgs.count(0), K]
    w = tab[plan.w_off:plan.w_off + plan.K].view(np.float32)
    assert np.array_equal(w, np.asarray(plan.w, dtype=np.float32))


def test_plan_zip_truncation_and_refusals():
    from mas_b200 import ops
    plan = ops.ObjectPlan((2, 3, 64, 64), (3, 3, 64, 64), [[[0, 0, 20, 20]], [], [[0, 0, 30, 30]]])
    assert plan.K == 1 and plan.n_img == [1, 0]
    # row ranges cover the larger batch (the rec side's third image has no rows)
    off = plan.classes[0][3]
    assert list(plan.tab.numpy()[off + ROW:off + ROW + 4]) == [0, 1, 1, 1]
    for bad in ([[[10, 0, 10, 32]]], [[[0, 20, 32, 5]]]):
        with pytest.raises(ValueError, match="extent"):
            ops.ObjectPlan((1, 3, 64, 64), (1, 3, 64, 64), bad)
    empty = ops.ObjectPlan((2, 3, 64, 64), (2, 3, 64, 64), [[], [[0, 0, 8, 40]]])
    assert empty.K == 0 and empty.tab is None and empty.classes == []


def _no_calls(monkeypatch):
    from mas_b200 import ops

    def refuse(name, *a):
        raise AssertionError("C-ABI call %s" % name)
    monkeypatch.setattr(ops.L, "call", refuse)
    monkeypatch.setattr(ops.L, "query", refuse)


def test_no_boxes_gives_new_tensor_zero_without_a_call(monkeypatch):
    from lpips_common import build_lpips
    from losses.object_loss import ObjectLoss
    _no_calls(monkeypatch)
    m = ObjectLoss(build_lpips())
    img = torch.zeros(2, 3, 32, 32, dtype=torch.float64)
    for boxes in ([[], []], [[[0, 0, 10, 40]], [[1, 1, 12, 12]]], torch.zeros(2, 0, 4)):
        z = m(img, img.clone().requires_grad_(True), boxes)
        assert z.dim() == 0 and z.dtype == torch.float64 and float(z) == 0.0 and not z.requires_grad


def test_refusals_and_shared_weights(monkeypatch):
    from lpips_common import build_lpips
    from losses.object_loss import ObjectLoss
    lp = build_lpips()
    m = ObjectLoss(lp)
    assert m.scorer is lp and list(m.state_dict()) == []          # shared, not registered: no second copy of the weights
    x = torch.zeros(1, 3, 32, 32)
    box = [[[0, 0, 16, 16]]]
    lp.train()
    with pytest.raises(RuntimeError, match=r"\.eval\(\)"):
        m(x, x, box)
    lp.eval()
    lp.lin2.model[1].weight.requires_grad_(True)
    with pytest.raises(RuntimeError, match="no weight gradients"):
        m(x, x, box)
    lp.lin2.model[1].weight.requires_grad_(False)
    with pytest.raises(ValueError, match="extent"):
        m(x, x, [[[4, 4, 4, 20]]])
    with pytest.raises(RuntimeError, match="CUDA"):                # no kernels on the CPU: refused loudly
        m(x, x, box)


def test_double_backward_is_refused():
    from mas_b200 import ops

    class Ctx:
        needs_input_grad = (False, True)
        J = None
    with torch.enable_grad(), pytest.raises(RuntimeError, match="double backward"):
        ops.ObjectLossFn.backward(Ctx(), torch.ones(()))


# ------------------------------------------------------------------------------------------------ emulated entries
class ObjectEmu(FaceEmu):
    """FaceEmu (the 3x3 family, edge layers, ReLU backward, Jacobian scaling) plus the mas_object_* entries, in fp64."""

    @staticmethod
    def _ext(rows, r, level):
        return int(rows[r, 3]) >> level, int(rows[r, 4]) >> level

    def mas_object_gather(self, tab, K, img, rec, shift, scale, out, H, W, Hc, Wc):
        rows = _rows(tab, K)
        nb = int(rows[:, 0].max()) + 1
        sh, sc = _f32(shift, 3).astype(np.float64), _f32(scale, 3).astype(np.float64)
        o = _f32(out, 2 * K * Hc * Wc * 3).reshape(2 * K, Hc, Wc, 3)
        o[...] = 0
        for side, src in enumerate((img, rec)):
            im = np.zeros((nb, 3, H + 2 * Hc, W + 2 * Wc))                  # the image inside a zero border
            im[:, :, Hc:Hc + H, Wc:Wc + W] = _f32(src, nb * 3 * H * W).reshape(nb, 3, H, W)
            for r in range(K):
                b, y0, x0, h, w, _ = rows[r]
                c = im[b, :, Hc + y0:Hc + y0 + h, Wc + x0:Wc + x0 + w].transpose(1, 2, 0)
                o[side * K + r, :h, :w] = (c - sh) / sc

    def mas_object_relu(self, y, tab, K, H, W, C, level, amax):
        rows = _rows(tab, K)
        v = _f32(y, 2 * K * H * W * C).reshape(2 * K, H, W, C)
        o = np.zeros_like(v)
        for n in range(2 * K):
            h, w = self._ext(rows, n % K, level)
            o[n, :h, :w] = np.maximum(v[n, :h, :w], 0)
        v[...] = o
        _f32(amax, 1)[0] = o.max()

    def mas_object_maxpool(self, x, y, tab, K, H, W, C, level, amax):
        rows = _rows(tab, K)
        X = _f32(x, 2 * K * H * W * C).reshape(2 * K, H, W, C)
        Y = _f32(y, 2 * K * (H // 2) * (W // 2) * C).reshape(2 * K, H // 2, W // 2, C)
        Y[...] = 0
        for n in range(2 * K):
            h, w = self._ext(rows, n % K, level + 1)
            Y[n, :h, :w] = X[n, :2 * h, :2 * w].reshape(h, 2, w, 2, C).max(axis=(1, 3))
        _f32(amax, 1)[0] = np.abs(Y).max()

    @staticmethod
    def _norm(t):
        return t / (np.sqrt((t * t).sum(-1, keepdims=True)) + 1e-10)

    def mas_object_head_forward(self, tap, wl, tab, K, H, W, C, level, part):
        rows = _rows(tab, K)
        T = _f32(tap, 2 * K * H * W * C).reshape(2 * K, H, W, C).astype(np.float64)
        wv = _f32(wl, C).astype(np.float64)
        P = _f64(part, K * 128).reshape(K, 128)
        P[...] = 0
        for r in range(K):
            h, w = self._ext(rows, r, level)
            d = self._norm(T[r, :h, :w]) - self._norm(T[K + r, :h, :w])
            P[r, 0] = (d * d * wv).sum()

    def mas_object_head_finalize(self, part, tab, K, p):
        rows = _rows(tab, K)
        P = _f64(part, 5 * K * 128).reshape(5, K, 128)
        out = _f32(p, int(rows[:, 5].max()) + 1)
        for r in range(K):
            out[rows[r, 5]] = sum(P[l, r].sum() / np.prod(self._ext(rows, r, l)) for l in range(5))

    def mas_object_tap_backward(self, tap, wl, tab, K, H, W, C, level, g0, G, dpool, dz, amax):
        rows = _rows(tab, K)
        T = torch.from_numpy(_f32(tap, 2 * K * H * W * C).reshape(2 * K, H, W, C).astype(np.float64))
        wv = torch.from_numpy(_f32(wl, C).astype(np.float64))
        out = np.zeros((G, H, W, C))
        for gi in range(G):
            t = g0 + gi
            o = (t + K) % (2 * K)
            h, w = self._ext(rows, t % K, level)
            with torch.enable_grad():                       # the autograd engine runs backward under no_grad
                g = self._tap_grad(T[t, :h, :w], T[o, :h, :w], wv, h, w, dpool, G, H, W, C, gi)
            x = T[t, :h, :w]
            out[gi, :h, :w] = torch.where(x > 0, g, torch.zeros_like(g)).numpy()
        _f32(dz, G * H * W * C)[...] = out.reshape(-1)
        _f32(amax, 1)[0] = np.abs(out).max()

    @staticmethod
    def _tap_grad(x, y, wv, h, w, dpool, G, H, W, C, gi):
        """fp64 autograd of the crop's head term (a unit seed) plus the pooled gradient inside the next level's extent."""
        x = x.clone().requires_grad_(True)

        def n(v):
            return v / (torch.sqrt((v * v).sum(-1, keepdim=True)) + 1e-10)
        loss = ((n(x) - n(y)) ** 2 * wv).sum() / (h * w)
        if dpool is not None:
            ph, pw = h // 2, w // 2
            D = _f32(dpool, G * (H // 2) * (W // 2) * C).reshape(G, H // 2, W // 2, C)[gi, :ph, :pw]
            pooled = torch.nn.functional.max_pool2d(x[:2 * ph, :2 * pw].permute(2, 0, 1)[None], 2)[0].permute(1, 2, 0)
            loss = loss + (pooled * torch.from_numpy(D.astype(np.float64))).sum()
        (g,) = torch.autograd.grad(loss, x)
        return torch.where(torch.isfinite(g), g, torch.zeros_like(g))   # a zero-norm pixel: masked by the ReLU select

    def mas_object_scatter(self, dxp, scale, tab, wts, K, g0, G, side, Hc, Wc, J, B, H, W, accumulate):
        rows = _rows(tab, K)
        offs = _i32(tab, ROW * K + B + 1)[ROW * K:]
        D = _f32(dxp, G * Hc * Wc * 3).reshape(G, Hc, Wc, 3).astype(np.float64) / _f32(scale, 3).astype(np.float64)
        wv = _f32(wts, int(rows[:, 5].max()) + 1)
        acc = np.zeros((B, 3, H + 2 * Hc, W + 2 * Wc))
        for b in range(B):
            for r in range(offs[b], offs[b + 1]):
                _, y0, x0, h, w, k = rows[r]
                acc[b, :, Hc + y0:Hc + y0 + h, Wc + x0:Wc + x0 + w] += wv[k] * D[side * K + r - g0, :h, :w].transpose(2, 0, 1)
        out = _f32(J, B * 3 * H * W).reshape(B, 3, H, W)
        s = acc[:, :, Hc:Hc + H, Wc:Wc + W]
        out[...] = out + s if accumulate else s

    def mas_object_loss(self, p, wts, K, out):
        _f32(out, 1)[0] = float((_f32(p, K).astype(np.float64) * _f32(wts, K)).sum())


@pytest.fixture
def obj_emu(monkeypatch):
    from mas_b200 import ops
    e = ObjectEmu()
    monkeypatch.setattr(ops.L, "call", e)

    def query(name, *a):
        if name == "mas_conv3x3_tc_eligible":        # dense NHWC, Cin % 8, Cout % 128, Hout % 16, Wout % 8, S1 / UP / ZS
            xs, ys, mode = a
            return int(_dense(xs) and _dense(ys) and xs.c % 8 == 0 and ys.c % 128 == 0 and ys.h % 16 == 0 and ys.w % 8 == 0
                       and mode in (0, 2, 3))
        if name == "mas_lpips_head_blocks":
            return 128
        raise AssertionError(name)
    monkeypatch.setattr(ops.L, "query", query)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: True)
    return e


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def test_module_72_against_golden_on_emulated_entries(obj_emu, golden):
    """Case b (three 72x72 images, one without boxes): per-box p, loss and d loss / d rec against the reference loop; the
    retained graph's second traversal is one scaling call; the class count, not the box count, sets the calls."""
    case = golden["b"]
    m, lp = case_module(case)
    img, rec = case_images(case)
    p, plan = m.per_box(img, rec, case["boxes"])
    assert plan.dropped == [] and len(plan.classes) == 3 and plan.K == 4
    assert rel_err(p, case["p"]) < 2e-3
    del obj_emu.names[:]
    r = rec.clone().requires_grad_(True)
    loss = m(img, r, case["boxes"])
    assert loss.dim() == 0 and loss.dtype == torch.float32
    assert float(loss.detach()) == pytest.approx(case["loss"], rel=2e-3)
    n = obj_emu.names
    assert n.count("mas_object_gather") == 3 and n.count("mas_object_head_finalize") == 3 and n.count("mas_object_loss") == 1
    (d1,) = torch.autograd.grad(loss, r, retain_graph=True)
    first = list(n)
    loss.backward()
    assert n[len(first):] == ["mas_lpips_scale_jacobian"] and torch.equal(r.grad, d1)
    assert first.count("mas_object_scatter") == 3 and first.count("mas_object_tap_backward") == 15
    assert rel_err(d1, case["drec"]["full"]) < 3e-2          # fp16 operands of the emulated tensor-core convolutions
    # against the fp64 loop itself (the image without boxes gets exactly zero)
    r64 = rec.double().requires_grad_(True)
    l64, p64 = restated_loop(lp, img.double(), r64, case["kept"])
    l64.backward()
    assert rel_err(p, p64) < 2e-3 and rel_err(d1, r64.grad) < 3e-2
    assert torch.count_nonzero(d1[1]) == 0


def test_module_256_against_golden_on_emulated_entries(obj_emu, golden):
    """Case a: mixed sizes, the whole image, edge-crossing and overlapping boxes, one box dropped; img and rec gradients."""
    case = golden["a"]
    m, _ = case_module(case)
    img, rec = case_images(case)
    i, r = img.clone().requires_grad_(True), rec.clone().requires_grad_(True)
    loss = m(i, r, case["boxes"])
    assert float(loss.detach()) == pytest.approx(case["loss"], rel=2e-3)
    loss.backward()
    d = case["drec"]
    assert abs(float(r.grad.norm()) - d["norm"]) <= 1e-2 * d["norm"]
    assert rel_err(r.grad.reshape(-1)[d["idx"]], d["val"]) < 2e-2
    assert i.grad is not None and float(i.grad.norm()) > 0
