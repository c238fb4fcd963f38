"""Object-aware loss (losses/object_loss.py) on the H100: every mas_object_* entry against fp64 on the same operands (odd
extents, boxes crossing the image edge, overlapping boxes), the per-box LPIPS of the canvases against LPIPS of each crop alone,
and the module against the per-box loop of the real reference (tests/golden/object_loss.pt) and against fp64 autograd."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from lpips_common import reference_lpips
from object_common import case_images, case_module, crop, load_golden, restated_loop

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SHIFT = torch.tensor([-.030, -.088, -.188]).view(1, 3, 1, 1)
SCALE = torch.tensor([.458, .448, .450]).view(1, 3, 1, 1)


@pytest.fixture(scope="module")
def mods():
    if not torch.cuda.is_available():
        pytest.skip("needs cuda:0")
    from mas_b200 import _lib, ops
    _lib.load()
    return _lib, ops


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def _cl(t):
    return t.to(DEV).contiguous(memory_format=torch.channels_last)


# boxes [x0, y0, x1, y1]: odd extents, both edges crossed, two overlapping boxes in image 0; all in one 32 x 32 class
BOXES = [[[3, 5, 26, 22], [-7, 9, 14, 36], [10, 14, 33, 31]], [[20, 19, 47, 36], [0, 0, 17, 29]]]
H = W = 40


def _plan(ops, boxes=BOXES, B=2):
    plan = ops.ObjectPlan((B, 3, H, W), (B, 3, H, W), boxes)
    assert len(plan.classes) == 1
    hc, wc, rows, off = plan.classes[0]
    tab, wts = plan.device_tables(DEV)
    return plan, (hc, wc), len(rows), tab[off:], wts


def _extents(plan, level):
    return [(h >> level, w >> level) for _, _, _, h, w in plan.boxes]


# ------------------------------------------------------------------------------------------------ kernels
def test_gather_fp64(mods):
    L, ops = mods
    g = torch.Generator().manual_seed(1)
    img, rec = torch.rand(2, 3, H, W, generator=g) * 2 - 1, torch.rand(2, 3, H, W, generator=g) * 2 - 1
    plan, (hc, wc), K, t, _ = _plan(ops)
    x = ops.empty_nhwc(2 * K, 3, hc, wc, img.to(DEV))
    L.call("mas_object_gather", t, K, img.to(DEV), rec.to(DEV), SHIFT.to(DEV), SCALE.to(DEV), x, H, W, hc, wc)
    want = torch.zeros(2 * K, 3, hc, wc, dtype=torch.float64)
    for side, src in enumerate((img, rec)):
        for r, (b, y0, x0, h, w) in enumerate(plan.boxes):
            c = crop(src[b].double(), y0, x0, h, w)
            want[side * K + r, :, :h, :w] = (c - SHIFT[0].double()) / SCALE[0].double()
    assert rel_err(x.cpu(), want) < 1e-7


def test_relu_maxpool_fp64(mods):
    L, ops = mods
    g = torch.Generator().manual_seed(2)
    plan, (hc, wc), K, t, _ = _plan(ops)
    for level in (0, 1, 2):
        hh, ww = hc >> level, wc >> level
        y0 = torch.randn(2 * K, 64, hh, ww, generator=g)
        y = _cl(y0)
        am = torch.empty(1, device=DEV)
        L.call("mas_object_relu", y, t, K, hh, ww, 64, level, am)
        want = torch.zeros_like(y0)
        for n in range(2 * K):
            h, w = _extents(plan, level)[n % K]
            want[n, :, :h, :w] = torch.relu(y0[n, :, :h, :w])
        assert torch.equal(y.cpu(), want) and float(am) == float(want.max())
        x0 = torch.randint(-2, 3, (2 * K, 32, hh, ww), generator=g).float()      # ties
        p = ops.empty_nhwc(2 * K, 32, hh // 2, ww // 2, x0.to(DEV))
        L.call("mas_object_maxpool", _cl(x0), p, t, K, hh, ww, 32, level, am)
        want = torch.zeros(2 * K, 32, hh // 2, ww // 2)
        for n in range(2 * K):
            h, w = _extents(plan, level + 1)[n % K]
            want[n, :, :h, :w] = F.max_pool2d(x0[n:n + 1], 2, 2)[0, :, :h, :w]
        assert torch.equal(p.cpu(), want) and float(am) == float(want.abs().max())


def _taps(g, plan, K, C, hh, ww, level):
    """Masked tap [2K, C, hh, ww]: ReLU values inside each canvas's extent, zero outside, with zero-norm pixels."""
    t = torch.relu(torch.randn(2 * K, C, hh, ww, generator=g))
    for n in range(2 * K):
        h, w = _extents(plan, level)[n % K]
        t[n, :, h:] = 0
        t[n, :, :, w:] = 0
    t[K, :, 0, 1] = 0
    t[0, :, 1, 0] = 0
    return t


def _head_fp64(tap, wl, plan, K, level, r):
    h, w = _extents(plan, level)[r]
    a, b = tap[r, :, :h, :w].double(), tap[K + r, :, :h, :w].double()
    na = a / (torch.sqrt((a ** 2).sum(0, keepdim=True)) + 1e-10)
    nb = b / (torch.sqrt((b ** 2).sum(0, keepdim=True)) + 1e-10)
    return (((na - nb) ** 2) * wl.double().view(-1, 1, 1)).sum(0).mean()


def test_head_forward_and_finalize_fp64(mods):
    L, ops = mods
    g = torch.Generator().manual_seed(3)
    plan, (hc, wc), K, t, _ = _plan(ops)
    nblk = int(L.query("mas_lpips_head_blocks"))
    part = torch.empty((5, K, nblk), dtype=torch.float64, device=DEV)
    want = torch.zeros(K, dtype=torch.float64)
    for level, C in enumerate((64, 128, 256, 512, 512)):
        tap = _taps(g, plan, K, C, hc >> level, wc >> level, level)
        wl = torch.rand(C, generator=g)
        L.call("mas_object_head_forward", _cl(tap), wl.to(DEV), t, K, hc >> level, wc >> level, C, level, part[level])
        for r in range(K):
            want[r] += _head_fp64(tap, wl, plan, K, level, r)
    p = torch.full((K + 2,), -1.0, device=DEV)
    L.call("mas_object_head_finalize", part, t, K, p[1:])
    assert rel_err(p[1:K + 1].cpu(), want) < 1e-6 and float(p[0]) == -1 and float(p[-1]) == -1


@pytest.mark.parametrize("level,C,g0,G,pool", [(0, 64, 0, 10, True), (1, 128, 5, 5, True), (3, 512, 0, 5, True),
                                               (4, 512, 5, 5, False)])
def test_tap_backward_fp64(mods, level, C, g0, G, pool):
    L, ops = mods
    g = torch.Generator().manual_seed(10 + level)
    plan, (hc, wc), K, t, _ = _plan(ops)
    hh, ww = hc >> level, wc >> level
    tap = _taps(g, plan, K, C, hh, ww, level)
    tap = torch.where(tap > 0, (tap * 2).round() / 2, tap)                 # ties in the pool windows
    wl = torch.rand(C, generator=g)
    dpool = torch.randn(G, C, hh // 2, ww // 2, generator=g) if pool else None
    want = torch.zeros(G, C, hh, ww, dtype=torch.float64)
    for gi in range(G):
        n = g0 + gi
        r = n % K
        h, w = _extents(plan, level)[r]
        x = tap.double().requires_grad_(True)
        s = _head_fp64(x, wl, plan, K, level, r)
        if pool:
            ph, pw = h // 2, w // 2
            s = s + (F.max_pool2d(x[n:n + 1, :, :2 * ph, :2 * pw], 2, 2) * dpool[gi:gi + 1, :, :ph, :pw].double()).sum()
        (gx,) = torch.autograd.grad(s, x)
        want[gi] = torch.where(tap[n] > 0, gx[n], torch.zeros_like(gx[n]))
    dz = ops.empty_nhwc(G, C, hh, ww, tap.to(DEV))
    am = torch.empty(1, device=DEV)
    L.call("mas_object_tap_backward", _cl(tap), wl.to(DEV), t, K, hh, ww, C, level, g0, G, _cl(dpool) if pool else None, dz, am)
    got = dz.cpu().double()
    assert torch.isfinite(got).all() and rel_err(got, want) < 1e-5
    assert float(am) == float(got.abs().max())


@pytest.mark.parametrize("g0,G,side", [(0, 10, 0), (0, 10, 1), (5, 5, 1), (0, 5, 0)])
def test_scatter_fp64_with_overlaps(mods, g0, G, side):
    L, ops = mods
    g = torch.Generator().manual_seed(20 + g0 + side)
    plan, (hc, wc), K, t, wts = _plan(ops)
    dxp = torch.randn(G, 3, hc, wc, generator=g)
    want = torch.zeros(2, 3, H, W, dtype=torch.float64)
    for r, (b, y0, x0, h, w) in enumerate(plan.boxes):
        full = torch.zeros(3, H + 2 * hc, W + 2 * wc, dtype=torch.float64)
        full[:, hc + y0:hc + y0 + h, wc + x0:wc + x0 + w] = dxp[side * K + r - g0, :, :h, :w].double() / SCALE[0].double()
        want[b] += plan.w[r] * full[:, hc:hc + H, wc:wc + W]
    J = torch.full((2, 3, H, W), 0.25, device=DEV)
    L.call("mas_object_scatter", _cl(dxp), SCALE.to(DEV), t, wts, K, g0, G, side, hc, wc, J, 2, H, W, 0)
    assert rel_err(J.cpu(), want) < 1e-6
    L.call("mas_object_scatter", _cl(dxp), SCALE.to(DEV), t, wts, K, g0, G, side, hc, wc, J, 2, H, W, 1)
    assert rel_err(J.cpu(), 2 * want) < 1e-6


def test_loss_finalize(mods):
    L, ops = mods
    p = torch.rand(7, generator=torch.Generator().manual_seed(4))
    w = torch.tensor([1 / 3, 1 / 3, 0.5, 0.25, 0.25, 0.25, 1.0])
    out = torch.empty((), device=DEV)
    L.call("mas_object_loss", p.to(DEV), w.to(DEV), 7, out)
    assert float(out) == float(torch.tensor(float((p.double() * w.double()).sum())))


# ------------------------------------------------------------------------------------------------ module
def test_per_box_against_crop_alone_and_fp64(mods, golden):
    """p of every box from the canvases against losses.lpips.LPIPS on the crop alone and against fp64 LPIPS of the crop."""
    case = golden["a"]
    m, lp = case_module(case)
    lp.to(DEV)
    img, rec = case_images(case)
    p, plan = m.per_box(img.to(DEV), rec.to(DEV), case["boxes"])
    alone, p64, pst = [], [], []
    lp64 = lp.cpu()
    for b, y0, x0, h, w in plan.boxes:
        ci, cr = crop(img[b], y0, x0, h, w)[None], crop(rec[b], y0, x0, h, w)[None]
        p64.append(float(reference_lpips(lp64, ci, cr)))
    lp.to(DEV)
    with torch.no_grad():
        for b, y0, x0, h, w in plan.boxes:
            ci, cr = crop(img[b], y0, x0, h, w)[None].to(DEV), crop(rec[b], y0, x0, h, w)[None].to(DEV)
            alone.append(float(lp(ci, cr)))
            pst.append(float(reference_lpips(lp, ci, cr, dtype=torch.float32)))
    p64, alone, pst = torch.tensor(p64, dtype=torch.float64), torch.tensor(alone), torch.tensor(pst)
    e_ours, e_alone, e_stock = rel_err(p.cpu(), p64), rel_err(alone, p64), rel_err(pst, p64)
    print("per-box p rel err: canvases %.3e, LPIPS per crop %.3e, stock %.3e; canvases vs per crop %.3e"
          % (e_ours, e_alone, e_stock, rel_err(p.cpu(), alone)))
    assert e_ours <= 2 * max(e_alone, e_stock) + 1e-4
    assert rel_err(p.cpu(), alone) < 1e-3
    assert rel_err(p.cpu(), case["p"]) < 1e-3


@pytest.mark.parametrize("name", ["a", "b"])
def test_module_against_golden(mods, golden, name):
    from mas_b200 import _lib
    case = golden[name]
    m, lp = case_module(case)
    lp.to(DEV)
    img, rec = case_images(case)
    img = img.to(DEV)
    r = rec.to(DEV).requires_grad_(True)
    loss = m(img, r, case["boxes"])
    assert loss.dim() == 0 and loss.dtype == torch.float32
    p, _ = m.per_box(img, r.detach(), case["boxes"])
    l0 = _lib.launch_count()
    (d1,) = torch.autograd.grad(loss, r, retain_graph=True)
    l1 = _lib.launch_count()
    loss.backward()
    l2 = _lib.launch_count()
    d = case["drec"]
    eg = rel_err(d1.cpu(), d["full"]) if "full" in d else rel_err(d1.detach().reshape(-1)[d["idx"].to(DEV)].cpu(), d["val"])
    print("%s: loss %.6e golden %.6e; p rel err %.3e; d rec rel err %.3e, norm %.6e golden %.6e"
          % (name, float(loss), case["loss"], rel_err(p.cpu(), case["p"]), eg, float(d1.norm()), d["norm"]))
    assert float(loss.detach()) == pytest.approx(case["loss"], rel=1e-3)
    assert rel_err(p.cpu(), case["p"]) < 1e-3
    assert eg < 2e-2 and abs(float(d1.norm()) - d["norm"]) <= 1e-2 * d["norm"]
    # the retained graph's second traversal is one scaling kernel and gives the same gradient bit for bit
    assert l2 - l1 == 1 and l1 - l0 > 13 and torch.equal(d1, r.grad)


def test_gradients_against_fp64_loop_with_overlaps(mods, golden):
    """img and rec both requiring grad, overlapping and edge-crossing boxes: against fp64 autograd of the restated loop."""
    case = golden["a"]
    m, lp = case_module(case)
    img, rec = case_images(case)
    i64, r64 = img.double().requires_grad_(True), rec.double().requires_grad_(True)
    l64, _ = restated_loop(lp, i64, r64, case["kept"])
    l64.backward()
    lp.to(DEV)
    i, r = img.to(DEV).requires_grad_(True), rec.to(DEV).requires_grad_(True)
    loss = m(i, r, case["boxes"])
    loss.backward()
    ei, er = rel_err(i.grad.cpu(), i64.grad), rel_err(r.grad.cpu(), r64.grad)
    print("fp64 loop: loss rel err %.3e, d img %.3e, d rec %.3e" % (abs(float(loss.detach()) / float(l64) - 1), ei, er))
    assert float(loss.detach()) == pytest.approx(float(l64), rel=1e-3)
    assert ei < 2e-2 and er < 2e-2


def test_deterministic_no_grad_and_double_backward(mods, golden):
    case = golden["b"]
    m, lp = case_module(case)
    lp.to(DEV)
    img, rec = (t.to(DEV) for t in case_images(case))
    outs = []
    for _ in range(2):
        r = rec.clone().requires_grad_(True)
        loss = m(img, r, case["boxes"])
        loss.backward()
        outs.append((loss.detach(), r.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        z = m(img, rec.clone().requires_grad_(True), case["boxes"])
    torch.cuda.synchronize()
    assert not z.requires_grad and z.grad_fn is None
    assert torch.cuda.memory_allocated() - base < 1 << 20          # no activations kept
    assert float(z) == float(outs[0][0])
    r = rec.clone().requires_grad_(True)
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(m(img, r, case["boxes"]), r, create_graph=True)


def test_launches_depend_on_classes_not_boxes(mods, golden):
    from mas_b200 import _lib
    m, lp = case_module(golden["a"])
    lp.to(DEV)
    img, rec = (t.to(DEV) for t in case_images(golden["a"]))
    few = [[[0, 0, 40, 20], [10, 10, 100, 70]], []]                          # classes (32, 64) and (64, 128)
    many = [[[0, 0, 40, 20], [10, 10, 100, 70], [5, 9, 40, 28], [100, 120, 190, 180]],
            [[3, 3, 60, 24], [30, 40, 140, 100], [200, 200, 290, 245]]]
    m(img, rec.clone().requires_grad_(True), few).backward()                 # weight images packed once, outside the count
    counts = []
    for boxes in (few, many):
        assert len(m.per_box(img, rec, boxes)[1].classes) == 2
        r = rec.clone().requires_grad_(True)
        l0 = _lib.launch_count()
        m(img, r, boxes).backward()
        counts.append(_lib.launch_count() - l0)
    assert counts[0] == counts[1]
