"""VGGFace2 face loss on the H100 kernels (csrc/face.cu + the row GEMMs and 3x3 family): the new entries against fp64, the
module against the golden (tests/golden/face_loss.pt) and the fp64 restatement of tests/face_common.py, the gradient with the
L1 signs pinned, determinism and the autograd behaviours."""
import copy

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from face_common import case_inputs, load_golden, restated_loss, seeded_face_loss

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def _model(case):
    m, _ = seeded_face_loss(case)
    return m.to(DEV)


def _cl(t):
    return t.to(DEV).contiguous(memory_format=torch.channels_last)


# ------------------------------------------------------------------------------------------------ entries against fp64
@pytest.mark.parametrize("size,boxes", [
    (128, [[[10, 5, 60, 75], [-20, 90, 40, 150]]]),     # upsampled; a box crossing two edges (zero fill)
    (640, [[[20, 30, 420, 330], [100, 200, 356, 600]]]),  # downsampled (short side 300), identity (short side 256)
])
def test_prepare_and_adjoint(size, boxes):
    from face_common import prepare
    from mas_b200 import _lib as L, ops
    g = torch.Generator().manual_seed(size)
    img = torch.rand(1, 3, size, size, generator=g) * 2 - 1
    rec = torch.rand(1, 3, size, size, generator=g) * 2 - 1
    plan = ops.FacePlan(img.shape, rec.shape, boxes)
    tab, wts = plan.tab.to(DEV), plan.wts.to(DEV)
    imgs = img.to(DEV).permute(0, 1, 3, 2)       # any strides: a transposed view
    recd = rec.to(DEV)
    x = ops.empty_nhwc(plan.F, 3, 254, 254, recd)
    L.call("mas_face_prepare", tab, wts, plan.F, imgs, L.t4(imgs), recd, L.t4(recd), x)
    ref = prepare(img.double().transpose(2, 3), rec.double(), boxes)
    assert rel_err(x.cpu(), ref) < 1e-6
    # adjoint: <A u, v> = <u, A^T v> per side
    v = torch.randn(plan.F, 3, 254, 254, generator=g).to(DEV).contiguous(memory_format=torch.channels_last)
    for side, src in ((0, imgs), (1, recd)):
        J = torch.empty(1, 3, src.shape[2], src.shape[3], device=DEV)
        L.call("mas_face_prepare_backward", tab, wts, 0, plan.F, side, v, J, 1, src.shape[2], src.shape[3])
        keep = torch.tensor([f[0] == side for f in plan.faces], device=DEV).view(-1, 1, 1, 1)
        ax = x.double() * keep
        lhs = float((ax * v.double()).sum())
        rhs = float((src.double() * J.double()).sum())
        assert abs(lhs - rhs) <= 1e-6 * float(ax.norm() * (v.double() * keep).norm())   # relative to the Cauchy-Schwarz bound


def test_stem_forward_and_data_gradient():
    from mas_b200 import _lib as L, ops
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 3, 254, 254, generator=g)
    w = torch.randn(64, 3, 7, 7, generator=g) / 147 ** 0.5
    xd = _cl(x)
    y = ops.empty_nhwc(2, 64, 127, 127, xd)
    L.call("mas_face_stem_forward", xd, w.to(DEV).contiguous(), y, 2, 254, 254)
    xr = x.double().requires_grad_(True)
    yr = F.conv2d(xr, w.double(), stride=2, padding=3)
    assert rel_err(y.cpu(), yr) < 1e-6
    dy = torch.randn(yr.shape, generator=g)
    yr.backward(dy.double())
    dx = ops.empty_nhwc(2, 3, 254, 254, xd)
    L.call("mas_face_stem_backward", _cl(dy), w.to(DEV).contiguous(), dx, 2, 254, 254)
    assert rel_err(dx.cpu(), xr.grad) < 1e-6


def test_pool_forward_backward_with_ties_and_seed():
    from mas_b200 import _lib as L, ops
    g = torch.Generator().manual_seed(4)
    N, C, H = 4, 64, 127
    x = torch.randint(-3, 4, (N, C, H, H), generator=g).float() * 0.5     # many ties, many non-positive values
    bn = torch.stack([1.0 + 0.1 * torch.rand(C, generator=g), 0.1 * torch.randn(C, generator=g)])
    xd = _cl(x)
    y = ops.empty_nhwc(N, C, 63, 63, xd)
    arg = torch.empty((N, 63, 63, C), dtype=torch.uint8, device=DEV)
    am = torch.empty(1, device=DEV)
    L.call("mas_face_pool_forward", xd, bn.to(DEV), y, arg, N, H, H, C, am)
    xr = x.double().requires_grad_(True)
    z = xr * bn[0].double().view(1, -1, 1, 1) + bn[1].double().view(1, -1, 1, 1)
    yr = F.max_pool2d(F.relu(z), 3, 2, 0, ceil_mode=True)
    assert rel_err(y.cpu(), yr) < 1e-6 and float(am) == pytest.approx(float(yr.max()), rel=1e-6)
    dp = torch.randn(yr.shape, generator=g)
    sgn = torch.randint(-1, 2, (N // 2, H, H, C), generator=g, dtype=torch.int8)
    coef = 0.37
    yr.backward(dp.double())
    # faces 1 .. 3 of the pair layout P = 2: seeds +coef * sgn[1], -coef * sgn[0], -coef * sgn[1]
    g0, G = 1, 3
    dx = ops.empty_nhwc(G, C, H, H, xd)
    L.call("mas_face_pool_backward", xd[g0:], bn.to(DEV), arg[g0:], _cl(dp)[g0:], sgn.to(DEV), coef, g0, 2, G, H, H, C, dx)
    s = sgn.permute(0, 3, 1, 2).double() * coef
    seed = torch.stack([s[1], -s[0], -s[1]])
    assert rel_err(dx.cpu(), xr.grad[g0:] + seed) < 1e-6


def test_l1_partials_terms_and_relu_seed():
    from mas_b200 import _lib as L, ops
    g = torch.Generator().manual_seed(5)
    feats = [torch.randn(4, c, h, h, generator=g) for c, h in ((64, 127), (256, 63), (512, 32), (1024, 16), (2048, 8))]
    feats[1][2:] = feats[1][:2]         # a level with a = b everywhere: sign 0
    nb = int(L.load().mas_face_l1_blocks())
    part = torch.empty((5, nb), dtype=torch.float64, device=DEV)
    alphas = [0.1, 0.0025, 0.025, 0.05, 0.005]
    signs = []
    for l, f in enumerate(feats):
        n = 2 * f[0].numel()
        sg = torch.empty(n, dtype=torch.int8, device=DEV)
        L.call("mas_face_l1_forward", _cl(f), n, sg, part[l])
        signs.append(sg)
        a, b = f[:2].permute(0, 2, 3, 1).double(), f[2:].permute(0, 2, 3, 1).double()
        assert torch.equal(sg.cpu().view(a.shape), torch.sign(a - b).to(torch.int8))
    terms = torch.empty(5, device=DEV)
    loss = torch.empty((), device=DEV)
    coef = [a / f[0].numel() for a, f in zip(alphas, feats)]
    L.call("mas_face_l1_finalize", part, *coef, terms, loss)
    ref = [a * (f[:2].double() - f[2:].double()).abs().sum(0).mean() for a, f in zip(alphas, feats)]
    assert rel_err(terms.cpu(), torch.stack(ref)) < 1e-6 and float(loss) == pytest.approx(float(sum(ref)), rel=1e-6)
    # block-output ReLU backward with the seed and a stride-2 consumer's gradient
    out = torch.relu(feats[2][1:])
    dh = torch.randn(3, 512, 16, 16, generator=g)
    dz = ops.empty_nhwc(3, 512, 32, 32, _cl(out))
    am = torch.empty(1, device=DEV)
    L.call("mas_face_relu_seed_backward", _cl(out), _cl(dh), 1, signs[2], coef[2], 1, 2, 3, 32, 32, 512, dz, am)
    full = torch.zeros(3, 512, 32, 32, dtype=torch.float64)
    full[:, :, ::2, ::2] = dh.double()
    s = signs[2].cpu().view(2, 32, 32, 512).permute(0, 3, 1, 2).double() * coef[2]
    want = torch.where(out > 0, full + torch.stack([s[1], -s[0], -s[1]]), torch.zeros_like(full))
    assert rel_err(dz.cpu(), want) < 1e-6 and float(am) == pytest.approx(float(want.abs().max()), rel=1e-6)


# ------------------------------------------------------------------------------------------------ the module
@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_module_against_golden_and_restatement(golden, name):
    case = golden[name]
    m = _model(case)
    img, rec = case_inputs(case)
    crops, feats, terms, loss = m.features(img.to(DEV), rec.to(DEV), case["boxes"])
    c = case["crops"]
    assert tuple(crops.shape) == case["crops_shape"]
    assert rel_err(crops.cpu().reshape(-1)[c["idx"]], c["val"]) < 1e-5
    mc = copy.deepcopy(m).cpu()
    ref_x, ref_f, ref_t, ref_l = restated_loss(mc, img.double(), rec.double(), case["boxes"])
    assert rel_err(crops.cpu(), ref_x) < 1e-6
    errs = [rel_err(f.cpu(), r) for f, r in zip(feats, ref_f)]
    print("feature rel err per level", ["%.2e" % e for e in errs])
    assert errs[0] < 1e-6 and max(errs) < 1.5e-3
    for f, halves in zip(feats, case["features"]):
        for h, r in zip(f.cpu().chunk(2), halves):
            assert rel_err(h.reshape(-1)[r["idx"]], r["val"]) < 1.5e-3
    assert float(loss) == pytest.approx(case["loss"], rel=1e-3)
    assert float(ref_l) == pytest.approx(case["loss"], rel=1e-5)
    assert rel_err(terms.cpu(), torch.stack(ref_t)) < 1e-3
    assert float(m(img.to(DEV), rec.to(DEV), case["boxes"])) == float(loss)


def _sign_pinned_check(case, m, img, rec):
    """Sign disagreements with fp64 only where |a - b| is within the level's forward error; then d rec against the
    restatement's gradient under OUR sign pattern."""
    boxes = case["boxes"]
    _, feats, _, _ = m.features(img.to(DEV), rec.to(DEV), boxes)
    mc = copy.deepcopy(m).cpu()
    ref_x, ref_f, _, _ = restated_loss(mc, img.double(), rec.double(), boxes)
    signs, flips, total = [], 0, 0
    for f, r in zip(feats, ref_f):
        a, b = f.cpu().double().chunk(2)
        ra, rb = r.chunk(2)
        s, s64 = torch.sign(a - b), torch.sign(ra - rb)
        err = float(((f.cpu().double() - r).pow(2).mean()).sqrt())     # the level's forward error (rms)
        bad = s != s64
        if bad.any():
            assert float((ra - rb)[bad].abs().max()) <= 20 * err
        print("level sign flips %d of %d (forward rms error %.2e)" % (int(bad.sum()), bad.numel(), err))
        flips += int(bad.sum())
        total += bad.numel()
        signs.append(s)
    # every flip is a near-tie (above); a ReLU output that is exactly 0 on one side and O(error) in fp64 is one
    assert flips < 2e-3 * total
    rg = rec.to(DEV).requires_grad_(True)
    loss = m(img.to(DEV), rg, boxes)
    loss.backward()
    rr = rec.double().requires_grad_(True)
    _, _, _, lr = restated_loss(mc, img.double(), rr, boxes, signs=signs)
    lr.backward()
    return rel_err(rg.grad.cpu(), rr.grad), flips, total


@pytest.mark.parametrize("name", ["a", "b"])
def test_gradient_with_signs_pinned(golden, name):
    case = golden[name]
    m = _model(case)
    img, rec = case_inputs(case)
    err, flips, total = _sign_pinned_check(case, m, img, rec)
    print("d rec rel err %.2e, sign flips %d of %d" % (err, flips, total))
    assert err < 3e-3


def test_determinism_retained_graph_and_gt_only(golden):
    case = golden["b"]
    m = _model(case)
    img, rec = case_inputs(case)
    res = []
    for _ in range(2):
        r = rec.to(DEV).requires_grad_(True)
        loss = m(img.to(DEV), r, case["boxes"])
        (d1,) = torch.autograd.grad(loss, r, retain_graph=True)
        loss.backward()
        assert torch.equal(d1, r.grad)
        res.append((loss.detach().clone(), d1))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    # both inputs wanted: the rec gradient is unchanged, img gets its own
    i2, r2 = img.to(DEV).requires_grad_(True), rec.to(DEV).requires_grad_(True)
    m(i2, r2, case["boxes"]).backward()
    assert torch.equal(r2.grad, res[0][1]) and i2.grad is not None and float(i2.grad.abs().sum()) > 0
    with pytest.raises(RuntimeError, match="create_graph"):
        r3 = rec.to(DEV).requires_grad_(True)
        torch.autograd.grad(m(img.to(DEV), r3, case["boxes"]), r3, create_graph=True)
    c = golden["c"]
    mc = _model(c)
    ic, rc = case_inputs(c)
    loss = mc(ic.to(DEV), rc.to(DEV).requires_grad_(True), c["boxes"])
    assert not loss.requires_grad and float(loss) == pytest.approx(c["loss"], rel=1e-3)
