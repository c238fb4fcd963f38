"""LPIPS (losses/lpips.py) on the H100: every csrc/lpips.cu kernel against fp64 on the same operands, and the drop-in module
through loss_img.py's call sequence (forward, autograd.grad(retain_graph=True), backward()) against the golden recorded
from the real reference (tests/golden/lpips.pt)."""
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, rel_err
from lpips_common import golden_tool, reference_lpips, seeded_lpips

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def mods():
    if not torch.cuda.is_available():
        pytest.skip("needs cuda:0")
    from mas_b200 import _lib, ops
    _lib.load()
    return _lib, ops


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "lpips.pt"), weights_only=False)


def _cl(t):
    return t.to(DEV).contiguous(memory_format=torch.channels_last)


# ------------------------------------------------------------------------------------------------ kernels
def test_prep_relu_maxpool_fp64(mods):
    L, ops = mods
    g = torch.Generator().manual_seed(5)
    B, H, W = 2, 18, 22
    real, fake = torch.rand(B, 3, H, W, generator=g) * 2 - 1, torch.rand(B, 3, H, W, generator=g) * 2 - 1
    shift = torch.tensor([-.030, -.088, -.188]).view(1, 3, 1, 1)
    scale = torch.tensor([.458, .448, .450]).view(1, 3, 1, 1)
    x = ops.empty_nhwc(2 * B, 3, H, W, real.to(DEV))
    L.call("mas_lpips_prep", real.to(DEV), fake.to(DEV), shift.to(DEV), scale.to(DEV), x, B, H, W)
    want = (torch.cat([real, fake]).double() - shift.double()) / scale.double()
    assert rel_err(x.cpu(), want) < 1e-7

    y0 = torch.randn(3, 64, 10, 12, generator=g)
    y = _cl(y0)
    am = torch.empty(1, device=DEV)
    L.call("mas_lpips_relu", y, y.numel(), am)
    assert torch.equal(y.cpu(), torch.relu(y0)) and float(am) == float(torch.relu(y0).max())

    # odd extents (floor mode) and many ties
    x0 = torch.randint(0, 3, (3, 32, 9, 7), generator=g).float()
    xp = _cl(x0)
    p = ops.empty_nhwc(3, 32, 4, 3, xp)
    L.call("mas_lpips_maxpool", xp, p, 3, 9, 7, 32, am)
    ref = F.max_pool2d(x0, 2, 2)
    assert torch.equal(p.cpu(), ref) and float(am) == float(ref.abs().max())


def _head_ref(tap, wl, B):
    t = tap.double()
    r, f = t[:B], t[B:]
    nr = r / (torch.sqrt((r ** 2).sum(1, keepdim=True)) + 1e-10)
    nf = f / (torch.sqrt((f ** 2).sum(1, keepdim=True)) + 1e-10)
    return F.conv2d((nr - nf) ** 2, wl.double()).mean([2, 3]).view(-1)


def _tap(g, B, C, H, W):
    t = torch.relu(torch.randn(2 * B, C, H, W, generator=g))
    t[B, :, 1, 2] = 0                                  # a zero-norm fake pixel
    t[0, :, 3, 3] = 0                                  # and a zero-norm real one
    return t


@pytest.mark.parametrize("C,H,W", [(64, 16, 16), (512, 9, 7)])
def test_head_forward_fp64(mods, C, H, W):
    L, ops = mods
    g = torch.Generator().manual_seed(C + H)
    B = 3
    tap = _tap(g, B, C, H, W)
    wl = torch.rand(1, C, 1, 1, generator=g)
    nblk = int(L.load().mas_lpips_head_blocks())
    part = torch.empty((5, B, nblk), dtype=torch.float64, device=DEV)
    L.call("mas_lpips_head_forward", _cl(tap), wl.to(DEV), B, H, W, C, part[0])
    got = part[0].sum(1).cpu() / (H * W)
    assert rel_err(got, _head_ref(tap, wl, B)) < 1e-6


@pytest.mark.parametrize("C,H,W,g0,G,pool", [(64, 16, 16, 3, 3, True), (256, 9, 7, 0, 6, True), (512, 4, 4, 3, 3, False)])
def test_tap_backward_fp64(mods, C, H, W, g0, G, pool):
    """Head gradient + max-pool gradient at the first maximum + ReLU select, against fp64 autograd."""
    L, ops = mods
    g = torch.Generator().manual_seed(C + W)
    B = 3
    tap = _tap(g, B, C, H, W)
    tap[g0:g0 + G, :, :2 * (H // 2), :2 * (W // 2)] = torch.relu(tap[g0:g0 + G, :, :2 * (H // 2), :2 * (W // 2)].round())  # ties
    wl = torch.rand(1, C, 1, 1, generator=g)
    dpool = torch.randn(G, C, H // 2, W // 2, generator=g) if pool else None
    # fp64: a unit seed on every p_b, gradient of the selected images' (pre-ReLU) tap
    t = tap.double().requires_grad_(True)
    p = _head_ref(t, wl, B).sum()
    if pool:
        p = p + (F.max_pool2d(t[g0:g0 + G], 2, 2) * dpool.double()).sum()
    (gt,) = torch.autograd.grad(p, t)
    sel = tap[g0:g0 + G].double()
    want = torch.where(sel > 0, gt[g0:g0 + G], torch.zeros_like(sel))
    dz = ops.empty_nhwc(G, C, H, W, tap.to(DEV))
    am = torch.empty(1, device=DEV)
    L.call("mas_lpips_tap_backward", _cl(tap), wl.to(DEV), B, H, W, C, g0, G, _cl(dpool) if pool else None, dz, am)
    got = dz.cpu().double()
    assert torch.isfinite(got).all()
    assert rel_err(got, want) < 1e-5
    assert float(am) == float(got.abs().max())


def test_tap_backward_pool_ties_go_to_first_maximum(mods):
    L, ops = mods
    B, C, H, W = 1, 32, 4, 6
    tap = torch.full((2 * B, C, H, W), 2.0)
    tap[:, :, 0, 0] = 1.0                 # window (0, 0): maxima at (0, 1), (1, 0), (1, 1) -> (0, 1)
    tap[:, :, 1, 3] = 3.0                 # window (0, 1): single maximum at (1, 3)
    dpool = torch.randn(B, C, H // 2, W // 2, generator=torch.Generator().manual_seed(0))
    want = torch.zeros(B, C, H, W)
    for i in range(H // 2):
        for j in range(W // 2):
            win = tap[B, :, 2 * i:2 * i + 2, 2 * j:2 * j + 2].reshape(C, 4)
            k = int(win[0].argmax())      # first maximum in row-major order
            want[0, :, 2 * i + k // 2, 2 * j + k % 2] = dpool[0, :, i, j]
    dz = ops.empty_nhwc(B, C, H, W, tap.to(DEV))
    L.call("mas_lpips_tap_backward", _cl(tap), torch.zeros(C, device=DEV), B, H, W, C, B, B, _cl(dpool), dz, None)
    assert torch.equal(dz.cpu(), want)
    assert float(dz[0, 0, 0, 1]) == float(dpool[0, 0, 0, 0])


def test_relu_backward_prep_backward_scale(mods):
    L, ops = mods
    g = torch.Generator().manual_seed(9)
    y = torch.relu(torch.randn(2, 64, 6, 8, generator=g))
    dy = torch.randn(2, 64, 6, 8, generator=g)
    dyd = _cl(dy)
    am = torch.empty(1, device=DEV)
    L.call("mas_lpips_relu_backward", dyd, _cl(y), dyd, dy.numel(), am)
    want = torch.where(y > 0, dy, torch.zeros_like(dy))
    assert torch.equal(dyd.cpu(), want) and float(am) == float(want.abs().max())
    dxp = torch.randn(2, 3, 6, 8, generator=g)
    scale = torch.tensor([.458, .448, .450])
    J = torch.empty(2, 3, 6, 8, device=DEV)
    L.call("mas_lpips_prep_backward", _cl(dxp), scale.to(DEV), J, 2, 6, 8)
    assert rel_err(J.cpu(), dxp.double() / scale.double().view(1, 3, 1, 1)) < 1e-7
    gg = torch.tensor([0.5, -2.0], device=DEV).view(2, 1, 1, 1)
    out = torch.empty_like(J)
    L.call("mas_lpips_scale_jacobian", J, gg, gg.stride(0), out, 2, 3 * 6 * 8)
    assert torch.equal(out.cpu(), (J * gg).cpu())


# ------------------------------------------------------------------------------------------------ module
def _run(m, case, want_real=False):
    from mas_b200 import _lib
    real, fake = golden_tool.images(case["seed"], case["size"], case["batch"])
    real = real.to(DEV).requires_grad_(want_real)
    rec = fake.to(DEV).requires_grad_(True)
    p = m(real, rec)
    coef = torch.tensor(case["coef"], device=DEV)
    loss = (p.view(-1) * coef).sum()
    l0 = _lib.launch_count()
    grads = torch.autograd.grad(loss, [rec, real] if want_real else [rec], retain_graph=True)
    l1 = _lib.launch_count()
    loss.backward()
    l2 = _lib.launch_count()
    torch.cuda.synchronize()
    return p, grads, rec.grad, real.grad, (l1 - l0, l2 - l1)


def _cmp_grad(got, rec):
    if "full" in rec:
        return rel_err(got.cpu(), rec["full"])
    return rel_err(got.detach().reshape(-1)[rec["idx"].to(DEV)].cpu(), rec["val"])


def test_module_72_matches_reference(mods, golden):
    case = golden["72"]
    m, _ = seeded_lpips(case)
    m.to(DEV)
    p, (d1,), d2, _, (n1, n2) = _run(m, case)
    assert p.shape == (2, 1, 1, 1) and p.dtype == torch.float32 and p.is_contiguous()
    print("72: p", p.view(-1).tolist(), "golden", case["p"].view(-1).tolist())
    assert rel_err(p.cpu(), case["p"]) < 1e-4
    assert _cmp_grad(d1, case["dfake_grad"]) < 1e-4
    assert _cmp_grad(d2, case["dfake_backward"]) < 1e-4
    # zero-norm relu5_3 pixels (dead share > 0 in the fixture) leave the gradient finite
    assert min(case["dead_relu5_3"]["fake"]) > 0 and torch.isfinite(d1).all()
    # the second traversal is one scaling kernel, and gives the first one's result bit for bit
    assert n2 == 1 and n1 > 13 and torch.equal(d1, d2)


def test_module_72_real_gradient_too(mods, golden):
    case = golden["72"]
    m, _ = seeded_lpips(case)
    m.to(DEV)
    real, fake = golden_tool.images(case["seed"], case["size"], case["batch"])
    coef = torch.tensor(case["coef"], dtype=torch.float64)
    r64, f64 = real.double().requires_grad_(True), fake.double().requires_grad_(True)
    m64 = m.cpu()
    (reference_lpips(m64, r64, f64).view(-1) * coef).sum().backward()
    m.to(DEV)
    _, (df, dr), _, _, _ = _run(m, case, want_real=True)
    assert rel_err(dr.cpu(), r64.grad) < 1e-4 and rel_err(df.cpu(), f64.grad) < 1e-4


def test_module_256_within_stock_deviation(mods, golden):
    case = golden["256"]
    m, _ = seeded_lpips(case)
    m.to(DEV)
    p, (d1,), d2, _, _ = _run(m, case)
    # stock: the same computation in torch ops on the GPU (cuDNN, PyTorch's default TF32 convolutions)
    real, fake = golden_tool.images(case["seed"], case["size"], case["batch"])
    rec = fake.to(DEV).requires_grad_(True)
    ps = reference_lpips(m, real.to(DEV), rec, dtype=torch.float32)
    (ds,) = torch.autograd.grad((ps.view(-1) * torch.tensor(case["coef"], device=DEV)).sum(), rec)
    ep, es = rel_err(p.cpu(), case["p"]), rel_err(ps.cpu(), case["p"])
    gp, gs = _cmp_grad(d1, case["dfake_grad"]), _cmp_grad(ds, case["dfake_grad"])
    print("256: p rel err ours %.3e stock %.3e; grad rel err ours %.3e stock %.3e" % (ep, es, gp, gs))
    assert ep <= 2 * es + 1e-5 and gp <= 2 * gs + 1e-5
    assert torch.equal(d1, d2)


def test_equal_images_give_zero(mods, golden):
    m, _ = seeded_lpips(golden["256"])
    m.to(DEV)
    x = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(3)).to(DEV)
    rec = x.clone().requires_grad_(True)
    p = m(x, rec)
    p.sum().backward()
    assert torch.count_nonzero(p) == 0 and torch.count_nonzero(rec.grad) == 0


def test_no_grad_saves_nothing_and_double_backward_is_refused(mods, golden):
    m, _ = seeded_lpips(golden["72"])
    m.to(DEV)
    x = torch.rand(1, 3, 32, 32, device=DEV)
    rec = x.flip(3).clone().requires_grad_(True)
    with torch.no_grad():
        p = m(x, rec)
    assert not p.requires_grad
    p = m(x, rec)
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(p.sum(), rec, create_graph=True)
