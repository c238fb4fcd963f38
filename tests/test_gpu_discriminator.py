"""PatchGAN discriminator (losses/discriminator.py) on the H100: the 4x4 convolution kernels against fp64 products, the
BatchNorm2d+LeakyReLU unit against torch's fp64 modules, and the whole drop-in module through the reference train.py call
sequence against the golden recorded from the real reference (tests/golden/discriminator.pt)."""
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, rel_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def mods():
    if not torch.cuda.is_available():
        pytest.skip("needs cuda:0")
    from mas_b200 import _lib, ops
    from losses import discriminator
    _lib.load()
    return _lib, ops, discriminator


# (cin, cout, h, w, stride, bias, slope, nchw input)
CONV_CASES = [
    (3, 64, 38, 30, 2, True, 0.2, True),      # model.0 shape family: image read through NCHW strides
    (64, 128, 19, 22, 2, False, None, False),
    (70, 33, 17, 17, 2, True, None, False),   # channel counts off every tile
    (96, 80, 9, 11, 1, False, None, False),
    (130, 1, 8, 9, 1, True, None, False),     # model.11: Cout = 1
    (256, 512, 10, 10, 1, False, None, False),
]


@pytest.mark.parametrize("cin,cout,h,w,stride,has_bias,slope,nchw", CONV_CASES)
def test_conv4x4_fwd_dgrad_wgrad_fp64(mods, cin, cout, h, w, stride, has_bias, slope, nchw):
    _lib, ops, _ = mods
    g = torch.Generator().manual_seed(cin * 1000 + cout + h)
    x = torch.randn(3, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 4, 4, generator=g) * (1.0 / (16 * cin) ** 0.5)
    b = torch.randn(cout, generator=g) if has_bias else None
    # fp64 reference
    x64 = x.double().requires_grad_(True)
    w64 = wt.double().requires_grad_(True)
    b64 = b.double().requires_grad_(True) if has_bias else None
    y64 = F.conv2d(x64, w64, b64, stride=stride, padding=1)
    if slope is not None:
        y64 = F.leaky_relu(y64, slope)
    dy = torch.randn(y64.shape, generator=g)
    y64.backward(dy.double())
    # device
    xd = x.to(DEV) if nchw else x.to(DEV).contiguous(memory_format=torch.channels_last)
    xd.requires_grad_(True)
    wd = wt.to(DEV).requires_grad_(True)
    bd = b.to(DEV).requires_grad_(True) if has_bias else None
    l0 = _lib.launch_count()
    y = ops.Conv4x4Fn.apply(xd, wd, bd, stride, slope)
    y.backward(dy.to(DEV))
    torch.cuda.synchronize()
    assert _lib.launch_count() > l0
    assert y.shape == y64.shape
    assert rel_err(y, y64) < 1e-5
    assert rel_err(xd.grad, x64.grad) < 1e-5
    assert rel_err(wd.grad, w64.grad) < 1e-5
    if has_bias:
        assert rel_err(bd.grad, b64.grad) < 1e-5


# (cin, cout, h, w, stride, batch): the discriminator's tensor-core layers at reduced size - Cin 64 forward and a 64-channel
# data-gradient destination (model.2), model.5, and the stride-1 layer whose 16x16 input gives a 15x15 output (model.8 at
# 32x32 -> 31x31: the dropped row / column of the 3x3 output, zero-padded output gradient)
TC_CASES = [(64, 128, 32, 32, 2, 3), (128, 256, 32, 64, 2, 2), (256, 512, 16, 16, 1, 3), (128, 128, 32, 16, 1, 2)]


@pytest.mark.parametrize("cin,cout,h,w,stride,batch", TC_CASES)
def test_conv4x4_tensor_core_route_fp64(mods, cin, cout, h, w, stride, batch):
    """The shift-map route on the fp16 wgmma kernels against fp64 (fp16 operands: 11-bit significands, fp32 accumulate),
    and against the exact-fp32 SIMT kernels of the same layer."""
    _lib, ops, _ = mods
    g = torch.Generator().manual_seed(cin + cout + h + stride)
    x = torch.randn(batch, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 4, 4, generator=g) * (1.0 / (16 * cin) ** 0.5)
    x64, w64 = x.double().requires_grad_(True), wt.double().requires_grad_(True)
    y64 = F.conv2d(x64, w64, stride=stride, padding=1)
    dy = torch.randn(y64.shape, generator=g)
    y64.backward(dy.double())
    res = {}
    for impl in ("tc", "simt"):
        ops.set_impl(ops.L.IMPL_AUTO if impl == "tc" else ops.L.IMPL_SIMT)
        try:
            xd = x.to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
            wd = wt.to(DEV).requires_grad_(True)
            assert ops.conv4x4_tc_route(xd, cout, stride) == (impl == "tc")
            tc0 = _lib.tc_launch_count()
            y = ops.Conv4x4Fn.apply(xd, wd, None, stride, None)
            y.backward(dy.to(DEV).contiguous(memory_format=torch.channels_last))
            torch.cuda.synchronize()
            assert (_lib.tc_launch_count() - tc0 >= 3) == (impl == "tc")
            res[impl] = (y.detach().cpu(), xd.grad.cpu(), wd.grad.cpu())
        finally:
            ops.set_impl(ops.L.IMPL_AUTO)
    tol = {"tc": 2e-3, "simt": 1e-5}
    for impl, (y, gx, gw) in res.items():
        assert y.shape == y64.shape
        assert rel_err(y, y64) < tol[impl] and rel_err(gx, x64.grad) < tol[impl] and rel_err(gw, w64.grad) < tol[impl], impl


def test_conv4x4_zero_stride_dy(mods):
    """The loss gradient of -mean(logits) arrives as an expanded tensor (all strides 0): read as is, no copy."""
    _lib, ops, _ = mods
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 40, 9, 9, generator=g)
    wt = torch.randn(1, 40, 4, 4, generator=g) * 0.05
    x64, w64 = x.double().requires_grad_(True), wt.double().requires_grad_(True)
    (-F.conv2d(x64, w64, padding=1).mean()).backward()
    xd = x.to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wd = wt.to(DEV).requires_grad_(True)
    (-ops.Conv4x4Fn.apply(xd, wd, None, 1, None).mean()).backward()
    assert rel_err(xd.grad, x64.grad) < 1e-5 and rel_err(wd.grad, w64.grad) < 1e-5


@pytest.mark.parametrize("train", [True, False])
def test_batchnorm_lrelu_fp64(mods, train):
    _lib, ops, D = mods
    g = torch.Generator().manual_seed(9)
    c = 96
    x = torch.randn(4, c, 7, 9, generator=g) * 3 + 1
    ref = torch.nn.BatchNorm2d(c).double()
    with torch.no_grad():
        ref.weight.normal_(1.0, 0.3, generator=g)
        ref.bias.normal_(0.0, 0.3, generator=g)
        ref.running_mean.normal_(generator=g)
        ref.running_var.uniform_(0.5, 2.0, generator=g)
    mine = D.BatchNorm2d(c).to(DEV)
    mine.load_state_dict({k: v.float() if v.is_floating_point() else v for k, v in ref.state_dict().items()})
    ref.train(train)
    mine.train(train)
    x64 = x.double().requires_grad_(True)
    y64 = F.leaky_relu(ref(x64), 0.2)
    dy = torch.randn(y64.shape, generator=g)
    y64.backward(dy.double())
    xd = x.to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = mine(xd, 0.2)
    assert rel_err(y, y64) < 1e-5
    for k in ("running_mean", "running_var"):
        assert rel_err(getattr(mine, k), getattr(ref, k)) < 1e-6
    if train:
        y.backward(dy.to(DEV))
        assert rel_err(xd.grad, x64.grad) < 1e-5
        assert rel_err(mine.weight.grad, ref.weight.grad) < 1e-5
        assert rel_err(mine.bias.grad, ref.bias.grad) < 1e-5
        assert int(mine.num_batches_tracked) == int(ref.num_batches_tracked)


def _golden():
    return torch.load(os.path.join(GOLDEN, "discriminator.pt"), weights_only=False)


def _images(case):
    gen = torch.Generator().manual_seed(case["seed"] + 1000)
    shape = (case["batch"], 3, case["size"], case["size"])
    return torch.rand(shape, generator=gen), torch.rand(shape, generator=gen)


def _err(rec, t):
    """Deviation of t from a golden record: the larger of the norm's relative difference and the norm-wise relative error of
    the full tensor (or of its recorded samples)."""
    t = t.detach().cpu().double()
    e = abs(float(t.norm()) - rec["norm"]) / rec["norm"]
    return max(e, rel_err(t, rec["full"]) if "full" in rec else rel_err(t.reshape(-1)[rec["idx"]], rec["val"]))


def _train_step_errors(m, case, real, fake):
    """train.py's discriminator work on module m: deviations of every golden quantity, and the two input gradients."""
    err = {}
    lr, lf = m(real), m(fake)
    err["logits"] = max(rel_err(lr, case["logits_real"]), rel_err(lf, case["logits_fake"]))
    (0.5 * (torch.relu(1.0 - lr).mean() + torch.relu(1.0 + lf).mean())).backward()
    for k, p in m.named_parameters():
        err[k] = _err(case["grads"][k], p.grad)
    for p in m.parameters():
        p.requires_grad_(False)
    rec = fake.clone().requires_grad_(True)
    lg = m(rec)
    g_loss = -torch.mean(lg)
    (d1,) = torch.autograd.grad(g_loss, rec, retain_graph=True)
    g_loss.backward()
    err["logits_g"] = rel_err(lg, case["logits_g"])
    err["drec_grad"], err["drec_backward"] = _err(case["drec_grad"], d1), _err(case["drec_backward"], rec.grad)
    sd = m.state_dict()
    for k, v in case["stats_g"].items():
        if "num_batches" in k:
            assert int(sd[k]) == int(v), k
        else:
            err[k] = rel_err(sd[k], v)
    return err, d1, rec.grad


def _stock(m):
    """The reference's own module graph (stock nn.Conv2d / BatchNorm2d / LeakyReLU: cuDNN with PyTorch's default TF32
    convolutions) holding m's weights."""
    layers = []
    for a in m.model:
        if isinstance(a, torch.nn.Conv2d):
            layers.append(torch.nn.Conv2d(a.in_channels, a.out_channels, 4, a.stride, 1, bias=a.bias is not None))
        elif isinstance(a, torch.nn.BatchNorm2d):
            layers.append(torch.nn.BatchNorm2d(a.num_features))
        else:
            layers.append(torch.nn.LeakyReLU(0.2))
    ref = torch.nn.Module()
    ref.model = torch.nn.Sequential(*layers)
    ref.load_state_dict(m.state_dict())
    ref.forward = lambda x: ref.model(x)
    return ref


@pytest.mark.parametrize("name", ["256", "72"])
def test_module_train_step_against_golden(mods, name):
    """train.py:84-98 order: D step (2 forwards, hinge loss, backward), then the generator step with D frozen:
    autograd.grad(retain_graph=True) followed by backward() through the same graph.  At 72^2 every layer runs on the
    exact-fp32 kernels: 1e-3 on the logits, 3e-3 on the gradients, 1e-5 on the running statistics.  At 256^2 model.2 / 5 / 8 run on fp16 operands
    (11-bit significands, like the TF32 convolutions the stock modules run on this GPU by default); a quantity may then
    also deviate from the fp32 golden by up to twice what the stock modules' own GPU run deviates."""
    _lib, ops, D = mods
    case = _golden()[name]
    torch.manual_seed(case["seed"])
    m = D.Discriminator()
    m.apply(D.weights_init)
    stock = _stock(m).to(DEV).train()
    m.to(DEV).train()
    real, fake = _images(case)
    real, fake = real.to(DEV), fake.to(DEV)

    calls = []
    real_call = ops.L.call

    def spy(name_, *a):
        calls.append(name_)
        return real_call(name_, *a)

    ops.L.call = spy
    try:
        tc0 = _lib.tc_launch_count()
        err, d1, d2 = _train_step_errors(m, case, real, fake)
        torch.cuda.synchronize()
        tc_launches = _lib.tc_launch_count() - tc0
    finally:
        ops.L.call = real_call
    tc = 3 if name == "256" else 0
    bound = {k: 1e-3 if k.startswith("logits") else 1e-5 if "running" in k else 3e-3 for k in err}
    if tc:
        stock_err, _, _ = _train_step_errors(stock, case, real, fake)
        bound = {k: max(v, 2 * stock_err[k]) for k, v in bound.items()}
        print("\n".join("%-24s ours %.2e  stock %.2e" % (k, err[k], stock_err[k]) for k in err))
    bad = {k: (err[k], bound[k]) for k in err if not err[k] <= bound[k]}
    assert not bad, bad
    assert torch.equal(d1, d2)
    # model.2 / 5 / 8 on the wgmma kernels in every pass at 256^2: forward, data and weight gradients of the discriminator
    # step (data gradients of model.2/5/8/11 only: the images are leaves), and the two data-gradient passes of the generator
    # step (no weight gradient: D is frozen); at 72^2 every layer on the SIMT kernels
    assert (tc_launches > 0) == (tc > 0)
    assert calls.count("mas_conv3x3_fprop_tc16") == 3 * tc + 2 * tc + 2 * tc
    assert calls.count("mas_conv3x3_wgrad_tc16") == 2 * tc
    assert calls.count("mas_conv4x4") == 3 * (5 - tc)
    assert calls.count("mas_conv4x4_wgrad") == 2 * (5 - tc)
    assert calls.count("mas_conv4x4_dgrad") == 2 * (4 - tc) + 2 * (5 - tc)


def test_eval_mode_matches_torch(mods):
    _lib, ops, D = mods
    torch.manual_seed(3)
    m = D.Discriminator()
    m.apply(D.weights_init)
    ref = torch.nn.Sequential(*[torch.nn.Conv2d(a.in_channels, a.out_channels, 4, a.stride, 1, bias=a.bias is not None)
                                if isinstance(a, torch.nn.Conv2d) else
                                torch.nn.BatchNorm2d(a.num_features) if isinstance(a, torch.nn.BatchNorm2d) else
                                torch.nn.LeakyReLU(0.2) for a in m.model])
    with torch.no_grad():
        for b in m.modules():
            if isinstance(b, torch.nn.BatchNorm2d):
                b.running_mean.normal_(0, 0.1)
                b.running_var.uniform_(0.5, 1.5)
    ref.load_state_dict({k[len("model."):]: v for k, v in m.state_dict().items()})
    ref.double().eval()
    m.to(DEV).eval()
    x = torch.rand(2, 3, 40, 40)
    with torch.no_grad():
        assert rel_err(m(x.to(DEV)), ref(x.double())) < 1e-5
