"""The FP8 Linear route on the H100 (csrc/gemm_f8.cu): the cast pass bit for bit against torch's float8 casts, the three GEMMs
against fp64 of their dequantised operands (also at long K, where only promoted partial sums stay accurate), LinearFn against the fp64
restatement of the quantised computation, a MakeAScene step against the fp16 route, convergence, and no change anywhere the
flag is off or no graph is recorded."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FMT = {0: (torch.float8_e4m3fn, 448.0, 7), 1: (torch.float8_e5m2, 57344.0, 14)}


def scale_of(amax, fmt):
    """tc::operand_scale<top> on the host (amax a normal fp32 number here)."""
    import math
    return 2.0 ** (FMT[fmt][2] - math.floor(math.log2(float(amax))))


def ref_codes(x, fmt, amax=None):
    """uint8 codes of torch's float8 cast of clamp(x * s) (computed on the CPU)."""
    dt, vmax, _ = FMT[fmt]
    s = scale_of(x.abs().max() if amax is None else amax, fmt)
    return (x.float().cpu() * s).clamp(-vmax, vmax).to(dt).view(torch.uint8), s


def dq(codes, fmt, s):
    return codes.cpu().view(FMT[fmt][0]).double() / s


@pytest.mark.parametrize("M,K,fmt", [(640, 1024, 0), (37, 3072, 1), (1408, 4096, 0), (5, 16, 1)])
def test_cast_pass_matches_torch_bit_for_bit(M, K, fmt):
    from mas_b200 import ops
    g = torch.Generator().manual_seed(M + K)
    x = torch.randn(M, K, generator=g) * torch.logspace(-3, 2, K)
    x[0, :3] = torch.tensor([0.0, -0.0, 1e-30])
    xd = x.to(DEV)
    r, c, s, am = ops.to_fp8(xd, fmt, rows=True, cols=True, colsum=True)
    want, _ = ref_codes(x, fmt)
    assert float(am) == float(x.abs().max())
    assert torch.equal(r.cpu(), want)
    Mp = (M + 15) // 16 * 16
    assert c.shape == (K, Mp) and torch.equal(c[:, :M].cpu(), want.T) and not c[:, M:].any()
    assert rel_err(s, x.double().sum(0)) < 1e-6
    # each layout alone gives the same bytes; two calls give the same bits
    r2 = ops.to_fp8(xd, fmt, rows=True)[0]
    c2, s2 = ops.to_fp8(xd, fmt, rows=False, cols=True, colsum=True)[1:3]
    assert torch.equal(r, r2) and torch.equal(c, c2) and torch.equal(s, s2)


def test_cast_pass_keeps_nan_and_scales_one_for_zero_or_inf_amax():
    from mas_b200 import ops
    x = torch.randn(64, 32, device=DEV)
    x[3, 5] = float("nan")
    r = ops.to_fp8(x, 0, am=torch.tensor([float("nan")], device=DEV))[0]
    assert torch.isnan(r.view(torch.float8_e4m3fn).float()[3, 5]) and torch.isnan(r.view(torch.float8_e4m3fn).float()).sum() == 1
    z = torch.zeros(64, 32, device=DEV)
    assert not ops.to_fp8(z, 1)[0].any()
    r = ops.to_fp8(x.nan_to_num(), 0, am=torch.tensor([float("inf")], device=DEV))[0]   # scale 1
    assert torch.equal(r.cpu(), x.nan_to_num().cpu().clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8))


# Hopper's FP8 MMA does not keep an fp32 sum while it accumulates: on all-positive operands, partial sums carried through
# the MMAs for the whole contraction miss fp64 by 1.1e-2 of the result at K = 16384 in the weight gradient and by 7.2e-2 at
# K = 4096 in the forward form, growing with K. Promoted into fp32 registers every 128 K elements, the error is 3e-4 .. 5.7e-4 at any K (1024 ..
# 65536), and 1.5e-4 on operands of both signs (an fp32 matmul: 5e-8). GEMM_TOL bounds the promoted kernel with a margin.
GEMM_TOL = 1e-3


def _check_gemm(y, a, b, bias=None):
    """y == a . b^T (+bias) of the dequantised fp64 operands within GEMM_TOL of the result, norm-wise and on the worst row."""
    ref = a @ b.T + (0 if bias is None else bias.double().cpu())
    torch.backends.cuda.matmul.allow_tf32 = False
    f32 = (a.float().to(DEV) @ b.float().to(DEV).T).double().cpu() + (0 if bias is None else bias.double().cpu())
    e, t = y.double().cpu() - ref, f32 - ref
    en, tn = float(e.norm() / ref.norm()), float(t.norm() / ref.norm())
    er, tr = float((e.norm(dim=1) / ref.norm(dim=1)).max()), float((t.norm(dim=1) / ref.norm(dim=1)).max())
    print("gemm %s: kernel %.3e / fp32 %.3e norm-wise, worst row %.3e / %.3e" % (tuple(y.shape), en, tn, er, tr))
    assert en <= GEMM_TOL and er <= GEMM_TOL, (en, tn, er, tr)


@pytest.mark.parametrize("M,N,K,positive", [(5120, 3072, 1024, False), (5120, 1024, 4096, False), (300, 1024, 4096, True),
                                             (1408, 384, 4096, True)])
def test_forward_and_data_gradient_gemms(M, N, K, positive):
    """Forward (x e4m3) and data-gradient form (dy e5m2) of mas_gemm_rows_f8; the positive cases are lin2's K = 4096."""
    from mas_b200 import ops
    g = torch.Generator().manual_seed(M + N)
    x = torch.rand(M, K, generator=g) if positive else torch.randn(M, K, generator=g)
    W = torch.rand(N, K, generator=g) * 0.05 if positive else torch.randn(N, K, generator=g) * 0.05
    bias = torch.randn(N, generator=g).to(DEV)
    Wd = W.to(DEV).requires_grad_(True)
    w8, w8t, am_w = ops.fp8_weight(Wd)
    assert torch.equal(w8t, w8.T.contiguous())
    wcodes, sw = ref_codes(W, 0)
    assert torch.equal(w8.cpu(), wcodes)
    for fmt in (0, 1):
        x8, _, _, am = ops.to_fp8(x.to(DEV), fmt)
        y = ops.gemm_rows_f8(x8, am, fmt, w8, am_w, bias)
        _check_gemm(y, dq(x8, fmt, scale_of(am, fmt)), dq(w8, 0, sw), bias)
        assert torch.equal(y, ops.gemm_rows_f8(x8, am, fmt, w8, am_w, bias))


@pytest.mark.parametrize("M,N,K,positive", [(5120, 1024, 1024, False), (22528, 3072, 1024, False), (16384, 256, 384, True),
                                             (1000, 1024, 4096, False)])
def test_weight_gradient_gemm(M, N, K, positive):
    """mas_wgrad_rows_f8 from the transposed copies; K = 16384 rows of all-positive operands checks the accumulation."""
    from mas_b200 import ops
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.rand(M, K, generator=g) if positive else torch.randn(M, K, generator=g)
    dy = torch.rand(M, N, generator=g) * 1e-3 if positive else torch.randn(M, N, generator=g) * 1e-3
    _, x8t, _, amx = ops.to_fp8(x.to(DEV), 0, rows=False, cols=True)
    _, d8t, _, amd = ops.to_fp8(dy.to(DEV), 1, rows=False, cols=True)
    dw = ops.wgrad_rows_f8(x8t, amx, d8t, amd, M)
    _check_gemm(dw, dq(d8t, 1, scale_of(amd, 1)), dq(x8t, 0, scale_of(amx, 0)))
    assert torch.equal(dw, ops.wgrad_rows_f8(x8t, amx, d8t, amd, M))


@pytest.mark.parametrize("shape", [(2, 640, 1024), (3, 37, 1024)])
def test_linear_fn_fp8_route_against_the_quantised_computation(shape, monkeypatch):
    from mas_b200 import ops
    monkeypatch.setenv("MAS_LINEAR_F16", "1")
    g = torch.Generator().manual_seed(shape[1])
    K, N = shape[-1], 4096
    x = torch.randn(shape, generator=g).to(DEV).requires_grad_(True)
    W = (torch.randn(N, K, generator=g) * 0.03).to(DEV).requires_grad_(True)
    b = torch.randn(N, generator=g).to(DEV).requires_grad_(True)
    dy = torch.randn(shape[:-1] + (N,), generator=g).to(DEV) * 1e-2
    with torch.cuda.device(DEV), ops.L.launch_trace() as names:
        y = ops.linear(x, W, b, True)
        y.backward(dy)
    assert any("rows_gemm_f8" in n for n in names) and not any("t16" in n for n in names)
    R = x.numel() // K

    def q(t, fmt):
        c, s = ref_codes(t.detach().reshape(-1, t.shape[-1]), fmt)
        return dq(c, fmt, s)
    xq, wq, dyq = q(x, 0), q(W, 0), q(dy, 1)
    for got, ref in ((y.reshape(R, N), xq @ wq.T + b.detach().double().cpu()), (x.grad.reshape(R, K), dyq @ wq),
                     (W.grad, dyq.T @ xq), (b.grad, dy.reshape(R, N).double().cpu().sum(0))):
        assert rel_err(got, ref) < GEMM_TOL          # 8.9e-5 measured for y


def _bench_model(fp8, layers=24, hidden=1024, heads=16, img_dim=16, seg_vocab=1024, img_vocab=8192, text=128, seg_dim=16):
    from models.transformer import MakeAScene
    torch.manual_seed(0)
    m = MakeAScene(layers, hidden, heads, img_vocab, seg_vocab, 49408, img_dim, seg_dim, text, fp8_linear=fp8).to(DEV).train()
    m.device = DEV
    return m


def test_make_a_scene_step_against_the_fp16_route():
    """The bench configuration (24 layers, 1024 wide, 640 tokens) at batch 2: loss and every parameter gradient of the FP8 step
    against the fp16 step on the same weights and tokens."""
    g = torch.Generator().manual_seed(7)
    text = torch.randint(1, 40000, (2, 128), generator=g).to(DEV)
    seg = torch.randint(0, 1024, (2, 256), generator=g).to(DEV)
    img = torch.randint(0, 8192, (2, 256), generator=g).to(DEV)
    out = {}
    for fp8 in (False, True):
        m = _bench_model(fp8)
        loss = m.loss(text, seg, img)
        loss.backward()
        out[fp8] = (float(loss), {k: p.grad.clone() for k, p in m.named_parameters()})
        del m
    dl = abs(out[True][0] - out[False][0]) / out[False][0]
    errs = {k: rel_err(out[True][1][k], v) for k, v in out[False][1].items()}
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    lin = max(v for k, v in errs.items() if k.endswith("weight") and any(s in k for s in ("qkv", "out_proj", "lin1", "lin2")))
    print("step: loss %.6f fp16 %.6f rel diff %.2e; worst gradients %s; worst Linear weight %.3e" % (
        out[True][0], out[False][0], dl, worst, lin))
    # measured on an H100: loss 6.5e-6 apart; worst gradient 0.139 (text_pos_embeddings), worst Linear weight 0.132
    assert dl < 1e-4
    assert max(errs.values()) < 0.25 and lin < 0.25


def test_training_converges_like_the_fp16_route():
    """4 layers, 512 wide, 300 Adam steps from the same initialisation and data; image tokens are a fixed function of the seg
    tokens, so the loss can fall far below its initial value."""
    from models.transformer import MakeAScene
    g = torch.Generator().manual_seed(3)
    B, steps = 8, 300
    text = torch.randint(1, 100, (steps, B, 128), generator=g)
    seg = torch.randint(0, 64, (steps, B, 64), generator=g)
    img = (seg * 5 + 3) % 128
    final = {}
    for fp8 in (False, True):
        torch.manual_seed(11)
        m = MakeAScene(4, 512, 8, 128, 64, 100, 8, 8, 128, fp8_linear=fp8).to(DEV).train()
        m.device = DEV
        opt = torch.optim.Adam(m.parameters(), lr=3e-4)
        losses = []
        for i in range(steps):
            opt.zero_grad(set_to_none=True)
            loss = m.loss(text[i].to(DEV), seg[i].to(DEV), img[i].to(DEV))
            loss.backward()
            opt.step()
            losses.append(float(loss))
        final[fp8] = (losses[0], sum(losses[-20:]) / 20)
    print("convergence: fp16 %.4f -> %.4f, fp8 %.4f -> %.4f" % (final[False] + final[True]))
    assert final[True][0] == pytest.approx(final[False][0], rel=1e-2)
    # measured on an H100: fp16 5.031 -> 3.746, FP8 5.030 -> 3.747
    for f in (False, True):
        assert final[f][1] < 0.85 * final[f][0]
    assert abs(final[True][1] - final[False][1]) < 0.02 * final[False][1]


def test_no_grad_calls_generate_and_score_are_unchanged_by_the_flag():
    from models.transformer import MakeAScene
    from mas_b200 import _lib
    cfg = (2, 512, 8, 256, 64, 100, 8, 8, 128)
    torch.manual_seed(5)
    a = MakeAScene(*cfg).to(DEV).eval()
    b = MakeAScene(*cfg, fp8_linear=True).to(DEV).eval()
    b.load_state_dict(a.state_dict())
    a.device = b.device = DEV
    g = torch.Generator().manual_seed(2)
    text = torch.randint(1, 100, (3, 128), generator=g).to(DEV)
    seg = torch.randint(0, 64, (3, 64), generator=g).to(DEV)
    img = torch.randint(0, 256, (3, 64), generator=g).to(DEV)
    with _lib.launch_trace() as names:
        with torch.no_grad():
            fa, fb = a(text, seg, img), b(text, seg, img)
        ta, la = a.generate(text, seg, img_tokens=img, return_logits=True)
        tb, lb = b.generate(text, seg, img_tokens=img, return_logits=True)
        sa, sb = a.score(text, seg, img), b.score(text, seg, img)
        ga = a.generate(text, seg, temperature=1.0, top_k=8, generator=torch.Generator(device=DEV).manual_seed(4))
        gb = b.generate(text, seg, temperature=1.0, top_k=8, generator=torch.Generator(device=DEV).manual_seed(4))
    assert torch.equal(fa, fb) and torch.equal(ta, tb) and torch.equal(la, lb) and torch.equal(ga, gb)
    assert all(torch.equal(u, v) for u, v in zip(sa if isinstance(sa, tuple) else (sa,), sb if isinstance(sb, tuple) else (sb,)))
    assert not any("f8" in n or "fp8" in n for n in names)
    # a training step with the flag off launches no FP8 kernel either
    a.train()
    with _lib.launch_trace() as names:
        a.loss(text, seg, img).backward()
    assert names and not any("f8" in n or "fp8" in n for n in names)


def test_fp8_training_step_replays_in_a_cuda_graph():
    """Forward and backward of a 2-layer FP8 Transformer captured in a CUDA graph: each replay gives the eager step's bits."""
    from models.transformer import Transformer
    torch.manual_seed(1)
    t = Transformer(2, 512, 8, 8, 8, 128, fp8_linear=True).to(DEV).train()
    x = torch.randn(2, 256, 512, device=DEV, requires_grad=True)
    w = torch.randn(2, 256, 512, device=DEV)
    params = [x] + list(t.parameters())

    def step():
        for p in params:
            if p.grad is not None:
                p.grad.zero_()
        out, _ = t(x)
        (out * w).sum().backward()
        return out

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    eager_out = step().detach().clone()
    eager = [p.grad.clone() for p in params]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager_out)
        assert all(torch.equal(p.grad, e) for p, e in zip(params, eager))
