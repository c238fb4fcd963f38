"""Training-step throughput of the token transformer (BASELINE.json configs[4] model: 24 layers, 1024 wide, 16 heads of 64,
128 text + 256 segmentation + 256 image tokens, 8192-code image vocabulary; random-init weights, synthetic tokens):
forward + cross-entropy over the image tokens + backward (train.py:136-153; no optimizer), CUDA-event timed.
One JSON line; beside bench.py's headline (tier 2, SURVEY.md 8f-2).
--image-tokens-per-dim 32 runs the sequence the VQ configs produce (128 + 16^2 + 32^2 = 1408 tokens); --recompute-attention
trains with MakeAScene(recompute_attention=True) (no stored attention probabilities); --hidden / --heads change the width and
the head count (--hidden 2048 --heads 16 and --hidden 1024 --heads 8: heads of 128).
--fp8-linear also times the same model and tokens with the four Linear layers of every TransformerLayer on the FP8 route
(MakeAScene(fp8_linear=True)), the two forms alternated over --rounds rounds (medians), and adds their step times, tokens/s,
peak memory and loss, with the SM clocks sampled during the rounds, under "fp8_linear".
Usage: python tools/bench_transformer.py [--batch B] [--steps K] [--warmup W] [--layers L] [--dropout P]
       [--image-tokens-per-dim N] [--recompute-attention] [--hidden H] [--heads N] [--fp8-linear [--rounds R]]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]
import torch  # noqa: E402
from mas_b200 import _lib  # noqa: E402
from models.transformer import MakeAScene  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=8)
ap.add_argument("--steps", type=int, default=4)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--layers", type=int, default=24)
ap.add_argument("--dropout", type=float, default=0.0, help="attention and residual dropout probability (both)")
ap.add_argument("--profile", action="store_true", help="per-entry-point CUDA-event times of one extra step (stderr)")
ap.add_argument("--torch-ce", action="store_true", help="F.cross_entropy on the logits instead of MakeAScene.loss (A/B of the fused entry)")
ap.add_argument("--image-tokens-per-dim", type=int, default=16, help="image tokens per side (sequence = 128 + 256 + N^2)")
ap.add_argument("--recompute-attention", action="store_true", help="store no attention probabilities; the backward recomputes them")
ap.add_argument("--hidden", type=int, default=1024, help="model width")
ap.add_argument("--heads", type=int, default=16, help="attention heads (head dim = hidden / heads)")
ap.add_argument("--fp8-linear", action="store_true", help="also time the FP8 Linear route, alternated with the default")
ap.add_argument("--rounds", type=int, default=3, help="alternated rounds of --fp8-linear")
args = ap.parse_args()
dev = torch.device("cuda:0")
torch.manual_seed(0)
cfg = dict(num_layers=args.layers, hidden_dim=args.hidden, num_attn_heads=args.heads, image_vocab_size=8192, seg_vocab_size=1024, text_vocab_size=49408,
           image_tokens_per_dim=args.image_tokens_per_dim, seg_tokens_per_dim=16, text_length=128)
m = MakeAScene(**cfg, attn_dropout_prob=args.dropout, out_dropout_prob=args.dropout,
               recompute_attention=args.recompute_attention).to(dev).train()
IMG = args.image_tokens_per_dim ** 2
m.device = dev
B = args.batch
g = torch.Generator().manual_seed(1234)
text = torch.randint(1, 40000, (B, 128), generator=g).to(dev)
seg = torch.randint(0, 1024, (B, 256), generator=g).to(dev)
img = torch.randint(0, 8192, (B, IMG), generator=g).to(dev)


def step():
    m.zero_grad(set_to_none=True)
    if args.torch_ce:
        lg = m(text, seg, img)
        loss = torch.nn.functional.cross_entropy(lg.view(-1, lg.shape[-1]), img.view(-1))
    else:
        loss = m.loss(text, seg, img)
    loss.backward()
    return loss


for _ in range(args.warmup):
    step()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
l0, t0 = _lib.launch_count(), _lib.tc_launch_count()
e0.record()
for _ in range(args.steps):
    loss = step()
e1.record()
torch.cuda.synchronize()
sec = e0.elapsed_time(e1) * 1e-3 / args.steps
if args.profile:
    _lib.profile_start()
    step()
    rep = _lib.profile_report()
    tot = sum(t for _, t in rep.values())
    for k, (c, t) in sorted(rep.items(), key=lambda kv: -kv[1][1])[:24]:
        print("  %-36s n=%4d  %8.2f ms  %5.1f%%  %7.3f ms/call" % (k, c, t, 100 * t / tot, t / c), file=sys.stderr)
    print("  total %.2f ms in %d calls" % (tot, sum(c for c, _ in rep.values())), file=sys.stderr)
S, H, L, V = 128 + 256 + IMG, args.hidden, args.layers, 8192
fp8 = None
if args.fp8_linear:
    import bench  # noqa: E402
    lins = [lin for layer in m.transformer.layers for lin in (layer.attn.qkv, layer.attn.out_proj, layer.mlp.lin1, layer.mlp.lin2)]

    def timed(on):
        for lin in lins:
            lin.fp8 = on
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.steps):
            lv = step()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.steps, torch.cuda.max_memory_allocated() / 1e9, float(lv.detach())

    sampler = bench.ClockSampler(0)
    sampler.start()
    res = {False: [], True: []}
    for _ in range(args.rounds):
        for on in (False, True):
            res[on].append(timed(on))
    clocks = sampler.stop()
    for lin in lins:
        lin.fp8 = False
    fp8 = {"clocks": clocks, "gpu": torch.cuda.get_device_name(0)}
    for on, tag in ((False, "fp16"), (True, "fp8")):
        ms = sorted(r[0] for r in res[on])[len(res[on]) // 2]
        fp8[tag] = {"ms_per_step": ms, "tokens_per_s": B * S / ms * 1e3, "peak_mem_gb": max(r[1] for r in res[on]),
                    "loss": res[on][-1][2]}
    fp8["speedup"] = fp8["fp16"]["ms_per_step"] / fp8["fp8"]["ms_per_step"]
lin = 2 * S * (12 * H * H) * L + 2 * IMG * H * V           # Linear layers, forward, per sequence
att = 2 * 2 * S * S * H * L                                # QK^T and PV over the full (masked) square, forward
print(json.dumps({"metric": "token transformer training step (fwd + cross-entropy + bwd), sequence tokens/s", "value": B * S / sec,
                  "unit": "tokens/s", "batch": B, "seq_len": S, "ms_per_step": sec * 1e3, "loss": float(loss),
                  "model_tflops": 3 * (lin + att) * B / sec / 1e12, "gpu_launches_per_step": (_lib.launch_count() - l0) // args.steps,
                  "tensor_core_launches_per_step": (_lib.tc_launch_count() - t0) // args.steps,
                  "peak_mem_gb": torch.cuda.max_memory_allocated() / 1e9, "dropout": args.dropout,
                  "attention": ("recomputed P (attn_causal_fwd_stats + attn_causal_bwd)" if args.recompute_attention else
                                "fused core (attn_causal_fwd)" if os.environ.get("MAS_ATTN_FUSED", "1") != "0" else "GEMM / softmax / GEMM"),
                  "loss_entry": "F.cross_entropy (torch)" if args.torch_ce else "MakeAScene.loss (mas_ce_*)", "config": cfg,
                  **({"fp8_linear": fp8} if fp8 else {})}))
