"""Candidates/s of MakeAScene.score(num_samples=n), the shared-prefix form, against the repeat_interleave call it equals bit for
bit, at the bench's model (24 layers, 1024 wide, 128 text + 256 segmentation tokens -> 256 image tokens of an 8192-code
vocabulary; random-init weights), 16 heads of 64 and 8 heads of 128.
Per workload (B prompts x n candidates, unguided and guided at scale 3): both forms warmed up, then --reps calls of each,
alternating; candidates/s from the median call (device synchronised), the spread as min / max call time, the peak memory of
each form (torch.cuda.max_memory_allocated over one call, minus what was allocated before it), and a bitwise check of the two
results. Then the kernel alone: mas_attn_causal_prefix_forward against mas_attn_causal_forward and
mas_attn_causal_forward_stats over the concatenated rows, CUDA events over --kreps launches, in us and TFLOP/s of the
algorithmic work (4 hd per query-key pair at or below the diagonal, each kernel's own queries).
One JSON line per workload and kernel shape, preceded by the card's name, power limit and max SM clock.
Usage: python tools/bench_score.py [--reps N] [--kreps N] [--layers N] [--workloads 1x8,8x8,4x32]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]
import torch  # noqa: E402
from mas_b200 import ops  # noqa: E402
from models.transformer import MakeAScene  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--kreps", type=int, default=50)
ap.add_argument("--layers", type=int, default=24)
ap.add_argument("--workloads", default="1x8,8x8,4x32")
ap.add_argument("--heads", default="16,8", help="head counts of the models (16: hd 64, 8: hd 128)")
ap.add_argument("--no-kernel", action="store_true", help="skip the kernel timings")
args = ap.parse_args()
dev = torch.device("cuda:0")
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True, check=True).stdout.strip()
card = dict(gpu=torch.cuda.get_device_name(0), smi=smi)
print(json.dumps(card), flush=True)
CFG = dict(num_layers=args.layers, hidden_dim=1024, image_vocab_size=8192, seg_vocab_size=1024, text_vocab_size=49408,
           image_tokens_per_dim=16, seg_tokens_per_dim=16, text_length=128)


def timed(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1) / 1e3, (torch.cuda.max_memory_allocated() - base) / 2 ** 30


for heads in (int(h) for h in args.heads.split(",")):
    torch.manual_seed(0)
    m = MakeAScene(num_attn_heads=heads, **CFG).to(dev).eval()
    assert m._score_shares_prefix()
    for wl in args.workloads.split(","):
        B, n = (int(v) for v in wl.split("x"))
        for scale in (None, 3.0):
            g = torch.Generator().manual_seed(B * 1000 + n)
            text = torch.randint(1, CFG["text_vocab_size"], (B, 128), generator=g).to(dev)
            seg = torch.randint(0, CFG["seg_vocab_size"], (B, 256), generator=g).to(dev)
            img = torch.randint(0, CFG["image_vocab_size"], (B * n, 256), generator=g).to(dev)
            tr, sr = text.repeat_interleave(n, 0), seg.repeat_interleave(n, 0)
            forms = dict(shared=lambda: m.score(text, seg, img, guidance_scale=scale, num_samples=n),
                         repeated=lambda: m.score(tr, sr, img, guidance_scale=scale))
            outs = {k: timed(f)[0] for k, f in forms.items()}                  # warm-up (weight images, modules)
            times, peaks = {k: [] for k in forms}, {}
            for _ in range(args.reps):
                for k, f in forms.items():
                    _, t, mem = timed(f)
                    times[k].append(t)
                    peaks[k] = mem
            med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            print(json.dumps(dict(
                heads=heads, hd=1024 // heads, B=B, n=n, guidance=scale, rows=B * n * (2 if scale else 1),
                equal=bool(torch.equal(outs["shared"], outs["repeated"])),
                cand_per_s={k: round(B * n / v, 2) for k, v in med.items()},
                median_s={k: round(v, 4) for k, v in med.items()},
                min_max_s={k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
                speedup=round(med["repeated"] / med["shared"], 3),
                peak_gib={k: round(v, 2) for k, v in peaks.items()})), flush=True)
    del m
    torch.cuda.empty_cache()


def pairs(q_from, q_to):
    """Query-key pairs at or below the diagonal for queries q_from .. q_to - 1 (keys 0 .. q)."""
    return (q_to * (q_to + 1) - q_from * (q_from + 1)) // 2


def ktime(fn):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.kreps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / args.kreps


for heads, hd in (() if args.no_kernel else ((16, 64), (8, 128))):
    for P, n in ((1, 8), (8, 8), (8, 32)):          # prefix rows (4 prompts x 2 streams = 8 for the guided 4x32)
        Lp, L, H = 384, 256, heads * hd
        g = torch.Generator().manual_seed(P * n)
        qp = torch.randn(P, Lp, 3 * H, generator=g).to(dev)
        qs = torch.randn(P * n, L, 3 * H, generator=g).to(dev)
        cat = torch.cat([qp.repeat_interleave(n, 0), qs], 1).contiguous()
        R, S = P * n, Lp + L
        am = ops.amax_joint(qp, qs)
        ctx_s = torch.empty(R, L, H, device=dev)
        ctx_c = torch.empty(R, S, H, device=dev)
        stats = torch.empty(2, R, heads, S, device=dev)
        alpha = 1.0 / hd ** 0.5
        res = dict(heads=heads, hd=hd, P=P, n=n, Lp=Lp, L=L)
        t = ktime(lambda: ops.L.call("mas_attn_causal_prefix_forward", qp, qs, am, ctx_s, P, n, Lp, L, heads, hd, alpha))
        fl = 4.0 * hd * heads * R * pairs(Lp, S)
        res["prefix_us"], res["prefix_tflops"] = round(t, 1), round(fl / t / 1e6, 1)
        t = ktime(lambda: ops.L.call("mas_attn_causal_forward_stats", cat, am, stats, ctx_c, R, S, heads, hd, alpha, 0.0, None))
        fl = 4.0 * hd * heads * R * pairs(0, S)
        res["concat_stats_us"], res["concat_stats_tflops"] = round(t, 1), round(fl / t / 1e6, 1)
        if R * heads * S * S * 4 < 8 * 2 ** 30:
            Pm = torch.empty(R, heads, S, S, device=dev)
            t = ktime(lambda: ops.L.call("mas_attn_causal_forward", cat, am, Pm, ctx_c, R, S, heads, hd, alpha))
            res["concat_forward_us"], res["concat_forward_tflops"] = round(t, 1), round(fl / t / 1e6, 1)
            del Pm
        ops.L.call("mas_attn_causal_prefix_forward", qp, qs, am, ctx_s, P, n, Lp, L, heads, hd, alpha)
        ops.L.call("mas_attn_causal_forward_stats", cat, am, stats, ctx_c, R, S, heads, hd, alpha, 0.0, None)
        res["equal"] = bool(torch.equal(ctx_s, ctx_c[:, Lp:]))
        print(json.dumps(res), flush=True)
