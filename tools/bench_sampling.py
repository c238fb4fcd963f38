"""Tokens/s of classifier-free-guided sampling with the KV cache (BASELINE.json configs[4]: 24 layers, 1024 wide, 16
heads, 128 text + 256 segmentation tokens -> 256 image tokens of an 8192-code vocabulary; random-init weights).
One JSON line; not part of bench.py's headline (the reference has no sampler to compare with: SURVEY.md 8f-3). It carries the
GPU's name and power limit, and the HBM bytes a decode step streams on the path actually taken: up to 8 rows fp32 weights and
fp32 KV cache, above 8 rows fp16 weights and fp16 cache (the cache read at the mean cache length of the image positions).
--top-p adds the nucleus filter to the draw (top-k 64 stays); --prompt-frac F forces a random share F of the image positions
(an image prompt, random tokens): the forced positions are still decoded one step each, so tokens/s counts every position.
--samples N draws N images per prompt (generate(num_samples=N)): B prompts give R = 2 B N rows that share each prompt's prefix
cache, and cache_gb_per_step counts a prompt's prefix once per step, as the shared-prefix attention reads it.
--logprobs also times the same call with return_logprobs=True next to the plain one (alternating, --reps each, after both
are warmed up) and adds both times and the relative cost to the line; without it the line is unchanged.
--sweep N times a guidance sweep over N scales two ways, alternating, --reps each after both are warmed up: one call with
num_samples=N and one guidance scale per sample (per-row controls: one prefix pass, N x the decode rows) against N calls at
num_samples=1, one per scale. It also times the draw kernel alone, mas_sample_rows (per-row values, u or seeds) against
mas_sample_filtered_logp with the same values as scalars, at R = 8, 128, 256 rows of V = 8192 (the bench's top-k 64).
Usage: python tools/bench_sampling.py [--batch B] [--samples N] [--reps N] [--graphs] [--top-p P] [--prompt-frac F] [--logprobs]
                                      [--sweep N]"""
import argparse
import copy
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]
import torch  # noqa: E402
from mas_b200 import _lib, ops  # noqa: E402
from models.transformer import MakeAScene  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=1)
ap.add_argument("--samples", type=int, default=1, help="images per prompt (generate's num_samples)")
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--layers", type=int, default=24)
ap.add_argument("--graphs", action="store_true", help="replay each position's decode step from a CUDA graph")
ap.add_argument("--top-p", type=float, default=None, help="nucleus filter of the draw (default: off)")
ap.add_argument("--prompt-frac", type=float, default=0.0, help="share of image positions forced by a random image prompt")
ap.add_argument("--logprobs", action="store_true", help="also time generate(return_logprobs=True) against the plain call")
ap.add_argument("--sweep", type=int, default=0, help="time a sweep over N guidance scales: one per-row call against N calls")
args = ap.parse_args()
dev = torch.device("cuda:0")
torch.manual_seed(0)
cfg = dict(num_layers=args.layers, hidden_dim=1024, num_attn_heads=16, image_vocab_size=8192, seg_vocab_size=1024, text_vocab_size=49408,
           image_tokens_per_dim=16, seg_tokens_per_dim=16, text_length=128)
m = MakeAScene(**cfg).to(dev).eval()
m.device = dev
B, N = args.batch, args.samples
text = torch.randint(1, 40000, (B, 128), device=dev)
seg = torch.randint(0, 1024, (B, 256), device=dev)
gen = torch.Generator(device=dev).manual_seed(1)
kw = dict(guidance_scale=3.0, temperature=1.0, top_k=64, top_p=args.top_p, generator=gen, use_graphs=args.graphs, num_samples=N)
if args.prompt_frac > 0:
    kw["img_tokens"] = torch.randint(0, cfg["image_vocab_size"], (B * N, 256), device=dev)
    kw["img_mask"] = torch.rand(B * N, 256, device=dev) < args.prompt_frac
m.generate(text, seg, **kw)     # warm-up (captures)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
l0 = _lib.launch_count()
e0.record()
for _ in range(args.reps):
    toks = m.generate(text, seg, **kw)
e1.record()
torch.cuda.synchronize()
sec = e0.elapsed_time(e1) * 1e-3 / args.reps
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
R = 2 * B * N
elem = 4 if R <= ops.DECODE_F32_ROWS else 2
params = sum(p.numel() for n, p in m.named_parameters() if "embedding" not in n)
prefix, steps = 128 + 256, 255
mean_suffix = (steps + 1) / 2        # the step of image position t reads prefix + t + 1 positions; its prompt's prefix once per group
weight_bytes = params * elem
cache_bytes = args.layers * 2 * cfg["hidden_dim"] * (R // N * prefix + R * mean_suffix) * elem
res = {"metric": "image tokens/s, classifier-free guided sampling with KV cache", "value": B * N * 256 / sec, "unit": "tokens/s",
       "images_per_s": B * N / sec, "gpu": gpu.stdout.strip().splitlines()[0], "batch": B, "prompts": B, "samples": N,
       "rows": R, "cuda_graphs": bool(args.graphs),
       "top_k": 64, "top_p": args.top_p, "prompt_frac": args.prompt_frac,
       "seconds_per_image": sec, "launches_per_image": (_lib.launch_count() - l0) // args.reps,
       "operand_bytes": elem, "weight_stream_gb_per_step": weight_bytes / 1e9, "cache_gb_per_step": cache_bytes / 1e9,
       "hbm_stream_gbs": (weight_bytes + cache_bytes) * steps / sec / 1e9, "config": cfg}
if args.logprobs:
    m.generate(text, seg, return_logprobs=True, **kw)     # warm-up of the logp entry
    times = {False: [], True: []}
    for i in range(args.reps):
        for flag in ((False, True) if i % 2 == 0 else (True, False)):
            torch.cuda.synchronize()
            e0.record()
            m.generate(text, seg, return_logprobs=flag, **kw)
            e1.record()
            torch.cuda.synchronize()
            times[flag].append(e0.elapsed_time(e1) * 1e-3)
    plain, logp = (sorted(times[f])[len(times[f]) // 2] for f in (False, True))
    res.update({"logprobs_seconds_per_call_median": logp, "plain_seconds_per_call_median": plain,
                "logprobs_relative_cost": logp / plain - 1, "logprobs_seconds_all": times[True], "plain_seconds_all": times[False]})
if args.sweep:
    scales = [1.5 + 3.5 * j / max(args.sweep - 1, 1) for j in range(args.sweep)]
    sweep_kw = dict(kw, num_samples=args.sweep, guidance_scale=torch.tensor([s for _ in range(B) for s in scales], device=dev))
    m_rows = copy.copy(m)     # the same parameters, its own sampler cache: with --graphs neither arm recaptures the other's graphs
    arms = {"per_row": lambda: m_rows.generate(text, seg, **sweep_kw),
            "scalar_calls": lambda: [m.generate(text, seg, **dict(kw, num_samples=1, guidance_scale=s)) for s in scales]}
    for f in arms.values():                                          # warm-up (and graph captures) of both arms
        f()
    times = {k: [] for k in arms}
    for i in range(args.reps):
        for k in (("per_row", "scalar_calls") if i % 2 == 0 else ("scalar_calls", "per_row")):
            torch.cuda.synchronize()
            e0.record()
            arms[k]()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e-3)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    # the draw kernel alone: per-row arrays (u or seeds) against the scalar entry at the same values, alternating
    kern = {}
    V = cfg["image_vocab_size"]
    for Rk in (8, 128, 256):
        lg = torch.randn(Rk, V, device=dev) * 2.5
        u = torch.rand(Rk, device=dev)
        tok, lp = torch.empty(Rk, dtype=torch.int64, device=dev), torch.empty(Rk, device=dev)
        tt, kk, pp = (torch.full((Rk,), 1.0, device=dev), torch.full((Rk,), 64, dtype=torch.int32, device=dev),
                      torch.full((Rk,), 1.0 if args.top_p is None else args.top_p, device=dev))
        sd = torch.arange(Rk, dtype=torch.int64, device=dev)
        p = 1.0 if args.top_p is None else args.top_p
        calls = {"scalar": lambda: _lib.call("mas_sample_filtered_logp", lg, V, Rk, V, 1.0, 64, p, u, None, None, 0, tok, lp, 1),
                 "rows_u": lambda: _lib.call("mas_sample_rows", lg, V, Rk, V, tt, kk, pp, u, None, 0, None, None, 0, tok, lp, 1),
                 "rows_seeds": lambda: _lib.call("mas_sample_rows", lg, V, Rk, V, tt, kk, pp, None, sd, 7, None, None, 0, tok, lp, 1)}
        per = {k: [] for k in calls}
        for f in calls.values():
            for _ in range(20):
                f()
        for i in range(7):
            for k in (list(calls) if i % 2 == 0 else list(calls)[::-1]):
                torch.cuda.synchronize()
                e0.record()
                for _ in range(200):
                    calls[k]()
                e1.record()
                torch.cuda.synchronize()
                per[k].append(e0.elapsed_time(e1) * 1e3 / 200)
        kern[str(Rk)] = {k: sorted(v)[len(v) // 2] for k, v in per.items()}
    res.update({"sweep": args.sweep, "sweep_scales": scales, "sweep_images": B * args.sweep,
                "sweep_per_row_seconds_median": med["per_row"], "sweep_scalar_calls_seconds_median": med["scalar_calls"],
                "sweep_per_row_images_per_s": B * args.sweep / med["per_row"],
                "sweep_scalar_calls_images_per_s": B * args.sweep / med["scalar_calls"],
                "sweep_seconds_all": times, "sampler_us_per_launch_median_V8192": kern})
print(json.dumps(res))
