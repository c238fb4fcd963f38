"""Tokens/s of classifier-free-guided sampling with the KV cache (BASELINE.json configs[4]: 24 layers, 1024 wide, 16
heads, 128 text + 256 segmentation tokens -> 256 image tokens of an 8192-code vocabulary; random-init weights).
One JSON line; not part of bench.py's headline (the reference has no sampler to compare with: SURVEY.md 8f-3). It carries the
GPU's name and power limit, and the HBM bytes a decode step streams on the path actually taken: up to 8 rows fp32 weights and
fp32 KV cache, above 8 rows fp16 weights and fp16 cache (the cache read at the mean cache length of the image positions).
--top-p adds the nucleus filter to the draw (top-k 64 stays); --prompt-frac F forces a random share F of the image positions
(an image prompt, random tokens): the forced positions are still decoded one step each, so tokens/s counts every position.
Usage: python tools/bench_sampling.py [--batch B] [--reps N] [--graphs] [--top-p P] [--prompt-frac F]"""
import argparse
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
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--layers", type=int, default=24)
ap.add_argument("--graphs", action="store_true", help="replay each position's decode step from a CUDA graph")
ap.add_argument("--top-p", type=float, default=None, help="nucleus filter of the draw (default: off)")
ap.add_argument("--prompt-frac", type=float, default=0.0, help="share of image positions forced by a random image prompt")
args = ap.parse_args()
dev = torch.device("cuda:0")
torch.manual_seed(0)
cfg = dict(num_layers=args.layers, hidden_dim=1024, num_attn_heads=16, image_vocab_size=8192, seg_vocab_size=1024, text_vocab_size=49408,
           image_tokens_per_dim=16, seg_tokens_per_dim=16, text_length=128)
m = MakeAScene(**cfg).to(dev).eval()
m.device = dev
B = args.batch
text = torch.randint(1, 40000, (B, 128), device=dev)
seg = torch.randint(0, 1024, (B, 256), device=dev)
gen = torch.Generator(device=dev).manual_seed(1)
kw = dict(guidance_scale=3.0, temperature=1.0, top_k=64, top_p=args.top_p, generator=gen, use_graphs=args.graphs)
if args.prompt_frac > 0:
    kw["img_tokens"] = torch.randint(0, cfg["image_vocab_size"], (B, 256), device=dev)
    kw["img_mask"] = torch.rand(B, 256, device=dev) < args.prompt_frac
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
R = 2 * B
elem = 4 if R <= ops.DECODE_F32_ROWS else 2
params = sum(p.numel() for n, p in m.named_parameters() if "embedding" not in n)
prefix, steps = 128 + 256, 255
mean_len = prefix + (steps + 1) / 2                       # cache positions read by the step of image position t: prefix + t + 1
weight_bytes = params * elem
cache_bytes = args.layers * R * 2 * cfg["hidden_dim"] * mean_len * elem
print(json.dumps({"metric": "image tokens/s, classifier-free guided sampling with KV cache", "value": B * 256 / sec, "unit": "tokens/s",
                  "gpu": gpu.stdout.strip().splitlines()[0], "batch": B, "rows": R, "cuda_graphs": bool(args.graphs),
                  "top_k": 64, "top_p": args.top_p, "prompt_frac": args.prompt_frac,
                  "seconds_per_image": sec, "launches_per_image": (_lib.launch_count() - l0) // args.reps,
                  "operand_bytes": elem, "weight_stream_gb_per_step": weight_bytes / 1e9, "cache_gb_per_step": cache_bytes / 1e9,
                  "hbm_stream_gbs": (weight_bytes + cache_bytes) * steps / sec / 1e9, "config": cfg}))
