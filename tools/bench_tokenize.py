"""Images per second and peak memory of VQBASE.encode_code, against `model.eval(); model.encode(x)` (under no_grad) on the
same inputs, the two arms alternated within one run:

    python tools/bench_tokenize.py [--rounds 5] [--iters 10] [--out FILE]

Shapes: the img_config model at 256 x 256, batch 1, 8 and 64; the seg_config model (out_channels=159) at 256 x 256 fed
compact scene planes (uint8 [B, 4, H, W]) and fed the dense fp32 map they expand to, batch 8 and 32. Prints the card's name
and power limit first. Each arm: one warm-up call, then --rounds rounds of --iters calls timed with CUDA events; the median
and spread (min - max) over rounds are reported. Peak memory: torch.cuda.max_memory_allocated over one call, the model and
the input included. Needs a CUDA device; there is no CPU arm."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]

IMG = dict(z_channels=256, in_channels=3, out_channels=3, channels=[128, 128, 128, 256, 512, 512], num_res_blocks=2,
           resolution=512, attn_resolutions=[32], dropout=0.0)
SEG = dict(z_channels=256, in_channels=159, out_channels=159, resolution=256, num_res_blocks=2, attn_resolutions=[16],
           dropout=0.0)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s)" % e


def events_ms(fn, iters):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def peak_mb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / 2 ** 20


def model(dd, n_embed, dev):
    from models import VQBASE
    torch.manual_seed(0)
    m = VQBASE(dd, n_embed, 256, 3000, 12500)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    return m.to(dev).eval()


def labels(b, size, seed=0):
    g = torch.Generator().manual_seed(seed)
    lab = torch.stack([torch.randint(0, 134, (b, size // 8, size // 8), generator=g),
                       torch.randint(0, 21, (b, size // 8, size // 8), generator=g),
                       torch.randint(0, 6, (b, size // 8, size // 8), generator=g),
                       torch.randint(0, 3, (b, size // 8, size // 8), generator=g)], 1)
    return lab.repeat_interleave(8, 2).repeat_interleave(8, 3).to(torch.uint8)


def bench(m, x, rounds, iters):
    arms = {"encode_code": lambda: m.encode_code(x)}

    def encode():
        with torch.no_grad():
            return m.encode(x)
    arms["eval encode"] = encode
    out = {}
    tok = m.encode_code(x)
    with torch.no_grad():
        seen = {}
        h = m.quantize.register_forward_hook(lambda _m, _i, o: seen.__setitem__("idx", o[2]))
        encode()
        h.remove()
    same = bool(torch.equal(tok.flatten(), seen["idx"].view(-1)))
    mem = {k: peak_mb(f) for k, f in arms.items()}
    times = {k: [] for k in arms}
    for _ in range(rounds):                                    # alternated: every round times both arms
        for k, f in arms.items():
            times[k].append(events_ms(f, iters))
    b = x.shape[0]
    for k in arms:
        med = statistics.median(times[k])
        out[k] = {"ms": round(med, 3), "ms_min": round(min(times[k]), 3), "ms_max": round(max(times[k]), 3),
                  "images_per_s": round(1000.0 * b / med, 1), "peak_mb": round(mem[k], 1)}
    out["tokens_equal"] = same
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tokenize.py needs a CUDA device: there is no CPU arm (not measured)")
    dev = torch.device("cuda:0")
    info = card()
    print("card:", info, flush=True)
    results = {"card": info, "runs": []}
    m = model(IMG, 8192, dev)
    for b in (1, 8, 64):
        x = (torch.rand(b, 3, 256, 256, generator=torch.Generator().manual_seed(b)) * 2 - 1).to(dev)
        r = dict(model="img_config", input="image fp32", batch=b, **bench(m, x, a.rounds, a.iters))
        print(json.dumps(r), flush=True)
        results["runs"].append(r)
    del m
    torch.cuda.empty_cache()
    from mas_b200 import ops
    m = model(SEG, 1024, dev)
    for b in (8, 32):
        lab = labels(b, 256).to(dev)
        for kind, x in (("compact uint8", lab), ("dense fp32", None)):
            if x is None:
                x = ops.scene_expand(ops.scene_labels(lab))      # the dense [B, 159, H, W] map of the same labels
            r = dict(model="seg_config", input=kind, batch=b, **bench(m, x, a.rounds, a.iters))
            print(json.dumps(r), flush=True)
            results["runs"].append(r)
            del x
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
