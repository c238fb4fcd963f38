"""Kernels of a decode step above 8 rows, timed with CUDA events around a CUDA graph of many launches (device time, no host
launch overhead), at BASELINE.json configs[4] extents: 1024 wide, 16 heads of 64, 640-token cache, mean cache length 512.
Consecutive launches rotate through enough copies of the weights / caches to exceed the 50 MB L2, so the operands stream
from HBM as they do in a decode step. One JSON line per measurement:
  * the five decode Linear shapes (qkv, out_proj, lin1 + GELU, lin2, to_logits) at R rows: the narrow split form
    mas_linear_rows_f16 against the training kernel mas_gemm_rows_f16 (+ mas_gelu_forward for lin1) on the same fp16 copy,
    as ms and weight-stream GB/s, and the form ops.linear_small selects;
  * attention decode on the fp16 cache against the fp32 one, as ms and cache GB/s (k and v bytes read);
  * the shared-prefix decode attention of generate(num_samples=n) (a 384-position prefix cache per group of n rows, a
    256-position suffix cache per row) against mas_attn_decode_append on the concatenated cache, at position 511 (cache length
    512, the mean of the image positions), fp16 caches: us per launch, and GB/s of the cache bytes the step needs (the
    shared form needs each group's prefix once). The launcher's rows per block ("auto") is timed beside one row per block,
    where a group's prefix can only be shared through L2 hits between adjacent blocks.
Usage: python tools/bench_decode.py [--rows 16 32 64 128 256] [--iters N] [--only linear|attn|shared] [--shared-rows 16 64 256]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]
import torch  # noqa: E402
from mas_b200 import _lib as L, ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, nargs="+", default=[16, 32, 64, 128, 256])
ap.add_argument("--iters", type=int, default=200)
ap.add_argument("--only", choices=["linear", "attn", "shared"], default=None)
ap.add_argument("--shared-rows", type=int, nargs="+", default=[16, 64, 256])
ap.add_argument("--samples", type=int, nargs="+", default=[1, 4, 8, 16])
args = ap.parse_args()
dev = torch.device("cuda:0")
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
print(json.dumps({"gpu": gpu.stdout.strip().splitlines()[0]}), flush=True)
L2_COLD = 160 << 20          # bytes touched between two uses of the same copy: over three times the H100's 50 MB L2


def copies(nbytes):
    return max(1, -(-L2_COLD // nbytes))


def timed(fn):
    """fn(i): the i-th launch of the window. Milliseconds per launch."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i in range(3):
            fn(i)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(args.iters):
            fn(i)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (5 * args.iters)


H = 1024
SHAPES = [("qkv", 3 * H, H, 0), ("out_proj", H, H, 0), ("lin1", 4 * H, H, 1), ("lin2", H, 4 * H, 0), ("to_logits", 8192, H, 0)]
torch.manual_seed(0)
for name, N, K, act in (SHAPES if args.only in (None, "linear") else []):
    wb = N * K * 2
    ws_ = [torch.randn(N, K, device=dev) / K ** 0.5 for _ in range(copies(wb))]
    wpk = [ops._packed_linear_weight(w, False, dev) for w in ws_]
    b = torch.randn(N, device=dev)
    for R in args.rows:
        x16, am = ops.rows_to_half(torch.randn(R, K, device=dev))
        y = torch.empty(R, N, device=dev)
        g = torch.empty(R, N, device=dev)
        ws = torch.empty(max(int(L.query("mas_linear_rows_f16_ws_bytes", R, N, K)), 16), dtype=torch.uint8, device=dev)

        def narrow(i):
            L.call("mas_linear_rows_f16", x16, R, K, wpk[i % len(wpk)], y, N, N, b, am, act, ws, ws.numel())

        def training(i):
            L.call("mas_gemm_rows_f16", x16, R, K, wpk[i % len(wpk)], y, N, N, b, None, am, 1.0)
            if act:
                L.call("mas_gelu_forward", y, g, y.numel())
        t_new, t_old = timed(narrow), timed(training)
        print(json.dumps({"kernel": "linear", "shape": name, "N": N, "K": K, "rows": R, "gelu": bool(act), "weight_copies": len(wpk),
                          "narrow_ms": round(t_new, 5), "training_ms": round(t_old, 5),
                          "narrow_weight_gbs": round(wb / t_new / 1e6, 1), "training_weight_gbs": round(wb / t_old / 1e6, 1),
                          "narrow_faster": t_new < t_old, "selected": "narrow" if ops.decode_narrow_rows(R, N, K) else "training"}),
              flush=True)
    del ws_, wpk

heads, hd, tmax, length = 16, 64, 640, 512
for R in (args.rows if args.only in (None, "attn") else []):
    qkv = torch.randn(R, 3 * heads * hd, device=dev)
    ctx = torch.empty(R, heads * hd, device=dev)
    res = {"kernel": "attn_decode", "rows": R, "heads": heads, "hd": hd, "len": length}
    for tag, dt, entry in (("f16", torch.float16, "mas_attn_decode_f16"), ("f32", torch.float32, "mas_attn_decode")):
        nb = 2 * R * heads * tmax * hd * torch.tensor([], dtype=dt).element_size()
        caches = [(torch.randn(R, heads, tmax, hd, device=dev).to(dt), torch.randn(R, heads, tmax, hd, device=dev).to(dt))
                  for _ in range(copies(nb))]
        t = timed(lambda i: L.call(entry, qkv, caches[i % len(caches)][0], caches[i % len(caches)][1], ctx, R, heads, hd, tmax, length))
        cache_bytes = 2 * R * heads * length * hd * caches[0][0].element_size()
        res[tag + "_ms"] = round(t, 5)
        res[tag + "_cache_gbs"] = round(cache_bytes / t / 1e6, 1)
        res[tag + "_copies"] = len(caches)
        del caches
    res["f16_share_of_3350_gbs"] = round(res["f16_cache_gbs"] / 3350, 3)
    print(json.dumps(res), flush=True)

prefix, tsuf, pos = 384, 256, 511
for R in (args.shared_rows if args.only in (None, "shared") else []):
    qkv = torch.randn(R, 3 * heads * hd, device=dev)
    ctx = torch.empty(R, heads * hd, device=dev)
    full = 2 * R * heads * (pos + 1) * hd * 2                                     # k + v bytes of the unshared step
    cc = [(torch.randn(R, heads, tmax, hd, device=dev).half(), torch.randn(R, heads, tmax, hd, device=dev).half()) for _ in range(copies(full))]
    t_ref = timed(lambda i: L.call("mas_attn_decode_append_f16", qkv, cc[i % len(cc)][0], cc[i % len(cc)][1], ctx, R, heads, hd, tmax, pos))
    del cc
    for n in args.samples:
        if R % n:
            continue
        need = 2 * heads * hd * 2 * (R // n * prefix + R * (pos + 1 - prefix))   # each group's prefix once, every row's suffix
        sc = [tuple(torch.randn(r, heads, t, hd, device=dev).half() for r, t in ((R // n, prefix), (R // n, prefix), (R, tsuf), (R, tsuf)))
              for _ in range(copies(need))]
        res = {"kernel": "attn_decode_shared_append_f16", "rows": R, "samples": n, "heads": heads, "hd": hd, "len": pos + 1,
               "unshared_us": round(t_ref * 1e3, 2), "unshared_needed_gbs": round(full / t_ref / 1e6, 1), "copies": len(sc)}
        for tag, rpb in (("auto", 0), ("one_row_per_block", 1)):
            t = timed(lambda i: L.call("mas_attn_decode_shared_append_f16", qkv, *sc[i % len(sc)][:2], *sc[i % len(sc)][2:], ctx, R, n, heads,
                                       hd, prefix, tsuf, pos, rpb))
            res[tag + "_us"] = round(t * 1e3, 2)
            res[tag + "_needed_gbs"] = round(need / t / 1e6, 1)
            res[tag + "_speedup"] = round(t_ref / t, 3)
        res["needed_bytes_share"] = round(need / full, 3)
        print(json.dumps(res), flush=True)
        del sc
