"""VQ-SEG training step fed compact scene maps (uint8 [B, 4, H, W] labels, mas_b200.scene) against the same step fed the
dense 159-channel fp32 map they expand to, at the seg_config model (bench.py's SEG_CFG) and batch 32 at 256 x 256.

    python tools/bench_scene_maps.py [--batch 32] [--steps 5] [--rounds 3] [--iters 50]

Prints the card and its power limit, then, with the arms alternated over --rounds rounds of --steps steps each:
  device:  step time with the input already on the device;
  e2e:     step time from a pinned host batch (the host-to-device copy included, loss read back);
  memory:  torch.cuda.max_memory_allocated over one step of each arm, the input counted;
  kernels: mas_scene_expand against mas_nchw_to_nhwc_pad (the padded conv_in operand), and mas_bce_scene_* against
           mas_bce_cl_* (the weighted BCE), CUDA events over --iters launches.
The labels are random valid maps; the dense arm gets their expansion, so both arms compute the same step (the first loss
of each is printed). No optimizer: the weights stay put, only BatchNorm's running statistics move."""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s)" % e


def labels(b, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    planes = []
    for hi in (133, 20, 5):
        code = torch.randint(1, hi + 1, (b, h, w), generator=g)
        planes.append(torch.where(torch.rand(b, h, w, generator=g) < 0.5, code, torch.zeros_like(code)))
    planes.append(torch.randint(0, 3, (b, h, w), generator=g))
    return torch.stack(planes, 1).to(torch.uint8)


def events_ms(fn, iters):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from bench import build_model
    from mas_b200 import _lib as L, ops
    dev = torch.device("cuda:0")
    B, R = args.batch, args.res
    print("card: %s (name, power limit, max SM clock)" % card())
    print("VQ-SEG seg_config model, batch %d, %dx%d, operands %s" % (B, R, R, ops.get_operand_format()))
    model = build_model("vqseg").to(dev)
    pw = torch.ones(159, device=dev)
    pw[153:158] = 20
    lab_host = labels(B, R, R).pin_memory()
    lab_dev = lab_host.to(dev)
    dense_dev = ops.scene_expand(lab_dev)
    dense_host = dense_dev.cpu().pin_memory()
    arms = {"dense": (dense_host, dense_dev), "compact": (lab_host, lab_dev)}
    print("input bytes per step: dense %d, compact %d" % (dense_host.numel() * 4, lab_host.numel()))

    def step(x):
        model.zero_grad(set_to_none=True)
        dec, diff = model(x)
        loss = ops.BCELogitsFn.apply(dec, x, pw) + diff
        loss.backward()
        return loss

    # memory of one step (after a warm-up step of each arm has sized the library's workspace), input counted
    first = {}
    for name, (_, xd) in arms.items():
        first[name] = float(step(xd))
    for name, (_, xd) in arms.items():
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev) - xd.numel() * xd.element_size()
        step(xd)
        torch.cuda.synchronize()
        print("memory  %-8s max_memory_allocated over one step: %9.1f MB" % (name, (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20))
    print("first loss: dense %.9g  compact %.9g  (%s)" % (first["dense"], first["compact"],
                                                         "identical" if first["dense"] == first["compact"] else "DIFFERENT"))

    def e2e(xh):
        x = xh.to(dev, non_blocking=True)
        return float(step(x).item())
    times = {(k, a): [] for k in ("device", "e2e") for a in arms}
    for r in range(args.rounds):
        for kind in ("device", "e2e"):
            for name, (xh, xd) in (list(arms.items()) if r % 2 == 0 else list(arms.items())[::-1]):
                fn = (lambda: step(xd)) if kind == "device" else (lambda: e2e(xh))
                fn()
                times[(kind, name)].append(events_ms(fn, args.steps))
    for kind in ("device", "e2e"):
        for name in arms:
            t = sorted(times[(kind, name)])
            print("%-6s  %-8s ms/step: median %8.2f  min %8.2f  max %8.2f  (%d rounds x %d steps)  %.1f images/s"
                  % (kind, name, t[len(t) // 2], t[0], t[-1], len(t), args.steps, B * 1e3 / t[len(t) // 2]))

    # kernels, CUDA events over many launches at the step's shapes
    del arms, dense_host
    model.zero_grad(set_to_none=True)
    torch.cuda.empty_cache()
    n, c, cp = B, 159, 160
    padded = torch.empty((n, R, R, cp), device=dev)
    k = {}
    k["mas_nchw_to_nhwc_pad"] = events_ms(lambda: L.call("mas_nchw_to_nhwc_pad", dense_dev, padded, n, c, cp, R, R), args.iters)
    pv = padded.permute(0, 3, 1, 2)
    k["mas_scene_expand (padded channels-last)"] = events_ms(lambda: L.call("mas_scene_expand", lab_dev, n, R, R, pv, L.t4(pv)), args.iters)
    k["mas_scene_expand (NCHW)"] = events_ms(lambda: L.call("mas_scene_expand", lab_dev, n, R, R, dense_dev, L.t4(dense_dev)), args.iters)
    logits = torch.randn((n, R, R, cp), device=dev)
    grad = torch.empty_like(logits)
    loss = torch.empty((), device=dev)
    ws = L.workspace(L.query("mas_bce_cl_ws_bytes", n, R, R), dev)
    k["mas_bce_cl_forward"] = events_ms(lambda: L.call("mas_bce_cl_forward", logits, dense_dev, pw, n, c, cp, R, R, loss, ws, ws.numel()), args.iters)
    k["mas_bce_scene_forward"] = events_ms(lambda: L.call("mas_bce_scene_forward", logits, lab_dev, pw, n, cp, R, R, loss, ws, ws.numel()), args.iters)
    k["mas_bce_cl_backward"] = events_ms(lambda: L.call("mas_bce_cl_backward", logits, dense_dev, pw, None, n, c, cp, R, R, grad), args.iters)
    k["mas_bce_scene_backward"] = events_ms(lambda: L.call("mas_bce_scene_backward", logits, lab_dev, pw, None, n, cp, R, R, grad), args.iters)
    for name, ms in k.items():
        print("kernel  %-42s %8.3f ms/launch  (%d launches)" % (name, ms, args.iters))


if __name__ == "__main__":
    main()
