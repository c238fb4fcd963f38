"""The VQ-SEG objective VQVAEWithBCELoss (losses/loss_seg.py:25-41) three ways, on logits of the model's shape (the padded
channels-last view [B, 159, H, W] with channel pitch 160 that the decoder's last convolution returns):

  reference:       the reference's own class (torch: sigmoid, MSE, BCE and their backward over the logits);
  kernel dense:    losses.scene_loss.VQVAEWithBCELoss on the dense fp32 [B, 159, H, W] map (mas_bce_mse_cl_*);
  kernel compact:  the same module on the compact uint8 [B, 4, H, W] map (mas_bce_mse_scene_*).

    python tools/bench_seg_loss.py [--batches 8,32] [--res 256] [--iters 20] [--rounds 5] [--steps 3]

Prints the card and its power limit, then per batch:
  loss:    forward + backward of the loss alone (torch.autograd.grad to the logits, as the decoder's backward receives it),
           CUDA events over --iters calls, the arms alternated over --rounds rounds, median / min / max of the rounds; the
           loss of each arm;
  memory:  torch.cuda.max_memory_allocated over one forward + backward of the loss, above what was allocated before it
           (logits, targets and the model's buffers not counted);
  step:    a whole VQ-SEG training step of the seg_config model (bench.py's SEG_CFG) with each objective, the reference fed the
           dense map, CUDA events over --steps steps, alternated over --rounds rounds.
The reference class is loaded from the copy of losses/loss_seg.py under oracle/_ref/ (python oracle/vendor_ref.py, or
build()). The labels are random valid maps; the dense arms get their expansion, so every arm computes the same loss."""
import argparse
import importlib.util
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


def reference_loss_seg():
    path = os.path.join(ROOT, "oracle", "_ref", "losses", "loss_seg.py")
    if not os.path.exists(path):
        raise SystemExit("%s is missing: run build() or `python oracle/vendor_ref.py` first" % path)
    spec = importlib.util.spec_from_file_location("_ref_loss_seg_bench", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


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


def alternate(arms, iters, rounds):
    """{name: sorted per-round ms} with the arms' order reversed every other round."""
    times = {name: [] for name in arms}
    names = list(arms)
    for r in range(rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
            arms[name]()
            times[name].append(events_ms(arms[name], iters))
    return {k: sorted(v) for k, v in times.items()}


def report(kind, times, extra=""):
    for name, t in times.items():
        print("%-5s %-15s ms: median %8.3f  min %8.3f  max %8.3f  (%d rounds)%s"
              % (kind, name, t[len(t) // 2], t[0], t[-1], len(t), extra))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8,32")
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from bench import build_model
    from losses import scene_loss
    from mas_b200 import ops
    ref = reference_loss_seg()
    dev = torch.device("cuda:0")
    R = args.res
    print("card: %s (name, power limit, max SM clock)" % card())
    ref_fn = ref.VQVAEWithBCELoss().to(dev)
    ker_fn = scene_loss.VQVAEWithBCELoss().to(dev)
    model = build_model("vqseg").to(dev)
    q = torch.tensor(0.25, device=dev)
    for B in (int(b) for b in args.batches.split(",")):
        print("---- batch %d, %dx%d, logits [%d, 159, %d, %d] channels-last, pitch 160" % (B, R, R, B, R, R))
        lab = labels(B, R, R, seed=B).to(dev)
        dense = ops.scene_expand(lab)
        base = torch.randn(B, R, R, 160, device=dev) * 3
        base[..., 159:] = 0
        logits = base.permute(0, 3, 1, 2)[:, :159].requires_grad_(True)
        arms = {"reference": lambda: ref_fn(q, dense, logits), "kernel dense": lambda: ker_fn(q, dense, logits),
                "kernel compact": lambda: ker_fn(q, lab, logits)}
        values = {}

        def fwd_bwd(fn, name=None):
            loss = fn()
            torch.autograd.grad(loss, logits)      # the gradient as the decoder's backward receives it: no .grad copy
            if name:
                values[name] = float(loss.detach())

        for name, fn in arms.items():                    # warm-up, sizes the library's workspace, records the loss
            fwd_bwd(fn, name)
        print("loss values: " + "  ".join("%s %.9g" % kv for kv in values.items()))
        report("loss", alternate({k: (lambda fn=fn: fwd_bwd(fn)) for k, fn in arms.items()}, args.iters, args.rounds),
               "  fwd+bwd")
        for name, fn in arms.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            before = torch.cuda.memory_allocated(dev)
            fwd_bwd(fn)
            torch.cuda.synchronize()
            print("mem   %-15s max_memory_allocated over fwd+bwd: %9.1f MB above the inputs"
                  % (name, (torch.cuda.max_memory_allocated(dev) - before) / 2 ** 20))
        del logits, base
        torch.cuda.empty_cache()

        def step(loss_fn, x):
            model.zero_grad(set_to_none=True)
            dec, diff = model(x)
            loss_fn(diff, x, dec).backward()
        steps = {"reference": lambda: step(ref_fn, dense), "kernel dense": lambda: step(ker_fn, dense),
                 "kernel compact": lambda: step(ker_fn, lab)}
        report("step", alternate(steps, args.steps, args.rounds), "  whole VQ-SEG step")
        model.zero_grad(set_to_none=True)
        del dense, lab
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
