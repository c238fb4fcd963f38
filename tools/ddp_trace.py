"""Where does the multi-GPU step time go?  Run under torchrun (world_size >= 2) on the GPU box:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29544 tools/ddp_trace.py
(1) times the bench step under several DistributedDataParallel / NCCL configurations (CUDA events, max over ranks);
(2) traces two steps of the default configuration with torch.profiler (CUPTI) and prints, for rank 0, the NCCL kernels, the
    busy / idle time of the compute stream and the kernels that slowed down relative to a single-GPU step.
No nsys in the image: the kineto trace is the timeline."""
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import bench  # noqa: E402


def main():
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    img = torch.rand(bench.BATCH, 3, bench.RES, bench.RES, generator=torch.Generator().manual_seed(1234 + rank)).to(dev)

    def make(kind):
        m = bench.build_model().to(dev)
        if world == 1 or kind == "nosync":
            return m, m
        kw = dict(device_ids=[local], gradient_as_bucket_view=True)
        if kind == "static":
            kw.update(static_graph=True)
        if kind == "nobcast":
            kw.update(broadcast_buffers=False)
        if kind == "bucket100":
            kw.update(bucket_cap_mb=100, broadcast_buffers=False)
        if kind == "bucket400":
            kw.update(bucket_cap_mb=400, broadcast_buffers=False)
        return m, torch.nn.parallel.DistributedDataParallel(m, **kw)

    def step(net):
        net.zero_grad(set_to_none=True)
        dec, diff = net(img)
        loss = (img - dec).abs().mean() + diff
        loss.backward()
        return loss

    def timed(net, steps=4, warm=3):
        for _ in range(warm):
            step(net)
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            step(net)
        e1.record()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1) / steps], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms)

    kinds = ["default", "nosync", "nobcast", "static", "bucket100", "bucket400"] if world > 1 else ["default"]
    res = {}
    for k in kinds:
        m, net = make(k)
        res[k] = timed(net)
        if rank == 0:
            print("config %-10s %8.2f ms/step" % (k, res[k]), flush=True)
        del m, net
        torch.cuda.empty_cache()

    # ---- trace of the default configuration
    from torch.profiler import ProfilerActivity, profile
    m, net = make("default")
    for _ in range(3):
        step(net)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        for _ in range(2):
            step(net)
        torch.cuda.synchronize()
    if rank == 0:
        evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        ks = {}
        for e in evs:
            c, t = ks.get(e.name, (0, 0.0))
            ks[e.name] = (c + 1, t + e.device_time)
        tot = sum(t for _, t in ks.values())
        print("\nCUDA activity over 2 traced steps (rank 0): %.2f ms of kernels+memcpy" % (tot / 1e3))
        for name, (c, t) in sorted(ks.items(), key=lambda kv: -kv[1][1])[:14]:
            print("  %-70s n=%5d %9.2f ms" % (name[:70], c, t / 1e3))
        nccl = {k: v for k, v in ks.items() if "nccl" in k.lower()}
        print("NCCL kernels:", {k[:60]: (c, round(t / 1e3, 2)) for k, (c, t) in nccl.items()})
        # busy / idle of the union of all device activity
        iv = sorted((e.time_range.start, e.time_range.end) for e in evs)
        busy, cur_s, cur_e = 0.0, None, None
        for s, e in iv:
            if cur_e is None or s > cur_e:
                if cur_e is not None:
                    busy += cur_e - cur_s
                cur_s, cur_e = s, e
            else:
                cur_e = max(cur_e, e)
        busy += cur_e - cur_s
        span = iv[-1][1] - iv[0][0]
        print("device span %.2f ms, busy (union) %.2f ms, idle %.2f ms over 2 steps" % (span / 1e3, busy / 1e3, (span - busy) / 1e3))
        out = os.path.join(tempfile.gettempdir(), "ddp_trace_w%d.json" % world)
        try:
            prof.export_chrome_trace(out)
        except Exception as e:  # noqa: BLE001
            print("trace export failed:", e)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
