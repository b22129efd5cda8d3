"""Device time per batch of the bench workload's response-key chain: ingest_kernel (which fills the radix passes' digit
histograms), the radix passes over the keys, segs_mark_kernel, long_sum_kernel and bins_merge_kernel.

    python scripts/slot_keys_probe.py [--batches 8] [--warmup 3]

Builds the bench's two batches (bench.gen_events_gpu, same seeds, same engine sizes), ingests them once (registration) and runs
the warm-up steps, then times --batches more batches under torch.profiler. Prints one JSON line: ms per batch of each kernel, the
number of radix-pass launches per batch, the engine's kernel launches in all, and the card, its power limit and SM clock before and after
the run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """name, power limit and current SM clock of GPU 0 as nvidia-smi reports them (read only)"""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi failed: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--events", type=int, default=100_000_000)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from gyeeta_b200 import engine as ge

    res = {"card": card()}
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = args.events
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23)
    ev_devs = [bench.gen_events_gpu(torch, n, 1234 + 7919 * b, 0, 1, dev) for b in range(2)]
    torch.cuda.synchronize()
    for ev in ev_devs:                      # registers the services and tasks, as bench.py does
        eng.ingest_device_ptr(ev.data_ptr(), n)
    for i in range(args.warmup):
        eng.ingest_device_ptr(ev_devs[i % 2].data_ptr(), n)
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.batches):
            eng.ingest_device_ptr(ev_devs[i % 2].data_ptr(), n)
        eng.sync()
        torch.cuda.synchronize()
    names = ["ingest_kernel", "os_pass_kernel", "segs_mark_kernel", "long_sum_kernel", "bins_merge_kernel"]
    out = {k: 0.0 for k in names}
    passes = 0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        for k in names:
            if k in e.key:
                out[k] += us
                if k == "os_pass_kernel":
                    passes += e.count
    launches = eng.stats()["kernel_launches"]
    eng.close()
    res.update({k: round(v / 1000.0 / args.batches, 4) for k, v in out.items()})
    res["radix_passes_per_batch"] = passes / args.batches
    res["kernel_launches_total"] = launches
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
