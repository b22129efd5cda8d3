"""The count-min table the bench workload leaves behind, whole, and where a batch's device time goes.

    python scripts/flow_agg_probe.py [--steps 20 --warmup 3] [--profile 8]

Builds the bench's two batches (bench.gen_events_gpu, same seeds, same engine sizes), registers them, runs the same warm-up and
timed steps, then prints one JSON line with the SHA-256 of the whole export_cms() table (`bench.py --dump-outputs` writes only a
sample of its cells): two builds that apply the connection records the same way print the same hash. With --profile N, N more
batches run under torch.profiler afterwards and the line also holds the device time per batch of every kernel, in ms."""
import argparse
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from gyeeta_b200 import engine as ge  # noqa: E402


def profile_batches(eng, ev_devs, n, nbatches):
    """device ms per batch of each kernel over nbatches batches (torch.profiler), the radix passes summed under one name"""
    from torch.profiler import ProfilerActivity, profile
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(nbatches):
            eng.ingest_device_ptr(ev_devs[i % len(ev_devs)].data_ptr(), n)
        eng.sync()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        key = e.key
        if "drain_kernel<true" in key or "drain_kernelILb1" in key:
            key = "task_pass"
        elif "drain_kernel<false" in key or "drain_kernelILb0" in key:
            key = "tcp_pass"
        elif "os_pass_kernel" in key:
            key = "radix_passes"
        else:
            for name in ("ingest_kernel", "bins_merge_kernel", "segs_mark_kernel", "long_sum_kernel", "os_hist_kernel"):
                if name in key:
                    key = name
        out[key] = out.get(key, 0.0) + us
    return {k: round(v / 1000.0 / nbatches, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1]) if v > 0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--profile", type=int, default=0, metavar="N", help="afterwards, time N more batches with torch.profiler")
    args = ap.parse_args()

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = args.events
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23)
    ev_devs = [bench.gen_events_gpu(torch, n, 1234 + 7919 * b, 0, 1, dev) for b in range(2)]
    torch.cuda.synchronize()
    for ev in ev_devs:                      # registers the services and tasks, as bench.py does
        eng.ingest_device_ptr(ev.data_ptr(), n)
    for i in range(args.warmup + args.steps):
        eng.ingest_device_ptr(ev_devs[i % 2].data_ptr(), n)
    eng.sync()

    cms = eng.export_cms()
    res = {"cms_sha256": hashlib.sha256(cms.tobytes()).hexdigest(), "cms_cells": int(len(cms)),
           "connection_events": int(eng.stats()["events_tcp"])}
    if hasattr(eng, "last_batch_flow_direct"):         # absent from builds before the flow table, which the probe also compares
        res["flow_direct_last_batch"] = eng.last_batch_flow_direct()
    if args.profile:
        res["ms_per_batch"] = profile_batches(eng, ev_devs, n, args.profile)
        res["gpu"] = torch.cuda.get_device_name(0)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
