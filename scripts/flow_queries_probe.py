"""What GYSK_FLAG_FLOW_QUERIES costs on the bench workload, and the tables it leaves behind.

    python scripts/flow_queries_probe.py [--steps 10 --warmup 2] [--profile 8]

Runs the bench's two batches of 100 M mixed events (bench.gen_events_gpu, same seeds and engine sizes as bench.py) through an engine
without the flag and one with it, one after the other. For each it prints one JSON line: the SHA-256 of the whole connection count-min
(export_cms, which the flag must leave alone) and, with the flag, of both flow query tables; the direct-path counts of the last batch;
the wall time per batch over the timed steps; with --profile N the device ms per batch of each kernel over N more batches
(torch.profiler), including one gysk_flush and one gysk_merge_prepare. The card's name and power limit are read in the same run."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.flow_agg_probe import profile_batches  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def profile_flush_merge(eng):
    """device ms of one gysk_flush and one gysk_merge_prepare (torch.profiler), per kernel"""
    from torch.profiler import ProfilerActivity, profile
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.flush(5)
        eng.merge_prepare()
        eng.sync()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        out[e.key[:60]] = round(us / 1000.0, 4)
    return {k: v for k, v in sorted(out.items(), key=lambda kv: -kv[1]) if v > 0}


def run(flag, args, ev_devs, n):
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23, flow_queries=flag)
    eng.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    for ev in ev_devs:                      # registers the services and tasks, as bench.py does
        eng.ingest_device_ptr(ev.data_ptr(), n)
    for i in range(args.warmup):
        eng.ingest_device_ptr(ev_devs[i % 2].data_ptr(), n)
    eng.sync()
    t0 = time.perf_counter()
    for i in range(args.steps):
        eng.ingest_device_ptr(ev_devs[i % 2].data_ptr(), n)
    eng.sync()
    ms = (time.perf_counter() - t0) * 1000.0 / args.steps
    res = {"flow_queries": flag, "ms_per_batch_wall": round(ms, 3), "cms_sha256": hashlib.sha256(eng.export_cms().tobytes()).hexdigest(),
           "flow_direct_last_batch": eng.last_batch_flow_direct(), "events_resp": int(eng.stats()["events_resp"])}
    if flag:
        res["cmsq_cur_sha256"] = hashlib.sha256(eng.export_cms_queries().tobytes()).hexdigest()
        res["cmsq_last_sha256"] = hashlib.sha256(eng.export_cms_queries(True).tobytes()).hexdigest()
        res["flow_query_direct_last_batch"] = eng.last_batch_flow_query_direct()
    if args.profile:
        res["ms_per_batch"] = profile_batches(eng, ev_devs, n, args.profile)
        res["ms_flush_merge"] = profile_flush_merge(eng)
    res["gpu"] = card()
    print(json.dumps(res), flush=True)
    del eng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--profile", type=int, default=0, metavar="N", help="afterwards, time N more batches with torch.profiler")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = args.events
    ev_devs = [bench.gen_events_gpu(torch, n, 1234 + 7919 * b, 0, 1, dev) for b in range(2)]
    torch.cuda.synchronize()
    for flag in (False, True):
        run(flag, args, ev_devs, n)


if __name__ == "__main__":
    main()
