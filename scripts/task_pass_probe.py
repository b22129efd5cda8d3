"""The process histograms the bench workload leaves behind, which `bench.py --dump-outputs` does not write.

    python scripts/task_pass_probe.py --out DIR [--steps 20 --warmup 3] [--profile 8]

Builds the bench's two batches (bench.gen_events_gpu, same seeds, same engine sizes), registers them, runs the same warm-up and
timed steps, then writes every registered task's three histograms (cpu %, cpu delay, blkio delay; export_hist) as
DIR/task_hist_{count,sum,total_max}.npy (int64 / uint64, exact), with the task ids in DIR/task_ids.npy. Two builds that apply the
process records the same way write byte-identical files. With --profile N, N more batches run under torch.profiler afterwards and
the per-batch device time of each drain pass and of ingest_kernel is printed as one JSON line."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from gyeeta_b200 import engine as ge  # noqa: E402
from gyeeta_b200 import synth  # noqa: E402

TASK_HISTS = (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY)


def task_ids(rank=0):
    """the bench's process ids (bench.gen_events_gpu)"""
    return synth.splitmix64(np.arange(1, bench.NTASK + 1, dtype=np.uint64) + np.uint64((1 << 40) + rank * bench.NTASK))


def export_task_hists(eng, ids):
    """-> (ids found, counts [k, 3, 15] uint64, sums [k, 3, 15] int64, {total, max} [k, 3, 2] int64)"""
    found, cnt, sm, tm = [], [], [], []
    for id_ in ids.tolist():
        hs = [eng.export_hist(id_, w) for w in TASK_HISTS]
        if any(h is None for h in hs):
            assert all(h is None for h in hs), hex(id_)
            continue
        found.append(id_)
        cnt.append([h[0]["count"].astype(np.uint64) for h in hs])
        sm.append([h[0]["sum"].astype(np.int64) for h in hs])
        tm.append([[np.int64(h[1]), np.int64(h[2])] for h in hs])
    return (np.array(found, dtype=np.uint64), np.array(cnt, dtype=np.uint64).reshape(-1, 3, 15),
            np.array(sm, dtype=np.int64).reshape(-1, 3, 15), np.array(tm, dtype=np.int64).reshape(-1, 3, 2))


def profile_batches(eng, ev_devs, n, nbatches):
    """device time per batch of ingest_kernel and of each drain pass over nbatches batches, torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(nbatches):
            eng.ingest_device_ptr(ev_devs[i % len(ev_devs)].data_ptr(), n)
        eng.sync()
        torch.cuda.synchronize()
    out = {"ingest_kernel": 0.0, "tcp_pass": 0.0, "task_pass": 0.0}
    for e in prof.key_averages():
        key = e.key
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if "drain_kernel<true" in key or "drain_kernelILb1" in key:
            out["task_pass"] += us
        elif "drain_kernel<false" in key or "drain_kernelILb0" in key:
            out["tcp_pass"] += us
        elif "ingest_kernel" in key:
            out["ingest_kernel"] += us
    return {k: round(v / 1000.0 / nbatches, 4) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the .npy files")
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

    ids, cnt, sm, tm = export_task_hists(eng, task_ids())
    os.makedirs(args.out, exist_ok=True)
    for name, a in (("task_ids", ids), ("task_hist_count", cnt), ("task_hist_sum", sm), ("task_hist_total_max", tm)):
        np.save(os.path.join(args.out, name + ".npy"), a)
    res = {"tasks": int(len(ids)), "process_events": int(eng.stats()["events_task"])}
    if args.profile:
        res["ms_per_batch"] = profile_batches(eng, ev_devs, n, args.profile)
        res["gpu"] = torch.cuda.get_device_name(0)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
