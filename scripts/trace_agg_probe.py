"""Where the time of a window with request traces goes: ingest, the sort + t-digest chain and the flush, with trace rows off and on.

    python scripts/trace_agg_probe.py [--svcs 1000] [--samples 10000000] [--batches 4] [--reps 3]

A window of `samples` request traces over `svcs` traced services with a Zipf(1.1) head, sent as the engine receives an API_TRAN
stream: a GYSK_EV_RESP and a GYSK_EV_TRACE event per record, in `batches` device batches, then gysk_flush. The same RESP events go
through an engine without trace rows for the baseline. Prints one JSON line: per configuration the device ms of the ingest kernel and of
the sort + t-digest chain per window (gysk_profile_read), the flush ms (CUDA events), the radix passes of the batch sort, and with
--profile the device time of bins_merge_kernel and trace_keys_kernel (torch.profiler). The line also names the GPU and its power
limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gyeeta_b200 import engine as ge  # noqa: E402
from tests import trace_agg as ta  # noqa: E402


def gpu_desc():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def window_events(rng, svcs, samples):
    ids = (np.arange(1, svcs + 1, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15 >> 20)) | np.uint64(1)
    z = rng.zipf(1.1, size=samples)
    gid = ids[(z - 1) % svcs]
    usec = np.exp(rng.normal(8.0, 1.5, size=samples)).astype(np.uint64)
    rec = ta.api_tran(gid, usec, rng.integers(0, 1 << 16, size=samples).astype(np.uint64),
                      rng.integers(0, 1 << 20, size=samples).astype(np.uint64), np.ones(samples, np.uint64))
    ev = np.empty(2 * samples, dtype=ge.EVENT_DTYPE)
    ev[0::2], ev[1::2] = ta.resp_events(rec), ta.trace_events(rec)
    return ev


def run(ev, rows, batches, reps, prof):
    per = (len(ev) + batches - 1) // batches
    eng = ge.Engine(max_svcs=1 << 14, max_tasks=1 << 10, max_batch=per + 1024, stage_batch=per + 1024, max_trace_svcs=rows)
    dev = [torch.from_numpy(ev[i * per:(i + 1) * per].view(np.uint8)).cuda() for i in range(batches)]
    s = torch.cuda.Stream()
    res = dict(ingest_ms=[], chain_ms=[], flush_ms=[])
    for rep in range(reps + 1):
        eng.profile_enable(True)
        for i, d in enumerate(dev):
            eng.ingest_device_ptr(d.data_ptr(), len(d) // 32)
        eng.sync()
        ms_ing, ms_td, _ = eng.profile_read()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        eng.flush(100 + 5 * rep)
        eng.sync()
        b.record()
        torch.cuda.synchronize()
        if rep:                                     # the first window warms up
            res["ingest_ms"].append(ms_ing); res["chain_ms"].append(ms_td); res["flush_ms"].append(a.elapsed_time(b))
    out = {k: float(np.median(v)) for k, v in res.items()}
    if prof:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            for d in dev:
                eng.ingest_device_ptr(d.data_ptr(), len(d) // 32)
            eng.sync()
            torch.cuda.synchronize()
        passes = 0
        for e in p.key_averages():
            us = getattr(e, "device_time_total", 0) or 0
            for name in ("bins_merge_kernel", "trace_keys_kernel", "ingest_kernel", "long_sum_kernel", "segs_mark_kernel"):
                if name in e.key:
                    out[name + "_ms"] = out.get(name + "_ms", 0.0) + us / 1000.0
            if "os_pass_kernel" in e.key:
                out["radix_ms"] = out.get("radix_ms", 0.0) + us / 1000.0
                passes += e.count
        out["radix_passes_per_batch"] = passes / batches
    if rows:
        out["trace_rows_in_use"], out["trace_dropped"] = eng.trace_info()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--svcs", type=int, default=1000)
    ap.add_argument("--samples", type=int, default=10_000_000)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    ev = window_events(rng, a.svcs, a.samples)
    off = run(ev[ev["type"] == ge.EV_RESP], 0, a.batches, a.reps, a.profile)
    on = run(ev, 1024, a.batches, a.reps, a.profile)
    print(json.dumps(dict(gpu=gpu_desc(), svcs=a.svcs, samples_per_window=a.samples, batches=a.batches, trace_off=off, trace_on=on)))


if __name__ == "__main__":
    main()
