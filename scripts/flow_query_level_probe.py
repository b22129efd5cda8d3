"""What GYSK_FLAG_FLOW_QUERY_LEVEL costs on the bench workload, with the flag off and on in the same run.

    python scripts/flow_query_level_probe.py [--reps 10] [--events 100000000] [--out DIR]

Two engines with the bench's sizes, one with GYSK_FLAG_FLOW_QUERIES and one with GYSK_FLAG_FLOW_QUERIES | GYSK_FLAG_FLOW_QUERY_LEVEL,
take the bench's two batches of 100 M mixed events (bench.gen_events_gpu, same seeds) one batch per 5-s window. Ten warm-up windows
30 s apart first fill every ring slot, so that each timed flush runs cms_level_roll_kernel at its most (the closing window and ten
slots read, one slot and the level written). Then, per window and engine in alternation: gysk_flush (host clock around flush + sync),
the next batch's ingest (host clock around ingest + sync) and gysk_merge_prepare (host clock around prepare + sync); medians and maxima
over the timed windows. Afterwards one flush of each engine under torch.profiler gives cms_level_roll_kernel's device time per ring.
Prints one JSON line with the SHA-256 of the query level and of the connection count-min (the same with the flag off and on), and the
card's name and power limit read in the same run."""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.flow_queries_probe import card  # noqa: E402


def make_engine(level):
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23, flow_queries=True,
                    flow_query_level=level)
    eng.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    return eng


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def roll_kernel_ms(eng, t):
    """device ms and launches of cms_level_roll_kernel in one gysk_flush (torch.profiler)"""
    from torch.profiler import ProfilerActivity, profile
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.flush(t)
        eng.sync()
        torch.cuda.synchronize()
    ms, n = 0.0, 0
    for e in prof.key_averages():
        if "cms_level_roll_kernel" in e.key:
            us = getattr(e, "device_time_total", None)
            ms += (us if us is not None else e.cuda_time_total) / 1000.0
            n += e.count
    return round(ms, 4), n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = a.events
    ev_devs = [bench.gen_events_gpu(torch, n, 1234 + 7919 * b, 0, 1, dev) for b in range(2)]
    torch.cuda.synchronize()
    engines = {False: make_engine(False), True: make_engine(True)}
    for eng in engines.values():
        for ev in ev_devs:                  # registers the services and tasks, as bench.py does
            eng.ingest_device_ptr(ev.data_ptr(), n)
        eng.sync()
    times = {flag: dict(flush=[], ingest=[], prepare=[]) for flag in engines}
    t = 0
    for w in range(10 + a.reps):
        t += 30 if w < 10 else 5                # ten warm-up windows in ten epochs: every ring slot live
        ev = ev_devs[w % 2]
        for flag, eng in engines.items():       # alternated window by window
            f = timed(lambda: (eng.flush(t), eng.sync()))
            i = timed(lambda: (eng.ingest_device_ptr(ev.data_ptr(), n), eng.sync()))
            p = timed(lambda: (eng.merge_prepare(), eng.sync()))
            if w >= 10:
                times[flag]["flush"].append(f); times[flag]["ingest"].append(i); times[flag]["prepare"].append(p)
    runs = []
    for flag, eng in engines.items():
        med = lambda v: round(float(np.median(v)), 3)
        r = dict(flow_query_level=flag, flush_ms_p50=med(times[flag]["flush"]), flush_ms_max=round(max(times[flag]["flush"]), 3),
                 next_ingest_ms_p50=med(times[flag]["ingest"]), next_ingest_ms_max=round(max(times[flag]["ingest"]), 3),
                 merge_prepare_ms_p50=med(times[flag]["prepare"]), device_bytes=eng.capacity()["device_bytes"],
                 cms_sha256=hashlib.sha256(eng.export_cms(True).tobytes()).hexdigest(),
                 cmsq_last_sha256=hashlib.sha256(eng.export_cms_queries(True).tobytes()).hexdigest())
        if flag:
            r["cmsq_5min_sha256"] = hashlib.sha256(eng.export_cms_queries_5min().tobytes()).hexdigest()
        ms, launches = roll_kernel_ms(eng, t + 5)
        r["roll_kernel_ms"], r["roll_launches"] = ms, launches
        r["roll_kernel_ms_per_ring"] = round(ms / launches, 4) if launches else 0.0
        runs.append(r)
    line = json.dumps(dict(card=card(), events_per_batch=n, timed_windows=a.reps, runs=runs))
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "flow_query_level_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
