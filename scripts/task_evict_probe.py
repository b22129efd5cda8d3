"""Times what process eviction (gysk_config.task_idle_evict_secs) adds, on one GPU, with it off and on. Prints one JSON line with the
card's name, power limit and clocks.

Each engine holds 256 K aggregated processes (max_tasks 2^18) on 4096 hosts. Every 5-s window brings one TASK sample of each live
process, in one device batch. A tenth of the processes stop after the first window; with eviction on (20 s) they leave at the flush
six windows later, and the next window brings as many new processes, which take the recycled slots (with eviction off, fresh ones).
Per setting, repeated over fresh engines:
1. gysk_flush, host clock around flush + sync: the median of the windows that evict nothing, and the flush that evicts 26 K processes.
2. The ingest batch right after that flush (host clock around ingest + sync), with the new processes in it.

    python scripts/task_evict_probe.py [--reps 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import engine as ge, synth  # noqa: E402
from scripts.window_read_probe import card  # noqa: E402

NTASK, NHOSTS, SECS = 1 << 18, 4096, 20


def clocks():
    r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,clocks.mem", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def window(rng, ids, t):
    ev = np.zeros(len(ids), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = ids; ev["type"] = ge.EV_TASK; ev["tsec"] = t
    ev["host_idx"] = (ids % np.uint64(NHOSTS)).astype(np.uint32)
    ev["value"] = rng.integers(0, 400, len(ev))
    ev["flow_key"] = rng.integers(0, 5000, len(ev)).astype(np.uint64) | (rng.integers(0, 5000, len(ev)).astype(np.uint64) << np.uint64(32))
    return ev


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def probe(on, rng):
    eng = ge.Engine(max_svcs=1 << 10, max_tasks=NTASK, max_batch=1 << 20, task_idle_evict_secs=SECS if on else 0)
    ids = synth.splitmix64(np.arange(1, NTASK + 1, dtype=np.uint64) + np.uint64(1 << 50)) >> np.uint64(8)
    idle, busy = ids[: NTASK // 10], ids[NTASK // 10:]
    fresh = synth.splitmix64(np.arange(1, NTASK // 10 + 1, dtype=np.uint64) + np.uint64(1 << 51)) >> np.uint64(8)
    flush_ms, evict_ms, next_ms = [], None, None
    for w, t in enumerate(range(5, 45, 5)):
        ev = window(rng, ids if w == 0 else (busy if t <= 5 + SECS + 5 else np.concatenate([busy, fresh])), t)
        if t == 5 + SECS + 10:
            next_ms = timed(lambda: (eng.ingest_events(ev), eng.sync()))
        else:
            eng.ingest_events(ev); eng.sync()
        f = timed(lambda: (eng.flush(t), eng.sync()))
        if t == 5 + SECS + 5:
            evict_ms = f
            if on:
                assert len(eng.evicted_task_ids(cap=NTASK)) == len(idle)
        elif w > 0:
            flush_ms.append(f)
    used = eng.capacity()["tasks_in_use"]
    dropped = eng.stats()["events_dropped"]
    eng.close()
    return dict(eviction=on, flush_ms_p50=round(float(np.median(flush_ms)), 3), evicting_flush_ms=round(evict_ms, 3),
                next_ingest_ms=round(next_ms, 3), tasks_in_use=used, events_dropped=dropped)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rng = np.random.default_rng(5)
    probe(False, rng)                                  # warm-up: module load, first allocations
    res = dict(card=card(), clocks_sm_maxsm_mem=clocks(), tasks=NTASK, idle_share=0.1, runs=[])
    for _ in range(a.reps):
        for on in (False, True):                       # alternated, so drift shows as a spread between the runs of a setting
            res["runs"].append(probe(on, rng))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "task_evict_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
