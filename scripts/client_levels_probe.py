"""What GYSK_FLAG_CLIENT_LEVELS costs on the bench workload.

    python scripts/client_levels_probe.py [--reps 8] [--profile 4] [--events 100000000] [--out DIR]

Per service capacity (the bench's 2^17 slots, and 2^20 = 1 M services), two engines, one with the flag, take the bench's two batches of
100 M mixed events (bench.gen_events_gpu, same seeds), alternated window by window in one run. Each engine maps every service it holds to
a logical service of its own, so gysk_merge_prepare folds every service. Per timed window: gysk_flush, the next batch's ingest and
gysk_merge_prepare (host clock around each call and a sync; medians), device_bytes against the device memory cudaMemGetInfo shows in use.
With --profile N the device ms per batch of each kernel over N more batches (torch.profiler: the TCP drain pass and ingest_kernel among
them). Each engine prints the SHA-256 of its window read, which must not differ. The card's name and power limit are read in the same run."""
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
from scripts.flow_agg_probe import profile_batches  # noqa: E402
from scripts.flow_queries_probe import card  # noqa: E402


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def in_use():
    free, total = torch.cuda.mem_get_info(0)
    return total - free


def costs(a, ev_devs, n, max_svcs):
    engines = {}
    for name, on in (("off", False), ("on", True)):
        before = in_use()
        eng = ge.Engine(device=0, max_svcs=max_svcs, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23, client_levels=on)
        for ev in ev_devs:                  # registers the services and tasks, as bench.py does
            eng.ingest_device_ptr(ev.data_ptr(), n)
        eng.sync()
        eng.flush(5)
        rows, _, _ = eng.query_window_hosts()
        ids = np.array(sorted(r.glob_id for r in rows), dtype=np.uint64)
        eng.set_logical_map(ids, ids)
        eng.sync()
        engines[name] = (eng, in_use() - before, len(ids))
    times = {k: dict(flush=[], ingest=[], prepare=[]) for k in engines}
    t = 5
    for w in range(2 + a.reps):
        t += 5
        for name, (eng, _, _) in engines.items():   # alternated window by window
            ev = ev_devs[w % 2]
            f = timed(lambda: (eng.flush(t), eng.sync()))
            i = timed(lambda: (eng.ingest_device_ptr(ev.data_ptr(), n), eng.sync()))
            p = timed(lambda: (eng.merge_prepare(), eng.sync()))
            if w >= 2:
                for k, v in zip(("flush", "ingest", "prepare"), (f, i, p)):
                    times[name][k].append(v)
    med = lambda v: round(float(np.median(v)), 3)
    out = []
    for name, (eng, used, nsvc) in engines.items():
        eng.flush(t + 5)
        rows, _, _ = eng.query_window_hosts()
        r = dict(config=name, max_svcs=max_svcs, services=nsvc, **{f"{k}_ms_p50": med(v) for k, v in times[name].items()},
                 device_bytes=eng.capacity()["device_bytes"], mem_get_info_in_use=used,
                 window_sha256=hashlib.sha256(b"".join(sorted(bytes(x) for x in rows))).hexdigest())
        if name == "on":
            c = eng.query_clients_window()[0]
            r["clients_last_5s_median"] = float(np.median([x.last_5s for x in c])) if len(c) else 0.0
            r["clients_last_5min_median"] = float(np.median([x.last_5min for x in c])) if len(c) else 0.0
        if a.profile:
            r["ms_per_batch"] = profile_batches(eng, ev_devs, n, a.profile)
        out.append(r)
    for eng, _, _ in engines.values():
        eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--profile", type=int, default=0, metavar="N")
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = a.events
    ev_devs = [bench.gen_events_gpu(torch, n, 1234 + 7919 * b, 0, 1, dev) for b in range(2)]
    torch.cuda.synchronize()
    lines = []
    for max_svcs in (1 << 17, 1 << 20):
        lines += [json.dumps(r) for r in costs(a, ev_devs, n, max_svcs)]
        print("\n".join(lines[-2:]), flush=True)
    lines.append(json.dumps(dict(card=card(), events_per_batch=n, timed_windows=a.reps)))
    print(lines[-1], flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "client_levels_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
