"""Times table growth on one GPU. Prints one JSON line with the card's name and power limit.

1. gysk_grow of the service table from 2^17 to 2^18 and from 2^20 to 2^21 slots (process table 2^14 -> 2^15), every service slot holding
   an id, histograms, connection counters, HLL registers and a digest, the level ring written by ten flushes. gysk_grow copies every
   array whole whatever it holds, so the time depends on the capacities only. Reports ms (host clock around the call, which ends in a
   stream sync), the bytes it moves (old arrays read, the new ones written) and those bytes over 3.35 TB/s.
2. A sustained-stream-shaped run: the live services grow by 30 % a window from 16 K to --services, then stay, 4 response samples and
   one connection event each per window. One engine starts at 2^16 service slots with auto-grow up to 2^21, the other is created at
   2^21. Window ms (ingest + flush, host clock) p50 / p95 / max of each, the windows in which the auto-grow engine grew and their ms,
   and the device bytes each holds at the end.

    python scripts/grow_probe.py [--services 1000000] [--windows 24] [--skip-big] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.window_read_probe import card  # noqa: E402

HBM_BPS = 3.35e12
BATCH = 1 << 22


def window(eng, ids, rng, t, per_resp=4):
    """per_resp response samples and one connection event of every id, in device batches of 4 M events, then the flush of t"""
    per = per_resp + 1
    step = BATCH // per
    for off in range(0, len(ids), step):
        part = ids[off: off + step]
        ev = np.zeros(len(part) * per, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = np.repeat(part, per)
        ev["type"] = np.tile(np.array([ge.EV_RESP] * per_resp + [ge.EV_ACCEPT], dtype=np.uint16), len(part))
        ev["value"] = rng.lognormal(8.0, 1.2, len(ev)).astype(np.uint32) + 1
        ev["flow_key"] = rng.integers(0, 1 << 62, len(ev), dtype=np.uint64)
        ev["host_idx"] = (ev["svc_id"] % np.uint64(4096)).astype(np.uint32)
        eng.ingest_events(ev)
    eng.flush(t)
    eng.sync()


def grow_once(log2_from):
    n = 1 << log2_from
    rng = np.random.default_rng(log2_from)
    eng = ge.Engine(max_svcs=n, max_tasks=1 << 14, max_batch=BATCH, idle_evict_secs=0)
    ids = (rng.choice(1 << 40, n, replace=False) + 1).astype(np.uint64)
    for k in range(10):                       # ten flushes, ten ring slots of each level written
        window(eng, ids if k == 0 else ids[: n // 16], rng, 43200 * (k + 1) + 30 * (k + 1), per_resp=8 if k == 0 else 1)
    before = eng.capacity()
    t0 = time.perf_counter()
    eng.grow(2 * n, 1 << 15)
    ms = (time.perf_counter() - t0) * 1e3
    after = eng.capacity()
    old_b, new_b = before["device_bytes"], after["device_bytes"]
    moved = old_b + new_b                     # (about) every old array read once, every new one written once
    res = dict(slots_from=n, slots_to=2 * n, ms=round(ms, 2), device_bytes_before=old_b, device_bytes_after=new_b, bytes_moved=moved,
               ms_at_3_35_TBps=round(moved / HBM_BPS * 1e3, 2))
    assert eng.query_svcs(ids[:4])[0]["found"]
    eng.close()
    return res


def stream(n_final, nwin, auto):
    import torch
    rng = np.random.default_rng(7)
    if auto:
        eng = ge.Engine(max_svcs=1 << 16, max_tasks=1 << 14, max_batch=BATCH)
        eng.set_auto_grow(1 << 21, 0)
    else:
        eng = ge.Engine(max_svcs=1 << 21, max_tasks=1 << 14, max_batch=BATCH)
    ids = (rng.choice(1 << 40, n_final, replace=False) + 1).astype(np.uint64)
    ms, grows, prev = [], [], eng.capacity()["ngrows"]
    for w in range(nwin):
        live = ids[: min(n_final, int(16384 * 1.3 ** w))]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        window(eng, live, rng, 5 * (w + 1))
        ms.append((time.perf_counter() - t0) * 1e3)
        c = eng.capacity()
        if c["ngrows"] != prev:
            grows.append(dict(window=w, ms=round(ms[-1], 2), max_svcs=c["max_svcs"]))
            prev = c["ngrows"]
    c, s = eng.capacity(), eng.stats()
    eng.close()
    a = np.array(ms)
    return dict(window_ms_p50=round(float(np.median(a)), 2), window_ms_p95=round(float(np.percentile(a, 95)), 2),
                window_ms_max=round(float(a.max()), 2), grows=grows, max_svcs=c["max_svcs"], device_bytes=c["device_bytes"],
                events_dropped=s["events_dropped"], nsvcs=s["nsvcs"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--services", type=int, default=1_000_000)
    ap.add_argument("--windows", type=int, default=24)
    ap.add_argument("--skip-big", action="store_true", help="only the 2^17 -> 2^18 growth")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card(), svc_slot_bytes=ge.slot_bytes(12)[0])
    res["grow"] = [grow_once(17)] + ([] if a.skip_big else [grow_once(20)])
    res["stream_auto"] = stream(a.services, a.windows, True)
    res["stream_fixed"] = stream(a.services, a.windows, False)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "grow_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
