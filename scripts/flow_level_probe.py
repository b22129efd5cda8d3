"""Times what GYSK_FLAG_FLOW_LEVEL adds, on one GPU, with the flag off and on. Prints one JSON line with the card's name and power limit.

Each engine first takes a config-3-sized window: 12.5 M mixed events (70 / 20 / 10 RESP / TCP / TASK, the share of one of four ranks of a
50 M-event batch) over 100 K services on 4096 hosts, in device batches of 4 M events. Then, per setting (count-min depth x width
4 x 2^20 and 8 x 2^22) and flag:
1. gysk_flush after that window, ten times over successive 5-s windows (host clock around flush + sync), median and max ms. Ten
   warm-up windows 30 s apart first fill every ring slot, so that with the flag each timed flush runs cms_level_roll_kernel at its
   most: it reads the closing window and all ten slots, and writes one slot and the level (13 tables of depth << log2_width cells).
2. The next window's ingest: gysk_profile_read's device time of the ingest kernel with its drain passes, and of the sort + t-digest
   chain, each summed over the window, median of the ten windows. A pass that pushed the count-min out of L2 would show in the first.
3. gysk_merge_prepare (one logical service per 16 services), host clock around prepare + sync, median of ten.

    python scripts/flow_level_probe.py [--events 12500000] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import engine as ge, synth  # noqa: E402
from scripts.window_read_probe import card  # noqa: E402

BATCH = 1 << 22
NSVC, NHOSTS = 100_000, 4096


def make_window(rng, n):
    return synth.gen_mixed(rng, n, NSVC, ntask=4096, nhosts=NHOSTS, nclients=200_000)


def feed(eng, ev):
    for off in range(0, len(ev), BATCH):
        eng.ingest_events(ev[off: off + BATCH])
    eng.sync()


def probe(depth, log2w, flag, windows, reps):
    eng = ge.Engine(max_svcs=1 << 17, max_tasks=1 << 13, max_batch=BATCH, cms_depth=depth, cms_log2_width=log2w, flow_level=flag)
    ids = synth.service_ids(NSVC)
    eng.set_logical_map(ids, ids // np.uint64(16))
    eng.profile_enable(True)
    flush_ms, ingest_ms, chain_ms, prep_ms = [], [], [], []
    t = 0
    for w in range(reps + 10):
        ev = windows[w % len(windows)]
        eng.profile_read()
        feed(eng, ev)
        ing, chain, _n = eng.profile_read()
        t += 30 if w < 10 else 5                # ten warm-up windows in ten epochs: every ring slot live
        t0 = time.perf_counter()
        eng.flush(t)
        eng.sync()
        f = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        eng.merge_prepare()
        eng.sync()
        p = (time.perf_counter() - t0) * 1e3
        if w >= 10:
            flush_ms.append(f); ingest_ms.append(ing); chain_ms.append(chain); prep_ms.append(p)
    dev = eng.capacity()["device_bytes"]
    eng.close()
    med = lambda a: round(float(np.median(a)), 3)
    return dict(depth=depth, log2_width=log2w, flow_level=flag, flush_ms_p50=med(flush_ms), flush_ms_max=round(max(flush_ms), 3),
                ingest_drain_ms_p50=med(ingest_ms), sort_tdigest_ms_p50=med(chain_ms), merge_prepare_ms_p50=med(prep_ms), device_bytes=dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--events", type=int, default=12_500_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rng = np.random.default_rng(3)
    windows = [make_window(rng, a.events) for _ in range(2)]
    res = dict(card=card(), events_per_window=a.events, runs=[])
    for depth, log2w in ((4, 20), (8, 22)):
        for flag in (False, True, False, True):          # alternated, so drift shows as a spread between the two runs of a flag
            res["runs"].append(probe(depth, log2w, flag, windows, a.reps))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "flow_level_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
