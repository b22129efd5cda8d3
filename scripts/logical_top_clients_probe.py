"""What merging each logical service's heaviest clients (GYSK_FLAG_SVC_TOP_CLIENTS with a logical map) costs in the merge step.

    python scripts/logical_top_clients_probe.py [--reps 7] [--out DIR]

At 6 250 and 62 500 logical services of 16 members each (100 000 and 1 000 000 services), two engines, one with the flag, take the same
two windows of seeded connection events (Zipf clients, every service with clients) and the same logical map. Then, alternating the two
engines rep by rep: gysk_merge_prepare and gysk_merge_finish at world 1 (the rank's own slab, no collective), each timed by the host clock
around the call and a device sync; and with the flag, gysk_query_logical_top_clients of every logical id and
gysk_query_logical_top_clients_all, beside gysk_query_logical and gysk_query_logical_all for scale. Medians in ms. It prints each engine's
slab bytes, and the card's name and power limit, read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.flow_queries_probe import card  # noqa: E402

MEMBERS = 16
GOLD = np.uint64(2654435761)


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def events(rng, nsvc, n):
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = (np.arange(n) % nsvc + 1).astype(np.uint64) * GOLD
    ev["flow_key"] = (rng.zipf(1.2, n) % 100_000).astype(np.uint64) * GOLD + np.uint64(1)
    ev["type"] = ge.EV_CLOSE_SER
    ev["value"] = rng.integers(0, 1 << 22, n)
    return ev


def run(a, nl):
    nsvc = nl * MEMBERS
    sids = np.arange(1, nsvc + 1, dtype=np.uint64) * GOLD
    lids = (np.arange(nsvc) % nl + 1).astype(np.uint64)
    batch = 1 << 22
    engines = {}
    for name, on in (("off", False), ("on", True)):
        eng = ge.Engine(device=0, max_svcs=1 << int(np.ceil(np.log2(nsvc + 1))), max_tasks=1 << 10, max_batch=batch, svc_top_clients=on)
        eng.set_logical_map(sids, lids)
        engines[name] = eng
    rng = {k: np.random.default_rng(3) for k in engines}
    for t in (5, 10):
        for name, eng in engines.items():
            for off in range(0, 2 * nsvc, batch):
                eng.ingest_events(events(rng[name], nsvc, min(batch, 2 * nsvc - off)))
                eng.sync()
            eng.flush(t)
    times = {k: dict(prepare=[], finish=[]) for k in engines}
    times["on"].update(read_by_id=[], read_all=[], query_logical=[], query_logical_all=[])
    ids = np.arange(1, nl + 1, dtype=np.uint64)
    for rep in range(a.reps + 1):
        for name, eng in engines.items():
            p = timed(lambda: (eng.merge_prepare(), eng.sync()))
            f = timed(lambda: (eng.merge_finish(), eng.sync()))
            if rep == 0:
                continue
            times[name]["prepare"].append(p)
            times[name]["finish"].append(f)
            if name == "on":
                times[name]["read_by_id"].append(timed(lambda: eng.query_logical_top_clients(ids, ge.TOPC_LAST)))
                times[name]["read_all"].append(timed(lambda: eng.query_logical_top_clients_all(ge.TOPC_LAST)))
                times[name]["query_logical"].append(timed(lambda: eng.query_logical(ids)))
                times[name]["query_logical_all"].append(timed(lambda: eng.query_logical_all()))
    out = []
    for name, eng in engines.items():
        r = dict(config=name, logical_services=nl, members=MEMBERS, services=nsvc, slab_bytes=eng.merge_tdigest_slab()[1],
                 **{f"{k}_ms_p50": round(float(np.median(v)), 3) for k, v in times[name].items()})
        if name == "on":
            rows = eng.query_logical_top_clients(ids, ge.TOPC_LAST)
            r["logical_with_clients"] = int((rows["n"] > 0).sum())
        out.append(r)
    for eng in engines.values():
        eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    lines = []
    for nl in (6250, 62500):
        for r in run(a, nl):
            lines.append(json.dumps(r))
            print(lines[-1], flush=True)
        torch.cuda.empty_cache()
    lines.append(json.dumps(dict(card=card(), reps=a.reps)))
    print(lines[-1], flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "logical_top_clients_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
