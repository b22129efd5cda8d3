"""Times gysk_merge_prepare with and without GYSK_FLAG_MERGE_LEVELS on one GPU, at 100 K and 1 M services in logical services of 16
members: ms per fold (prepare + stream sync), fold_levels_kernel's device time and bytes read over that time (torch.profiler) against the
3.35 TB/s HBM3 data-sheet figure of the H100 SXM, and the bytes the flag adds to the all-reduced regions. The services are flushed once
in each of ten 43 200-s slots of the 5-day level and, inside the last of them, once in each of ten 30-s slots of the 300-s level, so
every member has all ten slots of both rings live. Prints one JSON line per size and setting, with the card's name and power limit.

    python scripts/logical_levels_probe.py [--sizes 100000 1000000] [--out DIR]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.window_read_probe import HBM_TBS, card, fill, timed  # noqa: E402

MEMBERS = 16
SLOT5D, SLOT5M = 43200, 30


def flush_schedule():
    """ten 5-day slots (the first flush is fill's, at 5), then nine more 300-s slots inside the last 5-day slot"""
    last = 5 + 9 * SLOT5D
    return [5 + SLOT5D * k for k in range(1, 10)] + [last + SLOT5M * j for j in range(1, 10)]


def levels_kernel_bytes(n, nl):
    """what fold_levels_kernel reads and writes: 16 cells of 16 B of ten slots of both rings and the 40-byte aux word of every member,
    its slot and the CSR offsets; 2 x 16 cells of 16 B, the level maxima, four aux sums and the rtt of every logical service"""
    return n * (2 * 10 * 256 + 40 + 4) + (nl + 1) * 4 + nl * (2 * 256 + 16 + 32 + 8)


def probe(n, levels, name):
    import torch
    from torch.profiler import ProfilerActivity, profile

    rng = np.random.default_rng(n)
    eng = ge.Engine(max_svcs=n, max_tasks=1024, max_batch=1 << 22, merge_levels=levels)
    ids = fill(eng, n, rng)
    for t in flush_schedule():
        eng.flush(t)
    nl = (n + MEMBERS - 1) // MEMBERS
    eng.set_logical_map(ids, np.arange(n, dtype=np.uint64) // np.uint64(MEMBERS) + np.uint64(1))
    regions = {d[0].split(":")[0]: d[2] for d in eng.merge_buffers()}

    def prepare():
        eng.merge_prepare()
        eng.sync()

    ms, runs = timed(prepare, 5)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        prepare()
        torch.cuda.synchronize()
    kus = {"resolve_members_kernel": 0.0, "fold_hist_kernel": 0.0, "fold_hll_kernel": 0.0, "fold_td_kernel": 0.0, "fold_levels_kernel": 0.0}
    for e in prof.key_averages():
        for kn in kus:
            if kn in e.key:
                kus[kn] += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    eng.merge_finish(None, 1)
    rows = eng.query_logical([1, 2])
    assert rows[0]["nqrys_5day"] == (rows[0]["nqrys_all"] if levels else 0)
    eng.close()
    r = dict(services=n, logical=nl, members=MEMBERS, merge_levels=levels, card=name, prepare_ms=round(ms, 3), prepare_runs_ms=runs,
             allreduce_bytes=regions, kernels_ms={k: round(v / 1e3, 3) for k, v in kus.items()})
    kd = kus["fold_levels_kernel"]
    if levels and kd:
        kb = levels_kernel_bytes(n, nl)
        r.update(levels_kernel_bytes=kb, levels_kernel_tbs=round(kb / (kd * 1e-6) / 1e12, 3),
                 levels_kernel_share_of_3_35_tbs=round(kb / (kd * 1e-6) / 1e12 / HBM_TBS, 3))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--out", help="also write the JSON lines to DIR/logical_levels_probe.jsonl")
    a = ap.parse_args()
    name = card()
    lines = []
    for n in a.sizes:
        res = {lv: probe(n, lv, name) for lv in (False, True)}
        res[True]["extra_prepare_ms"] = round(res[True]["prepare_ms"] - res[False]["prepare_ms"], 3)
        res[True]["extra_allreduce_bytes"] = sum(res[True]["allreduce_bytes"].values()) - sum(res[False]["allreduce_bytes"].values())
        for lv in (False, True):
            print(json.dumps(res[lv]), flush=True)
            lines.append(json.dumps(res[lv]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "logical_levels_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
