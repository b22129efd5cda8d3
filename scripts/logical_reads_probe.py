"""Times the reads over every merged logical service on one GPU, at 100 K and 1 M services in logical services of 16 members (6 250 and
62 500 logical services, the layout of logical_levels_probe.py), GYSK_FLAG_MERGE_LEVELS on: gysk_query_logical_all (every row, and the
ACTIVE_ONLY read with half of the logical services active) and gysk_topn_logical, against gysk_query_logical over the same ids in the
same order. ms per call (host clock around calls that end in a stream sync, median of 5), the device time of the new kernels
(torch.profiler), and the largest relative gap between gysk_query_logical_quantiles and the rows' td_p50_us / td_p95_us / td_p99_us next
to the same gap of the per-service pair (gysk_query_quantiles against gysk_query_window rows), over up to 2000 ids each. Prints one JSON
line per size, with the card's name and power limit.

    python scripts/logical_reads_probe.py [--sizes 100000 1000000] [--out DIR]
"""
import argparse
import ctypes as C
import json
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.window_read_probe import card, fill, timed  # noqa: E402

MEMBERS = 16
QS = [0.5, 0.95, 0.99]
KERNELS = ("logical_select_kernel", "logical_summary_kernel", "logical_topn_score_kernel", "topn_pick_kernel")


def gap(rows, quantiles, limit=2000):
    g = 0.0
    for r in [r for r in rows if r.td_count][:limit]:
        for a, b in zip(quantiles(r.glob_id, QS), (r.td_p50_us, r.td_p95_us, r.td_p99_us)):
            if not (math.isnan(a) and math.isnan(b)):
                g = max(g, abs(float(a) - b) / abs(b) if b else abs(float(a) - b))
    return g


def probe(n, name):
    import torch
    from torch.profiler import ProfilerActivity, profile

    rng = np.random.default_rng(n)
    eng = ge.Engine(max_svcs=n, max_tasks=1024, max_batch=1 << 22, merge_levels=True)
    ids = fill(eng, n, rng)
    # a second window in which only the services of odd logical services have events: half of the logical services are active
    lof = np.arange(n, dtype=np.uint64) // np.uint64(MEMBERS) + np.uint64(1)
    eng.flush(5)
    keep = ids[(lof % np.uint64(2)) == 1]
    ev = np.zeros(len(keep), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["type"], ev["value"] = keep, ge.EV_RESP, 2000
    ev["host_idx"] = (keep % np.uint64(64)).astype(np.uint32)
    eng.ingest_events(ev)
    eng.flush(10)
    eng.set_logical_map(ids, lof)
    eng.merge_prepare()
    eng.merge_finish(None, 1)
    eng.sync()
    nl = (n + MEMBERS - 1) // MEMBERS
    lids = np.arange(1, nl + 1, dtype=np.uint64)
    out_all, out_act, out_id = (ge.SvcSummary * nl)(), (ge.SvcSummary * nl)(), (ge.SvcSummary * nl)()
    k = C.c_uint32()
    top = (ge.TopnEntry * 64)()

    def read_all():
        assert eng.L.gysk_query_logical_all(eng.h, 0, out_all, nl, C.byref(k)) == 0 and k.value == nl

    def read_active():
        assert eng.L.gysk_query_logical_all(eng.h, ge.WINDOW_ACTIVE_ONLY, out_act, nl, C.byref(k)) == 0 and k.value == nl // 2

    def read_by_id():
        assert eng.L.gysk_query_logical(eng.h, ge._p(lids), nl, out_id) == 0

    def topn():
        assert eng.L.gysk_topn_logical(eng.h, ge.TOPN_QPS, 64, top, C.byref(k)) == 0 and k.value == 64

    ms = {name_: timed(fn, 5) for name_, fn in (("query_logical_all", read_all), ("query_logical_all_active", read_active),
                                                 ("query_logical_same_ids", read_by_id), ("topn_logical_64", topn))}
    assert all(bytes(a) == bytes(b) for a, b in zip(out_all, out_id))            # the same rows, byte for byte
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        read_all()
        read_active()
        topn()
        torch.cuda.synchronize()
    kus = dict.fromkeys(KERNELS, 0.0)
    for e in prof.key_averages():
        for kn in kus:
            if kn in e.key:
                kus[kn] += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    logical_gap = gap(list(out_all), eng.logical_quantiles)
    svc_gap = gap(eng.query_window(cap=2000)[0], eng.quantiles)
    eng.close()
    return dict(services=n, logical=nl, members=MEMBERS, card=name, ms={k_: round(v[0], 3) for k_, v in ms.items()},
                runs_ms={k_: v[1] for k_, v in ms.items()}, kernels_ms={k_: round(v / 1e3, 3) for k_, v in kus.items()},
                quantile_gap_logical=logical_gap, quantile_gap_service=svc_gap)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--out", help="also write the JSON lines to DIR/logical_reads_probe.jsonl")
    a = ap.parse_args()
    name = card()
    lines = []
    for n in a.sizes:
        line = json.dumps(probe(n, name))
        print(line, flush=True)
        lines.append(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "logical_reads_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
