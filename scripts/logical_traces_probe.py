"""Times the merged request traces of logical services (GYSK_FLAG_MERGE_TRACES) on one GPU, at 6 250 and 62 500 logical services of 8
members (50 K and 500 K services) with 65 536 trace rows, each held by a service that had 32 trace samples in the last window: gysk_merge_prepare
and gysk_merge_finish (world 1) with and without the flag, gysk_query_logical_traces_all and gysk_query_logical_traces over every id.
ms per call (host clock around calls that end in a stream sync, median of 5) and the device time of the kernels the flag adds or
widens (torch.profiler). Also prints the bytes the flag adds to each rank's regions and slab and to an all-gather at world 8, computed
from the layout. One JSON line per size, with the card's name and power limit.

    python scripts/logical_traces_probe.py [--logical 6250 62500] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.window_read_probe import card, fill, timed  # noqa: E402
from tests import trace_agg as ta  # noqa: E402

MEMBERS, ROWS, PER = 8, 65_536, 32
KERNELS = ("fold_traces_kernel", "fold_td_kernel", "finish_td_kernel", "logical_trace_kernel", "fold_levels_kernel")
SLAB_ENTRY, TRACE_SLAB = 32 + 256 * 16, 32 + 100 * 16


def align256(v):
    return (v + 255) & ~255


def added_bytes(nl, world=8):
    """what the flag adds: SUM words, i64 MAX words and the flush tsec pair, slab entries per rank; the all-gather carries world slabs"""
    slab = -(-nl * TRACE_SLAB // SLAB_ENTRY) * SLAB_ENTRY
    return dict(sum=align256(nl * 16 * 8), max_i64=256 + align256(nl * 3 * 8), slab_per_rank=slab, gathered_at_world=world,
                gathered=world * slab, gathered_digest_slab=world * nl * SLAB_ENTRY)


def engine(n, rng, traces):
    eng = ge.Engine(max_svcs=n, max_tasks=1024, max_batch=1 << 22, max_trace_svcs=ROWS, merge_traces=traces)
    ids = fill(eng, n, rng)
    traced = ids[:: max(1, n // ROWS)][:ROWS]
    for off in range(0, len(traced), (1 << 21) // PER):
        part = np.repeat(traced[off: off + (1 << 21) // PER], PER)
        rec = ta.api_tran(part, np.exp(rng.normal(8.0, 1.5, len(part))).astype(np.uint64), 300, 2000)
        ev = ta.trace_events(rec)
        ev["host_idx"] = (ev["svc_id"] % np.uint64(64)).astype(np.uint32)
        eng.ingest_events(ev)
    eng.flush(10)
    eng.set_logical_map(ids, np.arange(n, dtype=np.uint64) // np.uint64(MEMBERS) + np.uint64(1))
    eng.sync()
    return eng


def merge_ms(eng):
    def prep():
        eng.merge_prepare()
        eng.sync()

    def fin():
        eng.merge_finish(None, 1)
        eng.sync()
    a = timed(prep, 5)
    b = timed(fin, 5)
    return a, b


def probe(nl, name):
    import torch
    from torch.profiler import ProfilerActivity, profile

    n = nl * MEMBERS
    off = engine(n, np.random.default_rng(n), False)
    ms = {}
    ms["prepare_without_flag"], ms["finish_without_flag"] = merge_ms(off)
    off.close()
    eng = engine(n, np.random.default_rng(n), True)
    ms["prepare_with_flag"], ms["finish_with_flag"] = merge_ms(eng)
    lids = np.arange(1, nl + 1, dtype=np.uint64)
    out_all, out_id = (ge.LogicalTrace * nl)(), (ge.LogicalTrace * nl)()
    k = C.c_uint32()

    def read_all():
        assert eng.L.gysk_query_logical_traces_all(eng.h, 0, out_all, nl, C.byref(k)) == 0 and k.value == nl

    def read_by_id():
        assert eng.L.gysk_query_logical_traces(eng.h, ge._p(lids), nl, out_id) == 0

    ms["query_logical_traces_all"] = timed(read_all, 5)
    ms["query_logical_traces_same_ids"] = timed(read_by_id, 5)
    assert all(bytes(a) == bytes(b) for a, b in zip(out_all, out_id))
    traced = sum(r.ntraced for r in out_all)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.merge_prepare()
        eng.merge_finish(None, 1)
        read_all()
        torch.cuda.synchronize()
    kus = dict.fromkeys(KERNELS, 0.0)
    for e in prof.key_averages():
        for kn in kus:
            if kn in e.key:
                kus[kn] += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    eng.close()
    return dict(logical=nl, services=n, members=MEMBERS, trace_rows=ROWS, members_traced=traced, card=name,
                ms={k_: round(v[0], 3) for k_, v in ms.items()}, runs_ms={k_: v[1] for k_, v in ms.items()},
                kernels_ms={k_: round(v / 1e3, 3) for k_, v in kus.items()}, added_bytes=added_bytes(nl))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logical", type=int, nargs="+", default=[6_250, 62_500])
    ap.add_argument("--out", help="also write the JSON lines to DIR/logical_traces_probe.jsonl")
    a = ap.parse_args()
    name = card()
    lines = []
    for nl in a.logical:
        line = json.dumps(probe(nl, name))
        print(line, flush=True)
        lines.append(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "logical_traces_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
