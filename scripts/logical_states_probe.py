"""Times the listener-state roll-up of logical services (GYSK_FLAG_MERGE_STATES) on one GPU, at 100 K and 1 M services in logical
services of 16 members (6 250 and 62 500 logical services, the layout of logical_reads_probe.py): the merge (gysk_merge_prepare +
gysk_merge_finish at world 1) with and without the flag, gysk_query_logical_states_all, gysk_query_logical_states over every id and the
GYSK_TOPN_ISSUE top-64. Four of every 16 members turn slow and error-prone in the last window so that their states reach BAD or worse
(SEVERE in the CPU oracle). ms per call (host clock
around calls that end in a stream sync, median of 5) and the device time of the new kernels (torch.profiler). Prints one JSON line
per size, with the card's name and power limit.

    python scripts/logical_states_probe.py [--sizes 100000 1000000] [--out DIR]
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

MEMBERS = 16
KERNELS = ("fold_states_kernel", "logical_state_kernel", "logical_topn_score_kernel", "fold_levels_kernel", "fold_hist_kernel")


def engine(n, rng, states):
    eng = ge.Engine(max_svcs=n, max_tasks=1024, max_batch=1 << 22, merge_states=states)
    ids = fill(eng, n, rng)
    slow = ids[(np.arange(n) % MEMBERS) < 4]
    for t in range(5, 215, 10):                  # past the 100-s rule the slow members' last window turns 100 x slower, with server errors
        ev = np.zeros(2 * n, dtype=ge.EVENT_DTYPE)
        ev["svc_id"][:n], ev["svc_id"][n:] = ids, np.resize(slow, n)
        ev["type"] = ge.EV_RESP
        ev["value"][:n], ev["value"][n:] = 20_000, 20_000 if t < 200 else 2_000_000
        ev["flags"][n:] = 0 if t < 200 else ge.EVF_SER_ERROR
        ev["host_idx"] = (ev["svc_id"] % np.uint64(64)).astype(np.uint32)
        eng.ingest_events(ev)
        eng.flush(t)
    eng.set_logical_map(ids, np.arange(n, dtype=np.uint64) // np.uint64(MEMBERS) + np.uint64(1))
    eng.sync()
    return eng


def merge(eng):
    eng.merge_prepare()
    eng.merge_finish(None, 1)
    eng.sync()


def probe(n, name):
    import torch
    from torch.profiler import ProfilerActivity, profile

    nl = (n + MEMBERS - 1) // MEMBERS
    off = engine(n, np.random.default_rng(n), False)
    ms = {"merge_without_flag": timed(lambda: merge(off), 5)}
    off.close()
    eng = engine(n, np.random.default_rng(n), True)
    ms["merge_with_flag"] = timed(lambda: merge(eng), 5)
    lids = np.arange(1, nl + 1, dtype=np.uint64)
    out_all, out_id = (ge.LogicalState * nl)(), (ge.LogicalState * nl)()
    k = C.c_uint32()
    top = (ge.TopnEntry * 64)()

    def read_all():
        assert eng.L.gysk_query_logical_states_all(eng.h, 0, out_all, nl, C.byref(k)) == 0 and k.value == nl

    def read_by_id():
        assert eng.L.gysk_query_logical_states(eng.h, ge._p(lids), nl, out_id) == 0

    def topn():
        assert eng.L.gysk_topn_logical(eng.h, ge.TOPN_ISSUE, 64, top, C.byref(k)) == 0

    for key, fn in (("query_logical_states_all", read_all), ("query_logical_states_same_ids", read_by_id), ("topn_logical_issue_64", topn)):
        ms[key] = timed(fn, 5)
    assert all(bytes(a) == bytes(b) for a, b in zip(out_all, out_id))            # the same rows, byte for byte
    issue = [r.nsvc_issue for r in out_all]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        merge(eng)
        read_all()
        topn()
        torch.cuda.synchronize()
    kus = dict.fromkeys(KERNELS, 0.0)
    for e in prof.key_averages():
        for kn in kus:
            if kn in e.key:
                kus[kn] += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    eng.close()
    return dict(services=n, logical=nl, members=MEMBERS, card=name, ms={k_: round(v[0], 3) for k_, v in ms.items()},
                runs_ms={k_: v[1] for k_, v in ms.items()}, kernels_ms={k_: round(v / 1e3, 3) for k_, v in kus.items()},
                logical_with_issue=sum(1 for x in issue if x), max_nsvc_issue=max(issue), top_issue_entries=k.value)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--out", help="also write the JSON lines to DIR/logical_states_probe.jsonl")
    a = ap.parse_args()
    name = card()
    lines = []
    for n in a.sizes:
        line = json.dumps(probe(n, name))
        print(line, flush=True)
        lines.append(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "logical_states_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
