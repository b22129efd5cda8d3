"""What GYSK_FLAG_FLOW_ERRORS costs on the bench workload, and how many of the exact top flows by server errors its sets name.

    python scripts/flow_errors_probe.py [--reps 6] [--profile 4] [--events 100000000] [--acc-events 20000000] [--out DIR]

The bench stream carries no error bits (its events have flags = 0), so for each error share (0 %, 1 %, 100 %) the probe sets them on a
seeded share of the RESP events of the bench's two batches of 100 M mixed events (bench.gen_events_gpu, same seeds) in device memory:
GYSK_EVF_CLI_ERROR, GYSK_EVF_SER_ERROR or both, in the ratio 5 : 4 : 1. At 1 % it also turns 400 RESP events into 8 low-volume
clients that always get server errors. Two engines with the bench's sizes and GYSK_FLAG_FLOW_QUERIES and GYSK_FLAG_FLOW_TOPK, one with
GYSK_FLAG_FLOW_ERRORS, take the batches alternated window by window. Per timed window: gysk_flush, the next batch's ingest,
gysk_merge_prepare and gysk_merge_finish at world 1 (host clock around each call and a sync; medians), and device_bytes. With --profile N
the device ms per batch of each kernel over N more batches (torch.profiler: the TCP and TASK drain passes, the selections' kernels). Each
engine prints the SHA-256 of its last-window flow query table, which must not differ.
Recall: the first --acc-events events of the first batch at the 1 % share go through an engine with the flag (depth 4, width 2^20); the
1000 flows with the most exact server errors are looked up in the first 1000 entries of gysk_topk_flow_errors. The card's name and power
limit are read in the same run."""
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
from tests import flow_errors as fe  # noqa: E402
from tests import flow_queries as fq  # noqa: E402


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def with_errors(ev_dev, n, share, seed):
    """a copy of a device batch with the error bits set on a seeded share of its RESP events (flags: u16 at byte 30, type at byte 28)"""
    out = ev_dev.clone()
    w16 = out.view(torch.int16).reshape(n, 16)
    g = torch.Generator(device=out.device).manual_seed(seed)
    resp = w16[:, 14] == ge.EV_RESP
    u = torch.rand(n, device=out.device, generator=g)
    bits = torch.where(u < 0.5 * share, 1, torch.where(u < 0.9 * share, 2, 3)).to(torch.int16)
    w16[:, 15] = torch.where(resp & (u < share), bits, w16[:, 15])
    if 0 < share < 1:
        idx = torch.nonzero(resp).reshape(-1)[:400]
        out.view(torch.int64).reshape(n, 4)[idx, 1] = (1 << 50) + torch.arange(len(idx), device=out.device) % 8
        w16[idx, 15] = ge.EVF_SER_ERROR
    return out


def make(err):
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23, flow_queries=True,
                    flow_topk=True, flow_errors=err)
    eng.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    return eng


def costs(a, ev_devs, n, share):
    engines = {"off": make(False), "on": make(True)}
    for eng in engines.values():
        for ev in ev_devs:                  # registers the services and tasks, as bench.py does
            eng.ingest_device_ptr(ev.data_ptr(), n)
        eng.sync()
    times = {k: dict(flush=[], ingest=[], prepare=[], finish=[]) for k in engines}
    t = 0
    for w in range(2 + a.reps):
        t += 5
        for name, eng in engines.items():   # alternated window by window
            ev = ev_devs[w % 2]
            f = timed(lambda: (eng.flush(t), eng.sync()))
            i = timed(lambda: (eng.ingest_device_ptr(ev.data_ptr(), n), eng.sync()))
            p = timed(lambda: (eng.merge_prepare(), eng.sync()))
            q = timed(lambda: (eng.merge_finish(None, 1), eng.sync()))
            if w >= 2:
                for k, v in zip(("flush", "ingest", "prepare", "finish"), (f, i, p, q)):
                    times[name][k].append(v)
    med = lambda v: round(float(np.median(v)), 3)
    out = []
    for name, eng in engines.items():
        r = dict(share=share, config=name, **{f"{k}_ms_p50": med(v) for k, v in times[name].items()},
                 device_bytes=eng.capacity()["device_bytes"], cmsq_sha256=sha(eng.export_cms_queries(True)))
        if name == "on":
            r["err_direct_last_batch"] = eng.last_batch_flow_err_direct()
            r["topk_flow_errors_last"] = len(eng.topk_flow_errors(fe.K, True))
        if a.profile:
            r["ms_per_batch"] = profile_batches(eng, ev_devs, n, a.profile)
        out.append(r)
    del engines
    torch.cuda.empty_cache()
    return out


def recall(ev_dev, m):
    ev = ev_dev[:m].cpu().numpy().view(ge.EVENT_DTYPE).reshape(-1)
    s = fq.counted(ev, None)
    keys = np.unique(s["flow_key"])
    ex = fe.exact(s, keys)[:, 1]
    order = np.lexsort((keys, -ex))
    top = keys[order[:1000]]
    top = top[ex[order[:1000]] > 0]
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=1 << 25, stage_batch=1 << 25, flow_queries=True,
                    flow_topk=True, flow_errors=True, cms_depth=4, cms_log2_width=20)
    eng.ingest_device_ptr(ev_dev.data_ptr(), m)
    eng.sync()
    got = set(eng.topk_flow_errors(1000)["flow_key"].tolist())
    return dict(batches=eng.stats()["batches"], ser_error_flows=int((ex > 0).sum()), ser_errors=int(ex.sum()),
                top1000_min_exact=int(ex[order[min(999, len(order) - 1)]]) if len(order) else 0,
                recall_top1000=float(np.mean([int(k) in got for k in top])) if len(top) else 1.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--profile", type=int, default=0, metavar="N")
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--acc-events", type=int, default=20_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = a.events
    base = [bench.gen_events_gpu(torch, n, 1234 + 7919 * b, 0, 1, dev) for b in range(2)]
    torch.cuda.synchronize()
    lines = []
    for share in (0.0, 0.01, 1.0):
        ev_devs = [with_errors(ev, n, share, 77 + b) for b, ev in enumerate(base)]
        lines += [json.dumps(r) for r in costs(a, ev_devs, n, share)]
        if share == 0.01:
            lines.append(json.dumps(dict(recall=recall(ev_devs[0], a.acc_events))))
        del ev_devs
        torch.cuda.empty_cache()
    lines.append(json.dumps(dict(card=card(), events_per_batch=n, timed_windows=a.reps)))
    print("\n".join(lines), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "flow_errors_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
