"""What GYSK_FLAG_FLOW_TOPK_5MIN costs on the bench workload, and how much of the five minutes' heaviest flows its sets name.

    python scripts/flow_topk_5min_probe.py [--reps 10] [--events 100000000] [--acc-events 12000000] [--out DIR]

Two engines with the bench's sizes and GYSK_FLAG_FLOW_QUERIES, GYSK_FLAG_FLOW_TOPK and both 300-s levels, one with
GYSK_FLAG_FLOW_TOPK_5MIN, take the bench's two batches of 100 M mixed events (bench.gen_events_gpu, same seeds), alternated window by
window in one run. Per timed window: gysk_flush, the next batch's ingest, gysk_merge_prepare and gysk_merge_finish at world 1 (host
clock around each call and a sync; medians). Each engine prints the SHA-256 of its level tables, which must not differ.
Recall, on two workloads of --acc-events events spread over 60 windows 5 s apart (the level then holds every one): the bench-shaped
Zipf workload, and a steady-client one (many clients sending the same moderate bytes every window, beside each window's own bursts that
fill its window set). The 1000 flows with the most exact 5-minute kbytes (and, on the Zipf workload, counted response samples) are
looked up in the first 1000 entries of gysk_topk_flows_5min / gysk_topk_flow_queries_5min, and B_L is printed beside the 1000th exact
score: a bound above it guarantees less than the list's length. The card's name and power limit are read in the same run."""
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
from scripts.flow_queries_probe import card  # noqa: E402
from tests import flow_queries as fq  # noqa: E402
from tests import flow_topk as ft  # noqa: E402

FLAGS = dict(flow_queries=True, flow_topk=True, flow_level=True, flow_query_level=True)


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def make(on):
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23, flow_topk_5min=on, **FLAGS)
    eng.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    return eng


def costs(a, ev_devs, n):
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
        r = dict(config=name, **{f"{k}_ms_p50": med(v) for k, v in times[name].items()}, device_bytes=eng.capacity()["device_bytes"],
                 cms_5min_sha256=sha(eng.export_cms_5min()), cmsq_5min_sha256=sha(eng.export_cms_queries_5min()))
        if name == "on":
            r["topk_flows_5min"] = len(eng.topk_flows_5min()[0])
            r["topk_flow_queries_5min"] = len(eng.topk_flow_queries_5min()[0])
        out.append(r)
    del engines
    torch.cuda.empty_cache()
    return out


def steady_events(rng, m, nwin, nsteady=150_000, nburst=8192):
    """nwin windows of m / nwin events: each steady client once a window with 150 kB, the rest the window's own bursts of 400 kB (each
    burst flow a few events: more than any steady client in its window, less over the five minutes)"""
    per = m // nwin
    out = []
    for w in range(nwin):
        ev = np.zeros(per, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = rng.integers(1, 1001, per).astype(np.uint64) * np.uint64(2654435761)
        ev["host_idx"] = rng.integers(0, 16, per)
        ev["type"] = ge.EV_CLOSE_CLI
        s = min(nsteady, per)
        ev["flow_key"][:s], ev["value"][:s] = np.arange(1, s + 1, dtype=np.uint64), 150 << 10
        b = per - s
        ev["flow_key"][s:] = np.uint64(10**9 + w * nburst) + rng.integers(0, nburst, b).astype(np.uint64)
        ev["value"][s:] = 400 << 10
        out.append(ev)
    return out


def top_exact(ev, which):
    if which == ft.QRY:
        s = fq.counted(ev, None)
        u, cnt = np.unique(s["flow_key"], return_counts=True)
        score = cnt.astype(np.int64)
    else:
        conn = ev[np.isin(ev["type"], ft.TCP_TYPES)]
        u = np.unique(conn["flow_key"])
        score = ft.exact_scores(u, conn["flow_key"], ft.conn_increments(conn), 1)
    order = np.argsort(-score, kind="stable")[:1000]
    return u[order], int(score[order[-1]])


def recall(windows, name, which_list):
    """the share of the exact 1000 heaviest 5-minute flows that the first 1000 entries of L name, B_L and the 1000th exact score"""
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=1 << 22, stage_batch=1 << 22, flow_topk_5min=True, **FLAGS)
    for i, ev in enumerate(windows):
        eng.ingest_events(ev)
        eng.flush(5 * i)                    # t = 0 ... 295: epochs 0 ... 9, all held
    eng.sync()
    allev = np.concatenate(windows)
    out = dict(workload=name, windows=len(windows), events=len(allev))
    for which in which_list:
        top, kth = top_exact(allev, which)
        rows, bound = eng.topk_flows_5min(1000) if which == ft.CONN else eng.topk_flow_queries_5min(1000)
        got = set(rows["flow_key"].tolist())
        tag = "kbytes" if which == ft.CONN else "queries"
        out.update({f"recall_{tag}": float(np.mean([int(k) in got for k in top])), f"bound_{tag}": int(bound), f"exact_1000th_{tag}": kth})
    del eng
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--acc-events", type=int, default=12_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = a.events
    ev_devs = [bench.gen_events_gpu(torch, n, 1234 + 7919 * b, 0, 1, dev) for b in range(2)]
    torch.cuda.synchronize()
    lines = [json.dumps(r) for r in costs(a, ev_devs, n)]
    zipf = ev_devs[0][: a.acc_events].cpu().numpy().view(ge.EVENT_DTYPE).reshape(-1)
    del ev_devs
    torch.cuda.empty_cache()
    lines.append(json.dumps(recall(np.array_split(zipf, 60), "zipf", (ft.CONN, ft.QRY))))
    lines.append(json.dumps(recall(steady_events(np.random.default_rng(5), a.acc_events, 60), "steady", (ft.CONN,))))
    lines.append(json.dumps(dict(card=card(), events_per_batch=n, timed_windows=a.reps)))
    print("\n".join(lines), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "flow_topk_5min_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
