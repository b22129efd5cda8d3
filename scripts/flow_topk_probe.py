"""What GYSK_FLAG_FLOW_TOPK costs on the bench workload, and how many of the exact heaviest flows its sets name.

    python scripts/flow_topk_probe.py [--reps 10] [--profile 8] [--events 100000000] [--acc-events 20000000] [--out DIR]

Two engines with the bench's sizes and GYSK_FLAG_FLOW_QUERIES, one with GYSK_FLAG_FLOW_TOPK, take the bench's two batches of 100 M mixed
events (bench.gen_events_gpu, same seeds), alternated window by window in one run. Per timed window: gysk_flush, the next batch's ingest,
gysk_merge_prepare and gysk_merge_finish at world 1 (host clock around each call and a sync; medians). With --profile N the device ms per
batch of each kernel over N more batches (torch.profiler: the TCP and TASK drain passes apart, the radix passes of the batch sort and of
the selection summed), and of one gysk_flush + gysk_merge_prepare. Each engine prints the SHA-256 of its connection count-min and query
table, which must not differ.
Recall: the first --acc-events events of the first batch go through an engine with the flag at widths 2^16 and 2^20 (depth 4); the 1000
flows with the most exact kbytes (connection records) and the most counted response samples are looked up in the first 1000 entries of
gysk_topk_flows / gysk_topk_flow_queries. The card's name and power limit are read in the same run."""
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
from scripts.flow_queries_probe import card, profile_flush_merge  # noqa: E402
from tests import flow_queries as fq  # noqa: E402
from tests import flow_topk as ft  # noqa: E402


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def make(topk):
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23, flow_queries=True, flow_topk=topk)
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
                 cms_sha256=sha(eng.export_cms(True)), cmsq_sha256=sha(eng.export_cms_queries(True)))
        if name == "on":
            r["topk_flows_last"] = len(eng.topk_flows(ft.K, True))
            r["topk_flow_queries_last"] = len(eng.topk_flow_queries(ft.K, True))
        if a.profile:
            r["ms_per_batch"] = profile_batches(eng, ev_devs, n, a.profile)
            r["ms_flush_merge"] = profile_flush_merge(eng)
        out.append(r)
    del engines
    torch.cuda.empty_cache()
    return out


def recall(ev_dev, m):
    """per width: the share of the exact 1000 heaviest flows by kbytes and by queries that the sets name among their first 1000"""
    ev = ev_dev[:m].cpu().numpy().view(ge.EVENT_DTYPE).reshape(-1)
    conn = ev[np.isin(ev["type"], ft.TCP_TYPES)]
    fk, inc = conn["flow_key"], ft.conn_increments(conn)
    u = np.unique(fk)
    top_kb = u[np.argsort(-ft.exact_scores(u, fk, inc, 1), kind="stable")[:1000]]
    s = fq.counted(ev, None)
    uq, cnt = np.unique(s["flow_key"], return_counts=True)
    top_q = uq[np.argsort(-cnt, kind="stable")[:1000]]
    out = []
    for log2w in (16, 20):
        eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=1 << 25, stage_batch=1 << 25, flow_queries=True, flow_topk=True,
                        cms_depth=4, cms_log2_width=log2w)
        eng.ingest_device_ptr(ev_dev.data_ptr(), m)
        eng.sync()
        got_kb, got_q = set(eng.topk_flows(1000)["flow_key"].tolist()), set(eng.topk_flow_queries(1000)["flow_key"].tolist())
        out.append(dict(log2_width=log2w, batches=eng.stats()["batches"], flows_kbytes=len(u), flows_queries=len(uq),
                        recall_kbytes=float(np.mean([int(k) in got_kb for k in top_kb])),
                        recall_queries=float(np.mean([int(k) in got_q for k in top_q]))))
        del eng
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--profile", type=int, default=0, metavar="N")
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--acc-events", type=int, default=20_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = a.events
    ev_devs = [bench.gen_events_gpu(torch, n, 1234 + 7919 * b, 0, 1, dev) for b in range(2)]
    torch.cuda.synchronize()
    lines = [json.dumps(r) for r in costs(a, ev_devs, n)]
    lines.append(json.dumps(dict(recall=recall(ev_devs[0], a.acc_events))))
    lines.append(json.dumps(dict(card=card(), events_per_batch=n, timed_windows=a.reps)))
    print("\n".join(lines), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "flow_topk_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
