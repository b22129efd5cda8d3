"""What GYSK_FLAG_FLOW_RESP_HIST costs on the bench workload, the tables it leaves behind, and how close its per-flow percentiles are.

    python scripts/flow_resp_hist_probe.py [--reps 10] [--profile 8] [--events 100000000] [--acc-events 20000000] [--out DIR]

Three engines with the bench's sizes take the bench's two batches of 100 M mixed events (bench.gen_events_gpu, same seeds), one after the
other: GYSK_FLAG_FLOW_QUERIES; that and GYSK_FLAG_FLOW_RESP_HIST; both and GYSK_FLAG_FLOW_QUERY_LEVEL. Ten warm-up windows 30 s apart
first fill every ring slot. Then per timed window: gysk_flush, the next batch's ingest and gysk_merge_prepare (host clock around each call
and a sync; medians). With --profile N the device ms per batch of each kernel over N more batches (torch.profiler: the TCP and TASK drain
passes apart) and of one gysk_flush + gysk_merge_prepare. Each engine prints one JSON line with the SHA-256 of the connection count-min,
the query tables and the response histograms.
Accuracy: the first --acc-events events of the first batch go through an engine with the flag at widths 2^16 and 2^20 (depth 4); for the
1000 flows with the most counted samples, gysk_query_flow_resp's p95 / p99 are compared with the same rule on the flow's exact bucket
counts. The card's name and power limit are read in the same run."""
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
from tests import flow_resp_hist as fr  # noqa: E402

CONFIGS = {"flow_queries": {}, "resp_hist": dict(flow_resp_hist=True), "resp_hist_level": dict(flow_resp_hist=True, flow_query_level=True)}


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def run(name, a, ev_devs, n):
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23, flow_queries=True,
                    **CONFIGS[name])
    eng.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    for ev in ev_devs:                      # registers the services and tasks, as bench.py does
        eng.ingest_device_ptr(ev.data_ptr(), n)
    eng.sync()
    times = dict(flush=[], ingest=[], prepare=[])
    t = 0
    for w in range(10 + a.reps):
        t += 30 if w < 10 else 5
        ev = ev_devs[w % 2]
        f = timed(lambda: (eng.flush(t), eng.sync()))
        i = timed(lambda: (eng.ingest_device_ptr(ev.data_ptr(), n), eng.sync()))
        p = timed(lambda: (eng.merge_prepare(), eng.sync()))
        if w >= 10:
            times["flush"].append(f); times["ingest"].append(i); times["prepare"].append(p)
    med = lambda v: round(float(np.median(v)), 3)
    r = dict(config=name, flush_ms_p50=med(times["flush"]), next_ingest_ms_p50=med(times["ingest"]), merge_prepare_ms_p50=med(times["prepare"]),
             device_bytes=eng.capacity()["device_bytes"], cms_sha256=sha(eng.export_cms(True)), cmsq_last_sha256=sha(eng.export_cms_queries(True)),
             flow_query_direct_last_batch=eng.last_batch_flow_query_direct())
    if CONFIGS[name]:
        r["cmsr_cur_sha256"], r["cmsr_last_sha256"] = sha(eng.export_cms_resp()), sha(eng.export_cms_resp(True))
        r["flow_resp_direct_last_batch"] = eng.last_batch_flow_resp_direct()
    if "flow_query_level" in CONFIGS[name]:
        r["cmsr_5min_sha256"] = sha(eng.export_cms_resp_5min())
    if a.profile:
        r["ms_per_batch"] = profile_batches(eng, ev_devs, n, a.profile)
        r["ms_flush_merge"] = profile_flush_merge(eng)
    del eng
    return r


def accuracy(ev_dev, m):
    """per width: how often the estimated p95 / p99 of the 1000 heaviest flows equal those of their exact counts"""
    ev = ev_dev[:m].cpu().numpy().view(ge.EVENT_DTYPE).reshape(-1)
    s = fq.counted(ev, None)
    u, inv, cnt = np.unique(s["flow_key"], return_inverse=True, return_counts=True)
    top = np.sort(u[np.argsort(-cnt, kind="stable")[:1000]])
    exact = fr.exact(s, top)
    want = np.array([fr.percentiles(c) for c in exact], dtype=np.int64)
    out = []
    for log2w in (16, 20):
        eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=1 << 25, stage_batch=1 << 23, flow_queries=True,
                        flow_resp_hist=True, cms_depth=4, cms_log2_width=log2w)
        eng.ingest_device_ptr(ev_dev.data_ptr(), m)
        eng.sync()
        got = eng.query_flow_resp(top)
        over = got["counts"].astype(np.int64) - exact
        assert (over >= 0).all()
        out.append(dict(log2_width=log2w, flows=len(top), samples_min=int(exact.sum(axis=1).min()),
                        p95_equal=float(np.mean(got["p95_ms"] == want[:, 1])), p99_equal=float(np.mean(got["p99_ms"] == want[:, 2])),
                        p95_over=float(np.mean(got["p95_ms"] > want[:, 1])), p99_over=float(np.mean(got["p99_ms"] > want[:, 2])),
                        count_overestimate_mean=float(over.sum(axis=1).mean()), counts_exact=float(np.mean((over == 0).all(axis=1)))))
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
    lines = [json.dumps(run(name, a, ev_devs, n)) for name in CONFIGS]
    lines.append(json.dumps(dict(accuracy=accuracy(ev_devs[0], a.acc_events))))
    lines.append(json.dumps(dict(card=card(), events_per_batch=n, timed_windows=a.reps)))
    print("\n".join(lines), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "flow_resp_hist_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
