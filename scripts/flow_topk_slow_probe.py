"""What GYSK_FLAG_FLOW_TOPK_SLOW costs on the bench workload, and how many of the exact top slow flows its sets name.

    python scripts/flow_topk_slow_probe.py [--reps 8] [--profile 4] [--events 100000000] [--acc-events 20000000] [--out DIR]

Two engines with the bench's sizes and GYSK_FLAG_FLOW_QUERIES, GYSK_FLAG_FLOW_RESP_HIST and GYSK_FLAG_FLOW_TOPK, one with
GYSK_FLAG_FLOW_TOPK_SLOW, take the bench's two batches of 100 M mixed events (bench.gen_events_gpu, same seeds), alternated window by
window in one run. Per timed window: gysk_flush, the next batch's ingest, gysk_merge_prepare and gysk_merge_finish at world 1 (host clock
around each call and a sync; medians), and device_bytes. With --profile N the device ms per batch of each kernel over N more batches
(torch.profiler: the TCP drain pass, and the slow set's score kernel beside the radix passes of every selection summed). Each engine prints
the SHA-256 of its last-window response table, which must not differ.
Recall: the first --acc-events events of the first batch go through an engine with the flag (depth 4, width 2^20), alone and with 300
clients added that take a slow path (40 requests each, 30 of them above 300 ms); the 1000 flows with the most exact slow samples are looked
up in the first 1000 entries of gysk_topk_flow_slow. The card's name and power limit are read in the same run."""
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
from tests import flow_queries as fq  # noqa: E402
from tests import flow_topk_slow as fs  # noqa: E402

BS = fs.b_slow(300)


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def make(slow):
    eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23, flow_queries=True,
                    flow_resp_hist=True, flow_topk=True, flow_topk_slow=slow)
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
                 cmsr_sha256=sha(eng.export_cms_resp(True)))
        if name == "on":
            r["topk_flow_slow_last"] = len(eng.topk_flow_slow(fs.K, True))
        if a.profile:
            r["ms_per_batch"] = profile_batches(eng, ev_devs, n, a.profile)
        out.append(r)
    del engines
    torch.cuda.empty_cache()
    return out


def slow_clients(rng, ev):
    """300 clients of the workload's services, 40 requests each, 30 of them above 300 ms"""
    resp = ev[ev["type"] == ge.EV_RESP]
    out = np.zeros(300 * 40, dtype=ge.EVENT_DTYPE)
    out["svc_id"] = rng.choice(resp["svc_id"], len(out))
    out["host_idx"] = rng.choice(resp["host_idx"], len(out))
    out["type"] = ge.EV_RESP
    out["flow_key"] = np.repeat(rng.integers(1 << 50, 1 << 51, 300).astype(np.uint64), 40)
    slow = np.tile(np.arange(40) < 30, 300)
    out["value"] = np.where(slow, rng.integers(301_000, 3_000_000, len(out)), rng.integers(0, 100_000, len(out)))
    return out


def recall(ev_dev, m):
    ev = ev_dev[:m].cpu().numpy().view(ge.EVENT_DTYPE).reshape(-1)
    rng = np.random.default_rng(11)
    out = []
    for name, batch in (("bench", ev), ("bench_plus_slow_clients", np.concatenate([ev, slow_clients(rng, ev)]))):
        s = fq.counted(batch, None)
        keys = np.unique(s["flow_key"])
        ex = fs.exact_slow(s, keys, BS)
        order = np.lexsort((keys, -ex))
        top = keys[order[:1000]]
        eng = ge.Engine(device=0, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=1 << 25, stage_batch=1 << 25, flow_queries=True,
                        flow_resp_hist=True, flow_topk=True, flow_topk_slow=True, cms_depth=4, cms_log2_width=20)
        d = torch.from_numpy(batch.view(np.uint8).copy()).to(ev_dev.device)
        eng.ingest_device_ptr(d.data_ptr(), len(batch))
        eng.sync()
        got = set(eng.topk_flow_slow(1000)["flow_key"].tolist())
        out.append(dict(workload=name, batches=eng.stats()["batches"], slow_flows=int((ex > 0).sum()), slow_samples=int(ex.sum()),
                        top1000_min_exact=int(ex[order[min(999, len(order) - 1)]]) if len(order) else 0,
                        recall_top1000=float(np.mean([int(k) in got for k in top])) if len(top) else 1.0))
        del eng, d
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=8)
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
        with open(os.path.join(a.out, "flow_topk_slow_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
