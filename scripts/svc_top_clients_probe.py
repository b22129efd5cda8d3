"""What GYSK_FLAG_SVC_TOP_CLIENTS costs on the bench workload, and how well the summaries name each service's heaviest clients.

    python scripts/svc_top_clients_probe.py [--reps 6] [--profile 3] [--events 100000000] [--out DIR]

Per service capacity (the bench's 2^17 slots, and 2^20), two engines, one with the flag, take the bench's two batches of 100 M mixed
events (bench.gen_events_gpu, same seeds), alternated window by window in one run. Per timed window: gysk_flush and the next batch
(host clock around each call and a sync; medians), and device_bytes. With --profile N the device ms per batch of each kernel over N more
batches (torch.profiler: topc_pairs_kernel, the radix passes, topc_merge_kernel among them). Each engine prints the SHA-256 of its window
read, which must not differ. Then the one-hot-service case: one service with 2^20 clients in a batch of 2^22 events. Then accuracy on a
seeded CPU stream (Zipf clients of Zipf services, 8 batches in one window): the recall of each service's exact 16 heaviest clients among
its listed ones, and the median delta / N_s. The card's name and power limit are read in the same run."""
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


def timed(f):
    t0 = time.perf_counter()
    f()
    return (time.perf_counter() - t0) * 1e3


def costs(a, ev_devs, n, max_svcs):
    engines = {}
    for name, on in (("off", False), ("on", True)):
        eng = ge.Engine(device=0, max_svcs=max_svcs, max_tasks=1 << 15, max_batch=(1 << 27) - 1, stage_batch=1 << 23, svc_top_clients=on)
        for ev in ev_devs:
            eng.ingest_device_ptr(ev.data_ptr(), n)
        eng.sync()
        eng.flush(5)
        engines[name] = eng
    times = {k: dict(flush=[], batch=[]) for k in engines}
    t = 5
    for w in range(2 + a.reps):
        t += 5
        for name, eng in engines.items():
            ev = ev_devs[w % 2]
            f = timed(lambda: (eng.flush(t), eng.sync()))
            b = timed(lambda: (eng.ingest_device_ptr(ev.data_ptr(), n), eng.sync()))
            if w >= 2:
                times[name]["flush"].append(f)
                times[name]["batch"].append(b)
    med = lambda v: round(float(np.median(v)), 3)
    out = []
    for name, eng in engines.items():
        eng.flush(t + 5)
        rows, _, nrows = eng.query_window_hosts()
        r = dict(config=name, max_svcs=max_svcs, services=nrows, **{f"{k}_ms_p50": med(v) for k, v in times[name].items()},
                 device_bytes=eng.capacity()["device_bytes"],
                 window_sha256=hashlib.sha256(b"".join(sorted(bytes(x) for x in rows))).hexdigest())
        if name == "on":
            tcr = eng.query_top_clients_window(ge.TOPC_LAST)[0]
            r["services_with_clients"] = int((tcr["n"] > 0).sum())
        if a.profile:
            r["ms_per_batch"] = profile_batches(eng, ev_devs, n, a.profile)
        out.append(r)
    for eng in engines.values():
        eng.close()
    return out


def one_hot(a):
    """one service with 2^20 distinct clients in each batch of 2^22 connection events (the split path), flag off and on"""
    rng = np.random.default_rng(5)
    n = 1 << 22
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["type"] = 77, ge.EV_CLOSE_SER
    ev["flow_key"] = (np.arange(n) % (1 << 20)).astype(np.uint64) + np.uint64(1 << 40)
    ev["value"] = (rng.zipf(1.3, n) % 100000) << 10
    dev = torch.from_numpy(ev.view(np.uint8)).cuda()
    out = []
    for on in (False, True):
        eng = ge.Engine(device=0, max_svcs=1 << 10, max_tasks=1 << 10, max_batch=n, svc_top_clients=on)
        eng.ingest_device_ptr(dev.data_ptr(), n)
        eng.sync()
        b = [timed(lambda: (eng.ingest_device_ptr(dev.data_ptr(), n), eng.sync())) for _ in range(a.reps)]
        out.append(dict(case="one_hot_service", config="on" if on else "off", batch_ms_p50=round(float(np.median(b)), 3)))
        eng.close()
    return out


def accuracy():
    """recall of each service's exact 16 heaviest clients (by kbytes) and the median delta / N_s, one window of 8 batches"""
    from tests import svc_top_clients as tc
    rng = np.random.default_rng(9)
    nsvc, n = 2000, 1 << 20
    eng = ge.Engine(device=0, max_svcs=4096, max_tasks=64, max_batch=n, svc_top_clients=True)
    evs = []
    for _ in range(8):
        ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = (rng.zipf(1.2, n) % nsvc + 1).astype(np.uint64)
        ev["flow_key"] = (rng.zipf(1.1, n) % 200000).astype(np.uint64) * np.uint64(2654435761) + ev["svc_id"]
        ev["type"] = ge.EV_CONNECT
        ev["value"] = rng.integers(0, 1 << 20, n)
        eng.ingest_events(ev)
        eng.sync()
        evs.append(ev)
    eng.flush(5)
    exact = tc.batch_sums(np.concatenate(evs))
    ids = np.array(sorted(exact), dtype=np.uint64)
    rows = eng.query_svc_top_clients(ids, ge.TOPC_LAST)
    recall, ratio = [], []
    for sid, r in zip(ids.tolist(), rows):
        ex = exact[sid]
        top = sorted(((kb, k) for k, (kb, _) in ex.items() if kb > 0), key=lambda t: (-t[0], t[1]))[: tc.K]
        if not top:
            continue
        listed = set(r["entries"]["flow_key"][: r["n"]].tolist())
        recall.append(sum(k in listed for _, k in top) / len(top))
        ratio.append(int(r["delta"]) / sum(kb for kb, _ in ex.values()))
    eng.close()
    return dict(case="accuracy", services=len(recall), recall_top16_mean=round(float(np.mean(recall)), 4),
                recall_top16_min=round(float(np.min(recall)), 4), delta_over_ns_median=float(np.median(ratio)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--profile", type=int, default=0, metavar="N")
    ap.add_argument("--events", type=int, default=100_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    n = a.events
    ev_devs = [bench.gen_events_gpu(torch, n, 1234 + 7919 * b, 0, 1, dev) for b in range(2)]
    torch.cuda.synchronize()
    lines = []
    for max_svcs in (1 << 17, 1 << 20):
        lines += [json.dumps(r) for r in costs(a, ev_devs, n, max_svcs)]
        print("\n".join(lines[-2:]), flush=True)
    del ev_devs
    torch.cuda.empty_cache()
    for r in one_hot(a) + [accuracy()]:
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    lines.append(json.dumps(dict(card=card(), events_per_batch=n, timed_windows=a.reps)))
    print(lines[-1], flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "svc_top_clients_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
