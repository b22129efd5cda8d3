"""Times the host-cluster roll-up (GYSK_FLAG_MERGE_CLUSTERS) on one GPU: 1 M services on 4096 hosts in 512 clusters (MAX_NUM_CLUSTERS of
MS_CLUSTER_STATE), beside 62 500 logical services of 16 members. gysk_merge_prepare with and without the flag (two engines fed the same
stream, timed in alternation), gysk_query_cluster_states_all and gysk_query_cluster_states over every cluster id. ms per call (host clock
around calls that end in a stream sync, median of 7) and the device time of the two cluster fold kernels (torch.profiler). Prints one
JSON line with the card's name and power limit.

    python scripts/cluster_states_probe.py [--services 1000000] [--hosts 4096] [--clusters 512] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.window_read_probe import card, timed  # noqa: E402

MEMBERS = 16
KERNELS = ("fold_cluster_hosts_kernel", "fold_clusters_kernel", "cluster_row_kernel", "fold_levels_kernel", "fold_hist_kernel",
           "fold_td_kernel", "fold_hll_kernel")


def engine(n, nhosts, nclusters, clusters):
    """n services, 8 response samples and 2 connection events each per window over two windows, host = id % nhosts"""
    rng = np.random.default_rng(n)
    eng = ge.Engine(max_svcs=n, max_tasks=1024, max_batch=1 << 22, merge_clusters=clusters)
    ids = (rng.choice(1 << 40, n, replace=False) + 1).astype(np.uint64)
    per = 10
    for t in (5, 10):
        for off in range(0, n, (1 << 22) // per):
            part = ids[off: off + (1 << 22) // per]
            ev = np.zeros(len(part) * per, dtype=ge.EVENT_DTYPE)
            ev["svc_id"] = np.repeat(part, per)
            ev["type"] = np.tile(np.array([ge.EV_RESP] * 8 + [ge.EV_ACCEPT] * 2, dtype=np.uint16), len(part))
            ev["value"] = rng.lognormal(9.0, 1.5, len(ev)).astype(np.uint32) + 1
            ev["flow_key"] = rng.integers(0, 1 << 62, len(ev), dtype=np.uint64)
            ev["host_idx"] = (ev["svc_id"] % np.uint64(nhosts)).astype(np.uint32)
            eng.ingest_events(ev)
        eng.flush(t)
    eng.set_logical_map(ids, np.arange(n, dtype=np.uint64) // np.uint64(MEMBERS) + np.uint64(1))
    if clusters:
        hosts = np.arange(nhosts, dtype=np.uint32)
        eng.set_cluster_map(hosts, (hosts % nclusters).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15 >> 8) + np.uint64(1))
    eng.sync()
    return eng


def prepare(eng):
    eng.merge_prepare()
    eng.sync()


def probe(n, nhosts, nclusters, name):
    import torch
    from torch.profiler import ProfilerActivity, profile

    off, eng = engine(n, nhosts, nclusters, False), engine(n, nhosts, nclusters, True)
    prepare(off); prepare(eng)
    runs = {"merge_prepare_without_flag": [], "merge_prepare_with_flag": []}
    for _ in range(7):                                       # alternated: other work on the machine hits both alike
        for key, e in (("merge_prepare_without_flag", off), ("merge_prepare_with_flag", eng)):
            t0 = time.perf_counter()
            prepare(e)
            runs[key].append((time.perf_counter() - t0) * 1e3)
    ms = {k: (float(np.median(v)), [round(x, 3) for x in v]) for k, v in runs.items()}
    eng.merge_finish(None, 1)
    rows, nc = eng.query_cluster_states_all()
    cids = np.array([r.cluster_id for r in rows], dtype=np.uint64)
    out_all, out_id = (ge.ClusterRow * nc)(), (ge.ClusterRow * nc)()
    k = C.c_uint32()

    def read_all():
        assert eng.L.gysk_query_cluster_states_all(eng.h, 0, out_all, nc, C.byref(k)) == 0 and k.value == nc

    def read_by_id():
        assert eng.L.gysk_query_cluster_states(eng.h, ge._p(cids), nc, out_id) == 0

    ms["query_cluster_states_all"] = timed(read_all, 7)
    ms["query_cluster_states_every_id"] = timed(read_by_id, 7)
    assert all(bytes(a) == bytes(b) for a, b in zip(out_all, out_id))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        prepare(eng)
        eng.merge_finish(None, 1)
        read_all()
        torch.cuda.synchronize()
    kus = dict.fromkeys(KERNELS, 0.0)
    for e in prof.key_averages():
        for kn in kus:
            if kn in e.key:
                kus[kn] += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    totals = dict(nhosts=sum(r.st.nhosts for r in out_all), nsvc=sum(r.st.nsvc for r in out_all))
    off.close(); eng.close()
    return dict(services=n, hosts=nhosts, clusters=nc, logical=(n + MEMBERS - 1) // MEMBERS, card=name,
                ms={k_: round(v[0], 3) for k_, v in ms.items()}, runs_ms={k_: v[1] for k_, v in ms.items()},
                kernels_ms={k_: round(v / 1e3, 3) for k_, v in kus.items()}, totals=totals)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--services", type=int, default=1_000_000)
    ap.add_argument("--hosts", type=int, default=4096)
    ap.add_argument("--clusters", type=int, default=512)
    ap.add_argument("--out", help="also write the JSON line to DIR/cluster_states_probe.jsonl")
    a = ap.parse_args()
    line = json.dumps(probe(a.services, a.hosts, a.clusters, card()))
    print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "cluster_states_probe.jsonl"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
