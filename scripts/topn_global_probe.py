"""Times the cross-GPU top listeners and top processes (GYSK_FLAG_MERGE_TOPN) on one GPU: 1 M services on 4096 hosts and 256 K processes,
beside 62 500 logical services of 16 members. gysk_merge_prepare and gysk_merge_finish with and without the flag (two engines fed the same
stream, timed in alternation; the finish over `world` copies of the engine's own slab, the all-gather emulated), then gysk_topn_global
and gysk_topn_global_tasks (n = 64 with rows). ms per call (host clock around calls that end in a stream sync, median of 7) and the
device time of the kernels of the flag (torch.profiler): the eight lists' score kernels, radix sorts and picks, the two row passes and
the global pick. Prints one JSON line with the card's name and power limit.

    python scripts/topn_global_probe.py [--services 1000000] [--hosts 4096] [--tasks 262144] [--world 8] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import dist as gd  # noqa: E402
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.window_read_probe import card, timed  # noqa: E402

MEMBERS = 16
BATCH = 1 << 22
# the kernels GYSK_FLAG_MERGE_TOPN adds; os_hist / os_pass are the radix sort's
KERNELS = ("topn_score_kernel", "topn_task_score_kernel", "os_hist_kernel", "os_pass_kernel", "topn_pick_kernel", "svc_summary_kernel",
           "task_summary_kernel", "topn_global_kernel", "finish_td_kernel", "fold_td_kernel", "fold_hist_kernel", "fold_hll_kernel")
SORT = ("topn_score_kernel", "topn_task_score_kernel", "os_hist_kernel", "os_pass_kernel", "topn_pick_kernel")


def engine(n, nhosts, ntasks, topn):
    """n services, 8 response samples and 2 connection events each per window, ntasks processes with one sample each, over two
    windows; host = id % nhosts"""
    rng = np.random.default_rng(n)
    eng = ge.Engine(max_svcs=n, max_tasks=ntasks, max_batch=BATCH, merge_topn=topn)
    ids = (rng.choice(1 << 40, n, replace=False) + 1).astype(np.uint64)
    tids = (rng.choice(1 << 40, ntasks, replace=False) + (1 << 41)).astype(np.uint64)
    per = 10
    for t in (5, 10):
        for off in range(0, n, BATCH // per):
            part = ids[off: off + BATCH // per]
            ev = np.zeros(len(part) * per, dtype=ge.EVENT_DTYPE)
            ev["svc_id"] = np.repeat(part, per)
            ev["type"] = np.tile(np.array([ge.EV_RESP] * 8 + [ge.EV_ACCEPT] * 2, dtype=np.uint16), len(part))
            ev["value"] = rng.lognormal(9.0, 1.5, len(ev)).astype(np.uint32) + 1
            ev["flow_key"] = rng.integers(0, 1 << 62, len(ev), dtype=np.uint64)
            ev["host_idx"] = (ev["svc_id"] % np.uint64(nhosts)).astype(np.uint32)
            ev["tsec"] = t
            eng.ingest_events(ev)
        ev = np.zeros(ntasks, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = tids; ev["type"] = ge.EV_TASK; ev["value"] = rng.integers(0, 400, ntasks); ev["tsec"] = t
        ev["flow_key"] = rng.integers(0, 1000, ntasks).astype(np.uint64) | (rng.integers(0, 1000, ntasks).astype(np.uint64) << np.uint64(32))
        ev["host_idx"] = (tids % np.uint64(nhosts)).astype(np.uint32)
        eng.ingest_events(ev)
        eng.flush(t)
    eng.set_logical_map(ids, np.arange(n, dtype=np.uint64) // np.uint64(MEMBERS) + np.uint64(1))
    eng.sync()
    return eng


def prepare(eng):
    eng.merge_prepare()
    eng.sync()


def probe(n, nhosts, ntasks, world, name):
    import torch
    from torch.profiler import ProfilerActivity, profile

    off, eng = engine(n, nhosts, ntasks, False), engine(n, nhosts, ntasks, True)
    gathered = {}
    for key, e in (("off", off), ("on", eng)):
        prepare(e)
        p, nb = e.merge_tdigest_slab()
        slab = torch.as_tensor(gd._DevBuf(p, nb, "|u1", 1), device="cuda:0")
        gathered[key] = (torch.cat([slab] * world).contiguous(), nb)

    def finish(key, e):
        e.merge_finish(gathered[key][0].data_ptr(), world)
        e.sync()

    finish("off", off); finish("on", eng)
    runs = {k: [] for k in ("merge_prepare_without_flag", "merge_prepare_with_flag", "merge_finish_without_flag", "merge_finish_with_flag")}
    for _ in range(7):                                       # alternated: other work on the machine hits both alike
        for suffix, key, e in (("without_flag", "off", off), ("with_flag", "on", eng)):
            t0 = time.perf_counter()
            prepare(e)
            t1 = time.perf_counter()
            finish(key, e)
            t2 = time.perf_counter()
            runs["merge_prepare_" + suffix].append((t1 - t0) * 1e3)
            runs["merge_finish_" + suffix].append((t2 - t1) * 1e3)
    ms = {k: (float(np.median(v)), [round(x, 3) for x in v]) for k, v in runs.items()}
    ms["topn_global_qps_64_rows"] = timed(lambda: eng.topn_global(ge.TOPN_QPS, 64), 7)
    ms["topn_global_tasks_cpu_64_rows"] = timed(lambda: eng.topn_global_tasks(ge.TOPN_TASK_CPU, 64), 7)
    got = {m: len(eng.topn_global(m, 64)[0]) for m in (ge.TOPN_QPS, ge.TOPN_CONNS, ge.TOPN_NET)}
    got_tasks = {m: len(eng.topn_global_tasks(m, 64)[0]) for m in (ge.TOPN_TASK_CPU, ge.TOPN_TASK_CPU_DELAY, ge.TOPN_TASK_BLKIO_DELAY)}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        prepare(eng)
        finish("on", eng)
        torch.cuda.synchronize()
    kus = dict.fromkeys(KERNELS, 0.0)
    for e in prof.key_averages():
        for kn in kus:
            if kn in e.key:
                kus[kn] += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    kernels_ms = {k: round(v / 1e3, 3) for k, v in kus.items()}
    prep_ms = ms["merge_prepare_with_flag"][0]
    off.close(); eng.close()
    return dict(services=n, hosts=nhosts, tasks=ntasks, logical=(n + MEMBERS - 1) // MEMBERS, world=world, card=name,
                ms={k: round(v[0], 3) for k, v in ms.items()}, runs_ms={k: v[1] for k, v in ms.items()}, kernels_ms=kernels_ms,
                topn_sorts_ms=round(sum(kernels_ms[k] for k in SORT), 3),
                topn_sorts_share_of_prepare=round(sum(kernels_ms[k] for k in SORT) / prep_ms, 3) if prep_ms else None,
                nonzero_entries=dict(svc=got, task=got_tasks))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--services", type=int, default=1_000_000)
    ap.add_argument("--hosts", type=int, default=4096)
    ap.add_argument("--tasks", type=int, default=262_144)
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--out", help="also write the JSON line to DIR/topn_global_probe.jsonl")
    a = ap.parse_args()
    line = json.dumps(probe(a.services, a.hosts, a.tasks, a.world, card()))
    print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "topn_global_probe.jsonl"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
