"""BASELINE.json configs[3] (SURVEY.md §8d "Config 4") at spec: 1 B mixed events (70 / 20 / 10 RESP / TCP / TASK), 100 K services on 4096
hosts, sharded by host_idx % N over N GPUs (N = 4), one NCCL sketch merge (gysk_merge_global) for the global per-logical-service
answers (16 instances per logical service, spread over the ranks), compared with the CPU aggregation of the SAME stream: every rank
copies its batches back to the host and feeds them to the CPU oracle port on its share of the host cores; the logical answers of the
CPU side (sums of the member histograms / conn cells, max of the HLL registers, summed over the ranks) must equal the GPUs' merged
answers bit for bit. Lives under tests/ because it runs the oracle (the checker) next to the product.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 4 --master-addr 127.0.0.1 tests/run_config3.py [--events 1e9]

Prints one JSON line (rank 0)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from gyeeta_b200 import dist as gd  # noqa: E402
from gyeeta_b200 import engine as ge  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--events", type=float, default=1e9, help="over all GPUs")
ap.add_argument("--batch", type=int, default=50_000_000)
ap.add_argument("--services", type=int, default=100_000, help="over all GPUs")
ap.add_argument("--cpu-threads", type=int, default=0, help="per rank; 0 = host cores / world")
args = ap.parse_args()

rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); local = int(os.environ.get("LOCAL_RANK", "0"))
os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)

nsvc = args.services // world
bench.NSVC = nsvc
per_rank = int(args.events) // world
nb = (per_rank + args.batch - 1) // args.batch
ids = bench.rank_service_ids(rank)
ids_all = np.concatenate([bench.rank_service_ids(r) for r in range(world)])
g_all = np.concatenate([np.arange(nsvc, dtype=np.uint64) * np.uint64(world) + np.uint64(r) for r in range(world)])
logical_all = g_all // np.uint64(16) + np.uint64(1)
my_logical = (np.arange(nsvc, dtype=np.uint64) * np.uint64(world) + np.uint64(rank)) // np.uint64(16)      # 0-based, per local service
nlogical = int(g_all.max() // 16 + 1)

batches = [bench.gen_events_gpu(torch, min(args.batch, per_rank - b * args.batch), 4242 + rank + 7919 * b, rank, world, dev) for b in range(nb)]
torch.cuda.synchronize()


def barrier():
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()


# ---- GPU: ids registered up front (the CPU side's first touch of an id is inside its timed pass; registration is not the point here)
eng = ge.Engine(device=local, max_svcs=1 << 17, max_tasks=1 << 15, max_batch=(1 << 27) - 1, rank=rank, world=world)
eng.register_ids(ids)
eng.set_logical_map(ids_all, logical_all)
if world > 1:
    gd.nccl_comm_init(eng, dist)
    eng.merge_global()                 # NCCL sets up its channels inside the first collective of a communicator (~1.2 s on 4 GPUs):
    eng.sync()                         # an empty merge before the timed window, as a long-running madhava has long done
stream = torch.cuda.ExternalStream(eng.stream(), device=dev)
barrier()
t0, t1, t2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
w0 = time.perf_counter()
with torch.cuda.stream(stream):
    t0.record()
for b_ in batches:
    eng.ingest_device_ptr(b_.data_ptr(), len(b_))
eng.flush(5)
with torch.cuda.stream(stream):
    t1.record()
if world > 1:
    eng.merge_global()
else:
    eng.merge_prepare(); eng.merge_finish(None, 1)
with torch.cuda.stream(stream):
    t2.record()
eng.sync()
barrier()
gpu_wall = time.perf_counter() - w0
tg = torch.tensor([t0.elapsed_time(t2), t1.elapsed_time(t2), gpu_wall * 1e3], device=dev, dtype=torch.float64)
if world > 1:
    dist.all_reduce(tg, op=dist.ReduceOp.MAX)
lids = np.arange(1, nlogical + 1, dtype=np.uint64)
gq = eng.query_logical(lids)

# ---- CPU: the same batches through the oracle port, pre-sharded by service over this rank's share of the cores
nthr = args.cpu_threads or max(1, (os.cpu_count() or 1) // world)
L = po.lib()
engines = [po.OracleEngine(max_svcs=nsvc + 16, max_tasks=bench.NTASK + 16) for _ in range(nthr)]
eh = (C.c_void_p * nthr)(*[e.h for e in engines])
own = bench.shard_owner(np.rec.fromarrays([ids], names="svc_id"), nthr, "svc") if nthr > 1 else np.zeros(nsvc, dtype=np.int32)
for t in range(nthr):
    engines[t].register_ids(ids[own == t])                 # untimed on both sides
cpu_sec = 0.0
for b_ in batches:
    ev = b_.cpu().numpy().view(np.uint8).reshape(-1).view(ge.EVENT_DTYPE)
    owner = bench.shard_owner(ev, nthr, "svc")
    order = np.argsort(owner, kind="stable")
    cuts = np.searchsorted(owner[order], np.arange(1, nthr))
    shards = [np.ascontiguousarray(a) for a in np.split(ev[order], cuts)]
    sp = (C.c_void_p * nthr)(*[s.ctypes.data for s in shards])
    cn = (C.c_uint64 * nthr)(*[len(s) for s in shards])
    cpu_sec += L.gyo_bench_ingest(eh, sp, cn, nthr, 1 << 22)
    del shards, ev
tm0 = time.perf_counter()
for e in engines:
    e.flush(5)
# logical roll-up on the CPU: per member the last-window histogram / conn cell / HLL registers, folded into its logical service
hist = np.zeros((nlogical, 15, 2), dtype=np.int64)
tot = np.zeros(nlogical, dtype=np.int64)
maxv = np.zeros(nlogical, dtype=np.int64)
conn = np.zeros((nlogical, 2), dtype=np.int64)
regs = np.zeros((nlogical, 4096), dtype=np.uint8)
for i in range(nsvc):
    e = engines[own[i]]
    h = e.export_hist(int(ids[i]), ge.HIST_RESP_LAST)
    lg = int(my_logical[i])
    if h is not None:
        cells, total, mx = h
        hist[lg, :, 0] += cells["count"].astype(np.int64); hist[lg, :, 1] += cells["sum"]
        tot[lg] += total; maxv[lg] = max(maxv[lg], mx)
    c = e.export_conn(int(ids[i]))
    if c is not None:
        conn[lg, 0] += c[1] & 0xFFFFFFFF; conn[lg, 1] += c[1] >> 32
    r = e.export_hll(int(ids[i]))
    if r is not None:
        np.maximum(regs[lg], r, out=regs[lg])
cpu_merge_sec = time.perf_counter() - tm0
tc = torch.tensor([cpu_sec, cpu_merge_sec], device=dev, dtype=torch.float64)
T = [torch.from_numpy(a).to(dev) for a in (hist, tot, conn)]
Tm = [torch.from_numpy(maxv).to(dev), torch.from_numpy(regs).to(dev)]
if world > 1:
    dist.all_reduce(tc, op=dist.ReduceOp.MAX)
    for t in T:
        dist.all_reduce(t)
    for t in Tm:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
hist, tot, conn = (t.cpu().numpy() for t in T)
maxv, regs = (t.cpu().numpy() for t in Tm)

# ---- compare (every rank checks the merged answers it holds)
bad = 0
checked = 0
for k, s in enumerate(gq):
    if tot[k] == 0 and conn[k, 0] == 0:
        continue
    checked += 1
    ok = (s["found"] == 1 and s["nqrys_5s"] == tot[k] and s["total_resp_5sec"] == int(hist[k, :, 1].sum()) and s["max_resp_ms"] == maxv[k]
          and s["nconns_5s"] == conn[k, 0] and s["kbytes_5s"] == conn[k, 1] and s["td_count"] == tot[k]
          and s["distinct_clients"] == L.gyo_hll_estimate(po._p(np.ascontiguousarray(regs[k])), 12))
    if ok and po.ref() is not None:                         # p95 / p99 / p25 of the merged histogram by the reference's own get_percentiles
        ser = np.zeros(16, dtype=po.SERIAL_DTYPE)
        ser["count"][:15] = hist[k, :, 0]; ser["sum"][:15] = hist[k, :, 1]
        out = np.zeros(3, dtype=np.int64)
        po.ref().gyref_hist_pct_from_serial(0, 0, po._p(ser), int(tot[k]), int(maxv[k]), po._p(np.array([95, 99, 25], dtype=np.float32)), 3, po._p(out), None)
        ok = [s["p95_5s_resp_ms"], s["p99_5s_resp_ms"], s["p25_5s_resp_ms"]] == out.tolist()
    bad += 0 if ok else 1
tb = torch.tensor([bad, checked], device=dev, dtype=torch.int64)
if world > 1:
    dist.all_reduce(tb, op=dist.ReduceOp.MAX)

# t-digest of the merged logical services against the exact quantiles of their samples (the three busiest logical services)
hot = np.argsort(-tot)[:3]
tdrows, td_bad = [], 0
for k in hot:
    members = torch.from_numpy(ids[my_logical == k].view(np.int64)).to(dev)
    vals = torch.cat([(b_[:, 2][torch.isin(b_[:, 0], members) & (((b_[:, 3] >> 32) & 0xFFFF) == 5)] & 0xFFFFFFFF) for b_ in batches]).to(torch.int32)
    if world > 1:
        nmine = torch.tensor([vals.numel()], device=dev, dtype=torch.int64)
        ns = [torch.zeros_like(nmine) for _ in range(world)]
        dist.all_gather(ns, nmine)
        mx = int(max(int(x) for x in ns))
        pad = torch.full((mx,), -1, device=dev, dtype=torch.int32); pad[: vals.numel()] = vals
        allv = [torch.empty_like(pad) for _ in range(world)]
        dist.all_gather(allv, pad)
        vals = torch.cat([a[: int(n_)] for a, n_ in zip(allv, ns)])
    if rank == 0 and vals.numel() >= 10_000:
        ex = torch.quantile(vals[: 16_000_000].double(), torch.tensor([0.5, 0.95, 0.99], device=dev, dtype=torch.float64), interpolation="lower").cpu().numpy()
        s = gq[int(k)]
        got = np.array([s["td_p50_us"], s["td_p95_us"], s["td_p99_us"]])
        # rank error: distance of q from [#{v < g}, #{v <= g}] / n; bound: two K_1 cells at q plus 1 / n (tests/test_gpu_td_accuracy.py)
        n_ = vals.numel()
        rk, bd = [], []
        for q, g in zip((0.5, 0.95, 0.99), got.tolist()):
            lo, hi = int((vals < g).sum()) / n_, int((vals <= g).sum()) / n_
            rk.append(max(0.0, lo - q, q - hi))
            bd.append(2.0 * (np.pi / 200) * np.sqrt(q * (1.0 - q)) + 1.0 / n_)
        td_bad += int(any(r > b for r, b in zip(rk, bd)))
        tdrows.append({"logical": int(k) + 1, "samples": int(n_), "rel_err_p50_p95_p99": (np.abs(got - ex) / ex).tolist(),
                       "rank_err_p50_p95_p99": rk, "rank_bound": bd})

if rank == 0:
    total = per_rank * world
    gpu_ms, merge_ms, gpu_wall_ms = (float(x) for x in tg)
    cs, cms_ = (float(x) for x in tc)
    print(json.dumps({
        "config": "BASELINE configs[3]: 1 B mixed events over N GPUs by host_idx % N, NCCL sketch merge, vs CPU aggregation of the same stream",
        "n_gpus": world, "events_total": total, "services_total": nsvc * world, "logical_services": nlogical,
        "gpu": {"device_ms_ingest_flush_merge": gpu_ms, "merge_global_ms": merge_ms, "wall_ms_incl_launch": gpu_wall_ms,
                "events_per_s": total / (gpu_ms * 1e-3), "input": "device-resident batches of %d events" % args.batch},
        "cpu": {"kind": "port (oracle/gysk_oracle.c), pre-sharded by service", "threads_total": nthr * world, "cpu_model": bench.cpu_model(),
                "ingest_sec_max_over_ranks": cs, "events_per_s": total / cs, "logical_rollup_sec_python": cms_},
        "speedup_gpu_over_cpu_ingest": (total / (gpu_ms * 1e-3)) / (total / cs),
        "parity": {"logical_services_checked": int(tb[1]), "mismatches": int(tb[0]),
                   "fields": "found, nqrys_5s, total_resp_5sec, max_resp_ms, nconns_5s, kbytes_5s, td_count, distinct_clients (HLL estimate of the "
                             "max-merged registers), p95/p99/p25 via the reference's get_percentiles on the summed histogram"},
        "tdigest_vs_exact_hot_logical": tdrows, "tdigest_rank_bound_exceeded": td_bad}))
if world > 1:
    dist.destroy_process_group()
sys.exit(0 if int(tb[0]) == 0 and td_bad == 0 else 1)
