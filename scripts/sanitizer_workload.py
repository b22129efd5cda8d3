"""a small pass over every kernel of the hot path, for compute-sanitizer (memcheck / racecheck / synccheck):

    compute-sanitizer --tool racecheck python scripts/sanitizer_workload.py

ingest_kernel (all five event kinds, auto-registration), the one-sweep radix passes with 6- to 8-bit digits (the batches' key
sorts, the top-N sorts) and 9-bit digits (a group-by of 100 000 samples), segs_mark / long_sum / bins_merge (small and > 512-entry
merged lists), flush + eviction + table rebuild, the raw decode kernel, the merge step's fold / finish kernels, the read-side
gathers. Sizes keep a racecheck run within a few minutes."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gyeeta_b200 import engine as ge  # noqa: E402
from gyeeta_b200 import synth  # noqa: E402

rng = np.random.default_rng(3)
eng = ge.Engine(max_svcs=2048, max_tasks=128, max_batch=1 << 17, cms_log2_width=12, idle_evict_secs=20)
tsec = 1000
for w in range(4):
    ev = synth.gen_mixed(rng, 60_000, 600 if w < 2 else 300, ntask=32, nhosts=16, nclients=3000)
    hot = ev["type"] == ge.EV_RESP
    ev["svc_id"][np.flatnonzero(hot)[:30_000]] = ev["svc_id"][np.flatnonzero(hot)[0]]     # one service with a long merged list
    act = np.zeros(64, dtype=ge.EVENT_DTYPE)
    act["svc_id"] = ev["svc_id"][:64]; act["flow_key"] = rng.integers(1, 1 << 40, 64); act["value"] = 100; act["type"] = ge.EV_ACTIVE
    act["flags"] = 3; act["tsec"] = np.float32(1.5).view(np.uint32)
    eng.ingest_events(np.concatenate([ev, act]))
    r16 = np.zeros(20_000, dtype=ge.RESP16_DTYPE)
    r16["svc_id"] = ev["svc_id"][hot][:20_000]; r16["usec"] = rng.integers(1, 1 << 20, 20_000); r16["cli_port"] = rng.integers(0, 256, 20_000)
    eng.ingest_raw(ge.RAW_RESP16, r16, len(r16))
    eng.sync()
    tsec += 5 if w != 2 else 100                     # one jump past the idle limit: eviction, slot reuse, table rebuild
    eng.flush(tsec)
    eng.evicted_ids()
    ids = np.unique(ev["svc_id"][hot])[:50]
    eng.query_svcs(ids)
    eng.topn(0, 10); eng.topn(1, 10, host_idx=3); eng.topn_tasks(0, 5)
    eng.export_hll(int(ids[0])); eng.export_tdigest(int(ids[0])); eng.query_flows(ev["flow_key"][:100])
ids = np.unique(ev["svc_id"][ev["type"] == ge.EV_RESP])
eng.set_logical_map(ids, np.arange(len(ids), dtype=np.uint64) // np.uint64(8) + np.uint64(1))
eng.merge_prepare(); eng.merge_finish(None, 1)
eng.query_logical(np.arange(1, 10, dtype=np.uint64))
# 100 000 samples (<= max_batch): group numbers of 17 bits, sorted in a 9-bit and an 8-bit pass
s = np.zeros(100_000, dtype=ge.PROC_SAMPLE_DTYPE)
s["aggr_task_id"] = rng.integers(1, 20_000, len(s)); s["pid"] = rng.integers(2, 1 << 22, len(s)); s["cpu_pct"] = rng.random(len(s))
_, ngroups = eng.task_groupby(s)
assert ngroups == len(np.unique(s["aggr_task_id"]))
print(eng.stats())
eng.close()
print("sanitizer workload ok")
