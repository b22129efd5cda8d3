"""Every flow, client and merge flag on, a long run: three ranks (the merge emulated on one GPU), 64 trace rows, service and process
tables that start small under an auto-grow ceiling and one explicit gysk_grow between a batch and its flush, idle eviction of services and
processes with a part of the stream that goes quiet and returns under the same ids, and the flush sequences of tests/flow_level.py one after
the other (over 100 flushes, several wraps of the ten-slot rings). Between batches gysk_task_groupby borrows the batch's sort buffers and
the logical map changes once. After every flush each rank's tests/all_flags.Model checks every answer family, and after every merge the
_global reads, the logical services' rows, client registers and trace rows are held to their restatement from the ranks' models."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge, synth, wire
from oracle import pyoracle as po
from tests import all_flags as af
from tests.flow_level import SEQUENCES
from tests.test_gpu_boundary import _proc_samples
from tests.test_gpu_flag_matrix import _stream
from tests.test_gpu_flow_topk import _shard
from tests.test_gpu_merge import _emulate_collectives
from tests.trace_agg import api_tran, trace_events

pytestmark = pytest.mark.gpu

WORLD = 3
FLAGS = {k: True for k in af.FLAGS}
MERGE = dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, merge_traces=True)
CFG = dict(max_svcs=128, max_tasks=64, max_batch=1 << 16, cms_depth=4, cms_log2_width=11, max_trace_svcs=64, idle_evict_secs=30,
           task_idle_evict_secs=30)
LIMIT_SVCS, LIMIT_TASKS = 1024, 256
QUIET_SVCS, QUIET_TASKS = range(20, 36), range(60, 72)         # flush indices in which a part of the ids sends nothing
# the services with trace events: fewer than the trace rows, so that a new one always finds a row (which ids win the last rows when they
# run out depends on the order the device meets them in). Those of them that go quiet are evicted, free their rows and take rows again
# when they return.
TRACED = synth.service_ids(40)


def stream(rng, i):
    """the events of flush i: a service count that grows with i, a fifth of the services (and a quarter of the processes) quiet during
    QUIET_SVCS (QUIET_TASKS) and back afterwards under the same ids, and API_TRAN trace events of the TRACED services"""
    nsvc = min(40 + 3 * i, 220)
    ev = _stream(rng, int(rng.integers(9_000, 15_000)), nsvc=nsvc)
    task = ev["type"] == ge.EV_TASK
    drop = np.zeros(len(ev), dtype=bool)
    if i in QUIET_SVCS:
        drop |= ~task & (ev["svc_id"] % np.uint64(5) == 0)
    if i in QUIET_TASKS:
        drop |= task & (ev["svc_id"] % np.uint64(4) == 0)
    ev = ev[~drop]
    ev["svc_id"][ev["type"] == ge.EV_TASK] >>= np.uint64(17)     # below 2^48, where tests/task_evict.py numbers a process's incarnations
    ids = TRACED[np.isin(TRACED, ev["svc_id"])]
    n = 1500
    rec = api_tran(rng.choice(ids, n), rng.integers(100, 3_000_000, n).astype(np.uint64), reqlen=rng.integers(0, 5000, n),
                   reslen=rng.integers(0, 50_000, n), reqnum=rng.integers(0, 3, n), errorcode=rng.choice([0, 0, 0, 1, 500], n))
    tr = trace_events(rec)
    tr["host_idx"] = rng.integers(0, 16, n)
    return np.concatenate([ev, tr])


def timeline():
    """steps_5s, gaps, same_tsec and step_back, each shifted to start 100 s after the previous one's largest tsec"""
    out, end = [], 0
    for name in ("steps_5s", "gaps", "same_tsec", "step_back"):
        seq = SEQUENCES[name]
        shift = max(0, end + 100 - seq[0])
        out += [(name, t + shift) for t in seq]
        end = max(t for _, t in out)
    return out


def test_every_flag_over_a_long_run():
    import torch
    rng = np.random.default_rng(2026)
    models = [af.Model(cap_svcs=LIMIT_SVCS, cap_tasks=LIMIT_TASKS, rank=r, world=WORLD, **CFG, **FLAGS, **MERGE) for r in range(WORLD)]
    for m in models:
        m.eng.set_auto_grow(LIMIT_SVCS, LIMIT_TASKS)
    tl = timeline()
    assert len(tl) > 100
    glob = logical = None
    traced_evicted = set()
    for i, (seq, t) in enumerate(tl):
        what = (seq, i, t)
        ev = stream(rng, i)
        ev["tsec"] = t
        if i in (3, len(tl) // 2):                              # the logical map, once set and once changed
            glob = np.unique(ev["svc_id"][ev["type"] != ge.EV_TASK])
            logical = glob % np.uint64(7 if i == 3 else 11) + np.uint64(50)
            for m in models:
                m.eng.set_logical_map(glob, logical)
        halves = np.array_split(ev, 2)
        for m, sh in zip(models, _shard(halves[0], WORLD)):
            m.ingest(sh)
        if i % 9 == 4:
            s = _proc_samples(rng, 3000, 400)
            want = po.task_groupby(s, wire.TASK)
            for m in models:
                got, ng = m.eng.task_groupby(s)
                assert ng == len(want) and got.tobytes() == want.tobytes(), what
        for m, sh in zip(models, _shard(halves[1], WORLD)):
            m.ingest(sh)
        if i % 10 == 7:
            models[i % WORLD].check(what)                       # reads between a batch and its flush
        if i == 50:
            for m in models:
                c = m.eng.capacity()
                m.grow(c["max_svcs"] * 2, c["max_tasks"])
        for m in models:
            m.flush(t)
            m.check(what)
        traced_evicted |= {g for m in models for g in m.evicted} & set(TRACED.tolist())
        _emulate_collectives(torch, [m.eng for m in models])
        af.check_merged(models, what)
        if glob is not None:
            af.check_logical(models, glob, logical, what)
    st = [m.eng.stats() for m in models]
    cap = [m.eng.capacity() for m in models]
    assert all(s["svcs_evicted"] > 0 for s in st) and all(m.eng.task_evict_count() > 0 or m.tasks.total > 0 for m in models)
    assert all(c["ngrows"] >= 2 for c in cap), cap
    assert all(m.eng.trace_info()[0] > 0 for m in models)
    assert traced_evicted                                       # trace rows were freed and taken again
