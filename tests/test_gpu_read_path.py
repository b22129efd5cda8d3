"""The read path: every read of the engine goes through one device stage and one page-locked stage. Two things must hold.

1. Each read issues a fixed number of kernel launches: one per 1024-id piece of a by-id read, one per single-id export (none for the
   merged logical services' exports, which copy from the merge arena), and for the window reads the list-and-sort launches plus one
   per 8192 rows; the reads over every logical service take one select launch under ACTIVE_ONLY, then one per 8192 rows (bench.py
   reports kernel_launches).
2. No read sees what another read left in the stage: every read, interleaved with all the others, answers what it answers when the
   reads run in another order on a second engine fed the same stream (top-N up to the order of tied entries), and an unknown id
   gives None or the not-found row."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests.test_gpu_window_read import _stream

pytestmark = pytest.mark.gpu

NAN = float("nan")
# window_list of a non-empty table with rows wanted: window_select_kernel, one radix sort of the 32 host bits (os_hist_kernel and
# four 8-bit os_pass_kernel passes: plain_sort_plan(32, 64)) and window_ids_kernel; a count-only call (cap 0) runs
# window_select_kernel alone. Then one summary launch per 8192 rows.
WINDOW_LIST_LAUNCHES, WINDOW_COUNT_LAUNCHES, WIN_ROWS = 7, 1, 8192
# top-N: the score kernel, the same 32-bit radix sort (5 launches) and the pick kernel
TOPN_LAUNCHES = 7


def _engine(seed):
    """services, processes and flows over two windows, the first one closed; a world-1 merge of the services into logical ids, with
    their listener states"""
    rng = np.random.default_rng(seed)
    eng = ge.Engine(max_svcs=1 << 14, max_tasks=1 << 12, merge_states=True)
    svc_ids = (rng.choice(1 << 40, 1500, replace=False) + 1).astype(np.uint64)
    task_ids = (rng.choice(1 << 40, 1200, replace=False) + (1 << 41)).astype(np.uint64)
    ev = _stream(rng, svc_ids, task_ids, 60000)
    eng.ingest_events(ev)
    eng.sync()
    eng.flush(5)
    ev2 = _stream(rng, svc_ids[:1000], task_ids[:800], 20000)
    eng.ingest_events(ev2)
    eng.sync()
    logical = svc_ids % np.uint64(97) + np.uint64(1 << 50)
    eng.set_logical_map(svc_ids, logical)
    eng.merge_prepare()
    eng.merge_finish()
    flows = np.unique(np.concatenate([ev, ev2])["flow_key"])
    live_tasks = np.array([r.aggr_task_id for r in eng.query_task_window()[0]], dtype=np.uint64)    # the ones the stream reached
    return eng, svc_ids, live_tasks, np.unique(logical), flows


def _launches(eng, fn):
    before = eng.stats()["kernel_launches"]
    fn()
    return eng.stats()["kernel_launches"] - before


def _raw_rows(eng, fn, ids, row_type):
    ids = np.ascontiguousarray(ids, dtype=np.uint64)
    out = (row_type * max(len(ids), 1))()
    eng._chk(fn(eng.h, ids.ctypes.data_as(C.c_void_p), len(ids), out))
    return out[: len(ids)]


def test_launch_counts_of_every_read():
    eng, svc_ids, task_ids, logical, flows = _engine(11)
    rng = np.random.default_rng(12)
    pool = np.concatenate([svc_ids, rng.choice(1 << 40, 1000, replace=False).astype(np.uint64) + (1 << 42)])
    nsvc_rows, ntask_rows = eng.query_window(cap=0)[1], eng.query_task_window(cap=0)[1]
    assert nsvc_rows > 1000 and ntask_rows > 1000
    for n in (0, 1, 1024, 1025, 2051):
        ids, pieces = pool[:n], math.ceil(n / 1024)
        assert _launches(eng, lambda: eng.query_svcs(ids)) == pieces, n
        assert _launches(eng, lambda: eng.query_tasks(ids)) == pieces, n
        assert _launches(eng, lambda: eng.query_flows(flows[:n])) == pieces, n
        assert _launches(eng, lambda: eng.query_flows_global(flows[:n])) == pieces, n
        assert _launches(eng, lambda: eng.query_logical(np.resize(logical, n))) == pieces, n
        assert _launches(eng, lambda: eng.query_logical_states(np.resize(logical, n))) == pieces, n
        fresh = rng.choice(1 << 40, n, replace=False).astype(np.uint64) + (1 << 43)
        assert _launches(eng, lambda: eng.register_ids(fresh)) == pieces, n
        # window reads: n rows wanted (cap), the table holds more than 1000
        for read, rows in ((eng.query_window, nsvc_rows), (eng.query_task_window, ntask_rows)):
            want = WINDOW_COUNT_LAUNCHES if n == 0 else WINDOW_LIST_LAUNCHES + math.ceil(min(n, rows) / WIN_ROWS)
            assert _launches(eng, lambda: read(cap=n)) == want, (read, n)
    for id_ in (int(svc_ids[0]), 0xDEAD0001):
        assert _launches(eng, lambda: eng.export_hist(id_, ge.HIST_RESP_ALL)) == 1
        assert _launches(eng, lambda: eng.export_conn_bitmap(id_)) == 1
        assert _launches(eng, lambda: eng.export_hll(id_)) == 1
        assert _launches(eng, lambda: eng.export_tdigest(id_)) == 1
    for id_ in (int(task_ids[0]), 0xDEAD0001):
        assert _launches(eng, lambda: eng.export_hist(id_, ge.HIST_TASK_CPU_DELAY)) == 1
    assert _launches(eng, lambda: eng.topn(ge.TOPN_QPS)) == TOPN_LAUNCHES
    # every logical service: the select kernel under ACTIVE_ONLY, then one row launch per 8192 rows
    for cap in (0, 5, len(logical)):
        for active in (False, True):
            for read in (eng.query_logical_all, eng.query_logical_states_all):
                rows = read(active_only=active, cap=len(logical))[1]
                assert rows > 5
                assert _launches(eng, lambda: read(active_only=active, cap=cap)) == active + math.ceil(min(cap, rows) / WIN_ROWS), (read, cap, active)
    for metric in (ge.TOPN_QPS, ge.TOPN_ISSUE):
        assert _launches(eng, lambda: eng.topn_logical(metric)) == TOPN_LAUNCHES, metric
    for id_ in (int(logical[0]), 0xDEAD0001):
        assert _launches(eng, lambda: eng.export_logical_hist(id_, ge.HIST_RESP_ALL)) == 0
        assert _launches(eng, lambda: eng.export_logical_tdigest(id_)) == 0
        assert _launches(eng, lambda: eng.export_logical_hll(id_)) == 0
    assert _launches(eng, lambda: eng.topn_tasks(0)) == TOPN_LAUNCHES
    eng.close()


def _canon(x):
    """a comparable form of any answer: bytes for rows and arrays, doubles by their bits (NaN included)"""
    if isinstance(x, (C.Structure, np.ndarray)):
        return bytes(x) if isinstance(x, C.Structure) else (x.dtype.str, x.tobytes())
    if isinstance(x, float):
        return struct.pack("<d", x)
    if isinstance(x, (list, tuple)):
        return tuple(_canon(v) for v in x)
    return x


def _topn_canon(entries):
    """entries of equal score come in slot order, and slot numbers follow insertion races: the scores in order, and as a set the
    entries above the lowest score (which of the entries tied at the lowest score make the cut depends on their slots too)"""
    scores = [e[1] for e in entries]
    return tuple(scores), frozenset(e for e in entries if e[1] != min(scores))


def _quantiles(eng, id_):
    qs = np.array([0.5, 0.9, 0.99])
    out = np.zeros(3)
    rc = eng.L.gysk_query_quantiles(eng.h, id_, qs.ctypes.data_as(C.c_void_p), 3, out.ctypes.data_as(C.c_void_p))
    if rc == -2:
        return None
    eng._chk(rc)
    return out


def _round(eng, k, svc_ids, task_ids, logical, flows, unknown):
    """round k of every read: the single-id exports take a live id in even rounds and an unknown one in odd rounds, the by-id
    reads live ids among unknown ids and id 0"""
    L = eng.L
    sid = int(svc_ids[k]) if k % 2 == 0 else int(unknown[k])
    tid = int(task_ids[k]) if k % 2 == 0 else int(unknown[k])
    mix = np.concatenate([svc_ids[k * 300: k * 300 + 700], unknown[k * 100: k * 100 + 500], np.zeros(50, dtype=np.uint64)])
    tmix = np.concatenate([task_ids[k * 200: k * 200 + 500], unknown[: 300], np.zeros(30, dtype=np.uint64)])
    keys = np.concatenate([flows[k * 500: k * 500 + 1500], unknown[: 200]])
    lmix = np.concatenate([logical, unknown[: 40]])
    lid = int(logical[k]) if k % 2 == 0 else int(unknown[k])
    return [
        ("export_hist", sid, lambda: eng.export_hist(sid, ge.HIST_RESP_ALL)),
        ("export_task_hist", tid, lambda: eng.export_hist(tid, ge.HIST_TASK_CPU_PCT + k % 3)),
        ("export_conn_bitmap", sid, lambda: eng.export_conn_bitmap(sid, last_window=bool(k & 2))),
        ("export_hll", sid, lambda: eng.export_hll(sid)),
        ("export_tdigest", sid, lambda: eng.export_tdigest(sid)),
        ("quantiles", sid, lambda: _quantiles(eng, sid)),
        ("export_tdigest_pgtext", sid, lambda: eng.export_tdigest_pgtext(sid)),
        ("query_svcs", None, lambda: _raw_rows(eng, L.gysk_query_svcs, mix, ge.SvcSummary)),
        ("query_tasks", None, lambda: eng.query_tasks(tmix)),
        ("query_flows", None, lambda: eng.query_flows(keys, last_window=bool(k & 1))),
        ("topn", None, lambda: eng.topn(k % 4, n=20)),
        ("topn_tasks", None, lambda: eng.topn_tasks(k % 3, n=20)),
        ("query_window", None, lambda: eng.query_window(active_only=bool(k & 1))),
        ("query_task_window", None, lambda: eng.query_task_window(host_idx=k)),
        ("query_logical", None, lambda: _raw_rows(eng, L.gysk_query_logical, lmix, ge.SvcSummary)),
        ("query_logical_all", None, lambda: eng.query_logical_all(active_only=bool(k & 1))),
        ("query_logical_states", None, lambda: _raw_rows(eng, L.gysk_query_logical_states, lmix, ge.LogicalState)),
        ("query_logical_states_all", None, lambda: eng.query_logical_states_all(active_only=bool(k & 2))),
        ("topn_logical", None, lambda: eng.topn_logical(k % 4, n=20)),
        ("export_logical_hist", lid, lambda: eng.export_logical_hist(lid, ge.HIST_RESP_LAST + k % 2)),
        ("export_logical_tdigest", lid, lambda: eng.export_logical_tdigest(lid)),
        ("export_logical_hll", lid, lambda: eng.export_logical_hll(lid)),
    ]


def _reads(eng, svc_ids, task_ids, logical, flows, unknown):
    """four rounds of every read, in this interleaving: (round, name, the single id or None, the read)"""
    return [(k, name, id_, fn) for k in range(4) for name, id_, fn in _round(eng, k, svc_ids, task_ids, logical, flows, unknown)]


def test_interleaved_reads_equal_the_same_reads_in_another_order():
    engines = [_engine(21), _engine(21)]
    rng = np.random.default_rng(22)
    unknown = rng.choice(1 << 40, 1000, replace=False).astype(np.uint64) + (1 << 44)
    interleaved = {(k, name): fn() for k, name, _id, fn in _reads(engines[0][0], *engines[0][1:], unknown)}
    # the second engine: the reads grouped by kind, the kinds in the reverse order
    grouped = {}
    reads = _reads(engines[1][0], *engines[1][1:], unknown)
    for name in reversed(list(dict.fromkeys(name for _k, name, _id, _fn in reads))):
        for k, nm, _id, fn in reads:
            if nm == name:
                grouped[(k, nm)] = fn()
    assert interleaved.keys() == grouped.keys()
    for key in interleaved:
        canon = _topn_canon if key[1] in ("topn", "topn_tasks") else _canon
        assert canon(interleaved[key]) == canon(grouped[key]), key
    # unknown ids: None from the exports, the not-found row from the by-id reads
    svc_ids, task_ids, logical = engines[0][1], engines[0][2], engines[0][3]
    for k, name, id_, _fn in reads:
        if id_ is not None:
            assert (interleaved[(k, name)] is None) == (k % 2 == 1), (k, name)
    live = set(svc_ids.tolist()) | set(logical.tolist())
    for k in range(4):
        for name in ("query_svcs", "query_logical"):
            for r in interleaved[(k, name)]:
                if r.glob_id not in live:
                    assert bytes(r) == bytes(ge.SvcSummary(glob_id=r.glob_id, td_p50_us=NAN, td_p95_us=NAN, td_p99_us=NAN)), (k, name)
                else:
                    assert r.found == 1, (k, name, hex(r.glob_id))
        for r in interleaved[(k, "query_logical_states")]:
            if r.logical_id not in live:
                assert bytes(r) == bytes(ge.LogicalState(logical_id=r.logical_id)), k
            else:
                assert r.found == 1, (k, hex(r.logical_id))
        tlive = set(task_ids.tolist())
        for r in interleaved[(k, "query_tasks")]:
            if r.aggr_task_id not in tlive:
                assert bytes(r) == bytes(ge.TaskSummary(aggr_task_id=r.aggr_task_id)), k
    for eng, *_rest in engines:
        eng.close()
