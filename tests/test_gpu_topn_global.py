"""Services and processes ranked across GPUs (GYSK_FLAG_MERGE_TOPN): gysk_topn_global and gysk_topn_global_tasks at world 1 ... 8, with
and without the other merge flags. Each answer is restated from what every rank answers on its own right after the merge: its
gysk_topn_svcs / gysk_topn_tasks(metric, 64) lists (GYSK_TOPN_ACTIVE: the nconns_active of its gysk_query_window rows), merged by score
descending, then rank ascending, then the rank's own order; each row is the owner's gysk_query_svcs / gysk_query_tasks row."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from tests.test_gpu_cluster_states import cluster_map
from tests.test_gpu_logical_states import TIMES, _ids, state_events, state_map
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import _dev_bytes

INVAL, NOTSUP = -22, -95
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(max_svcs=512, max_tasks=256, max_batch=1 << 14, cms_log2_width=10)
ENT = struct.Struct("<QQII")
SVC_METRICS = [ge.TOPN_QPS, ge.TOPN_CONNS, ge.TOPN_NET, ge.TOPN_ISSUE, ge.TOPN_ACTIVE]
TASK_METRICS = [ge.TOPN_TASK_CPU, ge.TOPN_TASK_CPU_DELAY, ge.TOPN_TASK_BLKIO_DELAY]
NS = (1, 10, 50, 64)
NTIE, NTASK, NHOSTS = 120, 100, 40
TIE_IDS = synth.splitmix64(np.arange(1, NTIE + 1, dtype=np.uint64) + np.uint64(1 << 55))
TASK_IDS = synth.splitmix64(np.arange(1, NTASK + 1, dtype=np.uint64) + np.uint64(1 << 56))
QUIET_IDS = synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 57))     # registered, never an event


assert ENT.size == C.sizeof(ge.TopnEntry) == 24


def _code(fn):
    with pytest.raises(ge.GyskError) as ei:
        fn()
    return ei.value.code


def tie_events(rng, w):
    """services and processes on hosts 0 .. NHOSTS - 1 whose scores come from a few values, so equal scores meet across ranks and at the
    cut: response samples, connection events, kbytes and active connections of the tie services, cpu and delays of the processes"""
    nresp = rng.choice([0, 5, 10, 15], NTIE)
    nconn = rng.choice([0, 1, 2, 3], NTIE)
    host = np.arange(NTIE) % NHOSTS
    r = np.zeros(int(nresp.sum()), dtype=ge.EVENT_DTYPE)
    r["svc_id"] = np.repeat(TIE_IDS, nresp); r["host_idx"] = np.repeat(host, nresp); r["type"] = ge.EV_RESP
    r["value"] = rng.integers(1000, 90_000, len(r))
    c = np.zeros(int(nconn.sum()), dtype=ge.EVENT_DTYPE)
    c["svc_id"] = np.repeat(TIE_IDS, nconn); c["host_idx"] = np.repeat(host, nconn); c["type"] = ge.EV_ACCEPT
    c["value"] = rng.choice([1 << 10, 2 << 10], len(c)); c["flow_key"] = rng.integers(1, 1 << 62, len(c), dtype=np.uint64)
    a = np.zeros(NTIE, dtype=ge.EVENT_DTYPE)
    a["svc_id"] = TIE_IDS; a["host_idx"] = host; a["type"] = ge.EV_ACTIVE; a["flow_key"] = 77
    a["flags"] = rng.choice([0, 2, 4, 6], NTIE)
    a = a[a["flags"] > 0]
    ns = rng.choice([0, 1, 2], NTASK)
    t = np.zeros(int(ns.sum()), dtype=ge.EVENT_DTYPE)
    t["svc_id"] = np.repeat(TASK_IDS, ns); t["host_idx"] = np.repeat(np.arange(NTASK) % NHOSTS, ns); t["type"] = ge.EV_TASK
    t["value"] = rng.choice([10, 20, 30], len(t))
    t["flow_key"] = rng.choice([5, 50], len(t)).astype(np.uint64) | (rng.choice([0, 7, 70], len(t)).astype(np.uint64) << np.uint64(32))
    ev = np.concatenate([r, c, a, t])
    ev["tsec"][ev["type"] != ge.EV_ACTIVE] = TIMES[w]
    return ev[rng.permutation(len(ev))]


class Ranks:
    """world engines of one configuration, rank r = shard r"""

    def __init__(self, world, **kw):
        self.engines = [ge.Engine(rank=r, world=world, **{**KW, **kw}) for r in range(world)]

    def feed(self, ev):
        for e in self.engines:
            for off in range(0, len(ev), 1 << 14):
                e.ingest_events(ev[off: off + (1 << 14)])
                e.sync()

    def flush(self, t):
        for e in self.engines:
            e.flush(t)


def _local(e, fn, metric, n=64, *host):
    out = (ge.TopnEntry * n)()
    k = C.c_uint32()
    e._chk(fn(e.h, metric, *host, n, out, C.byref(k)))
    return [bytes(x) for x in out[: k.value]]


def local_svcs(e, metric, n=64):
    return _local(e, e.L.gysk_topn_svcs, metric, n, -1)


def local_tasks(e, metric, n=64):
    return _local(e, e.L.gysk_topn_tasks, metric, n)


def svc_rows(e, ids):
    out = (ge.SvcSummary * max(len(ids), 1))()
    a = np.ascontiguousarray(ids, dtype=np.uint64)
    e._chk(e.L.gysk_query_svcs(e.h, ge._p(a), len(a), out))
    return [bytes(x) for x in out[: len(ids)]]


def merged(lists, n):
    """(score desc, rank asc, local position) over every rank's list of entry bytes -> [(rank, entry bytes)] of the n best"""
    keyed = [(-ENT.unpack(b)[1], r, i, b) for r, lst in enumerate(lists) for i, b in enumerate(lst)]
    return [(r, b) for _, r, _, b in sorted(keyed)[:n]]


def check_topn(torch, engines):
    """merge with the collectives emulated, then every read on every rank against the restatement; returns the number of non-zero
    entries of each list at n = 64"""
    _emulate_collectives(torch, engines)
    counts = {}
    for kind, metrics, local, read, rows_of in (
            ("svc", SVC_METRICS[:4], local_svcs, "topn_global", lambda e, ids: svc_rows(e, ids)),
            ("task", TASK_METRICS, local_tasks, "topn_global_tasks", lambda e, ids: [bytes(x) for x in e.query_tasks(ids)])):
        for m in metrics:
            lists = [local(e, m) for e in engines]
            for n in NS:
                want = merged(lists, n)
                for r, e in enumerate(engines):
                    got, rows = getattr(e, read)(m, n)
                    assert [bytes(x) for x in got] == [b for _, b in want], (kind, m, n, r)
                    for (owner, b), row in zip(want, rows):
                        assert bytes(row) == rows_of(engines[owner], [ENT.unpack(b)[0]])[0], (kind, m, n, r)
                    assert [bytes(x) for x in getattr(e, read)(m, n, rows=False)[0]] == [bytes(x) for x in got]
            counts[(kind, m)] = len(merged(lists, 64))
            if len(engines) == 1:                                   # world 1: the local calls themselves
                for n in NS:
                    assert [bytes(x) for x in getattr(engines[0], read)(m, n)[0]] == local(engines[0], m, n), (kind, m, n)
    counts[("svc", ge.TOPN_ACTIVE)] = check_active(engines)
    return counts


def check_active(engines):
    """GYSK_TOPN_ACTIVE: equal scores on one rank rank by slot, which no read shows, so each rank's tied entries are checked as a set: the
    global list's (score, owner rank) sequence equals the restatement's and each entry is one of its owner's services with that score"""
    owner, by_rank = {}, []
    for r, e in enumerate(engines):
        rows, hosts, _ = e.query_window_hosts()
        mine = {}
        for x, h in zip(rows, hosts.tolist()):
            owner[x.glob_id] = (r, x.nconns_active, h)
            if x.nconns_active:
                mine.setdefault(x.nconns_active, set()).add(x.glob_id)
        by_rank.append(mine)
    keys = sorted((-s, r) for r, mine in enumerate(by_rank) for s, ids in mine.items() for _ in range(len(ids)))
    keys = [k for r in range(len(engines)) for k in sorted(k for k in keys if k[1] == r)[:64]]         # each rank's 64 best
    keys.sort()
    for r, e in enumerate(engines):
        for n in NS:
            got, rows = e.topn_global(ge.TOPN_ACTIVE, n)
            assert [(-x.score, owner[x.glob_id][0]) for x in got] == keys[:n], (r, n)
            assert len({x.glob_id for x in got}) == len(got)
            for x, row in zip(got, rows):
                o, s, h = owner[x.glob_id]
                assert x.glob_id in by_rank[o][x.score] and (x.host_idx, x.pad) == (h, 0)
                assert bytes(row) == svc_rows(engines[o], [x.glob_id])[0]
    return min(len(keys), 64)


@pytest.mark.gpu
@pytest.mark.parametrize("others", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_topn_equals_the_restatement(world, others):
    """a stream that turns slow and error-prone (ISSUE), with tie services and processes and registered services without events: every
    list on every rank equals the restatement at early and late flushes. Without the other flags no map call comes before the merge"""
    import torch
    rng = np.random.default_rng(4100 + 10 * world + others)
    ids, conn_ids, ghost_ids = _ids()
    sh = Ranks(world, merge_topn=True, merge_levels=others, merge_states=others, merge_clusters=others)
    if others:
        hosts, cids = cluster_map(rng)
        glob, logical = state_map(rng, ids, conn_ids, ghost_ids)
        for e in sh.engines:
            e.set_logical_map(glob, logical)
            e.set_cluster_map(hosts, cids)
    for e in sh.engines:
        e.register_ids(QUIET_IDS)
    seen = {}
    for w, t in enumerate(TIMES[:18]):
        sh.feed(np.concatenate([state_events(rng, w, ids, conn_ids), tie_events(rng, w)]))
        sh.flush(t)
        if w not in (0, 9, 17):
            continue
        counts = check_topn(torch, sh.engines)
        for k, v in counts.items():
            seen[k] = max(seen.get(k, 0), v)
        for e in sh.engines:
            for m in SVC_METRICS:
                assert not set(int(x.glob_id) for x in e.topn_global(m, 64)[0]) & set(QUIET_IDS.tolist())
    assert all(v > 0 for v in seen.values()), seen
    assert seen[("svc", ge.TOPN_QPS)] == 64 and seen[("task", ge.TOPN_TASK_CPU)] == 64


@pytest.mark.gpu
def test_fewer_entries_than_asked():
    """three services and one process: n = 10 gives what has a non-zero score, best first"""
    import torch
    e = ge.Engine(merge_topn=True, **KW)
    a, b, c, t = (int(x) for x in synth.splitmix64(np.arange(1, 5, dtype=np.uint64) + np.uint64(1 << 58)))
    ev = np.zeros(9, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = [a, a, a, b, b, c, t, t, t]; ev["host_idx"] = [1, 1, 1, 2, 2, 3, 4, 4, 4]
    ev["type"] = [ge.EV_RESP] * 6 + [ge.EV_TASK] * 3; ev["value"] = [100] * 6 + [7, 8, 9]; ev["tsec"] = 5
    e.ingest_events(ev)
    e.flush(5)
    check_topn(torch, [e])
    got, rows = e.topn_global(ge.TOPN_QPS, 10)
    assert [(x.glob_id, x.score, x.host_idx) for x in got] == [(a, 3, 1), (b, 2, 2), (c, 1, 3)]
    assert [r.glob_id for r in rows] == [a, b, c] and all(r.found for r in rows)
    got, rows = e.topn_global_tasks(ge.TOPN_TASK_CPU, 10)
    assert [(x.glob_id, x.score, x.host_idx) for x in got] == [(t, 24, 4)] and rows[0].aggr_task_id == t
    assert e.topn_global(ge.TOPN_CONNS, 10) == ([], [])


@pytest.mark.gpu
def test_topn_across_eviction_and_recycled_slots():
    """A is evicted and its slot goes to U, then A returns into G's slot after G is evicted: the lists follow the live services"""
    import torch
    sh = Ranks(2, max_svcs=3, max_tasks=8, idle_evict_secs=300, merge_topn=True)
    A, B, U, F, G = (int(x) for x in synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 53)))
    host = {A: 0, F: 2, G: 4, U: 6, B: 1}
    weight = {A: 5, B: 2, U: 3, F: 1, G: 4}
    rng = np.random.default_rng(59)

    def window(t, live):
        n = np.array([40 * weight[x] for x in live])
        ev = np.zeros(int(n.sum()), dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = np.repeat(np.array(live, dtype=np.uint64), n)
        ev["host_idx"] = np.repeat(np.array([host[x] for x in live], dtype=np.uint32), n)
        ev["type"] = ge.EV_RESP; ev["value"] = rng.integers(1000, 50_000, len(ev)); ev["tsec"] = t
        sh.feed(ev[rng.permutation(len(ev))])
        sh.flush(t)
        return set().union(*[set(int(i) for i in e.evicted_ids()) for e in sh.engines])

    def qps():
        check_topn(torch, sh.engines)
        return [(x.glob_id, x.score) for x in sh.engines[1].topn_global(ge.TOPN_QPS, 64)[0]]

    for t in (5, 10, 200, 400):
        window(t, [A, B, F, G] if t < 100 else [B, F, G])
    assert window(606, [B, F]) == {A}
    assert qps() == [(B, 80), (F, 40)]
    window(620, [B, F, U])                                      # U takes A's slot
    assert qps() == [(U, 120), (B, 80), (F, 40)]
    assert window(720, [B, F, U]) == {G}
    window(730, [A, B, F, U])                                   # A returns into G's slot
    assert qps() == [(A, 200), (U, 120), (B, 80), (F, 40)]


def _stream(engines, ids, conn_ids, nwin=8):
    rng = np.random.default_rng(91)
    for w, t in enumerate(TIMES[:nwin]):
        ev = np.concatenate([state_events(rng, w, ids, conn_ids), tie_events(rng, w)])
        for e in engines:
            for off in range(0, len(ev), 1 << 14):
                e.ingest_events(ev[off: off + (1 << 14)])
                e.sync()
            e.flush(t)


def _launches(e, fn):
    k0 = e.stats()["kernel_launches"]
    fn()
    return e.stats()["kernel_launches"] - k0


@pytest.mark.gpu
def test_flag_leaves_everything_else_unchanged():
    """with the other three flags: the merge arena, the logical rows and digests, the state and cluster rows are those of the engine
    without GYSK_FLAG_MERGE_TOPN; the slab grows by the candidates, the merge by the lists' launches. Without it the slab and the
    launches are as before and the new reads are GYSK_ERR_NOTSUP"""
    import torch
    rng = np.random.default_rng(33)
    ids, conn_ids, ghost_ids = _ids()
    glob, logical = state_map(rng, ids, conn_ids, ghost_ids)
    hosts, cids = cluster_map(rng)
    flags = dict(merge_levels=True, merge_states=True, merge_clusters=True)
    off, on = ge.Engine(**KW, **flags), ge.Engine(merge_topn=True, **KW, **flags)
    plain, only = ge.Engine(**KW), ge.Engine(merge_topn=True, **KW)
    for e in (off, on):
        e.set_logical_map(glob, logical)
        e.set_cluster_map(hosts, cids)
    plain.set_logical_map(glob, logical)
    _stream([off, on, plain, only], ids, conn_ids)
    per_list = _launches(off, lambda: off.topn(ge.TOPN_QPS, 64))      # score + sort + pick of one list
    assert _launches(only, lambda: only.topn_tasks(ge.TOPN_TASK_CPU, 64)) == per_list
    n_off, n_plain = (_launches(e, lambda: _emulate_collectives(torch, [e])) for e in (off, plain))
    assert (n_off, n_plain) == (9, 5)
    assert _launches(on, lambda: _emulate_collectives(torch, [on])) == n_off + 8 * per_list + 2 + 1
    assert _launches(only, lambda: _emulate_collectives(torch, [only])) == 8 * per_list + 2 + 1        # no map: no fold at all
    nl = len(set(logical.tolist()))
    assert off.merge_tdigest_slab()[1] == plain.merge_tdigest_slab()[1] == nl * 4128
    ncand = -(-(5 * 64 * (24 + 208) + 3 * 64 * (24 + 88)) // 4128)
    assert on.merge_tdigest_slab()[1] == (nl + ncand) * 4128 and only.merge_tdigest_slab()[1] == ncand * 4128
    bo, bn = off.merge_buffers(), on.merge_buffers()
    assert [(n, b, r) for n, _, b, r in bo] == [(n, b, r) for n, _, b, r in bn]
    for (_, pa, na, _), (_, pb, _, _) in zip(bo, bn):
        assert _dev_bytes(torch, pa, na).tobytes() == _dev_bytes(torch, pb, na).tobytes()
    pa, _ = off.merge_tdigest_slab()
    pb, _ = on.merge_tdigest_slab()
    assert _dev_bytes(torch, pa, nl * 4128).tobytes() == _dev_bytes(torch, pb, nl * 4128).tobytes()
    lids = list(dict.fromkeys(logical.tolist()))
    assert repr(on.query_logical(lids)) == repr(off.query_logical(lids))
    for lid in lids:
        a, b = off.export_logical_tdigest(lid), on.export_logical_tdigest(lid)
        assert all(np.array_equal(x, y) for x, y in zip(a[:2], b[:2])) and a[2:] == b[2:]
    assert [bytes(x) for x in on.query_logical_states(lids)] == [bytes(x) for x in off.query_logical_states(lids)]
    dense = list(dict.fromkeys(cids.tolist()))
    assert [bytes(x) for x in on.query_cluster_states(dense)] == [bytes(x) for x in off.query_cluster_states(dense)]
    check_topn(torch, [on])
    # reads leave the merge as it was
    got = [bytes(x) for x in on.topn_global(ge.TOPN_NET, 64)[0]]
    assert _launches(on, lambda: on.topn_global(ge.TOPN_NET, 64)) == 0
    assert [bytes(x) for x in on.topn_global(ge.TOPN_NET, 64)[0]] == got
    assert _code(lambda: off.topn_global(ge.TOPN_QPS, 10)) == NOTSUP
    assert _code(lambda: off.topn_global_tasks(ge.TOPN_TASK_CPU, 10)) == NOTSUP
    assert _code(lambda: plain.topn_global(ge.TOPN_QPS, 10)) == NOTSUP


@pytest.mark.gpu
def test_error_codes():
    """GYSK_ERR_INVAL before a finished merge and for a bad metric or n; gysk_topn_svcs keeps refusing GYSK_TOPN_ACTIVE"""
    e = ge.Engine(merge_topn=True, **KW)
    calls = [lambda: e.topn_global(ge.TOPN_QPS, 10), lambda: e.topn_global_tasks(ge.TOPN_TASK_CPU, 10)]
    assert [_code(c) for c in calls] == [INVAL, INVAL]                        # no merge
    e.ingest_events(tie_events(np.random.default_rng(1), 0))
    e.flush(TIMES[0])
    e.merge_prepare()
    e.sync()
    assert [_code(c) for c in calls] == [INVAL, INVAL]                        # prepared, not finished
    e.merge_finish(None, 1)
    assert len(e.topn_global(ge.TOPN_QPS, 64)[0]) == 64
    for m, n in ((5, 10), (-1, 10), (ge.TOPN_QPS, 0), (ge.TOPN_QPS, 65)):
        assert _code(lambda: e.topn_global(m, n)) == INVAL, (m, n)
    for m, n in ((3, 10), (-1, 10), (ge.TOPN_TASK_CPU, 0), (ge.TOPN_TASK_CPU, 65)):
        assert _code(lambda: e.topn_global_tasks(m, n)) == INVAL, (m, n)
    assert _code(lambda: e.topn(ge.TOPN_ACTIVE, 10)) == INVAL
    k = C.c_uint32()
    assert e.L.gysk_topn_global(e.h, ge.TOPN_QPS, 10, None, None, C.byref(k)) == INVAL
    assert e.L.gysk_topn_global(e.h, ge.TOPN_QPS, 10, (ge.TopnEntry * 10)(), None, None) == INVAL


def _nccl_uid():
    try:
        return ge.Engine(max_svcs=64, max_tasks=8, max_batch=4096, cms_log2_width=8).nccl_unique_id()
    except ge.GyskError as ex:
        pytest.skip(f"NCCL not loadable: {ex}")


def _answers(e):
    return [[bytes(x) for x in e.topn_global(m, 64)[0]] + [bytes(x) for x in e.topn_global(m, 64)[1]] for m in SVC_METRICS] + \
        [[bytes(x) for x in e.topn_global_tasks(m, 64)[0]] + [bytes(x) for x in e.topn_global_tasks(m, 64)[1]] for m in TASK_METRICS]


@pytest.mark.gpu
def test_library_nccl_merge_equals_the_emulation():
    """gysk_merge_global (NCCL inside the library) at world 1, with no map call, gives the lists and rows of the emulated collectives"""
    import torch
    uid = _nccl_uid()
    ids, conn_ids, _ = _ids()
    e = ge.Engine(merge_topn=True, **KW)
    e.nccl_comm_init(uid, 1, 0)
    _stream([e], ids, conn_ids)
    _emulate_collectives(torch, [e])
    want = _answers(e)
    e.merge_global()
    e.sync()
    assert _answers(e) == want and len(want[0]) == 128


@pytest.mark.gpu
def test_two_device_nccl_merge_equals_the_emulation():
    """two engines on two devices merged by gysk_merge_global equal two emulated shards on one device"""
    import threading

    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("the two-device NCCL merge needs two GPUs")
    _nccl_uid()
    ids, conn_ids, _ = _ids()
    emu = [ge.Engine(rank=r, world=2, merge_topn=True, **KW) for r in range(2)]
    lib = [ge.Engine(device=r, rank=r, world=2, merge_topn=True, **KW) for r in range(2)]
    _stream(emu + lib, ids, conn_ids)
    _emulate_collectives(torch, emu)
    uid2 = lib[0].nccl_unique_id()
    errs = []

    def merge(r):
        try:
            lib[r].nccl_comm_init(uid2, 2, r)
            lib[r].merge_global()
            lib[r].sync()
        except Exception as ex:      # noqa: BLE001
            errs.append(ex)
    th = [threading.Thread(target=merge, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errs, errs
    want = _answers(emu[0])
    assert _answers(lib[0]) == want and _answers(lib[1]) == want


def test_symbols_and_flag_match_the_header():
    """no device needed: the new entry points are exported and answer GYSK_ERR_INVAL without an engine; the flag is the header's"""
    L = ge.load_library()
    n = C.c_uint32()
    out = (ge.TopnEntry * 4)()
    assert L.gysk_topn_global(None, ge.TOPN_QPS, 4, out, None, C.byref(n)) == INVAL
    assert L.gysk_topn_global_tasks(None, ge.TOPN_TASK_CPU, 4, out, None, C.byref(n)) == INVAL
    hdr = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert int(re.search(r"#define GYSK_FLAG_MERGE_TOPN\s+(0x[0-9a-fA-F]+)u", hdr).group(1), 16) == ge.FLAG_MERGE_TOPN == 0x10
    assert re.search(r"int\s+gysk_topn_global\(gysk_engine \*e, int metric, uint32_t n, gysk_topn_entry \*out, gysk_svc_summary \*rows, uint32_t \*nout\);", hdr)
    assert re.search(r"int\s+gysk_topn_global_tasks\(gysk_engine \*e, int metric, uint32_t n, gysk_topn_entry \*out, gysk_task_summary \*rows, uint32_t \*nout\);", hdr)
