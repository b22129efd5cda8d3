"""Growing the service and process tables of a live engine (gysk_grow, gysk_set_auto_grow, gysk_capacity_info). An engine G that starts
small and grows is fed the same calls as an engine F created at G's final capacity; after every growth every read of G must answer as
F's does. Slot numbers inside a batch depend on atomics, so rows are compared by id byte for byte, id-ordered reads as arrays, eviction
lists as sets and rankings with their ties as sets."""
import ctypes as C
import threading

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po
from tests.test_gpu_merge import _emulate_collectives

pytestmark = pytest.mark.gpu

INVAL, NOMEM = -22, -12
KW = dict(max_batch=1 << 14, cms_log2_width=12, idle_evict_secs=20)
NHOSTS = 12
SVC_WHICH = [ge.HIST_RESP_CUR, ge.HIST_RESP_LAST, ge.HIST_RESP_ALL, ge.HIST_RESP_5MIN, ge.HIST_RESP_5DAY, ge.HIST_QPS, ge.HIST_ACTIVE_CONN]
TASK_WHICH = [ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY]
UNKNOWN = np.array([0, 12345, 0xFFFFFFFFFFFFFFFE], dtype=np.uint64)


def ids_of(base, n):
    return synth.splitmix64(np.arange(1, n + 1, dtype=np.uint64) + np.uint64(base << 40))


def events(rng, n, ids, tids, tsec=1):
    """RESP (some with client / server error flags), TCP accept / close, TASK and ACTIVE_CONN events over ids / tids; ids[0] and
    ids[1] take a quarter of the samples each, enough to take a hot row"""
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    k = rng.integers(0, len(ids), n)
    heavy = rng.random(n) < 0.5
    k[heavy] = rng.integers(0, min(2, len(ids)), int(heavy.sum()))
    ev["svc_id"] = ids[k]
    ev["host_idx"] = (k % NHOSTS).astype(np.uint32)
    u = rng.random(n)
    resp, tcp, close, task, act = u < 0.6, (u >= 0.6) & (u < 0.75), (u >= 0.75) & (u < 0.8), (u >= 0.8) & (u < 0.93), u >= 0.93
    ev["type"][resp] = ge.EV_RESP
    ev["value"][resp] = np.minimum(np.exp(rng.normal(np.log(3000.0), 1.5, int(resp.sum()))), 9.0e8).astype(np.uint32)
    ev["flags"][resp] = rng.choice([0, 0, 0, 0, ge.EVF_CLI_ERROR, ge.EVF_SER_ERROR], int(resp.sum()))
    ev["flow_key"][resp] = rng.integers(0, 64, int(resp.sum()))
    for m, t in ((tcp, ge.EV_ACCEPT), (close, ge.EV_CLOSE_SER)):
        ev["type"][m] = t
        ev["flow_key"][m] = synth.splitmix64(rng.integers(0, 3000, int(m.sum())).astype(np.uint64))
        ev["value"][m] = rng.integers(100, 1 << 16, int(m.sum()))
    nt = int(task.sum())
    tk = rng.integers(0, len(tids), nt)
    ev["svc_id"][task] = tids[tk]
    ev["host_idx"][task] = (tk % NHOSTS).astype(np.uint32)
    ev["type"][task] = ge.EV_TASK
    ev["value"][task] = rng.integers(0, 400, nt)
    ev["flow_key"][task] = rng.integers(0, 500, nt).astype(np.uint64) | (rng.integers(0, 90, nt).astype(np.uint64) << np.uint64(32))
    ev["type"][act] = ge.EV_ACTIVE
    ev["flow_key"][act] = 77
    ev["flags"][act] = rng.integers(1, 8, int(act.sum()))
    ev["tsec"] = tsec
    return ev


def feed(engines, ev, batch=2048):
    for off in range(0, len(ev), batch):
        for e in engines:
            e.ingest_events(ev[off: off + batch])
            e.sync()


def _entries(lst):
    """a ranking as (scores in order, the ids of every score but the last one as sets, the count of the last one): equal scores rank by
    slot, which no read shows"""
    scores = [x[1] for x in lst]
    groups = {}
    for x in lst:
        groups.setdefault(x[1], set()).add(x[0])
    last = scores[-1] if scores else None
    return scores, {s: g for s, g in groups.items() if s != last}


def same_ranking(a, b, what):
    assert _entries(a) == _entries(b), what


def answers_equal(G, F, ids, tids, keys):
    """every read of G against F's"""
    sg, sf = G.stats(), F.stats()
    for f in ("events_in", "events_dropped", "events_resp", "events_tcp", "events_task", "nsvcs", "ntasks", "svcs_evicted"):
        assert sg[f] == sf[f], (f, sg[f], sf[f])
    for host, active in ((-1, False), (-1, True), (3, False)):
        rg, hg, ng = G.query_window_hosts(host, active)
        rf, hf, nf = F.query_window_hosts(host, active)
        assert ng == nf and [bytes(x) for x in rg] == [bytes(x) for x in rf] and np.array_equal(hg, hf), (host, active)
    tg, tf = G.query_task_window()[0], F.query_task_window()[0]
    assert [bytes(x) for x in tg] == [bytes(x) for x in tf]
    q = np.concatenate([ids, UNKNOWN])
    a, b = (SvcRowsOf(G, q), SvcRowsOf(F, q))
    assert a == b
    tq = np.concatenate([tids, UNKNOWN])
    assert [bytes(x) for x in G.query_tasks(tq)] == [bytes(x) for x in F.query_tasks(tq)]
    sample = list(ids[:20]) + list(ids[-40:]) + list(UNKNOWN[1:2])      # the last ids: slots past the old capacity, recycled slots
    for i in tids[:10].tolist() + tids[-20:].tolist() + [12345]:
        for w in TASK_WHICH:
            x, y = task_hist(G, i, w), task_hist(F, i, w)
            assert x == y, (hex(i), w)
    for i in dict.fromkeys(sample):
        i = int(i)
        for w in SVC_WHICH:
            x, y = G.export_hist(i, w), F.export_hist(i, w)
            assert (x is None) == (y is None), (i, w)
            if x is not None:
                assert x[0].tobytes() == y[0].tobytes() and x[1:] == y[1:], (hex(i), w)
        x, y = G.export_tdigest(i), F.export_tdigest(i)
        assert (x is None) == (y is None)
        if x is not None:
            assert x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes() and np.float64(x[2]).tobytes() == np.float64(y[2]).tobytes()
            qs = [0.5, 0.9, 0.99]
            assert G.quantiles(i, qs).tobytes() == F.quantiles(i, qs).tobytes()
        x, y = G.export_hll(i), F.export_hll(i)
        assert (x is None) == (y is None) and (x is None or np.array_equal(x, y))
        for lw in (False, True):
            x, y = G.export_conn_bitmap(i, lw), F.export_conn_bitmap(i, lw)
            assert (x is None) == (y is None) and (x is None or (np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])))
    for lw in (False, True):
        assert np.array_equal(G.export_cms(lw), F.export_cms(lw))
        assert G.query_flows(keys, lw).tobytes() == F.query_flows(keys, lw).tobytes()
    dg, dhg, ndg = G.query_day_stats()
    df, dhf, ndf = F.query_day_stats()
    assert ndg == ndf and [bytes(x) for x in dg] == [bytes(x) for x in df] and np.array_equal(dhg, dhf)
    hg, nhg = G.query_host_listen()
    hf, nhf = F.query_host_listen()
    assert nhg == nhf and [bytes(x) for x in hg] == [bytes(x) for x in hf]
    assert set(G.evicted_ids().tolist()) == set(F.evicted_ids().tolist())
    for m in (ge.TOPN_QPS, ge.TOPN_CONNS, ge.TOPN_NET, ge.TOPN_ISSUE):
        same_ranking(G.topn(m, 64), F.topn(m, 64), ("svc", m))
        same_ranking(G.topn(m, 10, 2), F.topn(m, 10, 2), ("svc host", m))
    for m in (ge.TOPN_TASK_CPU, ge.TOPN_TASK_CPU_DELAY, ge.TOPN_TASK_BLKIO_DELAY):
        same_ranking(G.topn_tasks(m, 64), F.topn_tasks(m, 64), ("task", m))
    for w in range(11):
        assert G.topn_host(w, 10) == F.topn_host(w, 10), w


def task_hist(e, id_, which):
    """gysk_export_task_hist: (cells bytes, total, max), or the error code"""
    out = np.zeros(15, dtype=ge.SERIAL_DTYPE)
    total, mx = C.c_uint64(), C.c_int64()
    rc = e.L.gysk_export_task_hist(e.h, int(id_), which, ge._p(out), C.byref(total), C.byref(mx))
    return (out.tobytes(), total.value, mx.value) if rc == 0 else rc


def SvcRowsOf(e, q):
    out = (ge.SvcSummary * len(q))()
    a = np.ascontiguousarray(q, dtype=np.uint64)
    e._chk(e.L.gysk_query_svcs(e.h, ge._p(a), len(a), out))
    return [bytes(x) for x in out]


def _code(fn):
    with pytest.raises(ge.GyskError) as ei:
        fn()
    return ei.value.code


@pytest.mark.parametrize("which", ["svcs", "tasks", "both"])
def test_grown_engine_answers_as_one_created_at_its_capacity(monkeypatch, which):
    """grow before the first event, between two batches of one window, right after a flush, right after an eviction (slots on the free
    stack), while hot rows are in use, and twice in a row; after each, every read equals F's. Then new ids stream in past the old
    capacity with nothing dropped."""
    monkeypatch.setenv("GYSK_HOT_ROWS", "64")
    monkeypatch.setenv("GYSK_HOT_MIN", "200")
    rng = np.random.default_rng(11)
    s0, t0 = 96, 48
    final_s, final_t = (s0 << 7 if which != "tasks" else s0), (t0 << 7 if which != "svcs" else t0)
    G = ge.Engine(max_svcs=s0, max_tasks=t0, **KW)
    F = ge.Engine(max_svcs=final_s, max_tasks=final_t, **KW)
    cap = [s0, t0]

    def grow():
        cap[0] = cap[0] * 2 if which != "tasks" else cap[0]
        cap[1] = cap[1] * 2 if which != "svcs" else cap[1]
        G.grow(cap[0], cap[1])
        c = G.capacity()
        assert (c["max_svcs"], c["max_tasks"]) == tuple(cap)

    A, B, T = ids_of(1, 40), ids_of(2, 30), ids_of(3, 40)
    keys = synth.splitmix64(np.arange(0, 3000, dtype=np.uint64))
    allids, alltids = np.concatenate([A, B]), T
    grow()                                                           # 1: before the first event
    answers_equal(G, F, allids, alltids, keys)
    t = 0
    for w in range(4):                                               # A and B active, three batches per window
        t += 5
        feed([G, F], events(rng, 6000, allids, alltids, t))
        if w == 1:
            grow()                                                   # 2: between two batches of one window
            answers_equal(G, F, allids, alltids, keys)
        feed([G, F], events(rng, 6000, allids, alltids, t))
        for e in (G, F):
            e.flush(t)
        if w == 2:
            grow()                                                   # 3: right after a flush
            answers_equal(G, F, allids, alltids, keys)
    assert G.hot_rows_in_use() > 0
    grow()                                                           # 4: hot rows in use
    answers_equal(G, F, allids, alltids, keys)
    for w in range(8):                                               # B goes idle and is evicted
        t += 5
        feed([G, F], events(rng, 4000, A, alltids, t))
        for e in (G, F):
            e.flush(t)
    assert G.stats()["svcs_evicted"] == len(B)
    grow()                                                           # 5: slots on the free stack
    answers_equal(G, F, allids, alltids, keys)
    grow(); grow()                                                   # 6: twice in a row
    answers_equal(G, F, allids, alltids, keys)
    # new ids past the old capacity, and a jump past 900 s for the day stats
    Cn = ids_of(4, 3 * s0) if which != "tasks" else ids_of(4, 0)   # a table that did not grow takes no new ids: which of them would
    Tn = ids_of(5, 3 * t0) if which != "svcs" else ids_of(5, 0)     # win its last slots is a race
    for tt in (t + 5, t + 1000, t + 1005):
        feed([G, F], events(rng, 12000, np.concatenate([A, Cn]), np.concatenate([T, Tn]), tt))
        for e in (G, F):
            e.flush(tt)
    allids, alltids = np.concatenate([A, B, Cn]), np.concatenate([T, Tn])
    answers_equal(G, F, allids, alltids, keys)
    assert G.stats()["events_dropped"] == 0
    assert G.capacity()["ngrows"] == 7 and G.capacity()["svcs_in_use"] == F.capacity()["svcs_in_use"]


def _merge(torch, engines, between=None):
    """_emulate_collectives with a hook between gysk_merge_prepare and gysk_merge_finish"""
    import gyeeta_b200.dist as gd
    if between is None:
        return _emulate_collectives(torch, engines)
    dev = torch.device("cuda", 0)
    for e in engines:
        e.merge_prepare()
        e.sync()
    between()
    bufs = [e.merge_buffers() for e in engines]
    for k in range(len(bufs[0])):
        ts = [gd.wrap(torch, b[k][1], b[k][2], b[k][3], dev) for b in bufs]
        red = ts[0].clone()
        for x in ts[1:]:
            red = red + x if bufs[0][k][3] == gd.RED_SUM_U64 else torch.maximum(red, x)
        for x in ts:
            x.copy_(red)
    slabs = []
    for e in engines:
        p, nb = e.merge_tdigest_slab()
        slabs.append(torch.as_tensor(gd._DevBuf(p, nb, "|u1", 1), device=dev))
    gathered = torch.cat(slabs).contiguous()
    torch.cuda.synchronize()
    for e in engines:
        e.merge_finish(gathered.data_ptr(), len(engines))


@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_merge_with_grown_ranks(world):
    """some ranks grow, others do not, rank 0 once between gysk_merge_prepare and gysk_merge_finish (allowed: the prepared buffers do not
    depend on the capacity); every logical, logical-state, cluster and global top-N answer equals the ungrown large engines'"""
    import torch
    rng = np.random.default_rng(50 + world)
    flags = dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True)
    G = [ge.Engine(max_svcs=128, max_tasks=64, rank=r, world=world, **flags, **KW) for r in range(world)]
    F = [ge.Engine(max_svcs=512, max_tasks=256, rank=r, world=world, **flags, **KW) for r in range(world)]
    ids, tids = ids_of(6, 150), ids_of(7, 60)
    logical = np.arange(len(ids), dtype=np.uint64) // np.uint64(5) + np.uint64(900)
    hosts, clusters = np.arange(NHOSTS, dtype=np.uint32), np.arange(NHOSTS, dtype=np.uint64) // np.uint64(3) + np.uint64(70)
    for e in G + F:
        e.set_logical_map(ids, logical)
        e.set_cluster_map(hosts, clusters)
    for r, e in enumerate(G):
        if r % 2 == 0:
            e.grow(256, 128)
    for w in range(3):
        ev = events(rng, 9000, ids, tids, 5 * (w + 1))
        for r in range(world):
            sh = ev[(ev["host_idx"] % world) == r]
            feed([G[r], F[r]], sh)
        for e in G + F:
            e.flush(5 * (w + 1))
        if w == 1:
            for r, e in enumerate(G):
                if r % 2 == 0 or r == world - 1:
                    e.grow(512, 256)
        _merge(torch, G, between=(lambda: G[0].grow(512, 256)) if w == 0 else None)
        _merge(torch, F)
        lids, cids = np.unique(logical), np.unique(clusters)
        for g, f in zip(G, F):
            assert repr(g.query_logical(lids)) == repr(f.query_logical(lids))
            assert [bytes(x) for x in g.query_logical_all()[0]] == [bytes(x) for x in f.query_logical_all()[0]]
            assert [bytes(x) for x in g.query_logical_states_all()[0]] == [bytes(x) for x in f.query_logical_states_all()[0]]
            assert [bytes(x) for x in g.query_cluster_states_all()[0]] == [bytes(x) for x in f.query_cluster_states_all()[0]]
            assert [bytes(x) for x in g.query_cluster_states(cids)] == [bytes(x) for x in f.query_cluster_states(cids)]
            for l in lids[:10]:
                x, y = g.export_logical_tdigest(int(l)), f.export_logical_tdigest(int(l))
                assert (x is None) == (y is None) and (x is None or (x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes()))
            for m in (ge.TOPN_QPS, ge.TOPN_CONNS, ge.TOPN_NET):
                same_ranking(g.topn_logical(m, 30), f.topn_logical(m, 30), ("logical", m))
                a, b = g.topn_global(m, 64, rows=False)[0], f.topn_global(m, 64, rows=False)[0]
                same_ranking([(x.glob_id, x.score) for x in a], [(x.glob_id, x.score) for x in b], ("global", m))
            for m in (ge.TOPN_TASK_CPU, ge.TOPN_TASK_CPU_DELAY, ge.TOPN_TASK_BLKIO_DELAY):
                a, b = g.topn_global_tasks(m, 64, rows=False)[0], f.topn_global_tasks(m, 64, rows=False)[0]
                same_ranking([(x.glob_id, x.score) for x in a], [(x.glob_id, x.score) for x in b], ("global task", m))
    assert all(e.capacity()["max_svcs"] == 512 for e in G[::2])


def test_auto_grow_doubles_at_the_named_flush_and_stops_at_the_ceiling():
    """new services arrive window after window; a table doubles at the flush after the one whose count reached half its capacity, up
    to the ceiling; nothing is dropped below it, and past it the drops equal the oracle's at the ceiling capacity"""
    s0, limit, per_win, nwin = 32, 256, 8, 40                      # per_win <= s0 / 4: doubling keeps up
    G = ge.Engine(max_svcs=s0, max_tasks=16, max_batch=1 << 14, cms_log2_width=12)
    G.set_auto_grow(limit, 0)
    orc = po.OracleEngine(max_svcs=limit, max_tasks=16, cms_log2_width=12)
    ids = ids_of(8, per_win * nwin)
    rng = np.random.default_rng(3)
    cap, used, prev = s0, 0, None
    reached = None
    for w in range(nwin):
        live = ids[: per_win * (w + 1)]
        ev = np.zeros(3 * len(live), dtype=ge.EVENT_DTYPE)          # three samples per service and window: drops do not depend on
        ev["svc_id"] = np.repeat(live, 3)                             # which ids win the last slots
        ev["type"] = ge.EV_RESP
        ev["value"] = rng.integers(1000, 50_000, len(ev))
        ev["host_idx"] = 1
        ev = ev[rng.permutation(len(ev))]
        G.ingest_events(ev); G.sync()
        orc.ingest(ev)
        if cap < limit:
            assert G.stats()["events_dropped"] == 0, w
        G.flush(5 * (w + 1)); orc.flush(5 * (w + 1))
        # the rule, restated: at this flush the previous flush's count decides
        if prev is not None and cap < limit and 2 * prev >= cap:
            cap = min(2 * cap, limit)
        used = min(len(live), cap)
        prev = used
        c = G.capacity()
        assert c["max_svcs"] == cap and c["svcs_in_use"] == min(len(live), limit if cap == limit else cap), (w, c, cap)
        if cap == limit and reached is None:
            reached = w
    assert reached is not None and reached < nwin - 5
    assert G.capacity()["ngrows"] == int(np.log2(limit // s0))
    assert G.stats()["events_dropped"] == orc.counters()["dropped"] > 0


def test_limits_and_refused_growth_leave_the_engine_unchanged():
    import torch
    rng = np.random.default_rng(5)
    E = ge.Engine(max_svcs=64, max_tasks=32, **KW)
    ids, tids = ids_of(9, 100), ids_of(10, 50)
    ev = events(rng, 8000, ids, tids, 5)
    feed([E], ev)
    E.flush(5)
    def stats():
        d = E.stats()
        del d["kernel_launches"]                                     # the reads launch kernels of their own
        return d

    before = (stats(), SvcRowsOf(E, ids), [bytes(x) for x in E.query_window()[0]], E.export_cms().tobytes(), E.capacity())
    assert _code(lambda: E.grow(32, 32)) == INVAL
    assert _code(lambda: E.grow(64, 16)) == INVAL
    assert _code(lambda: E.grow((1 << 24) + 1, 32)) == INVAL
    assert E.L.gysk_set_auto_grow(E.h, (1 << 24) + 1, 0) == INVAL
    sb, _ = ge.slot_bytes(12)
    assert (1 << 24) * sb > torch.cuda.mem_get_info()[1]             # more than the device has: refused by the pre-check
    assert _code(lambda: E.grow(1 << 24, 32)) == NOMEM
    after = (stats(), SvcRowsOf(E, ids), [bytes(x) for x in E.query_window()[0]], E.export_cms().tobytes(), E.capacity())
    assert after == before and after[-1]["ngrows"] == 0
    E.grow(64, 32)                                                   # the same capacities: nothing to do
    assert E.capacity()["ngrows"] == 0


def test_full_engine_accepts_new_ids_after_a_grow():
    """an engine that filled its table dropped what the oracle of its capacity drops; after a grow it takes new ids"""
    rng = np.random.default_rng(6)
    E = ge.Engine(max_svcs=50, max_tasks=16, max_batch=1 << 14, cms_log2_width=12)
    orc = po.OracleEngine(max_svcs=50, max_tasks=16, cms_log2_width=12)
    ids = ids_of(11, 80)
    ev = np.zeros(4 * len(ids), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = np.repeat(ids, 4); ev["type"] = ge.EV_RESP; ev["value"] = rng.integers(1000, 9000, len(ev))
    ev = ev[rng.permutation(len(ev))]
    E.ingest_events(ev); E.sync(); orc.ingest(ev)
    assert E.stats()["events_dropped"] == orc.counters()["dropped"] == 4 * 30
    E.grow(200, 16)
    E.ingest_events(ev); E.sync()
    s = E.stats()
    assert s["events_dropped"] == 4 * 30 and s["nsvcs"] == 80
    assert all(r["found"] for r in E.query_svcs(ids))


def test_grow_while_eight_threads_ingest():
    """eight threads ingest through their page-locked stages while a ninth grows the engine once: every event is counted and the
    batch-independent state (histograms, HLL registers, count-min table) equals the oracle's"""
    rng = np.random.default_rng(8)
    E = ge.Engine(max_svcs=256, max_tasks=128, max_batch=1 << 14, cms_log2_width=12)
    ids, tids = ids_of(12, 200), ids_of(13, 100)
    parts = [events(rng, 20000, ids, tids, 1) for _ in range(8)]
    start = threading.Barrier(9)
    errs = []

    def ingest(p):
        try:
            start.wait()
            for off in range(0, len(p), 700):
                E.ingest_events(p[off: off + 700])
        except Exception as x:                      # noqa: BLE001
            errs.append(x)

    def grower():
        start.wait()
        E.grow(1024, 512)

    ths = [threading.Thread(target=ingest, args=(p,)) for p in parts] + [threading.Thread(target=grower)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errs
    E.sync()
    ev = np.concatenate(parts)
    orc = po.OracleEngine(max_svcs=1024, max_tasks=512, cms_log2_width=12)
    orc.ingest(ev)
    s = E.stats()
    assert s["events_in"] == len(ev) and s["events_dropped"] == orc.counters()["dropped"] == 0
    assert s["nsvcs"] == len(ids) and s["ntasks"] == len(tids)
    assert np.array_equal(E.export_cms(), orc.cms())
    for i in ids:
        a, b = E.export_hist(int(i), ge.HIST_RESP_CUR), orc.export_hist(int(i), 0)
        assert (a is None) == (b is None)
        if a is not None:
            assert a[0].tobytes() == b[0].tobytes() and a[1:] == b[1:]
            assert np.array_equal(E.export_hll(int(i)), orc.export_hll(int(i)))
    assert E.capacity()["max_svcs"] == 1024


def test_device_bytes_match_the_allocations():
    """device_bytes against cudaMemGetInfo around gysk_create / gysk_grow (within the allocator's granularity), and the difference of
    two engines against gysk_slot_bytes"""
    import torch
    torch.cuda.init()
    # Each cudaMalloc may be rounded up to the allocator's 2 MiB granularity. gysk_create makes 59 device allocations: 6 for the id
    # tables and counters, 32 per-slot arrays (tests/test_grow_host.py), 5 for the count-min tables, the t-digest grid and the hot rows,
    # 4 sort buffers, 6 batch buffers (long-segment rows, merge scratch, record queue), 4 event buffers and 2 read stages; 4 more
    # granules for kernel code loaded at a first launch. A growth of both tables (max_batch above the slots: the sort buffers stay)
    # makes 34 allocations and 34 frees, each pair off by less than one granule. An accounting slip in an array below a granule is
    # left to the exact comparison of two engines at the end.
    g = 2 << 20
    f0 = torch.cuda.mem_get_info()[0]
    E = ge.Engine(max_svcs=1 << 17, max_tasks=1 << 15, max_batch=1 << 20, cms_log2_width=12)
    f1 = torch.cuda.mem_get_info()[0]
    c = E.capacity()
    assert abs((f0 - f1) - c["device_bytes"]) <= (59 + 4) * g, (f0 - f1, c["device_bytes"])
    E.grow(1 << 18, 1 << 16)
    f2 = torch.cuda.mem_get_info()[0]
    c2 = E.capacity()
    assert abs((f1 - f2) - (c2["device_bytes"] - c["device_bytes"])) <= 34 * g, (f1 - f2, c2["device_bytes"] - c["device_bytes"])
    assert c2["device_bytes"] - c["device_bytes"] > 1 << 30
    sb, tb = ge.slot_bytes(12)
    E.close()
    B = ge.Engine(max_svcs=1 << 18, max_tasks=1 << 16, max_batch=1 << 20, cms_log2_width=12)
    A = ge.Engine(max_svcs=1 << 17, max_tasks=1 << 15, max_batch=1 << 20, cms_log2_width=12)
    tbl = 16 * ((1 << 20) - (1 << 19)) + 16 * ((1 << 17) - (1 << 16))  # both id tables double: 16-byte entries
    assert B.capacity()["device_bytes"] - A.capacity()["device_bytes"] == sb * (1 << 17) + tb * (1 << 15) + tbl
    assert c2["device_bytes"] == B.capacity()["device_bytes"]
