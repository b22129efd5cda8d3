"""The heaviest-flow sets on the device (GYSK_FLAG_FLOW_TOPK). Batches are driven one by one (one ingest of at most stage_batch events,
then sync, the batch count asserted), and after every batch and flush the four local reads at n = K must equal the restatement of
tests/flow_topk.py byte for byte, keys and both halves, scored on the engine's exported tables (pinned by the flow table tests). The
guarantee is asserted against exact per-flow scores at every check. Covered: the connection routes with ACTIVE records and the response
routes with hot rows on and off, set sizes around K and ties, zero scores, the direct path, the sketch edges and a wrapping kbytes half,
unknown ids, a full table and growth, the flag off against on, and the merge at world 1 ... 8 emulated on one GPU and once through NCCL."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge, synth
from tests import flow_queries as fq
from tests import flow_topk as ft
from tests.test_gpu_flow_level import _rowbytes
from tests.test_gpu_flow_query_level import _regions
from tests.test_gpu_merge import _emulate_collectives

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
K = ft.K
CFG = dict(max_svcs=1024, max_tasks=64, max_batch=1 << 17, cms_depth=4, cms_log2_width=12)


def _mixed(rng, n, nsvc=300, nclients=20_000, nactive=200):
    """gen_mixed with responses beyond the validity rule and ACTIVE records mixed in"""
    ev = synth.gen_mixed(rng, n, nsvc, ntask=32, nhosts=16, nclients=nclients)
    r = np.flatnonzero(ev["type"] == ge.EV_RESP)
    ev["value"][r[::211]] = fq.VALID_USEC + 5
    t = np.flatnonzero(np.isin(ev["type"], (ge.EV_CONNECT, ge.EV_ACCEPT, ge.EV_CLOSE_CLI, ge.EV_CLOSE_SER)))[:nactive]
    ev["type"][t] = ge.EV_ACTIVE
    ev["flags"][t] = rng.integers(1, 5, len(t))
    ev["value"][t] = rng.integers(1, 5000, len(t))
    return ev


def _tcp(keys, kbytes, svc=1000003, types=ge.EV_ACCEPT):
    """connection events, one per key, bytes = kbytes << 10"""
    ev = np.zeros(len(keys), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"], ev["value"], ev["type"] = svc, keys, np.asarray(kbytes, dtype=np.uint64) << np.uint64(10), types
    return ev


class Run:
    """one engine with the flag, the restated sets, and the window's events for the exact scores"""

    def __init__(self, queries=True, **kw):
        self.eng = ge.Engine(flow_topk=True, flow_queries=queries, **{**CFG, **kw})
        c = self.eng.cfg
        self.d, self.w, self.queries = c.cms_depth, c.cms_log2_width, queries
        self.sets = {ft.CONN: ft.Sets(1, self.d, self.w), ft.QRY: ft.Sets(0, self.d, self.w)}
        self.win = []
        self.nb = 0

    def tables(self, last=False):
        t = {ft.CONN: self.eng.export_cms(last)}
        if self.queries:
            t[ft.QRY] = self.eng.export_cms_queries(last)
        return t

    def batch(self, ev, known=None, ingest=None, what=None):
        assert len(ev) <= (self.eng.cfg.stage_batch or min(self.eng.cfg.max_batch, 1 << 22))      # one device batch
        (ingest or (lambda e: e.ingest_events(ev)))(self.eng)
        self.eng.sync()
        self.nb += 1
        assert self.eng.stats()["batches"] == self.nb, what
        tabs = self.tables()
        for w, tab in tabs.items():
            s = self.sets[w]
            floor = s.floor[-1] if s.floor else None
            s.batch(ft.batch_keys(ev, w, known), tab)
            if floor is not None and s.floor:
                assert s.floor[-1] >= floor, what      # the K-th score never falls within a window (no wrap in these streams)
        self.win.append((ev, known))
        self.check(what)

    def flush(self, t, what=None):
        self.eng.flush(t)
        for s in self.sets.values():
            s.flush()
        self.win = []
        self.check(what)

    def reads(self, last):
        out = {ft.CONN: self.eng.topk_flows(K, last)}
        if self.queries:
            out[ft.QRY] = self.eng.topk_flow_queries(K, last).view(ge.FLOW_EST_DTYPE)
        return out

    def check(self, what):
        for last in (False, True):
            tabs, got = self.tables(last), self.reads(last)
            for w, tab in tabs.items():
                keys = self.sets[w].last if last else self.sets[w].open
                want = ft.read(keys, tab, self.d, self.w, ft.HALF[w])
                assert got[w].tobytes() == want.tobytes(), (what, last, w, len(got[w]), len(want))
            keys = self.sets[ft.CONN].last if last else self.sets[ft.CONN].open
            assert self.eng.topk_flows(7, last).tobytes() == ft.read(keys, tabs[ft.CONN], self.d, self.w, 1, 7).tobytes(), (what, last)
        # the guarantee against the exact scores of the open window
        tabs = self.tables()
        for w, tab in tabs.items():
            if not self.win:
                break
            parts = [(ev, kn) for ev, kn in self.win]
            if w == ft.QRY:
                s = np.concatenate([fq.counted(ev, kn) for ev, kn in parts])
                fk, inc = s["flow_key"], fq.increments(s)
            else:
                evs = []
                for ev, kn in parts:
                    m = np.isin(ev["type"], ft.TCP_TYPES) & (ev["svc_id"] != 0)
                    if kn is not None:
                        m &= np.isin(ev["svc_id"], np.fromiter(kn, dtype=np.uint64, count=len(kn)))
                    evs.append(ev[m])
                e = np.concatenate(evs)
                fk, inc = e["flow_key"], ft.conn_increments(e)
            allk = np.unique(fk)
            ex = ft.exact_scores(allk, fk, inc, ft.HALF[w])
            assert ft.guarantee_holds(self.sets[w].open, tab, self.d, self.w, ft.HALF[w], allk, ex), (what, w)


@pytest.mark.parametrize("hot", ["on", "off"])
def test_mixed_routes_hot_rows_on_and_off(hot, monkeypatch):
    if hot == "on":
        monkeypatch.setenv("GYSK_HOT_MIN", "64")
    else:
        monkeypatch.setenv("GYSK_HOT_ROWS", "0")
    rng = np.random.default_rng(1 if hot == "on" else 2)
    run = Run()
    for i, step in enumerate(["b", "b", "b", 5, "b", "b", 10, 15, "b"]):
        if step == "b":
            run.batch(_mixed(rng, int(rng.integers(30_000, 90_000))), what=(hot, i))
        else:
            run.flush(step, what=(hot, i))
    assert (run.eng.hot_rows_in_use() > 0) == (hot == "on")


def test_raw_routes():
    """raw IPv4 connection and response records, and RESP16, reach the sets as they reach the tables"""
    from tests.test_gpu_flow_query_level import _route_batch
    rng = np.random.default_rng(3)
    run = Run()
    for i, route in enumerate(["ipv4", "ipv6", "resp16", "api_tran", "event32"]):
        ev, ingest = _route_batch(rng, route)
        run.batch(ev, ingest=ingest, what=route)
        if i == 2:
            run.flush(20, what=route)


def test_trace_events_never_enter():
    rng = np.random.default_rng(4)
    run = Run(max_trace_svcs=8)
    ev = _mixed(rng, 20_000)
    tr = ev[:500].copy()
    tr["type"] = ge.EV_TRACE
    tr["flow_key"] = np.arange(10**9, 10**9 + 500, dtype=np.uint64)
    run.batch(np.concatenate([ev, tr]), what="trace")
    keys = set(run.eng.topk_flows(K)["flow_key"].tolist()) | set(run.eng.topk_flow_queries(K)["flow_key"].tolist())
    assert not keys & set(tr["flow_key"].tolist())


@pytest.mark.parametrize("nflows", [K - 1, K, K + 1, 3 * K])
def test_set_sizes_and_ties(nflows):
    """fewer than, exactly and one more than K flows; equal scores cut inside a run; zero scores left out of the reads"""
    rng = np.random.default_rng(nflows)
    run = Run(queries=False, cms_log2_width=20)
    keys = rng.choice(1 << 40, nflows, replace=False).astype(np.uint64)
    kb = np.where(np.arange(nflows) % 3 == 0, 7, rng.integers(0, 3, nflows))       # a long run of score 7, many 0, 1 and 2
    run.batch(_tcp(keys, kb), what=nflows)
    got = run.eng.topk_flows(K)
    assert np.all(got["kbytes"] > 0) and len(got) == min(K, int((kb > 0).sum()))
    run.batch(_tcp(keys[: nflows // 2], np.ones(nflows // 2, dtype=np.int64)), what=nflows)
    run.flush(5)


def test_direct_path():
    """more than 2^21 distinct flows in one batch: most records take the direct path"""
    rng = np.random.default_rng(6)
    n = (1 << 21) + 300_000
    run = Run(queries=False, max_batch=1 << 22, cms_log2_width=20)
    keys = rng.integers(1, 1 << 62, n, dtype=np.uint64)
    run.batch(_tcp(keys, rng.integers(0, 64, n)), what="direct")
    assert run.eng.last_batch_flow_direct() > 0
    run.batch(_tcp(keys[:100_000], rng.integers(0, 4096, 100_000)), what="direct2")


@pytest.mark.parametrize("depth,log2w", [(1, 12), (8, 12), (4, 4), (4, 22)])
def test_sketch_edges(depth, log2w):
    rng = np.random.default_rng(depth * 100 + log2w)
    run = Run(cms_depth=depth, cms_log2_width=log2w)
    for i, step in enumerate(["b", "b", 5, "b"]):
        if step == "b":
            run.batch(_mixed(rng, 40_000), what=(depth, log2w, i))
        else:
            run.flush(step)


def test_wrapping_kbytes_half():
    """ACTIVE records near 2^32 kbytes: the estimates wrap and the sets follow them"""
    rng = np.random.default_rng(8)
    run = Run(queries=False)
    keys = np.arange(1, 6001, dtype=np.uint64)
    ev = np.zeros(len(keys), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"], ev["type"], ev["flags"] = 1000003, keys, ge.EV_ACTIVE, 1
    ev["value"] = rng.integers(0xF0000000, 0xFFFFFFFF, len(keys))
    run.sets[ft.CONN].floor = []
    for i in range(3):
        ev["value"] = rng.integers(0xC0000000, 0xFFFFFFFF, len(keys))
        run.eng.ingest_events(ev); run.eng.sync(); run.nb += 1
        run.sets[ft.CONN].batch(keys, run.eng.export_cms())
        tab = run.eng.export_cms()
        assert run.eng.topk_flows(K).tobytes() == ft.read(run.sets[ft.CONN].open, tab, run.d, run.w, 1).tobytes(), i


def test_unknown_ids_full_table_and_growth():
    rng = np.random.default_rng(9)
    run = Run(auto_register=False, max_svcs=64)
    ev = _mixed(rng, 30_000, nsvc=40)
    known = np.unique(ev["svc_id"][ev["type"] != ge.EV_TASK])[:20]
    run.eng.register_ids(known)
    run.batch(ev, known=set(known.tolist()), what="unknown")
    run.eng.grow(128, 64)
    run.batch(_mixed(rng, 30_000, nsvc=40), known=set(known.tolist()), what="grown")
    run.flush(5)
    # a full table: the ids beyond its slots are dropped, and their records never reach the sets
    full = Run(max_svcs=16)
    ev = _mixed(rng, 30_000, nsvc=40)
    ids = np.unique(ev["svc_id"][ev["type"] != ge.EV_TASK])
    full.eng.ingest_events(ev); full.eng.sync()
    held = {int(r["glob_id"]) for r in full.eng.query_svcs(ids) if r["found"]}
    assert 0 < len(held) <= 16 < len(ids)
    full.nb = 1
    for w, tab in full.tables().items():
        full.sets[w].batch(ft.batch_keys(ev, w, held), tab)
    full.win.append((ev, held))
    full.check("full")


OTHER = {"alone": {}, "queries": dict(flow_queries=True), "levels": dict(flow_queries=True, flow_level=True, flow_query_level=True),
         "resp_hist": dict(flow_queries=True, flow_resp_hist=True),
         "merge": dict(flow_queries=True, merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, merge_traces=True,
                       max_trace_svcs=64)}


@pytest.mark.parametrize("other", sorted(OTHER))
def test_flag_off_and_on_answer_alike(other):
    import torch
    rng = np.random.default_rng(17)
    flags = OTHER[other]
    off, on = ge.Engine(**CFG, **flags), ge.Engine(flow_topk=True, **CFG, **flags)
    ev0 = _mixed(np.random.default_rng(0), 20_000)
    sids = np.unique(ev0["svc_id"][ev0["type"] != ge.EV_TASK])
    for e in (off, on):
        e.set_logical_map(sids, sids % np.uint64(7) + np.uint64(50))
    lids = np.unique(sids % np.uint64(7) + np.uint64(50))
    for i, t in enumerate((5, 10, 40, 40)):
        ev = _mixed(rng, 40_000)
        for e in (off, on):
            e.ingest_events(ev); e.sync()
        keys = np.unique(ev["flow_key"])[:2000]
        for lw in (False, True):
            assert off.export_cms(lw).tobytes() == on.export_cms(lw).tobytes()
            assert off.query_flows(keys, lw).tobytes() == on.query_flows(keys, lw).tobytes()
            if flags.get("flow_queries"):
                assert off.export_cms_queries(lw).tobytes() == on.export_cms_queries(lw).tobytes()
        assert _rowbytes(off.query_svcs(sids)) == _rowbytes(on.query_svcs(sids))
        sa, sb = off.stats(), on.stats()
        sa.pop("kernel_launches"); sb.pop("kernel_launches")
        assert sa == sb
        assert off.last_batch_flow_direct() == on.last_batch_flow_direct()
        for e in (off, on):
            e.flush(t)
        for e in (off, on):
            _emulate_collectives(torch, [e])
        ra, rb = _regions(off, torch), _regions(on, torch)
        assert {k: (v[0], v[1].tobytes()) for k, v in ra.items()} == {k: (v[0], v[1].tobytes()) for k, v in rb.items()}
        assert _rowbytes(off.query_logical(lids)) == _rowbytes(on.query_logical(lids))
        for lw in (False, True):
            assert off.query_flows_global(keys, lw).tobytes() == on.query_flows_global(keys, lw).tobytes()
    for call in (lambda e: e.topk_flows(), lambda e: e.topk_flow_queries(), lambda e: e.topk_flows_global(), lambda e: e.topk_flow_queries_global()):
        with pytest.raises(ge.GyskError) as ex:
            call(off)
        assert ex.value.code == NOTSUP
    if not flags.get("flow_queries"):
        for call in (lambda e: e.topk_flow_queries(), lambda e: e.topk_flow_queries_global()):
            with pytest.raises(ge.GyskError) as ex:
                call(on)
            assert ex.value.code == NOTSUP
    fresh = ge.Engine(flow_topk=True, flow_queries=True, **CFG)
    for call in (fresh.topk_flows_global, fresh.topk_flow_queries_global):
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == INVAL


def _shard(ev, world):
    return [ev[ev["host_idx"] % world == r] for r in range(world)]


def _check_merge(engines, d, w, what):
    summed = {ft.CONN: sum((e.export_cms(True) for e in engines[1:]), engines[0].export_cms(True).copy()),
              ft.QRY: sum((e.export_cms_queries(True) for e in engines[1:]), engines[0].export_cms_queries(True).copy())}
    for wh, read in ((ft.CONN, lambda e: e.topk_flows_global()), (ft.QRY, lambda e: e.topk_flow_queries_global().view(ge.FLOW_EST_DTYPE))):
        local = [(e.topk_flows(K, True) if wh == ft.CONN else e.topk_flow_queries(K, True).view(ge.FLOW_EST_DTYPE)) for e in engines]
        # the last sets as the ranks hold them, zero scores included: every flow of a rank's window when it has at most K
        sets = [r["flow_key"] for r in local]
        want = ft.read(ft.merged(sets, summed[wh], d, w, ft.HALF[wh]), summed[wh], d, w, ft.HALF[wh])
        for e in engines:
            assert read(e).tobytes() == want.tobytes(), (what, wh)


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("others", ["alone", "merge"])
def test_merge_ranks_the_union(world, others):
    import torch
    rng = np.random.default_rng(world * 10 + 7)
    d, w = CFG["cms_depth"], CFG["cms_log2_width"]
    extra = OTHER["merge"] if others == "merge" else dict(flow_queries=True)
    engines = [ge.Engine(flow_topk=True, rank=r, world=world, **{**CFG, **extra}) for r in range(world)]
    for step, t in enumerate([30, 35, 60]):
        ev = _mixed(rng, 60_000, nclients=3000)
        ev["value"][np.isin(ev["type"], ft.TCP_TYPES[:4])] |= np.uint32(1024)      # every connection record scores: no zero to leave out
        for e, sh in zip(engines, _shard(ev, world)):
            e.ingest_events(sh); e.sync()
            e.flush(t)
        _emulate_collectives(torch, engines)
        _check_merge(engines, d, w, (world, others, step))


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(5)
    eng = ge.Engine(flow_topk=True, flow_queries=True, **CFG)
    for t in (30, 35):
        eng.ingest_events(_mixed(rng, 30_000)); eng.sync()
        eng.flush(t)
    _emulate_collectives(torch, [eng])
    emulated = eng.topk_flows_global().tobytes(), eng.topk_flow_queries_global().tobytes()
    assert emulated == (eng.topk_flows(K, True).tobytes(), eng.topk_flow_queries(K, True).tobytes())
    eng.nccl_comm_init(eng.nccl_unique_id(), 1, 0)
    eng.merge_global()
    eng.sync()
    assert (eng.topk_flows_global().tobytes(), eng.topk_flow_queries_global().tobytes()) == emulated
