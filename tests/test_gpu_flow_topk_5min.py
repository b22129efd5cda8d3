"""The heaviest-flow sets of the rolling 300-s levels on the device (GYSK_FLAG_FLOW_TOPK_5MIN). Batches are driven one by one as in
tests/test_gpu_flow_topk.py, whose window-set checks run at every batch and flush. After every flush both local reads at n = K and their
bounds must equal the restatement of tests/flow_topk_5min.py, fed the flush's closing tables (gysk_export_cms(last_window=1) /
gysk_export_cms_queries(last_window=1)) and the window sets restated from the events; every row must be byte-equal to the _5min point
query on its key, and the bound must hold against exact per-flow scores from the events. Covered: the flush sequences of
tests/flow_level.py, the connection and response routes with hot rows on and off, set sizes around K with ties and zero scores, the
direct path, the sketch edges, eviction and growth, the refusals, the flag off against on, and the merge at world 1 ... 8 emulated on
one GPU and once through NCCL."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import flow_level as fl
from tests import flow_queries as fq
from tests import flow_topk as ft
from tests import flow_topk_5min as f5
from tests.test_gpu_flow_level import _rowbytes
from tests.test_gpu_flow_query_level import _regions
from tests.test_gpu_flow_topk import CFG, Run, _mixed, _shard, _tcp
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import _dev_bytes

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
K = ft.K
LEVELS = dict(flow_level=True, flow_query_level=True)
SLAB_ENTRY = 4128                                                       # sizeof(SlabEntry)
TOPK_SLAB_BYTES = -(-2 * (K + 2) * 8 // SLAB_ENTRY) * SLAB_ENTRY       # two sets of K + 2 words, in whole slab entries


class Run5(Run):
    """Run with the 300-s sets: per held level its restated LevelSets, and per flush the exact scores of the window it closed"""

    def __init__(self, queries=True, level=True, qlevel=True, **kw):
        super().__init__(queries=queries, flow_topk_5min=True, flow_level=level, flow_query_level=qlevel, **kw)
        self.lv = {}
        if level:
            self.lv[ft.CONN] = f5.LevelSets(1, self.d, self.w)
        if qlevel:
            self.lv[ft.QRY] = f5.LevelSets(0, self.d, self.w)
        self.tsecs, self.exact = [], {w: [] for w in self.lv}
        self.check5("before the first flush")

    def _window_exact(self, w):
        if not self.win:
            return {}
        if w == ft.QRY:
            s = np.concatenate([fq.counted(ev, kn) for ev, kn in self.win])
            fk, inc = s["flow_key"], fq.increments(s)
        else:
            evs = []
            for ev, kn in self.win:
                m = np.isin(ev["type"], ft.TCP_TYPES) & (ev["svc_id"] != 0)
                if kn is not None:
                    m &= np.isin(ev["svc_id"], np.fromiter(kn, dtype=np.uint64, count=len(kn)))
                evs.append(ev[m])
            e = np.concatenate(evs)
            fk, inc = e["flow_key"], ft.conn_increments(e)
        allk = np.unique(fk)
        return dict(zip(allk.tolist(), ft.exact_scores(allk, fk, inc, ft.HALF[w]).tolist()))

    def flush(self, t, what=None):
        wins = {w: self.sets[w].open.copy() for w in self.lv}
        for w in self.lv:
            self.exact[w].append(self._window_exact(w))
        super().flush(t, what)
        self.tsecs.append(t)
        closed = self.tables(True)
        for w, lv in self.lv.items():
            lv.flush(t, wins[w], closed[w])
        self.check5(what)

    def reads5(self):
        out = {}
        if ft.CONN in self.lv:
            out[ft.CONN] = self.eng.topk_flows_5min(K)
        if ft.QRY in self.lv:
            rows, b = self.eng.topk_flow_queries_5min(K)
            out[ft.QRY] = rows.view(ge.FLOW_EST_DTYPE), b
        return out

    def check5(self, what):
        got = self.reads5()
        for w, lv in self.lv.items():
            rows, b = got[w]
            level = self.eng.export_cms_5min() if w == ft.CONN else self.eng.export_cms_queries_5min()
            assert level.tobytes() == lv.level.tobytes(), (what, w)
            want = ft.read(lv.L, lv.level, self.d, self.w, ft.HALF[w])
            assert rows.tobytes() == want.tobytes(), (what, w, len(rows), len(want))
            assert b == lv.B, (what, w, b, lv.B)
            point = self.eng.query_flows_5min(rows["flow_key"]) if w == ft.CONN else \
                self.eng.query_flow_queries_5min(rows["flow_key"]).view(ge.FLOW_EST_DTYPE)
            assert point.tobytes() == rows.tobytes(), (what, w)
            if self.tsecs:
                ex = f5.exact_level(self.tsecs, self.exact[w])
                assert f5.guarantee_holds(lv.L, lv.B, ex), (what, w)
            else:
                assert len(rows) == 0 and b == 0
        if ft.CONN in self.lv:
            assert self.eng.topk_flows_5min(7)[0].tobytes() == ft.read(self.lv[ft.CONN].L, self.lv[ft.CONN].level, self.d, self.w, 1,
                                                                       7).tobytes(), what


@pytest.mark.parametrize("seq", sorted(fl.SEQUENCES))
def test_flush_sequences(seq):
    rng = np.random.default_rng(sum(map(ord, seq)))
    run = Run5()
    for i, t in enumerate(fl.SEQUENCES[seq]):
        run.batch(_mixed(rng, int(rng.integers(5_000, 15_000)), nclients=6000), what=(seq, i))
        run.flush(t, what=(seq, i, t))


@pytest.mark.parametrize("hot", ["on", "off"])
def test_mixed_routes_hot_rows_on_and_off(hot, monkeypatch):
    monkeypatch.setenv(*(("GYSK_HOT_MIN", "64") if hot == "on" else ("GYSK_HOT_ROWS", "0")))
    rng = np.random.default_rng(11 if hot == "on" else 12)
    run = Run5()
    for i, t in enumerate([5, 10, 35, 65, 70]):
        for _ in range(2):
            run.batch(_mixed(rng, int(rng.integers(30_000, 60_000))), what=(hot, i))
        run.flush(t, what=(hot, i))
    assert (run.eng.hot_rows_in_use() > 0) == (hot == "on")


def test_raw_routes():
    """raw IPv4 / IPv6 response records, RESP16 and API_TRAN reach the level sets as they reach the levels"""
    from tests.test_gpu_flow_query_level import _route_batch
    rng = np.random.default_rng(13)
    run = Run5()
    for i, route in enumerate(["ipv4", "ipv6", "resp16", "api_tran", "event32"]):
        ev, ingest = _route_batch(rng, route)
        run.batch(ev, ingest=ingest, what=route)
        run.flush(30 * (i + 1), what=route)


@pytest.mark.parametrize("nflows", [K - 1, K, K + 1, 3 * K])
def test_set_sizes_ties_and_zero_scores(nflows):
    """K - 1 ... 3K flows over several windows and slots: long runs of equal scores cut inside the run, zero scores left out of the
    reads, and a slot that holds more than K of them across its windows"""
    rng = np.random.default_rng(nflows)
    run = Run5(queries=False, qlevel=False, cms_log2_width=20)
    keys = rng.choice(1 << 40, nflows, replace=False).astype(np.uint64)
    for i, t in enumerate([5, 10, 15, 40, 45, 400]):
        part = keys[rng.permutation(nflows)[: max(1, nflows * 2 // 3)]]
        kb = np.where(np.arange(len(part)) % 3 == 0, 7, rng.integers(0, 3, len(part)))
        run.batch(_tcp(part, kb), what=(nflows, i))
        run.flush(t, what=(nflows, i))
    rows, b = run.eng.topk_flows_5min(K)
    assert np.all(rows["kbytes"] > 0)


def test_direct_path():
    """more than 2^21 distinct flows in one batch: most records take the direct path"""
    rng = np.random.default_rng(16)
    n = (1 << 21) + 300_000
    run = Run5(queries=False, qlevel=False, max_batch=1 << 22, cms_log2_width=20)
    keys = rng.integers(1, 1 << 62, n, dtype=np.uint64)
    run.batch(_tcp(keys, rng.integers(0, 64, n)), what="direct")
    assert run.eng.last_batch_flow_direct() > 0
    run.flush(5, what="direct")
    run.batch(_tcp(keys[:100_000], rng.integers(0, 4096, 100_000)), what="direct2")
    run.flush(10, what="direct2")


@pytest.mark.parametrize("depth,log2w", [(1, 4), (8, 4), (1, 22), (8, 22)])
def test_sketch_edges(depth, log2w):
    rng = np.random.default_rng(depth * 100 + log2w)
    wide = dict(queries=False, qlevel=False) if log2w > 20 else {}       # one level at 2^22: the restated ring holds 10 tables
    run = Run5(cms_depth=depth, cms_log2_width=log2w, **wide)
    for i, t in enumerate([5, 35, 40]):
        run.batch(_mixed(rng, 20_000), what=(depth, log2w, i))
        run.flush(t, what=(depth, log2w, i))


def test_eviction_and_growth_between_flushes():
    rng = np.random.default_rng(19)
    run = Run5(max_svcs=256, idle_evict_secs=20)
    for i, t in enumerate([5, 10, 100, 105, 140]):
        run.batch(_mixed(rng, 20_000, nsvc=200 if i < 2 else 60), what=("evict", i))
        if i == 2:
            run.eng.grow(512, 128)
        run.flush(t, what=("evict", i))
    assert run.eng.stats()["svcs_evicted"] > 0


def test_refusals():
    for kw in (dict(flow_level=True), dict(flow_topk=True), dict(flow_topk=True, flow_queries=True)):
        with pytest.raises(ge.GyskError) as ex:
            ge.Engine(flow_topk_5min=True, **CFG, **kw)
        assert ex.value.code == INVAL
    conn_only = ge.Engine(flow_topk=True, flow_topk_5min=True, flow_level=True, flow_queries=True, **CFG)
    qry_only = ge.Engine(flow_topk=True, flow_topk_5min=True, flow_queries=True, flow_query_level=True, **CFG)
    without = ge.Engine(flow_topk=True, flow_queries=True, **LEVELS, **CFG)
    calls = {"c": lambda e: e.topk_flows_5min(), "q": lambda e: e.topk_flow_queries_5min(), "cg": lambda e: e.topk_flows_global_5min(),
             "qg": lambda e: e.topk_flow_queries_global_5min()}
    for eng, notsup in ((conn_only, ("q", "qg")), (qry_only, ("c", "cg")), (without, tuple(calls))):
        for name, call in calls.items():
            if name in notsup:
                with pytest.raises(ge.GyskError) as ex:
                    call(eng)
                assert ex.value.code == NOTSUP, name
            elif name.endswith("g"):
                with pytest.raises(ge.GyskError) as ex:
                    call(eng)
                assert ex.value.code == INVAL, name          # before the first merge finish
            else:
                rows, b = call(eng)
                assert len(rows) == 0 and b == 0


OTHER = {"levels": dict(flow_level=True), "both_levels": dict(flow_queries=True, **LEVELS),
         "every_flag": dict(flow_queries=True, flow_resp_hist=True, merge_levels=True, merge_states=True, merge_clusters=True,
                            merge_topn=True, merge_traces=True, max_trace_svcs=64, **LEVELS)}


@pytest.mark.parametrize("other", sorted(OTHER))
def test_flag_off_and_on_answer_alike(other):
    import torch
    rng = np.random.default_rng(27)
    flags = OTHER[other]
    off, on = ge.Engine(flow_topk=True, **CFG, **flags), ge.Engine(flow_topk=True, flow_topk_5min=True, **CFG, **flags)
    ev0 = _mixed(np.random.default_rng(0), 20_000)
    sids = np.unique(ev0["svc_id"][ev0["type"] != ge.EV_TASK])
    for e in (off, on):
        e.set_logical_map(sids, sids % np.uint64(7) + np.uint64(50))
    lids = np.unique(sids % np.uint64(7) + np.uint64(50))
    for i, t in enumerate((5, 10, 40, 40, 300)):
        ev = _mixed(rng, 40_000)
        for e in (off, on):
            e.ingest_events(ev); e.sync()
        keys = np.unique(ev["flow_key"])[:2000]
        for lw in (False, True):
            assert off.export_cms(lw).tobytes() == on.export_cms(lw).tobytes()
            assert off.query_flows(keys, lw).tobytes() == on.query_flows(keys, lw).tobytes()
            assert off.topk_flows(K, lw).tobytes() == on.topk_flows(K, lw).tobytes()
            if flags.get("flow_queries"):
                assert off.topk_flow_queries(K, lw).tobytes() == on.topk_flow_queries(K, lw).tobytes()
        assert off.query_flows_5min(keys).tobytes() == on.query_flows_5min(keys).tobytes()
        assert _rowbytes(off.query_svcs(sids)) == _rowbytes(on.query_svcs(sids))
        sa, sb = off.stats(), on.stats()
        sa.pop("kernel_launches"); sb.pop("kernel_launches")
        assert sa == sb
        for e in (off, on):
            e.flush(t)
        for e in (off, on):
            _emulate_collectives(torch, [e])
        ra, rb = _regions(off, torch), _regions(on, torch)
        assert {k: (v[0], v[1].tobytes()) for k, v in ra.items()} == {k: (v[0], v[1].tobytes()) for k, v in rb.items()}
        # the slab only grows by the level sets, in whole entries after the window sets. The logical digests and the window sets are
        # byte-equal; the top-N candidates and trace slabs between them depend on the order services took their slots, so an engine
        # differs from any other there, flag or not.
        pa, na = off.merge_tdigest_slab()
        pb, nb = on.merge_tdigest_slab()
        sa_, sb_ = _dev_bytes(torch, pa, na).tobytes(), _dev_bytes(torch, pb, nb).tobytes()
        assert nb - na == TOPK_SLAB_BYTES
        assert sa_[: len(lids) * SLAB_ENTRY] == sb_[: len(lids) * SLAB_ENTRY]
        assert sa_[na - TOPK_SLAB_BYTES:] == sb_[na - TOPK_SLAB_BYTES: na]
        new = np.frombuffer(sb_[na:], dtype=np.uint64)
        rows, bound = on.topk_flows_5min(K)
        assert new[1] == bound and new[0] >= len(rows) and new[2: 2 + len(rows)].tolist() == rows["flow_key"].tolist()
        assert _rowbytes(off.query_logical(lids)) == _rowbytes(on.query_logical(lids))
        assert off.topk_flows_global().tobytes() == on.topk_flows_global().tobytes()
        for lw in (False, True):
            assert off.query_flows_global(keys, lw).tobytes() == on.query_flows_global(keys, lw).tobytes()
        assert off.query_flows_global_5min(keys).tobytes() == on.query_flows_global_5min(keys).tobytes()
        assert off.merge_flush_range() == on.merge_flush_range()
    with pytest.raises(ge.GyskError) as ex:
        off.topk_flows_5min()
    assert ex.value.code == NOTSUP


def _check_merge(ranks, what):
    d, w = ranks[0].d, ranks[0].w
    for wh in ranks[0].lv:
        summed = sum((r.lv[wh].level for r in ranks[1:]), ranks[0].lv[wh].level.copy())
        g, bg = f5.merged([r.lv[wh].L for r in ranks], [r.lv[wh].B for r in ranks], summed, d, w, ft.HALF[wh])
        want = ft.read(g, summed, d, w, ft.HALF[wh])
        for r in ranks:
            if wh == ft.CONN:
                rows, b = r.eng.topk_flows_global_5min()
                point = r.eng.query_flows_global_5min(rows["flow_key"])
            else:
                rows, b = r.eng.topk_flow_queries_global_5min()
                rows = rows.view(ge.FLOW_EST_DTYPE)
                point = r.eng.query_flow_queries_global_5min(rows["flow_key"]).view(ge.FLOW_EST_DTYPE)
            assert rows.tobytes() == want.tobytes(), (what, wh)
            assert point.tobytes() == rows.tobytes(), (what, wh)
            assert b == bg, (what, wh, b, bg)
        ex = {}
        for r in ranks:
            for key, x in f5.exact_level(r.tsecs, r.exact[wh]).items():
                ex[key] = ex.get(key, 0) + x
        assert f5.guarantee_holds(g, bg, ex), (what, wh)


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("others", ["alone", "merge"])
def test_merge_ranks_the_union(world, others):
    import torch
    rng = np.random.default_rng(world * 10 + 9)
    extra = dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, merge_traces=True, max_trace_svcs=64) \
        if others == "merge" else {}
    ranks = [Run5(rank=r, world=world, **extra) for r in range(world)]
    for step, t in enumerate([30, 35, 60, 200]):
        ev = _mixed(rng, 40_000, nclients=3000)
        for run, sh in zip(ranks, _shard(ev, world)):
            run.batch(sh, what=(world, others, step))
            run.flush(t, what=(world, others, step))
        _emulate_collectives(torch, [r.eng for r in ranks])
        _check_merge(ranks, (world, others, step))


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(25)
    run = Run5()
    for t in (30, 35, 65):
        run.batch(_mixed(rng, 30_000), what=t)
        run.flush(t, what=t)
    _emulate_collectives(torch, [run.eng])
    emulated = run.eng.topk_flows_global_5min(), run.eng.topk_flow_queries_global_5min()
    _check_merge([run], "emulated")
    run.eng.nccl_comm_init(run.eng.nccl_unique_id(), 1, 0)
    run.eng.merge_global()
    run.eng.sync()
    got = run.eng.topk_flows_global_5min(), run.eng.topk_flow_queries_global_5min()
    for (ra, ba), (rb, bb) in zip(got, emulated):
        assert ra.tobytes() == rb.tobytes() and ba == bb
