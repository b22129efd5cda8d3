"""The slow-response sets on the device (GYSK_FLAG_FLOW_TOPK_SLOW). Batches are driven one by one, and after every batch and flush both
local reads at n = K must equal the restatement of tests/flow_topk_slow.py on the engine's exported response tables, key for key and byte
for byte; every row must equal its point query, its score must be the sum of its counts from b_slow on, and the guarantee must hold against
exact per-flow slow counts. With the 300-s level, L and B_L must equal the fold restated on the rolled response tables after every flush.
Covered: every response route with hot rows on and off, trace events, samples at T and T + 1 for three thresholds and beyond the validity
rule, set sizes around K with ties, fast-only flows, the direct path, the sketch edges, eviction and growth, the threshold call and its
refusals, the flag off against on, and the merge at world 1 ... 8 emulated on one GPU and once through NCCL."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import flow_level as fl
from tests import flow_queries as fq
from tests import flow_resp_hist as frh
from tests import flow_topk_slow as fs
from tests.test_gpu_flow_level import _rowbytes
from tests.test_gpu_flow_query_level import _regions, _route_batch
from tests.test_gpu_flow_topk import CFG, _mixed, _shard
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import _dev_bytes

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
K = fs.K
FLAGS = dict(flow_topk=True, flow_queries=True, flow_resp_hist=True)
LEVEL = dict(flow_topk_5min=True, flow_query_level=True)
SLAB_ENTRY = 4128                                                       # sizeof(SlabEntry)


def _slab_bytes(nsets):
    return -(-nsets * (K + 2) * 8 // SLAB_ENTRY) * SLAB_ENTRY


def _resp(keys, msec, svc=1000003):
    """response events, one per key, usec = msec * 1000 + 500 (the histogram takes msec = usec / 1000)"""
    ev = np.zeros(len(keys), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"], ev["type"] = svc, keys, ge.EV_RESP
    ev["value"] = np.asarray(msec, dtype=np.uint64) * np.uint64(1000) + np.uint64(500)
    return ev


def _slow_mixed(rng, n, t_ms=300, **kw):
    """gen_mixed with a share of its responses moved above t_ms, so that slow flows are a minority of the window's"""
    ev = _mixed(rng, n, **kw)
    r = np.flatnonzero((ev["type"] == ge.EV_RESP) & (ev["value"] < fq.VALID_USEC))
    pick = r[rng.random(len(r)) < 0.03]
    ev["value"][pick] = (np.uint32(t_ms + 1) + rng.integers(0, 3 * t_ms + 2, len(pick)).astype(np.uint32)) * np.uint32(1000)
    return ev


class Run:
    """one engine with the flag (and with level=True its 300-s sets), the restated sets and the window's counted samples"""

    def __init__(self, above_ms=None, level=False, **kw):
        self.eng = ge.Engine(flow_topk_slow=True, **{**CFG, **FLAGS, **(LEVEL if level else {}), **kw})
        if above_ms is not None:
            self.eng.set_flow_slow(above_ms)
        c = self.eng.cfg
        self.d, self.w = c.cms_depth, c.cms_log2_width
        self.bs = fs.b_slow(300 if above_ms is None else above_ms)
        self.score = fs.scorer(self.bs)
        self.sets = fs.Sets(self.bs, self.d, self.w)
        self.lv = fs.LevelSets(self.bs, self.d, self.w) if level else None
        self.win, self.tsecs, self.history = [], [], []
        self.nb = 0

    def table(self, last=False):
        return self.eng.export_cms_resp(last).reshape(-1)

    def batch(self, ev, known=None, ingest=None, what=None):
        assert len(ev) <= (self.eng.cfg.stage_batch or min(self.eng.cfg.max_batch, 1 << 22))      # one device batch
        (ingest or (lambda e: e.ingest_events(ev)))(self.eng)
        self.eng.sync()
        self.nb += 1
        assert self.eng.stats()["batches"] == self.nb, what
        s = fq.counted(ev, known)
        self.sets.batch(fs.slow_keys(s, self.bs), self.table())
        self.win.append(s)
        self.check(what)

    def flush(self, t, what=None):
        closing = self.table()
        self.eng.flush(t)
        if self.lv is not None:
            self.lv.flush(t, self.sets.open, closing)
            self.tsecs.append(t)
            self.history.append(np.concatenate(self.win) if self.win else np.zeros(0, dtype=self.win_dtype()))
        self.sets.flush()
        self.win = []
        self.check(what)

    def win_dtype(self):
        return fq.counted(np.zeros(0, dtype=ge.EVENT_DTYPE), None).dtype

    def check_rows(self, rows, point, what):
        assert rows.tobytes() == point(rows["flow_key"]).tobytes(), what                 # each row is its point query
        s = fs.score_of_counts(rows["counts"], self.bs)
        assert np.all(s > 0) and np.all(s[:-1] >= s[1:]), what                            # best first, no zero score

    def check(self, what):
        for last in (False, True):
            tab = self.table(last)
            got = self.eng.topk_flow_slow(K, last)
            keys = self.sets.last if last else self.sets.open
            want = fs.read(keys, tab, self.d, self.w, self.bs)
            assert got.tobytes() == want.tobytes(), (what, last, len(got), len(want))
            self.check_rows(got, lambda k: self.eng.query_flow_resp(k, last), (what, last))
            assert self.eng.topk_flow_slow(7, last).tobytes() == fs.read(keys, tab, self.d, self.w, self.bs, 7).tobytes(), (what, last)
        if self.win:
            s = np.concatenate(self.win)
            allk = np.unique(s["flow_key"])
            ex = fs.exact_slow(s, allk, self.bs)
            assert fs.guarantee_holds(self.sets.open, self.table(), self.d, self.w, self.score, allk, ex), what
        if self.lv is not None:
            level = self.eng.export_cms_resp_5min().reshape(-1)
            assert level.tobytes() == self.lv.level.tobytes(), what
            rows, bound = self.eng.topk_flow_slow_5min(K)
            assert rows.tobytes() == fs.read(self.lv.L, level, self.d, self.w, self.bs).tobytes(), what
            assert bound == self.lv.B, (what, bound, self.lv.B)
            self.check_rows(rows, self.eng.query_flow_resp_5min, what)
            if self.tsecs:
                held = [self.history[j] for j in fl.held_windows(self.tsecs)]
                held = np.concatenate(held) if held else np.zeros(0, dtype=self.win_dtype())
                keys = np.unique(held["flow_key"])
                ex = dict(zip(keys.tolist(), fs.exact_slow(held, keys, self.bs).tolist()))
                members = set(self.lv.L.tolist())
                assert all(x <= bound for key, x in ex.items() if key not in members), what


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
            run.batch(_slow_mixed(rng, int(rng.integers(30_000, 90_000))), what=(hot, i))
        else:
            run.flush(step, what=(hot, i))
    assert (run.eng.hot_rows_in_use() > 0) == (hot == "on")


def test_raw_routes():
    rng = np.random.default_rng(3)
    run = Run(above_ms=1000, max_trace_svcs=8)
    for i, route in enumerate(["ipv4", "ipv6", "resp16", "api_tran", "event32"]):
        ev, ingest = _route_batch(rng, route)
        run.batch(ev, ingest=ingest, what=route)
        if i == 2:
            run.flush(20, what=route)


def test_trace_events_never_enter():
    rng = np.random.default_rng(4)
    run = Run(max_trace_svcs=8)
    ev = _slow_mixed(rng, 20_000)
    tr = ev[:500].copy()
    tr["type"], tr["value"] = ge.EV_TRACE, 5_000_000
    tr["flow_key"] = np.arange(10**9, 10**9 + 500, dtype=np.uint64)
    run.batch(np.concatenate([ev, tr]), what="trace")
    assert not set(run.eng.topk_flow_slow(K)["flow_key"].tolist()) & set(tr["flow_key"].tolist())


@pytest.mark.parametrize("t_ms", [1, 300, 15000])
def test_samples_at_and_above_the_threshold(t_ms):
    """a flow with samples at T only is never listed, one with a sample at T + 1 is; samples beyond the validity rule never count"""
    run = Run(above_ms=t_ms, cms_log2_width=16)
    at = np.arange(1, 201, dtype=np.uint64)
    above = np.arange(1001, 1051, dtype=np.uint64)
    invalid = np.arange(5001, 5021, dtype=np.uint64)
    ev = np.concatenate([_resp(np.repeat(at, 3), t_ms), _resp(above, t_ms + 1), _resp(invalid, 0)])
    ev["value"][-len(invalid):] = fq.VALID_USEC + 5
    run.batch(ev, what=t_ms)
    got = set(run.eng.topk_flow_slow(K)["flow_key"].tolist())
    assert got == set(above.tolist()), t_ms
    run.flush(5)


@pytest.mark.parametrize("nflows", [K - 1, K, K + 1, 3 * K])
def test_set_sizes_and_ties(nflows):
    rng = np.random.default_rng(nflows)
    run = Run(cms_log2_width=20)
    keys = rng.choice(1 << 40, nflows, replace=False).astype(np.uint64)
    nslow = np.where(np.arange(nflows) % 3 == 0, 4, rng.integers(0, 3, nflows))      # a long run of score 4, many 0, 1 and 2
    ev = np.concatenate([_resp(np.repeat(keys, nslow), 500), _resp(keys, 10)])
    run.batch(ev, what=nflows)
    got = run.eng.topk_flow_slow(K)
    assert len(got) == min(K, int((nslow > 0).sum()))
    run.batch(_resp(keys[: nflows // 2], 2000), what=nflows)
    run.flush(5)


def test_fast_only_flows_never_listed():
    """heavy fast clients fill the query set; the slow set holds only the few slow clients"""
    rng = np.random.default_rng(5)
    run = Run(cms_log2_width=16)
    fast = rng.choice(1 << 40, 3000, replace=False).astype(np.uint64)
    slow = rng.choice(1 << 40, 20, replace=False).astype(np.uint64) | np.uint64(1 << 41)
    ev = np.concatenate([_resp(np.repeat(fast, 14), rng.integers(0, 300, 14 * len(fast))), _resp(np.repeat(slow, 4), 350)])
    run.batch(ev, what="fast")
    got = set(run.eng.topk_flow_slow(K)["flow_key"].tolist())
    assert got == set(slow.tolist())
    q = run.eng.topk_flow_queries(K)["flow_key"]
    assert set(q[:100].tolist()) <= set(fast.tolist()) and not set(q[:100].tolist()) & got


def test_direct_path():
    """more than 2^21 distinct flows in one batch: most slow samples take the direct path of the response flow table"""
    rng = np.random.default_rng(6)
    n = (1 << 21) + 300_000
    run = Run(max_batch=1 << 22, cms_log2_width=20)
    keys = rng.integers(1, 1 << 62, n, dtype=np.uint64)
    run.batch(_resp(keys, np.where(rng.random(n) < 0.01, 700, 20)), what="direct")
    assert run.eng.last_batch_flow_resp_direct() > 0


@pytest.mark.parametrize("depth,log2w", [(1, 12), (8, 12), (4, 4), (4, 22)])
def test_sketch_edges(depth, log2w):
    rng = np.random.default_rng(depth * 100 + log2w)
    run = Run(cms_depth=depth, cms_log2_width=log2w)
    for i, step in enumerate(["b", "b", 5, "b"]):
        if step == "b":
            run.batch(_slow_mixed(rng, 40_000), what=(depth, log2w, i))
        else:
            run.flush(step)


def test_eviction_and_growth():
    rng = np.random.default_rng(19)
    run = Run(max_svcs=256, idle_evict_secs=20)
    for i, t in enumerate([5, 10, 100, 105, 140]):
        run.batch(_slow_mixed(rng, 20_000, nsvc=200 if i < 2 else 60), what=("evict", i))
        if i == 2:
            run.eng.grow(512, 128)
            run.batch(_slow_mixed(rng, 20_000, nsvc=60), what=("grown", i))
        run.flush(t, what=("evict", i))
    assert run.eng.stats()["svcs_evicted"] > 0


@pytest.mark.parametrize("t_ms", fs.THR.tolist())
def test_every_threshold(t_ms):
    rng = np.random.default_rng(t_ms)
    run = Run(above_ms=t_ms)
    ev = _mixed(rng, 30_000)
    r = np.flatnonzero((ev["type"] == ge.EV_RESP) & (ev["value"] < fq.VALID_USEC))
    ev["value"][r] = rng.choice([t_ms, t_ms + 1, 0, 20000], len(r)).astype(np.uint32) * np.uint32(1000) + np.uint32(999)
    run.batch(ev, what=t_ms)
    run.flush(5)


def test_threshold_call_and_refusals():
    eng = ge.Engine(flow_topk_slow=True, **CFG, **FLAGS)
    for bad in (0, 2, 299, 301, 15001):
        with pytest.raises(ge.GyskError) as ex:
            eng.set_flow_slow(bad)
        assert ex.value.code == INVAL, bad
    eng.set_flow_slow(450)
    eng.set_flow_slow(300)                         # the default again; both before any event
    eng.ingest_events(_resp(np.arange(1, 4, dtype=np.uint64), 400)); eng.sync()
    with pytest.raises(ge.GyskError) as ex:
        eng.set_flow_slow(1000)
    assert ex.value.code == INVAL
    assert set(eng.topk_flow_slow(K)["flow_key"].tolist()) == {1, 2, 3}           # still 300: 400 ms is slow
    flushed = ge.Engine(flow_topk_slow=True, **CFG, **FLAGS)
    flushed.flush(5)
    with pytest.raises(ge.GyskError) as ex:
        flushed.set_flow_slow(1000)
    assert ex.value.code == INVAL
    without = ge.Engine(**CFG, **FLAGS)
    with pytest.raises(ge.GyskError) as ex:
        without.set_flow_slow(300)
    assert ex.value.code == NOTSUP
    for call in (lambda e: e.topk_flow_slow(), lambda e: e.topk_flow_slow_global(), lambda e: e.topk_flow_slow_5min(),
                 lambda e: e.topk_flow_slow_global_5min()):
        with pytest.raises(ge.GyskError) as ex:
            call(without)
        assert ex.value.code == NOTSUP
    for kw in (dict(flow_queries=True, flow_resp_hist=True), dict(flow_topk=True, flow_queries=True)):
        with pytest.raises(ge.GyskError) as ex:
            ge.Engine(flow_topk_slow=True, **CFG, **kw)
        assert ex.value.code == INVAL
    nolevel = ge.Engine(flow_topk_slow=True, **CFG, **FLAGS)
    with pytest.raises(ge.GyskError) as ex:
        nolevel.topk_flow_slow_5min()
    assert ex.value.code == NOTSUP
    with pytest.raises(ge.GyskError) as ex:
        nolevel.topk_flow_slow_global()
    assert ex.value.code == INVAL                  # before the first merge finish


@pytest.mark.parametrize("seq", sorted(fl.SEQUENCES))
def test_level_flush_sequences(seq):
    rng = np.random.default_rng(len(seq) + 40)
    run = Run(level=True, flow_level=True)
    for i, t in enumerate(fl.SEQUENCES[seq]):
        run.batch(_slow_mixed(rng, 20_000, nclients=3000), what=(seq, i))
        run.flush(t, what=(seq, i))


OTHER = {"alone": {}, "levels": dict(flow_level=True, **LEVEL),
         "merge": dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, merge_traces=True, max_trace_svcs=64,
                       flow_level=True, **LEVEL)}


@pytest.mark.parametrize("other", sorted(OTHER))
def test_flag_off_and_on_answer_alike(other):
    import torch
    rng = np.random.default_rng(27)
    flags = {**CFG, **FLAGS, **OTHER[other]}
    off, on = ge.Engine(**flags), ge.Engine(flow_topk_slow=True, **flags)
    level = "flow_topk_5min" in flags
    ev0 = _mixed(np.random.default_rng(0), 20_000)
    sids = np.unique(ev0["svc_id"][ev0["type"] != ge.EV_TASK])
    for e in (off, on):
        e.set_logical_map(sids, sids % np.uint64(7) + np.uint64(50))
    lids = np.unique(sids % np.uint64(7) + np.uint64(50))
    for i, t in enumerate((5, 10, 40, 40, 300)):
        ev = _slow_mixed(rng, 40_000)
        for e in (off, on):
            e.ingest_events(ev); e.sync()
        keys = np.unique(ev["flow_key"])[:2000]
        for lw in (False, True):
            for ex in (lambda e: e.export_cms(lw), lambda e: e.export_cms_queries(lw), lambda e: e.export_cms_resp(lw),
                       lambda e: e.topk_flows(K, lw), lambda e: e.topk_flow_queries(K, lw), lambda e: e.query_flow_resp(keys, lw)):
                assert ex(off).tobytes() == ex(on).tobytes()
        if level:
            for call in (lambda e: e.topk_flows_5min(K), lambda e: e.topk_flow_queries_5min(K)):
                a, b = call(off), call(on)
                assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1]
            assert off.export_cms_resp_5min().tobytes() == on.export_cms_resp_5min().tobytes()
        assert _rowbytes(off.query_svcs(sids)) == _rowbytes(on.query_svcs(sids))
        sa, sb = off.stats(), on.stats()
        sa.pop("kernel_launches"); sb.pop("kernel_launches")
        assert sa == sb
        assert off.last_batch_flow_resp_direct() == on.last_batch_flow_resp_direct()
        for e in (off, on):
            e.flush(t)
        for e in (off, on):
            _emulate_collectives(torch, [e])
        ra, rb = _regions(off, torch), _regions(on, torch)
        assert {k: (v[0], v[1].tobytes()) for k, v in ra.items()} == {k: (v[0], v[1].tobytes()) for k, v in rb.items()}
        # the slab only grows, by the slow sets in whole entries after everything else
        pa, na = off.merge_tdigest_slab()
        pb, nb = on.merge_tdigest_slab()
        sa_, sb_ = _dev_bytes(torch, pa, na).tobytes(), _dev_bytes(torch, pb, nb).tobytes()
        assert nb - na == _slab_bytes(2 if level else 1)
        assert sa_[: len(lids) * SLAB_ENTRY] == sb_[: len(lids) * SLAB_ENTRY]
        tk = _slab_bytes(2) * (2 if level else 1)          # the window sets, and with the level the level sets, before the slow ones
        assert sa_[na - tk:] == sb_[na - tk: na]
        new = np.frombuffer(sb_[na:], dtype=np.uint64)
        rows = on.topk_flow_slow(K, True)
        assert new[0] >= len(rows) and new[2: 2 + len(rows)].tolist() == rows["flow_key"].tolist()
        if level:
            rows5, bound = on.topk_flow_slow_5min(K)
            l5 = new[K + 2:]
            assert l5[1] == bound and l5[2: 2 + len(rows5)].tolist() == rows5["flow_key"].tolist()
        assert _rowbytes(off.query_logical(lids)) == _rowbytes(on.query_logical(lids))
        assert off.topk_flows_global().tobytes() == on.topk_flows_global().tobytes()
        assert off.topk_flow_queries_global().tobytes() == on.topk_flow_queries_global().tobytes()
        for lw in (False, True):
            assert off.query_flow_resp_global(keys, lw).tobytes() == on.query_flow_resp_global(keys, lw).tobytes()
        if level:
            for call in (lambda e: e.topk_flows_global_5min(K), lambda e: e.topk_flow_queries_global_5min(K)):
                a, b = call(off), call(on)
                assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1]
            assert off.merge_flush_range() == on.merge_flush_range()
    with pytest.raises(ge.GyskError) as ex:
        off.topk_flow_slow()
    assert ex.value.code == NOTSUP


def _check_merge(ranks, level, what):
    engines = [r.eng for r in ranks]
    d, w, bs = ranks[0].d, ranks[0].w, ranks[0].bs
    summed = sum((e.export_cms_resp(True).reshape(-1) for e in engines[1:]), engines[0].export_cms_resp(True).reshape(-1).copy())
    # the last sets as the ranks hold them: every slow flow of a rank's window when it has at most K
    g = fs.merged([r.sets.last for r in ranks], summed, d, w, bs)
    want = fs.read(g, summed, d, w, bs)
    for e in engines:
        got = e.topk_flow_slow_global()
        assert got.tobytes() == want.tobytes(), what
        assert got.tobytes() == e.query_flow_resp_global(got["flow_key"], True).tobytes(), what
    if level:
        summed5 = sum((e.export_cms_resp_5min().reshape(-1) for e in engines[1:]), engines[0].export_cms_resp_5min().reshape(-1).copy())
        g5, bg = fs.merged([r.lv.L for r in ranks], summed5, d, w, bs, bounds=[r.lv.B for r in ranks])
        want5 = fs.read(g5, summed5, d, w, bs)
        for e in engines:
            rows, bound = e.topk_flow_slow_global_5min()
            assert rows.tobytes() == want5.tobytes() and bound == bg, what
            assert rows.tobytes() == e.query_flow_resp_global_5min(rows["flow_key"]).tobytes(), what


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("others", ["alone", "merge"])
def test_merge_ranks_the_union(world, others):
    import torch
    rng = np.random.default_rng(world * 10 + 7)
    extra = {k: v for k, v in OTHER["merge"].items() if k not in LEVEL} if others == "merge" else {}
    level = others == "merge"
    ranks = [Run(level=level, rank=r, world=world, **extra) for r in range(world)]
    for step, t in enumerate([30, 35, 60]):
        ev = _slow_mixed(rng, 60_000, nclients=3000)
        for run, sh in zip(ranks, _shard(ev, world)):
            run.batch(sh, what=(world, others, step))
            run.flush(t, what=(world, others, step))
        _emulate_collectives(torch, [r.eng for r in ranks])
        _check_merge(ranks, level, (world, others, step))


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(5)
    run = Run(level=True, flow_level=True)
    for t in (30, 35):
        run.batch(_slow_mixed(rng, 30_000))
        run.flush(t)
    _emulate_collectives(torch, [run.eng])
    emulated = run.eng.topk_flow_slow_global().tobytes(), run.eng.topk_flow_slow_global_5min()
    assert emulated[0] == run.eng.topk_flow_slow(K, True).tobytes()
    run.eng.nccl_comm_init(run.eng.nccl_unique_id(), 1, 0)
    run.eng.merge_global()
    run.eng.sync()
    got = run.eng.topk_flow_slow_global().tobytes(), run.eng.topk_flow_slow_global_5min()
    assert got[0] == emulated[0] and got[1][0].tobytes() == emulated[1][0].tobytes() and got[1][1] == emulated[1][1]
