"""The flow response histograms on the device (GYSK_FLAG_FLOW_RESP_HIST). After every batch and flush the open and last
gysk_export_cms_resp tables must be byte-equal to the tables restated from the samples (tests/flow_resp_hist.py); every cell's 15 counts
sum to the query half of the same gysk_export_cms_queries cell; without eviction every row's bucket sums equal the services' response
histograms of the same window (GYSK_HIST_RESP_CUR / _LAST / _5MIN); gysk_query_flow_resp equals the min-over-rows restatement, never
falls below the exact per-key counts, and a key alone in its columns gets its exact counts and the reference's percentiles of its own
samples. With GYSK_FLAG_FLOW_QUERY_LEVEL the 300-s level must equal the held windows' tables and the rolled restatement after every flush of
the scripts of tests/flow_level.py. Covered: every response route, the bucket edges, the direct path, service-table churn, the sketch
edges, the flag off against on, and the merge at world 1 ... 8 with the collectives emulated on one GPU, and once through NCCL."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge, synth
from oracle import pyoracle as po
from tests import flow_queries as fq
from tests import flow_resp_hist as fr
from tests.flow_level import SEQUENCES, FlowLevelRing, held_windows, level_of_history
from tests.test_gpu_flow_level import _rowbytes
from tests.test_gpu_flow_queries import _mixed
from tests.test_gpu_flow_query_level import _regions, _route_batch
from tests.test_gpu_merge import _emulate_collectives

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
U32 = fq.U32
CFG = dict(max_svcs=1024, max_tasks=64, max_batch=1 << 17, cms_depth=4, cms_log2_width=12)
EMPTY = np.zeros(0, dtype=ge.EVENT_DTYPE)
RESP_NAMES = ["cms_resp_cur", "cms_resp_last", "cms_resp_5min"]


def _service_buckets(eng, which):
    """per bucket the sum over every service of its response histogram `which`, mod 2^32"""
    rows, _ = eng.query_window()
    tot = np.zeros(15, dtype=np.int64)
    for r in rows:
        h = eng.export_hist(int(r.glob_id), which)
        if h is not None:
            tot += h[0]["count"][:15].astype(np.int64)
    return tot & U32


def _ref_percentiles(samples):
    """the reference's get_percentiles (p25, p95, p99) of a key's own samples (msec), else the library's rule on their buckets"""
    ms = (samples["value"] // np.uint32(1000)).astype(np.int64)
    R = po.ref()
    if R is not None:
        return tuple(po.hist_run(R, "gyref_hist_run", 0, 0, ms, np.array([25, 95, 99], dtype=np.float32))["pct"].tolist())
    return fr.percentiles(np.bincount(fr.buckets(samples["value"]), minlength=15))


class Run:
    """one engine with the flag (and with level, GYSK_FLAG_FLOW_QUERY_LEVEL), the restated open table, the closed windows' history and,
    with the level, the ring fed the restated tables"""

    def __init__(self, restate=True, level=False, services=True, **kw):
        self.eng = ge.Engine(flow_queries=True, flow_resp_hist=True, flow_query_level=level, **kw)
        c = self.eng.cfg
        self.d, self.w, self.level, self.services = c.cms_depth, c.cms_log2_width, level, services
        self.cur = fr.empty(self.d, self.w) if restate else None
        self.ring = FlowLevelRing((self.d << self.w) * fr.WORDS) if restate and level else None
        self.tsecs, self.tables, self.windows, self.samples = [], [], [], []

    def batch(self, ev, known=None, ingest=None, what=None):
        (ingest or (lambda e: e.ingest_events(ev)))(self.eng)
        self.eng.sync()
        s = fq.counted(ev, known)
        if self.cur is not None:
            fr.add_samples(self.cur, s, self.d, self.w)
        self.samples.append(s)
        got = self.eng.export_cms_resp().reshape(-1)
        if self.cur is not None:
            assert got.tobytes() == self.cur.tobytes(), what
        self.tie(got, self.eng.export_cms_queries(), ge.HIST_RESP_CUR, what)
        self.points(got, np.concatenate(self.samples), self.eng.query_flow_resp, what)

    def flush(self, t, what=None):
        self.eng.flush(t)
        closed = self.eng.export_cms_resp(last_window=True).reshape(-1)
        if self.cur is not None:
            assert closed.tobytes() == self.cur.tobytes(), what
            if self.ring:
                self.ring.flush(t, self.cur)
            self.cur = fr.empty(self.d, self.w)
        assert not self.eng.export_cms_resp().any(), what
        self.tsecs.append(t)
        self.tables.append(closed if self.level else None)
        self.windows.append(np.concatenate(self.samples) if self.samples else EMPTY)
        self.samples = []
        self.tie(closed, self.eng.export_cms_queries(last_window=True), ge.HIST_RESP_LAST, what)
        self.points(closed, self.windows[-1], lambda k: self.eng.query_flow_resp(k, last_window=True), what)
        if self.level:
            self.check_level(what)

    def held(self):
        return np.concatenate([self.windows[j] for j in held_windows(self.tsecs)]) if self.tsecs else EMPTY

    def check_level(self, what):
        got = self.eng.export_cms_resp_5min().reshape(-1)
        want = level_of_history(self.tsecs, self.tables) if self.tsecs else np.zeros_like(got)
        assert got.tobytes() == want.tobytes(), what
        if self.ring:
            assert got.tobytes() == self.ring.level.tobytes(), what
        self.tie(got, self.eng.export_cms_queries_5min(), ge.HIST_RESP_5MIN, what)
        self.points(got, self.held(), self.eng.query_flow_resp_5min, what)

    def tie(self, table, qtable, which, what):
        assert np.array_equal(fr.cell_totals(table), qtable & np.uint64(U32)), what
        sums = fr.bucket_sums(table, self.d, self.w)
        assert not sums[:, 15].any(), what
        if self.services:
            svc = _service_buckets(self.eng, which)
            for row in range(self.d):
                assert np.array_equal(sums[row, :15], svc), (what, row, which)

    def points(self, table, samples, query, what):
        keys = np.unique(samples["flow_key"])
        if not len(keys):
            return
        q = keys[:2000]
        got = query(q)
        assert got.tobytes() == fr.point_query(table, q, self.d, self.w).tobytes(), what
        ex = fr.exact(samples, q)
        assert (got["counts"].astype(np.int64) >= ex).all(), what
        # a key alone in its column of every row: its exact counts and its own samples' percentiles
        cols = fq.columns(keys, self.d, self.w)
        alone = np.ones(len(keys), dtype=bool)
        for r in range(self.d):
            _, inv, cnt = np.unique(cols[r], return_inverse=True, return_counts=True)
            alone &= cnt[inv.reshape(-1)] == 1
        idx = np.flatnonzero(alone[: len(q)])[:20]
        for i in idx.tolist():
            assert np.array_equal(got["counts"][i], ex[i]), what
            own = samples[samples["flow_key"] == q[i]]
            assert (int(got["p25_ms"][i]), int(got["p95_ms"][i]), int(got["p99_ms"][i])) == _ref_percentiles(own), what


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_level_after_every_flush(name):
    tsecs = SEQUENCES[name]
    rng = np.random.default_rng(500 + len(tsecs))
    run = Run(level=True, **CFG)
    assert not run.eng.export_cms_resp_5min().any()                 # empty before the first flush
    for i, t in enumerate(tsecs):
        run.batch(_mixed(rng, int(rng.integers(1000, 8000)), nsvc=40, nclients=3000), what=(name, i))
        run.flush(t, what=(name, i, t))
    run.batch(_mixed(rng, 5000, nsvc=40, nclients=3000), what=(name, "open"))     # the open window stays out of the level
    run.check_level((name, "open"))


@pytest.mark.parametrize("route", ["event32", "event32_hot", "resp16", "ipv4", "ipv6", "api_tran", "api_tran_traced"])
def test_every_response_route(route, monkeypatch):
    if route == "event32_hot":
        monkeypatch.setenv("GYSK_HOT_MIN", "64")                    # busy services turn hot after their first batch
    elif route == "event32":
        monkeypatch.setenv("GYSK_HOT_ROWS", "0")
    rng = np.random.default_rng(sum(map(ord, route)) + 1)
    run = Run(level=True, max_trace_svcs=64 if route == "api_tran_traced" else 0, **CFG)
    for i, t in enumerate(SEQUENCES["gaps"][:6]):
        for _ in range(2):
            ev, ingest = _route_batch(rng, route)
            run.batch(ev, ingest=ingest, what=(route, i))
        run.flush(t, what=(route, i, t))
    if route.startswith("event32"):
        assert (run.eng.hot_rows_in_use() > 0) == (route == "event32_hot")
    assert run.eng.stats()["events_resp"] > 0


def test_bucket_edges():
    """samples at 0, 1, 1000, 15000 and 15001 ms, at the validity bound and beyond it, each on a key of its own"""
    run = Run(**CFG)
    usec = np.array([0, 999, 1000, 1999, 1_000_000, 15_000_999, 15_001_000, fq.VALID_USEC - 1, fq.VALID_USEC, 0xFFFFFFFF], dtype=np.uint32)
    ev = np.zeros(len(usec) * 7, dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["type"] = 4242, ge.EV_RESP
    ev["value"] = np.repeat(usec, 7)
    keys = np.arange(1, len(usec) + 1, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    ev["flow_key"] = np.repeat(keys, 7)
    run.batch(ev, what="edges")
    got = run.eng.query_flow_resp(keys)
    want_b = [1, 1, 1, 1, 11, 13, 14, 14, None, None]
    for i, b in enumerate(want_b):
        c = np.zeros(15, dtype=np.uint32)
        if b is not None:
            c[b] = 7
        assert np.array_equal(got["counts"][i], c), (i, got["counts"][i])
    run.flush(5, what="edges")


def test_direct_path():
    """more distinct (flow, bucket) pairs in one batch than the response flow table holds"""
    rng = np.random.default_rng(13)
    run = Run(max_svcs=1024, max_tasks=64, max_batch=1 << 22, stage_batch=1 << 22, cms_depth=4, cms_log2_width=16)
    n = 2_500_000
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = rng.integers(1, 200, n).astype(np.uint64) * np.uint64(7919)
    ev["flow_key"] = synth.splitmix64(np.arange(1, n + 1, dtype=np.uint64))
    ev["value"], ev["type"] = rng.integers(0, 1 << 25, n), ge.EV_RESP
    run.batch(ev, what="direct")
    assert run.eng.last_batch_flow_resp_direct() > 0
    assert run.eng.flow_table_used() == 0
    run.flush(5, what="direct")
    run.batch(_mixed(rng, 50_000), what="then the table")
    assert run.eng.last_batch_flow_resp_direct() == 0
    run.flush(10, what="then the table")


def test_service_table_churn():
    """eviction, recycled slots and a gysk_grow inside a window leave the tables alone"""
    rng = np.random.default_rng(14)
    run = Run(level=True, services=False, **dict(CFG, max_svcs=256, idle_evict_secs=10))

    def ev_of(lo, hi, n=20_000):
        ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = rng.integers(lo, hi, n).astype(np.uint64) * np.uint64(6151)
        ev["flow_key"], ev["value"], ev["type"] = rng.integers(1, 3000, n), rng.integers(0, 1 << 25, n), ge.EV_RESP
        return ev
    run.batch(ev_of(1, 150), what="first")
    for t in (5, 10, 20, 35, 60):
        run.flush(t, what=("idle", t))
    run.batch(ev_of(200, 380), what="recycled")                      # the first services were evicted: their slots taken by new ids
    assert run.eng.stats()["svcs_evicted"] > 0
    run.eng.grow(max_svcs=1024)                                        # inside the window
    run.batch(ev_of(400, 900), what="grown")
    run.flush(65, what="grow")
    run.batch(ev_of(400, 900), what="after grow")
    run.flush(70, what="after grow")
    assert run.eng.stats()["events_dropped"] == 0


# beyond 2^22 the batch key's column fields take the width's full 28 bits (24, 23): a wrong column would break the tie to the query table
@pytest.mark.parametrize("depth,log2w,level", [(1, 4, False), (8, 4, False), (1, 22, False), (8, 22, False), (8, 20, True), (1, 22, True),
                                               (1, 24, False), (1, 23, True)])
def test_sketch_edges(depth, log2w, level):
    rng = np.random.default_rng(depth * 100 + log2w + level)
    wide = log2w >= 20
    run = Run(restate=not wide, level=level, **dict(CFG, cms_depth=depth, cms_log2_width=log2w))
    for i, t in enumerate([5, 35, 40] if wide else [5, 35, 40, 299, 400]):
        run.batch(_mixed(rng, 20_000, nsvc=40, nclients=3000), what=(depth, log2w, i))
        run.flush(t, what=(depth, log2w, i))
    words = (depth << log2w) * fr.WORDS * 8
    assert run.eng.capacity()["device_bytes"] >= (13 if level else 2) * words


def _same_merge_arrays(off, on, torch):
    """on's merge arrays are off's with the response tables inserted after the last count-min table of the SUM region"""
    a, b = _regions(off, torch), _regions(on, torch)
    assert set(a) == set(b)
    cells = off.cfg.cms_depth << off.cfg.cms_log2_width
    for region, (names, buf) in a.items():
        names2, buf2 = b[region]
        if region != "sum_u64":
            assert names2 == names and buf2.tobytes() == buf.tobytes(), region
            continue
        k = max(i for i, n in enumerate(names) if n.startswith("cms_")) + 1
        extra = [n for n in RESP_NAMES if n in names2]
        assert len(extra) in (2, 3) and names2 == names[:k] + extra + names[k:]
        p = k * ((cells * 8 + 255) & ~255)
        ins = len(extra) * ((cells * 64 + 255) & ~255)
        assert buf2[:p].tobytes() == buf[:p].tobytes() and buf2[p + ins:].tobytes() == buf[p:].tobytes()


OTHER = {"alone": {}, "flow_level": dict(flow_level=True), "query_level": dict(flow_query_level=True),
         "merge": dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, merge_traces=True, max_trace_svcs=64)}


@pytest.mark.parametrize("other", sorted(OTHER))
def test_flag_off_and_on_answer_alike(other):
    import torch
    rng = np.random.default_rng(17)
    flags = OTHER[other]
    off, on = ge.Engine(flow_queries=True, **CFG, **flags), ge.Engine(flow_queries=True, flow_resp_hist=True, **CFG, **flags)
    cells = CFG["cms_depth"] << CFG["cms_log2_width"]
    ntab = 13 if flags.get("flow_query_level") else 2
    assert on.capacity()["device_bytes"] - off.capacity()["device_bytes"] == ntab * cells * 64 + (2 * CFG["max_batch"]) * 16
    ev0 = _mixed(np.random.default_rng(0), 20_000)
    sids = np.unique(ev0["svc_id"][ev0["type"] != ge.EV_TASK])
    for e in (off, on):
        e.set_logical_map(sids, sids % np.uint64(7) + np.uint64(50))
    lids = np.unique(sids % np.uint64(7) + np.uint64(50))
    for i, t in enumerate((5, 10, 40, 40, 400)):
        ev = _mixed(rng, 40_000)
        for e in (off, on):
            e.ingest_events(ev); e.sync()
        keys = np.unique(ev["flow_key"])[:2000]
        for lw in (False, True):
            assert off.export_cms(lw).tobytes() == on.export_cms(lw).tobytes()
            assert off.query_flows(keys, lw).tobytes() == on.query_flows(keys, lw).tobytes()
            assert off.export_cms_queries(lw).tobytes() == on.export_cms_queries(lw).tobytes()
            assert off.query_flow_queries(keys, lw).tobytes() == on.query_flow_queries(keys, lw).tobytes()
        if flags.get("flow_level"):
            assert off.export_cms_5min().tobytes() == on.export_cms_5min().tobytes()
        if flags.get("flow_query_level"):
            assert off.export_cms_queries_5min().tobytes() == on.export_cms_queries_5min().tobytes()
        assert _rowbytes(off.query_svcs(sids)) == _rowbytes(on.query_svcs(sids))
        for sid in sids[:40].tolist():
            for which in (ge.HIST_RESP_LAST, ge.HIST_RESP_5MIN):
                a, b = off.export_hist(sid, which), on.export_hist(sid, which)
                assert (a is None) == (b is None) and (a is None or (np.array_equal(a[0], b[0]) and a[1:] == b[1:]))
        sa, sb = off.stats(), on.stats()
        # one roll more per flush with the level
        assert sb.pop("kernel_launches") - sa.pop("kernel_launches") == (i if flags.get("flow_query_level") else 0)
        assert sa == sb
        assert off.last_batch_flow_query_direct() == on.last_batch_flow_query_direct() and on.last_batch_flow_resp_direct() == 0
        for e in (off, on):
            e.flush(t)
        for e in (off, on):
            _emulate_collectives(torch, [e])
        _same_merge_arrays(off, on, torch)
        assert _rowbytes(off.query_logical(lids)) == _rowbytes(on.query_logical(lids))
        for lw in (False, True):
            assert off.query_flows_global(keys, lw).tobytes() == on.query_flows_global(keys, lw).tobytes()
            assert off.query_flow_queries_global(keys, lw).tobytes() == on.query_flow_queries_global(keys, lw).tobytes()
    calls = [lambda e: e.query_flow_resp(keys), lambda e: e.export_cms_resp(), lambda e: e.query_flow_resp_global(keys),
             lambda e: e.query_flow_resp_5min(keys), lambda e: e.export_cms_resp_5min(), lambda e: e.query_flow_resp_global_5min(keys),
             lambda e: e.last_batch_flow_resp_direct()]
    for k, call in enumerate(calls):
        with pytest.raises(ge.GyskError) as ex:
            call(off)
        assert ex.value.code == NOTSUP
        if 3 <= k <= 5 and not flags.get("flow_query_level"):       # the level calls need GYSK_FLAG_FLOW_QUERY_LEVEL too
            with pytest.raises(ge.GyskError) as ex:
                call(on)
            assert ex.value.code == NOTSUP
    fresh = ge.Engine(flow_queries=True, flow_resp_hist=True, flow_query_level=True, **CFG)
    for call in (lambda: fresh.query_flow_resp_global(keys), lambda: fresh.query_flow_resp_global_5min(keys)):
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == INVAL
    with pytest.raises(ge.GyskError) as ex:
        ge.Engine(flow_resp_hist=True, **CFG, **flags)
    assert ex.value.code == INVAL


def _resp_slices(eng, torch):
    """{name: the merged table's words} of the response tables in the SUM region"""
    names, buf = _regions(eng, torch)["sum_u64"]
    cells = eng.cfg.cms_depth << eng.cfg.cms_log2_width
    out, off = {}, 0
    for n in names:
        if not n.startswith("cms_"):
            break
        nbytes = cells * (64 if n in RESP_NAMES else 8)
        if n in RESP_NAMES:
            out[n] = buf[off: off + nbytes].view(np.uint64)
        off += (nbytes + 255) & ~255
    return out


def _shard(ev, world):
    return [ev[ev["host_idx"] % world == r] for r in range(world)]


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_merge_sums_the_ranks(world):
    import torch
    rng = np.random.default_rng(world * 10 + 7)
    d, w = CFG["cms_depth"], CFG["cms_log2_width"]
    engines = [ge.Engine(flow_queries=True, flow_resp_hist=True, flow_query_level=True, rank=r, world=world, **CFG) for r in range(world)]
    for e in engines:
        e.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    for step, t in enumerate([30, 35, 60, 95, 300]):
        ev = _mixed(rng, 30_000)
        for e, sh in zip(engines, _shard(ev, world)):
            e.ingest_events(sh); e.sync()
            if step % 2 == 0:
                e.flush(t)
        _emulate_collectives(torch, engines)
        keys = np.unique(ev["flow_key"])[:500]
        tables = {"cms_resp_cur": [e.export_cms_resp().reshape(-1) for e in engines],
                  "cms_resp_last": [e.export_cms_resp(last_window=True).reshape(-1) for e in engines],
                  "cms_resp_5min": [e.export_cms_resp_5min().reshape(-1) for e in engines]}
        want = {k: sum(v[1:], v[0].copy()) for k, v in tables.items()}
        for e in engines:
            got = _resp_slices(e, torch)
            for k in RESP_NAMES:
                assert got[k].tobytes() == want[k].tobytes(), (world, step, k)
            for lw, k in ((False, "cms_resp_cur"), (True, "cms_resp_last")):
                assert e.query_flow_resp_global(keys, lw).tobytes() == fr.point_query(want[k], keys, d, w).tobytes(), (world, step, k)
            assert e.query_flow_resp_global_5min(keys).tobytes() == fr.point_query(want["cms_resp_5min"], keys, d, w).tobytes()


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(5)
    eng = ge.Engine(flow_queries=True, flow_resp_hist=True, flow_query_level=True, **CFG)
    eng.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    for t in (30, 35, 65):
        eng.ingest_events(_mixed(rng, 30_000)); eng.sync()
        eng.flush(t)
    eng.ingest_events(_mixed(rng, 30_000)); eng.sync()
    keys = rng.integers(1, 5000, 300).astype(np.uint64)
    _emulate_collectives(torch, [eng])
    emulated = [eng.query_flow_resp_global(keys, lw).tobytes() for lw in (False, True)] + [eng.query_flow_resp_global_5min(keys).tobytes()]
    slices = {k: v.tobytes() for k, v in _resp_slices(eng, torch).items()}
    eng.nccl_comm_init(eng.nccl_unique_id(), 1, 0)
    eng.merge_global()
    eng.sync()
    assert [eng.query_flow_resp_global(keys, lw).tobytes() for lw in (False, True)] + [eng.query_flow_resp_global_5min(keys).tobytes()] == emulated
    assert emulated == [eng.query_flow_resp(keys, lw).tobytes() for lw in (False, True)] + [eng.query_flow_resp_5min(keys).tobytes()]
    assert {k: v.tobytes() for k, v in _resp_slices(eng, torch).items()} == slices
    assert slices["cms_resp_5min"] == eng.export_cms_resp_5min().tobytes()
