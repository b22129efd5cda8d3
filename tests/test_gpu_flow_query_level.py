"""The rolling 300-s flow query level on the device (GYSK_FLAG_FLOW_QUERY_LEVEL). After every flush of the scripted sequences of
tests/flow_level.py, gysk_export_cms_queries_5min must be byte-equal to the sum of the held windows' gysk_export_cms_queries(last_window=1)
tables and to the flow query tables restated from the samples (tests/flow_queries.py) and rolled by FlowLevelRing, and
gysk_query_flow_queries_5min must equal the min-over-rows restatement and be at least the exact per-key counts. Without eviction, every
row's halves also sum to the services' 300-s response level: the nqrys_5min and the GYSK_HIST_RESP_5MIN bucket sums. Covered: every
response route, excluded samples, the sketch edges with a wrapping msec half, eviction, growth and the direct path, the flag off against
on over the same stream, and the merge at world 1 ... 8 with the collectives emulated on one GPU, and once through the library's NCCL
path."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge, synth
from gyeeta_b200.wire import RESP4, RESP6
from tests import flow_queries as fq
from tests.flow_level import SEQUENCES, FlowLevelRing, held_windows, level_of_history
from tests.test_gpu_flow_level import _rowbytes
from tests.test_gpu_flow_queries import _expanded, _mixed, _raw_resp
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import _dev_bytes
from tests.test_gpu_sketch_accuracy import fold_ip6, raw_svc_id
from tests.trace_agg import api_tran, resp_events, trace_events

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
U32 = fq.U32
CFG = dict(max_svcs=1024, max_tasks=64, max_batch=1 << 17, cms_depth=4, cms_log2_width=12)
EMPTY = np.zeros(0, dtype=ge.EVENT_DTYPE)


class Run:
    """one engine with the flag, the history of its closed windows (tsec, device table, counted samples) and, with restate, the open
    table restated from the samples and the ring fed those restated tables"""

    def __init__(self, restate=True, **kw):
        self.eng = ge.Engine(flow_queries=True, flow_query_level=True, **kw)
        c = self.eng.cfg
        self.d, self.w = c.cms_depth, c.cms_log2_width
        self.cur = np.zeros(self.d << self.w, dtype=np.uint64) if restate else None
        self.ring = FlowLevelRing(self.d << self.w) if restate else None
        self.tsecs, self.tables, self.windows, self.samples = [], [], [], []

    def batch(self, ev, known=None, ingest=None):
        """ev: the batch as the library expands it; known: the ids that have a slot (None: every id)"""
        (ingest or (lambda e: e.ingest_events(ev)))(self.eng)
        self.eng.sync()
        s = fq.counted(ev, known)
        if self.cur is not None:
            fq.add_samples(self.cur, s, self.d, self.w)
        self.samples.append(s)

    def flush(self, t, what=None, responses=False):
        self.eng.flush(t)
        closed = self.eng.export_cms_queries(last_window=True)
        if self.cur is not None:
            assert closed.tobytes() == self.cur.tobytes(), what
            self.ring.flush(t, self.cur)
            self.cur = np.zeros_like(self.cur)
        self.tsecs.append(t)
        self.tables.append(closed)
        self.windows.append(np.concatenate(self.samples) if self.samples else EMPTY)
        self.samples = []
        return self.check(what, responses)

    def held(self):
        return np.concatenate([self.windows[j] for j in held_windows(self.tsecs)]) if self.tsecs else EMPTY

    def check(self, what, responses=False):
        got = self.eng.export_cms_queries_5min()
        want = level_of_history(self.tsecs, self.tables) if self.tsecs else np.zeros_like(got)
        assert got.tobytes() == want.tobytes(), what
        if self.ring:
            assert got.tobytes() == self.ring.level.tobytes(), what
        held = self.held()
        keys = np.unique(held["flow_key"])[:2000]
        if len(keys):
            r = self.eng.query_flow_queries_5min(keys)
            q, m = fq.point_query(got, keys, self.d, self.w)
            assert np.array_equal(r["flow_key"], keys) and np.array_equal(r["queries"], q) and np.array_equal(r["resp_ms"], m), what
            for (eq, em), a, b in zip(fq.exact(held, keys), q.tolist(), m.tolist()):
                if eq <= U32 and em <= U32:
                    assert a >= eq and b >= em, what
        if responses:
            cross_check(self.eng, got, self.d, what)
        return got


def cross_check(eng, level, depth, what):
    """without eviction every row's query halves sum to the services' nqrys_5min and its msec halves to their GYSK_HIST_RESP_5MIN
    bucket sums (mod 2^32)"""
    rows, _ = eng.query_window()
    nq, ms = 0, 0
    for r in rows:
        nq += int(r.nqrys_5min)
        h = eng.export_hist(int(r.glob_id), ge.HIST_RESP_5MIN)
        if h is not None:
            ms += int(h[0]["sum"].astype(np.int64).sum())
    t = level.reshape(depth, -1)
    for row in range(depth):
        assert int((t[row] & np.uint64(U32)).sum(dtype=np.uint64)) & U32 == nq & U32, (what, row)
        assert int((t[row] >> np.uint64(32)).sum(dtype=np.uint64)) & U32 == ms & U32, (what, row)


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_level_after_every_flush(name):
    tsecs = SEQUENCES[name]
    rng = np.random.default_rng(300 + len(tsecs))
    run = Run(**CFG)
    assert not run.eng.export_cms_queries_5min().any()              # empty before the first flush
    for i, t in enumerate(tsecs):
        run.batch(_mixed(rng, int(rng.integers(1000, 8000)), nsvc=40, nclients=3000))
        run.flush(t, what=(name, i, t), responses=True)
    run.batch(_mixed(rng, 5000, nsvc=40, nclients=3000))              # the open window stays out of the level
    run.check((name, "open"), responses=True)


def _route_batch(rng, route, n=4000):
    """(the batch as the library expands it, a callable that ingests it) of one response route"""
    if route in ("event32", "event32_hot"):
        ev = _mixed(rng, n, nsvc=60, nclients=2000)
        return ev, None
    if route in ("ipv4", "ipv6"):
        rec = _raw_resp(rng, n, RESP6 if route == "ipv6" else RESP4, route == "ipv6")
        ms, ok = fq.resp_usec_raw(rec)
        keys = fq.route_key_ipv6(rec) if route == "ipv6" else fq.route_key_ipv4(rec)
        svc = raw_svc_id(fold_ip6([0x20010DB8, 0, 0, 1]) if route == "ipv6" else 0x0A000001, 8080)
        kind = ge.RAW_TCP_IPV6_RESP if route == "ipv6" else ge.RAW_TCP_IPV4_RESP
        return _expanded(svc, keys, ms * np.uint32(1000), ok), lambda e: e.ingest_raw(kind, rec, len(rec))
    if route == "resp16":
        rec = np.zeros(n, dtype=ge.RESP16_DTYPE)
        rec["svc_id"] = rng.integers(1, 40, n).astype(np.uint64) * np.uint64(1000003)
        rec["usec"], rec["cli_port"] = rng.integers(0, 3_000_000, n), rng.integers(0, 256, n)
        rec["usec"][::50] = fq.VALID_USEC + 1
        ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
        ev["svc_id"], ev["flow_key"], ev["value"], ev["type"] = rec["svc_id"], fq.route_key_resp16(rec), rec["usec"], ge.EV_RESP
        return ev, lambda e: e.ingest_raw(ge.RAW_RESP16, rec, len(rec))
    ids = rng.integers(1, 40, n).astype(np.uint64) * np.uint64(1000003)
    usec = rng.integers(0, 3_000_000, n).astype(np.uint64)
    usec[::50] = fq.VALID_USEC + 7
    rec = api_tran(ids, usec, reqlen=100, reslen=200, cliport=rng.integers(40000, 40100, n))
    return resp_events(rec), lambda e: e.ingest_raw(ge.RAW_API_TRAN, rec, len(rec))


@pytest.mark.parametrize("route", ["event32", "event32_hot", "resp16", "ipv4", "ipv6", "api_tran", "api_tran_traced"])
def test_every_response_route_feeds_the_level(route, monkeypatch):
    if route == "event32_hot":
        monkeypatch.setenv("GYSK_HOT_MIN", "64")                    # busy services turn hot after their first batch
    elif route == "event32":
        monkeypatch.setenv("GYSK_HOT_ROWS", "0")
    rng = np.random.default_rng(sum(map(ord, route)))
    run = Run(max_trace_svcs=64 if route == "api_tran_traced" else 0, **CFG)
    for i, t in enumerate(SEQUENCES["gaps"]):
        for _ in range(2):
            ev, ingest = _route_batch(rng, route)
            run.batch(ev, ingest=ingest)
        run.flush(t, what=(route, i, t), responses=True)
    if route.startswith("event32"):
        assert (run.eng.hot_rows_in_use() > 0) == (route == "event32_hot")
    assert run.eng.stats()["events_resp"] > 0


def test_excluded_samples_stay_out():
    """samples beyond the validity rule, unknown ids without auto-registration, ids beyond a full table and GYSK_EV_TRACE events of
    traced services never reach the level"""
    rng = np.random.default_rng(11)
    run = Run(**dict(CFG, auto_register=False, max_trace_svcs=64))
    ev = _mixed(rng, 30_000, nsvc=200)
    ids = np.unique(ev["svc_id"][ev["type"] == ge.EV_RESP])
    reg = ids[::2]
    run.eng.register_ids(reg)
    for i, t in enumerate((5, 35, 65, 95)):
        ev = _mixed(rng, 30_000, nsvc=200)
        tr = trace_events(api_tran(reg[rng.integers(0, len(reg), 2000)], rng.integers(0, 3_000_000, 2000).astype(np.uint64),
                                   cliport=rng.integers(1, 50, 2000)))
        run.batch(np.concatenate([ev, tr]), known=set(reg.tolist()))
        run.flush(t, what=("registered", i))
    full = Run(**dict(CFG, max_svcs=64))
    svc = (np.arange(64, dtype=np.uint64) + np.uint64(1)) * np.uint64(104729)
    for i, t in enumerate((5, 10, 40)):
        ev = np.zeros(20_000, dtype=ge.EVENT_DTYPE)
        ev["svc_id"], ev["type"] = svc[rng.integers(0, 64, len(ev))], ge.EV_RESP
        ev["svc_id"][:64] = svc                                      # every one of the 64 ids: the table is full after the first batch
        ev["flow_key"], ev["value"] = rng.integers(1, 5000, len(ev)), rng.integers(0, 1 << 22, len(ev))
        if i:
            ev["svc_id"][64::3] = (np.arange(len(ev[64::3]), dtype=np.uint64) % np.uint64(30) + np.uint64(100)) * np.uint64(7)
        full.batch(ev, known=set(svc.tolist()))
        full.flush(t, what=("full", i), responses=True)
    assert full.eng.stats()["events_dropped"] > 0


@pytest.mark.parametrize("depth,log2w", [(1, 4), (8, 4), (1, 22), (8, 22)])
def test_sketch_edges_and_a_wrapping_msec_half(depth, log2w):
    """1467 samples of 1 000 000 ms a window on one key: with three windows held its msec half passes 2^32 in the level"""
    rng = np.random.default_rng(depth * 100 + log2w)
    wide = log2w >= 20
    run = Run(restate=not wide, **dict(CFG, cms_depth=depth, cms_log2_width=log2w))
    hot = np.uint64(0x5EED0001)
    wrapped = False
    for i, t in enumerate([5, 35, 40] if wide else [5, 35, 40, 299, 400, 405]):
        ev = _mixed(rng, 20_000, nsvc=40, nclients=3000)
        big = np.zeros(1467, dtype=ge.EVENT_DTYPE)
        big["svc_id"], big["flow_key"], big["type"], big["value"] = ev["svc_id"][0], hot, ge.EV_RESP, 1_000_000_000
        run.batch(np.concatenate([ev, big]))
        run.flush(t, what=(depth, log2w, i), responses=True)
        wrapped |= fq.exact(run.held(), [hot])[0][1] > U32
    assert wrapped                                                    # the level held the key's msec half past 2^32
    if wide:
        assert run.eng.capacity()["device_bytes"] >= 15 * (depth << log2w) * 8


def test_eviction_recycled_slots_grow_and_the_direct_path():
    rng = np.random.default_rng(13)
    run = Run(**dict(CFG, max_svcs=256, idle_evict_secs=10))

    def ev_of(lo, hi, n=20_000):
        ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = rng.integers(lo, hi, n).astype(np.uint64) * np.uint64(6151)
        ev["flow_key"], ev["value"], ev["type"] = rng.integers(1, 3000, n), rng.integers(0, 1 << 22, n), ge.EV_RESP
        return ev
    run.batch(ev_of(1, 150))
    for t in (5, 10, 20, 35, 60):
        run.flush(t, what=("idle", t))
    run.batch(ev_of(200, 380))                                        # the first services were evicted: their slots taken by new ids
    assert run.eng.stats()["svcs_evicted"] > 0
    run.eng.grow(max_svcs=1024)                                        # inside the window
    run.batch(ev_of(400, 900))
    run.flush(65, what="grow")
    run.batch(ev_of(400, 900))
    run.flush(70, what="after grow")
    assert run.eng.stats()["events_dropped"] == 0

    big = Run(max_svcs=1024, max_tasks=64, max_batch=1 << 22, stage_batch=1 << 22, cms_depth=4, cms_log2_width=20)
    n = 2_500_000
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = rng.integers(1, 200, n).astype(np.uint64) * np.uint64(7919)
    ev["flow_key"] = synth.splitmix64(np.arange(1, n + 1, dtype=np.uint64))
    ev["value"], ev["type"] = rng.integers(0, 1 << 22, n), ge.EV_RESP
    big.batch(ev)
    assert big.eng.last_batch_flow_query_direct() >= n - (1 << 21)
    big.flush(5, what="direct", responses=True)
    big.batch(_mixed(rng, 50_000))
    big.flush(10, what="direct, then the table", responses=True)


def _regions(eng, torch):
    """{region: (array names, region bytes)} of gysk_merge_buffers"""
    out = {}
    for name, ptr, nbytes, _redop in eng.merge_buffers():
        region, arrays = name.split(": ")
        out[region] = (arrays.split("|"), _dev_bytes(torch, ptr, nbytes))
    return out


def _level_slice(eng, torch):
    names, buf = _regions(eng, torch)["sum_u64"]
    ncms = (eng.cfg.cms_depth << eng.cfg.cms_log2_width) * 8
    off = names.index("cms_qry_5min") * ((ncms + 255) & ~255)      # the count-min tables lead the SUM region
    return buf[off: off + ncms].view(np.uint64)


def _same_merge_arrays(off, on, torch):
    """on's merge arrays are off's with cms_qry_5min inserted after cms_qry_last in the SUM region and, when off has none, the flush
    tsec pair appended to the i64 MAX region"""
    a, b = _regions(off, torch), _regions(on, torch)
    assert set(a) == set(b)
    ncms = (off.cfg.cms_depth << off.cfg.cms_log2_width) * 8
    step = (ncms + 255) & ~255
    for region, (names, buf) in a.items():
        names2, buf2 = b[region]
        if region == "sum_u64":
            k = names.index("cms_qry_last") + 1
            assert names2 == names[:k] + ["cms_qry_5min"] + names[k:]
            p = k * step
            assert buf2[:p].tobytes() == buf[:p].tobytes() and buf2[p + step:].tobytes() == buf[p:].tobytes()
        elif region == "max_i64" and "flush tsec" not in names:
            assert names2 == names + ["flush tsec"]
            assert buf2[: len(buf)].tobytes() == buf.tobytes()
        else:
            assert names2 == names and buf2.tobytes() == buf.tobytes(), region


OTHER = {"alone": {}, "flow_level": dict(flow_level=True),
         "merge": dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, merge_traces=True, max_trace_svcs=64)}


@pytest.mark.parametrize("other", sorted(OTHER))
def test_flag_off_and_on_answer_alike(other):
    import torch
    rng = np.random.default_rng(17)
    flags = OTHER[other]
    off, on = ge.Engine(flow_queries=True, **CFG, **flags), ge.Engine(flow_queries=True, flow_query_level=True, **CFG, **flags)
    ncell = (CFG["cms_depth"] << CFG["cms_log2_width"])
    assert on.capacity()["device_bytes"] - off.capacity()["device_bytes"] == 11 * ncell * 8
    ev0 = _mixed(np.random.default_rng(0), 20_000)
    sids = np.unique(ev0["svc_id"][ev0["type"] != ge.EV_TASK])
    for e in (off, on):
        e.set_logical_map(sids, sids % np.uint64(7) + np.uint64(50))
    lids = np.unique(sids % np.uint64(7) + np.uint64(50))
    tsecs = (5, 10, 40, 40, 400)
    for i, t in enumerate(tsecs):
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
        assert _rowbytes(off.query_svcs(sids)) == _rowbytes(on.query_svcs(sids))
        for sid in sids[:40].tolist():
            for which in (ge.HIST_RESP_LAST, ge.HIST_RESP_5MIN):
                a, b = off.export_hist(sid, which), on.export_hist(sid, which)
                assert (a is None) == (b is None) and (a is None or (np.array_equal(a[0], b[0]) and a[1:] == b[1:]))
        sa, sb = off.stats(), on.stats()
        # one roll per flush so far and, where off has no flush tsec pair, one fold of the pair per merge
        assert sb.pop("kernel_launches") - sa.pop("kernel_launches") == i * (1 if flags else 2)
        assert sa == sb
        for e in (off, on):
            e.flush(t)
        for e in (off, on):
            _emulate_collectives(torch, [e])
        _same_merge_arrays(off, on, torch)
        assert _rowbytes(off.query_logical(lids)) == _rowbytes(on.query_logical(lids))
        for lw in (False, True):
            assert off.query_flows_global(keys, lw).tobytes() == on.query_flows_global(keys, lw).tobytes()
            assert off.query_flow_queries_global(keys, lw).tobytes() == on.query_flow_queries_global(keys, lw).tobytes()
        assert on.merge_flush_range() == (t, t)
        if flags:
            assert off.merge_flush_range() == (t, t)
    for call in (lambda: off.query_flow_queries_5min(keys), off.export_cms_queries_5min, lambda: off.query_flow_queries_global_5min(keys)):
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == NOTSUP
    if not flags:
        with pytest.raises(ge.GyskError) as ex:
            off.merge_flush_range()
        assert ex.value.code == NOTSUP
    fresh = ge.Engine(flow_queries=True, flow_query_level=True, **CFG)
    with pytest.raises(ge.GyskError) as ex:
        fresh.query_flow_queries_global_5min(keys)
    assert ex.value.code == INVAL
    with pytest.raises(ge.GyskError) as ex:
        ge.Engine(flow_query_level=True, **CFG, **flags)
    assert ex.value.code == INVAL


def _shard(ev, world):
    return [ev[ev["host_idx"] % world == r] for r in range(world)]


@pytest.mark.parametrize("other_flags", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_merge_sums_the_ranks_levels(world, other_flags):
    import torch
    rng = np.random.default_rng(world * 10 + other_flags)
    flags = dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, flow_level=True) if other_flags else {}
    engines = [ge.Engine(flow_queries=True, flow_query_level=True, rank=r, world=world, **flags, **CFG) for r in range(world)]
    ev0 = _mixed(np.random.default_rng(0), 20_000)
    sids = np.unique(ev0["svc_id"][ev0["type"] != ge.EV_TASK])
    for e in engines:
        e.set_logical_map(sids, sids % np.uint64(3) + np.uint64(10))
    for step, t in enumerate([30, 35, 60, 95, 300, 305]):
        ev = _mixed(rng, 30_000)
        last = step == 5
        tsec = [t + (5 * (r % 3) if last else 0) for r in range(world)]       # at the last flush the ranks close different windows
        for e, sh, ts in zip(engines, _shard(ev, world), tsec):
            e.ingest_events(sh); e.sync()
            e.flush(ts)
        _emulate_collectives(torch, engines)
        levels = [e.export_cms_queries_5min() for e in engines]
        want = sum(levels[1:], levels[0].copy())
        keys = np.unique(ev["flow_key"])[:500]
        q, m = fq.point_query(want, keys, CFG["cms_depth"], CFG["cms_log2_width"])
        for e in engines:
            assert _level_slice(e, torch).tobytes() == want.tobytes(), (world, step)
            got = e.query_flow_queries_global_5min(keys)
            assert np.array_equal(got["flow_key"], keys) and np.array_equal(got["queries"], q) and np.array_equal(got["resp_ms"], m), (world, step)
            assert e.merge_flush_range() == (min(tsec), max(tsec))


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(5)
    eng = ge.Engine(flow_queries=True, flow_query_level=True, **CFG)
    eng.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    for t in (30, 35, 65):
        eng.ingest_events(_mixed(rng, 30_000)); eng.sync()
        eng.flush(t)
    eng.ingest_events(_mixed(rng, 30_000)); eng.sync()
    keys = rng.integers(1, 5000, 300).astype(np.uint64)
    _emulate_collectives(torch, [eng])
    emulated = eng.query_flow_queries_global_5min(keys).tobytes()
    level = _level_slice(eng, torch).tobytes()
    eng.nccl_comm_init(eng.nccl_unique_id(), 1, 0)
    eng.merge_global()
    eng.sync()
    assert eng.query_flow_queries_global_5min(keys).tobytes() == emulated
    assert emulated == eng.query_flow_queries_5min(keys).tobytes()
    assert _level_slice(eng, torch).tobytes() == level == eng.export_cms_queries_5min().tobytes()
    assert eng.merge_flush_range() == (65, 65)
