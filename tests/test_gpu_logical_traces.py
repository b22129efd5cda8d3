"""Request traces of logical services (GYSK_FLAG_MERGE_TRACES): gysk_query_logical_traces, gysk_query_logical_traces_all and the merged
trace digest, at world 1 ... 8 with the collectives emulated on one device, with and without the other merge flags. After every merge
each rank's rows equal the restatement of tests/logical_traces.py byte for byte: each rank's TraceOracle, fed the events that rank owns,
gives every member's last window; counters are summed and maxima taken, the window digests folded with td_fold at compression 100 in
map order and then rank-ascending. Scenarios: members spread over ranks with a rank holding none, members without a trace row, logical
services with no traced member, a full trace table with dropped events, eviction and a recycled slot, a growth between prepare and
finish, ranks that flushed different windows, hot rows on and off; the p99 accuracy of a merged digest at world 8; the flag off and on
without traces; the library's NCCL path."""
import ctypes as C

import numpy as np
import pytest

from gyeeta_b200 import dist as gd
from gyeeta_b200 import engine as ge
from tests import logical_traces as lt
from tests import trace_agg as ta
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import _align256, _dev_bytes
from tests.util import exact_quantile, same_double, td_p99_tolerance

pytestmark = pytest.mark.gpu

INVAL, NOENT, NOTSUP = -22, -2, -95
UNKNOWN = 123456789
NHOSTS = 16
KW = dict(max_svcs=256, max_tasks=16, max_batch=1 << 14, cms_log2_width=10)
OTHERS = dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, flow_level=True)


def _code(fn):
    with pytest.raises(ge.GyskError) as ei:
        fn()
    return ei.value.code


class Ranks:
    """world engines with trace rows and the flag, rank r = shard r, and one TraceOracle per rank fed the events that rank owns"""

    def __init__(self, world, rows=64, others=False, **kw):
        self.world = world
        args = dict(KW, **kw)
        args.update(OTHERS if others else {})
        self.engines = [ge.Engine(rank=r, world=world, max_trace_svcs=rows, merge_traces=True, **args) for r in range(world)]
        self.oracles = [ta.TraceOracle(rows) for _ in range(world)]

    def set_map(self, glob, logical):
        self.glob, self.logical = glob, logical
        for e in self.engines:
            e.set_logical_map(glob, logical)

    def feed(self, ev, batch=KW["max_batch"]):
        for off in range(0, len(ev), batch):
            chunk = ev[off: off + batch]
            for r, (e, to) in enumerate(zip(self.engines, self.oracles)):
                e.ingest_events(chunk)
                e.sync()
                to.ingest(chunk[chunk["host_idx"] % self.world == r])

    def flush(self, t, per_rank=None):
        for r, (e, to) in enumerate(zip(self.engines, self.oracles)):
            e.flush(per_rank[r] if per_rank else t)
            to.flush()
            to.evict(e.evicted_ids())


def verify(rk):
    """every new read of every rank against the restatement; returns {logical id: (row, digest)}"""
    mem = lt.members_of(rk.glob, rk.logical)
    dense, lids = list(mem), sorted(mem)
    want = {l: lt.row(rk.oracles, l, gs) for l, gs in mem.items()}
    wb = {l: lt.row_bytes(r) for l, (r, _) in want.items()}
    active = [l for l in lids if want[l][0].last.nreq]
    for l, (r, d) in want.items():
        assert r.last.td_count == d.total and r.last.nreq == sum(r.last.resp_buckets), l
    for r, e in enumerate(rk.engines):
        got = e.query_logical_traces(dense + [UNKNOWN])
        assert [lt.row_bytes(x) for x in got] == [wb[l] for l in dense] + [lt.row_bytes(lt.missing(UNKNOWN))], \
            (r, [(x.asdict(), want[x.logical_id][0].asdict()) for x in got[:-1] if lt.row_bytes(x) != wb[x.logical_id]][:2])
        rows, n = e.query_logical_traces_all()
        assert n == len(lids) and [lt.row_bytes(x) for x in rows] == [wb[l] for l in lids], r
        assert [x.logical_id for x in rows] == [x.glob_id for x in e.query_logical_all()[0]]
        arows, an = e.query_logical_traces_all(active_only=True)
        assert an == len(active) and [lt.row_bytes(x) for x in arows] == [wb[l] for l in active], r
        assert e.query_logical_traces_all(cap=0) == ([], len(lids))
        part, pn = e.query_logical_traces_all(cap=max(1, len(lids) // 3))
        assert pn == len(lids) and [lt.row_bytes(x) for x in part] == [wb[l] for l in lids[: len(part)]]
        for l, (_, d) in want.items():
            m, w, mn, mx = e.export_logical_trace_tdigest(l)
            assert m.tobytes() == np.ascontiguousarray(d.cent["mean"]).tobytes() and np.array_equal(w, d.cent["weight"]), (r, l)
            assert same_double(mn, d.minv) and same_double(mx, d.maxv), (r, l, mn, mx, d.minv, d.maxv)
            assert int(w.sum()) == d.total
            assert e.export_logical_trace_tdigest_pgtext(l) == lt.pgtext(d), (r, l)
        assert e.export_logical_trace_tdigest(UNKNOWN) is None and e.export_logical_trace_tdigest_pgtext(UNKNOWN) is None
    return want


def merge_and_verify(torch, rk):
    _emulate_collectives(torch, rk.engines)
    return verify(rk)


def _ids(n, salt):
    return (np.arange(1, n + 1, dtype=np.uint64) * np.uint64(0x9E3779B1)) | np.uint64(salt << 40)


def trace_stream(rng, ids, n):
    """API_TRAN records of ids: log-normal response times with the bucket edges and samples beyond the validity rule, errors, new
    connections, saturated byte counts"""
    gid = rng.choice(ids, size=n)
    usec = np.exp(rng.normal(8.0, 1.8, size=n)).astype(np.uint64)
    edges = np.array([0, 299, 300, 999, 1000, 9999, 10000, 29999, 30000, 99999, 100000, 299999, 300000, 999999, 1000000, 1000000999,
                      1000001000, 5_000_000_000], dtype=np.uint64)
    k = min(len(edges), n)
    usec[:k] = edges[:k]
    reqlen = rng.integers(0, 1 << 20, size=n).astype(np.uint64)
    reqlen[rng.random(n) < 0.01] = np.uint64(1 << 40)
    reslen = rng.integers(0, 1 << 24, size=n).astype(np.uint64)
    reqnum = np.where(rng.random(n) < 0.1, 0, rng.integers(1, 100, size=n)).astype(np.uint64)
    err = rng.choice(np.array([0, 0, 0, 1, 500], dtype=np.int32), size=n)
    return ta.api_tran(gid, usec, reqlen, reslen, reqnum, err, cliport=rng.integers(0, 65536, size=n))


def events(rec, host):
    """each record's RESP and trace events on its service's host, interleaved as the wire walk stages them"""
    hosts = np.array([host[i] for i in rec["glob_id"].tolist()], dtype=np.uint32)
    tr, rs = ta.trace_events(rec), ta.resp_events(rec)
    tr["host_idx"], rs["host_idx"] = hosts, hosts
    out = np.empty(2 * len(rec), dtype=ge.EVENT_DTYPE)
    out[0::2], out[1::2] = rs, tr
    return out


def resp_only(rng, ids, host, n):
    """RESP events alone: services that hold a slot and no trace row"""
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = rng.choice(ids, size=n)
    ev["host_idx"] = [host[i] for i in ev["svc_id"].tolist()]
    ev["type"], ev["value"] = ge.EV_RESP, rng.integers(100, 100_000, size=n)
    return ev


def scenario():
    """(ids, host of each id, traced ids, untraced ids, glob ids, logical ids) of a shuffled map:
      9000: services 0..15, one per host => members on every rank; 12..15 never traced
      9001: services 16 and 32, both on host 0 => one rank; the others hold no member
      9002: services 17..19, never traced: found = 1, ntraced = 0
      9003: ids that never appear
      9004 + i: singletons 20..27
      9005: services 28..31 and 33..47"""
    ids = _ids(48, 3)
    ghosts = _ids(3, 4)
    host = {int(g): i % NHOSTS for i, g in enumerate(ids.tolist())}
    untraced = [int(ids[i]) for i in list(range(12, 16)) + [17, 18, 19]]
    traced = [int(g) for g in ids.tolist() if int(g) not in untraced]
    pairs = [(ids[i], 9000) for i in range(16)] + [(ids[16], 9001), (ids[32], 9001)] + [(ids[i], 9002) for i in (17, 18, 19)]
    pairs += [(g, 9003) for g in ghosts] + [(ids[i], 9004 + i) for i in range(20, 28)]
    pairs += [(ids[i], 9005) for i in list(range(28, 32)) + list(range(33, 48))]
    perm = np.random.default_rng(77).permutation(len(pairs))
    glob = np.array([int(pairs[i][0]) for i in perm], dtype=np.uint64)
    logical = np.array([pairs[i][1] for i in perm], dtype=np.uint64)
    return ids, host, traced, untraced, glob, logical


@pytest.mark.parametrize("others,hot", [(False, False), (True, True)], ids=["alone_hot_off", "other_flags_hot_rows"])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_traces_equal_the_restatement(monkeypatch, world, others, hot):
    """every rank's rows, the all-rows read, ACTIVE_ONLY and the merged digests equal the restatement after each merge, mid-window
    merges included"""
    import torch
    monkeypatch.setenv("GYSK_HOT_ROWS", "2048" if hot else "0")
    monkeypatch.setenv("GYSK_HOT_MIN", "8")
    rng = np.random.default_rng(300 + 10 * world + others)
    ids, host, traced, untraced, glob, logical = scenario()
    rk = Ranks(world, others=others)
    rk.set_map(glob, logical)
    seen = {}
    for w in range(6):
        n = 3000 if w != 3 else 40                      # a thin window: some members without requests
        ev = np.concatenate([events(trace_stream(rng, np.array(traced[:20 + 4 * w], dtype=np.uint64), n), host),
                             resp_only(rng, untraced, host, 500)])
        rk.feed(ev[rng.permutation(len(ev))])
        if w == 2:
            merge_and_verify(torch, rk)                 # mid-window: the last closed window only
        rk.flush(100 + 5 * w)
        if w in (0, 3, 5):
            seen = merge_and_verify(torch, rk)
    r = {l: x for l, (x, _) in seen.items()}
    assert r[9000].ntraced == 12 and r[9000].last.nreq > 0
    assert r[9001].ntraced == 2
    for l in (9002, 9003):
        assert r[l].found == 1 and r[l].ntraced == 0 and r[l].last.nreq == 0 and np.isnan(r[l].last.p99_resp_us)
    if world > 1:
        held = [sum(1 for g in lt.members_of(glob, logical)[9001] if g in to.in_use) for to in rk.oracles]
        assert held.count(0) == world - 1
    for e in rk.engines:
        assert e.merge_flush_range() == (125, 125)
        if others:
            assert e.query_logical_states([9000])[0].found == 1


def test_full_table_eviction_and_recycled_slot():
    """world 2, two trace rows per rank: a full table drops events; idle members are evicted and drop out; a new traced id takes a
    recycled slot and its row joins its logical service"""
    import torch
    rng = np.random.default_rng(5)
    rk = Ranks(2, rows=2, max_svcs=8, idle_evict_secs=10)
    host = {i: i % 2 for i in range(10, 20)}
    rk.set_map(np.array([11, 17, 12, 13, 14, 15, 16], dtype=np.uint64), np.array([7000, 7000, 7001, 7001, 7002, 7002, 7002], dtype=np.uint64))

    def batch(ids_, n=400):
        rk.feed(events(trace_stream(rng, np.array(ids_, dtype=np.uint64), n), host))

    def flush(t):
        rk.flush(t)
        return merge_and_verify(torch, rk)

    batch([11, 13, 12, 14])
    batch([11, 15, 12, 16])                 # both tables full: 15 and 16 dropped
    assert all(to.dropped > 0 for to in rk.oracles)
    assert [e.trace_info()[1] for e in rk.engines] == [to.dropped for to in rk.oracles]
    flush(100)
    batch([13, 14])
    flush(105)
    batch([13, 14])
    rows = flush(125)                       # 11 and 12 idle since 100: evicted, their rows freed
    assert rows[7000][0].ntraced == 0 and rows[7001][0].ntraced == 1
    batch([17, 13, 14])                     # 17 takes a freed slot and row
    batch([15])                             # table full again
    rows = flush(130)
    assert rows[7000][0].ntraced == 1 and rows[7000][0].last.nreq > 0


def test_grow_between_prepare_and_finish():
    """gysk_grow after the collectives and before gysk_merge_finish changes no row: finish reads only the slab"""
    import torch
    rng = np.random.default_rng(8)
    ids, host, traced, untraced, glob, logical = scenario()
    rk = Ranks(3, max_svcs=64)
    rk.set_map(glob, logical)
    rk.feed(np.concatenate([events(trace_stream(rng, np.array(traced, dtype=np.uint64), 4000), host), resp_only(rng, untraced, host, 300)]))
    rk.flush(100)

    class GrowBeforeFinish:
        def __init__(self, e):
            self.e = e

        def __getattr__(self, k):
            return getattr(self.e, k)

        def merge_finish(self, *a):
            self.e.grow(max_svcs=256)
            self.e.merge_finish(*a)

    _emulate_collectives(torch, [GrowBeforeFinish(e) for e in rk.engines])
    verify(rk)
    assert all(e.capacity()["max_svcs"] == 256 for e in rk.engines)


def test_ranks_that_flushed_different_windows():
    """each rank merges its own last closed window; gysk_merge_flush_range shows the spread"""
    import torch
    rng = np.random.default_rng(12)
    ids, host, traced, untraced, glob, logical = scenario()
    rk = Ranks(3)
    rk.set_map(glob, logical)
    rk.feed(events(trace_stream(rng, np.array(traced, dtype=np.uint64), 3000), host))
    rk.flush(0, per_rank=[100, 105, 110])
    merge_and_verify(torch, rk)
    assert all(e.merge_flush_range() == (100, 110) for e in rk.engines)


def test_merged_p99_accuracy_at_world_8():
    """8 members on 8 ranks, 120 K samples per logical service: the merged p99 within twice td_p99_tolerance of the exact p99 of the
    union of the members' samples"""
    import torch
    rng = np.random.default_rng(21)
    world, per = 8, 15_000
    engines = [ge.Engine(rank=r, world=world, max_svcs=64, max_tasks=16, max_batch=1 << 16, cms_log2_width=10, max_trace_svcs=16,
                         merge_traces=True) for r in range(world)]
    mids = {l: [int(x) for x in _ids(8, 10 + l)] for l in range(2)}
    glob = np.array(mids[0] + mids[1], dtype=np.uint64)
    logical = np.array([500] * 8 + [501] * 8, dtype=np.uint64)
    for e in engines:
        e.set_logical_map(glob, logical)
    host = {g: i % 8 for l in mids for i, g in enumerate(mids[l])}
    vals = {}
    for l, (mu, sigma) in enumerate(((np.log(20_000.0), 1.0), (np.log(3_000.0), 1.5))):
        usec = np.minimum(np.exp(rng.normal(mu, sigma, size=8 * per)), 9.0e8).astype(np.uint64)
        gid = np.repeat(np.array(mids[l], dtype=np.uint64), per)
        vals[500 + l] = usec
        ev = ta.trace_events(ta.api_tran(gid, usec))
        ev["host_idx"] = [host[g] for g in gid.tolist()]
        ev = ev[rng.permutation(len(ev))]
        for e in engines:
            for off in range(0, len(ev), 1 << 16):
                e.ingest_events(ev[off: off + (1 << 16)])
            e.sync()
    for e in engines:
        e.flush(100)
    _emulate_collectives(torch, engines)
    for lid, v in vals.items():
        rows = [e.query_logical_traces([lid])[0] for e in engines]
        assert len({lt.row_bytes(r) for r in rows}) == 1
        r = rows[0]
        assert r.ntraced == 8 and r.last.nreq == r.last.td_count == len(v) and r.last.sum_resp_us == int(v.sum())
        exact = exact_quantile(v, 0.99)
        assert abs(r.last.p99_resp_us - exact) <= 2 * td_p99_tolerance(len(v)) * exact, (lid, r.last.p99_resp_us, exact)


def _regions(torch, e):
    return [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in e.merge_buffers()]


def _slab(torch, e):
    p, nb = e.merge_tdigest_slab()
    return _dev_bytes(torch, p, nb).tobytes()


def test_flag_off_is_unchanged_and_reads_are_read_only():
    """an engine without the flag, one with it and no trace events, fed the same stream: without the flag the regions, names, slab and
    launches are today's and the new calls GYSK_ERR_NOTSUP; with it the trace words follow the old part of each region and slab, whose
    bytes and every existing logical read stay as they were, and every logical service reads found = 1, ntraced = 0. The reads change
    nothing the merge left"""
    import torch
    rng = np.random.default_rng(23)
    ids, host, traced, untraced, glob, logical = scenario()
    lids = list(dict.fromkeys(logical.tolist()))
    off, on = ge.Engine(max_trace_svcs=64, **KW), ge.Engine(max_trace_svcs=64, merge_traces=True, **KW)
    for e in (off, on):
        e.set_logical_map(glob, logical)
    ev = resp_only(rng, [int(g) for g in ids.tolist()], host, 20_000)
    for e in (off, on):
        e.ingest_events(ev)
        e.flush(100)

    def launches(e, fn):
        k0 = e.stats()["kernel_launches"]
        fn()
        return e.stats()["kernel_launches"] - k0

    assert [launches(e, lambda: _emulate_collectives(torch, [e])) for e in (off, on)] == [5, 7]
    nl, c = len(lids), off.cfg
    ncms = c.cms_depth << c.cms_log2_width
    sizes = [2 * _align256(ncms * 8) + 2 * _align256(nl * 16 * 16) + _align256(nl * 32), _align256(nl * 16), _align256(nl << c.hll_p)]
    assert [(n, b, r) for n, _, b, r in off.merge_buffers()] == [
        ("sum_u64: cms_cur|cms_last|hist_last|hist_all|conn", sizes[0], gd.RED_SUM_U64),
        ("max_i64: hist max_val_seen", sizes[1], gd.RED_MAX_I64), ("max_u8: hll registers", sizes[2], gd.RED_MAX_U8)]
    assert [(n, b, r) for n, _, b, r in on.merge_buffers()] == [
        ("sum_u64: cms_cur|cms_last|hist_last|hist_all|conn|traces", sizes[0] + _align256(nl * 16 * 8), gd.RED_SUM_U64),
        ("max_i64: hist max_val_seen|flush tsec|trace max", sizes[1] + 256 + _align256(nl * 3 * 8), gd.RED_MAX_I64),
        ("max_u8: hll registers", sizes[2], gd.RED_MAX_U8)]
    slab_entry = 32 + 256 * 16
    assert off.merge_tdigest_slab()[1] == nl * slab_entry
    assert on.merge_tdigest_slab()[1] == (nl + -(-nl * 1632 // slab_entry)) * slab_entry
    for a, b in zip(_regions(torch, off), _regions(torch, on)):
        assert b[: len(a)] == a
    assert _slab(torch, on)[: nl * slab_entry] == _slab(torch, off)
    assert repr(on.query_logical(lids)) == repr(off.query_logical(lids))
    for x in on.query_logical_traces(lids):
        assert x.found == 1 and x.ntraced == 0 and x.last.nreq == 0 and np.isnan(x.last.p99_resp_us)
    assert on.export_logical_trace_tdigest(lids[0])[0].size == 0
    # without the flag
    out, n = (ge.LogicalTrace * 1)(), C.c_uint32()
    m, w = np.zeros(100), np.zeros(100, dtype=np.uint64)
    d = C.c_double()
    L = off.L
    assert L.gysk_query_logical_traces(off.h, ge._p(np.array(lids, dtype=np.uint64)), 1, out) == NOTSUP
    assert L.gysk_query_logical_traces_all(off.h, 0, out, 1, C.byref(n)) == NOTSUP
    assert L.gysk_export_logical_trace_tdigest(off.h, lids[0], ge._p(m), ge._p(w), 100, C.byref(n), C.byref(d), C.byref(d)) == NOTSUP
    assert L.gysk_export_logical_trace_tdigest_pgtext(off.h, lids[0], C.create_string_buffer(64), 64) == NOTSUP
    assert _code(lambda: off.merge_flush_range()) == NOTSUP and on.merge_flush_range() == (100, 100)
    # read-only reads: one launch per by-id chunk, one per all-rows pass, the select under ACTIVE_ONLY (no row pass: nothing is active)
    regions, slab, rows = _regions(torch, on), _slab(torch, on), [lt.row_bytes(x) for x in on.query_logical_traces(lids)]
    assert launches(on, lambda: on.query_logical_traces(lids)) == 1
    assert launches(on, lambda: on.query_logical_traces_all(cap=nl)) == 1
    assert launches(on, lambda: on.query_logical_traces_all(cap=0)) == 0
    assert launches(on, lambda: on.query_logical_traces_all(active_only=True, cap=nl)) == 1
    assert on.query_logical_traces_all(active_only=True) == ([], 0)
    assert launches(on, lambda: on.export_logical_trace_tdigest_pgtext(lids[0])) == 0
    assert _regions(torch, on) == regions and _slab(torch, on) == slab
    assert [lt.row_bytes(x) for x in on.query_logical_traces(lids)] == rows


def test_create_refuses_the_flag_without_trace_rows():
    with pytest.raises(ge.GyskError) as ei:
        ge.Engine(merge_traces=True, **KW)
    assert ei.value.code == INVAL and "max_trace_svcs" in str(ei.value)
    with ge.Engine(merge_traces=True, max_trace_svcs=1, **KW) as e:
        assert e.cfg.flags & ge.FLAG_MERGE_TRACES


def test_every_read_needs_a_finished_merge():
    """GYSK_ERR_INVAL without a map, with a map before a merge, and after gysk_merge_prepare before gysk_merge_finish"""
    ids, host, traced, untraced, glob, logical = scenario()
    e = ge.Engine(merge_traces=True, max_trace_svcs=64, **KW)
    calls = [lambda: e.query_logical_traces([9000]), lambda: e.query_logical_traces_all(), lambda: e.query_logical_traces_all(True, cap=0),
             lambda: e.export_logical_trace_tdigest(9000), lambda: e.export_logical_trace_tdigest_pgtext(9000), lambda: e.merge_flush_range()]
    assert [_code(c) for c in calls] == [INVAL] * len(calls)
    e.set_logical_map(glob, logical)
    assert [_code(c) for c in calls] == [INVAL] * len(calls)
    e.ingest_events(events(trace_stream(np.random.default_rng(1), np.array(traced, dtype=np.uint64), 500), host))
    e.flush(5)
    e.merge_prepare()
    e.sync()
    assert [_code(c) for c in calls] == [INVAL] * len(calls)
    e.merge_finish()
    rows, n = e.query_logical_traces_all()
    assert n == len(rows) > 0 and e.query_logical_traces([9000])[0].found == 1
    e.close()


def _nccl_uid():
    try:
        return ge.Engine(max_svcs=64, max_tasks=8, max_batch=4096, cms_log2_width=8).nccl_unique_id()
    except ge.GyskError as ex:
        pytest.skip(f"NCCL not loadable: {ex}")


def _nccl_feed(engines):
    ids, host, traced, untraced, glob, logical = scenario()
    for e in engines:
        e.set_logical_map(glob, logical)
    for w in range(3):
        ev = events(trace_stream(np.random.default_rng(w), np.array(traced, dtype=np.uint64), 2000), host)
        for e in engines:
            e.ingest_events(ev)
            e.flush(100 + 5 * w)
    return list(dict.fromkeys(logical.tolist()))


def test_library_nccl_merge_equals_the_emulation():
    """gysk_merge_global (NCCL inside the library) at world 1 leaves the same region bytes, trace rows and digests as the emulation"""
    import torch
    uid = _nccl_uid()
    e = ge.Engine(merge_traces=True, max_trace_svcs=64, **KW)
    lids = _nccl_feed([e])
    _emulate_collectives(torch, [e])
    want = (_regions(torch, e), [lt.row_bytes(x) for x in e.query_logical_traces(lids)], [e.export_logical_trace_tdigest_pgtext(l) for l in lids])
    e.nccl_comm_init(uid, 1, 0)
    e.merge_global()
    e.sync()
    assert (_regions(torch, e), [lt.row_bytes(x) for x in e.query_logical_traces(lids)], [e.export_logical_trace_tdigest_pgtext(l) for l in lids]) == want


def test_two_device_nccl_merge_equals_the_emulation():
    """two engines on two devices merged by gysk_merge_global equal two emulated shards on one device"""
    import threading

    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("the two-device NCCL merge needs two GPUs")
    _nccl_uid()
    emu = [ge.Engine(rank=r, world=2, merge_traces=True, max_trace_svcs=64, **KW) for r in range(2)]
    lib = [ge.Engine(device=r, rank=r, world=2, merge_traces=True, max_trace_svcs=64, **KW) for r in range(2)]
    lids = _nccl_feed(emu + lib)
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
    want = [lt.row_bytes(x) for x in emu[0].query_logical_traces(lids)]
    assert [lt.row_bytes(x) for x in lib[0].query_logical_traces(lids)] == want == [lt.row_bytes(x) for x in lib[1].query_logical_traces(lids)]
