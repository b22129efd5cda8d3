"""Trace rows (gysk_config.max_trace_svcs) on the device against the restated trace view (tests/trace_agg.py): after every batch and
every flush, every row of gysk_query_traces and gysk_query_trace_window equals the restatement byte for byte, the two reads agree, the
exported digests are the CPU oracle's compression-100 centroids bit for bit and their pgtext is gysk_tdigest_to_pgtext of those.
Scenarios: a mixed stream with RESP and trace samples of the same services (hot rows forced on and off), a service with more than
LONG_SEG trace samples in one batch, samples beyond the validity rule, bucket edges and byte saturation; the API_TRAN wire walk; a full
table, then rows freed by service eviction and taken again; a growth between two batches of a window; the host filter and ACTIVE_ONLY;
and an engine with trace rows but no trace events, whose every other answer equals an engine without them."""
import ctypes as C

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po
from tests import trace_agg as ta
from tests.util import td_p99_tolerance

pytestmark = pytest.mark.gpu

NHOSTS = 4


def host_of(id_):
    return int(id_) % NHOSTS


def pgtext(means, weights):
    L = ge.load_library()
    buf = C.create_string_buffer(8192)
    rc = L.gysk_tdigest_to_pgtext(ge._p(np.ascontiguousarray(means)), ge._p(np.ascontiguousarray(weights, dtype=np.uint64)), len(means), 100,
                                  buf, len(buf))
    assert rc >= 0
    return buf.value.decode()


def check(eng, to):
    """every read of the trace rows against the restatement"""
    ids = sorted(to.in_use)
    probe = ids + [0xDEAD0000BEEF]                                  # an unknown id: found = 0
    rows = eng.query_traces(probe)
    for id_, r in zip(probe, rows):
        want = to.row(id_, host_of(id_))
        assert ta.row_bytes(r) == ta.row_bytes(want), (hex(id_), r.asdict(), want.asdict())
    win, n = eng.query_trace_window()
    assert n == len(ids) and [r.glob_id for r in win] == ids
    for r, b in zip(win, rows):
        assert ta.row_bytes(r) == ta.row_bytes(b)
    for id_ in ids:
        for last in (False, True):
            m, w, mn, mx = eng.export_trace_tdigest(id_, last)
            om, ow, omn, omx = to.digest(id_, last)
            assert m.tobytes() == np.asarray(om, dtype=np.float64).tobytes() and np.array_equal(w, ow), (hex(id_), last, len(m), len(om))
            if len(m):
                assert (mn, mx) == (omn, omx)
            assert eng.export_trace_tdigest_pgtext(id_, last) == pgtext(om, ow)
    assert eng.trace_info() == (len(to.in_use), to.dropped)


def stream(rng, ids, n, big=None, nbig=0):
    """API_TRAN records of ids: log-normal response times with every bucket edge, errors, new connections, saturated byte counts"""
    gid = rng.choice(ids, size=n)
    usec = np.exp(rng.normal(8.0, 1.8, size=n)).astype(np.uint64)
    edges = np.array([0, 299, 300, 999, 1000, 9999, 10000, 29999, 30000, 99999, 100000, 299999, 300000, 999999, 1000000, 1000000999,
                      1000001000, 5_000_000_000], dtype=np.uint64)
    k = min(len(edges), n)
    usec[:k] = edges[:k]
    reqlen = rng.integers(0, 1 << 20, size=n).astype(np.uint64)
    reqlen[rng.random(n) < 0.01] = np.uint64(1 << 40)                 # beyond 32 bits: saturated
    reslen = rng.integers(0, 1 << 24, size=n).astype(np.uint64)
    reslen[rng.random(n) < 0.01] = np.uint64((1 << 64) - 1)
    reqnum = np.where(rng.random(n) < 0.1, 0, rng.integers(1, 100, size=n)).astype(np.uint64)
    err = rng.choice(np.array([0, 0, 0, 0, 1, 499, 500], dtype=np.int32), size=n)
    if big is not None:
        gid = np.concatenate([gid, np.full(nbig, big, dtype=np.uint64)])
        usec = np.concatenate([usec, np.exp(rng.normal(7.0, 1.0, size=nbig)).astype(np.uint64)])
        reqlen, reslen = np.concatenate([reqlen, np.full(nbig, 100, np.uint64)]), np.concatenate([reslen, np.full(nbig, 200, np.uint64)])
        reqnum, err = np.concatenate([reqnum, np.ones(nbig, np.uint64)]), np.concatenate([err, np.zeros(nbig, np.int32)])
    return ta.api_tran(gid, usec, reqlen, reslen, reqnum, err, cliport=rng.integers(0, 65536, size=len(gid)))


def events_of(rec, with_resp=True):
    """each record's RESP and trace events on its service's host, interleaved as the wire walk stages them"""
    hosts = np.array([host_of(i) for i in rec["glob_id"].tolist()], dtype=np.uint32)
    tr = ta.trace_events(rec)
    tr["host_idx"] = hosts
    if not with_resp:
        return tr
    rs = ta.resp_events(rec)
    rs["host_idx"] = hosts
    out = np.empty(2 * len(rec), dtype=ge.EVENT_DTYPE)
    out[0::2], out[1::2] = rs, tr
    return out


def feed(eng, orc, to, ev):
    eng.ingest_events(ev)
    eng.sync()
    orc.ingest(ev)
    to.ingest(ev)


@pytest.mark.parametrize("hot", [False, True], ids=["hot_off", "hot_rows"])
def test_mixed_stream_matches_restatement(monkeypatch, hot):
    monkeypatch.setenv("GYSK_HOT_ROWS", "2048" if hot else "0")
    monkeypatch.setenv("GYSK_HOT_MIN", "8")
    rng = np.random.default_rng(7)
    ids = (np.arange(1, 41, dtype=np.uint64) * np.uint64(0x9E3779B1)) | np.uint64(1 << 40)
    eng = ge.Engine(max_svcs=256, max_tasks=64, max_batch=1 << 18, max_trace_svcs=64)
    orc = po.OracleEngine(max_svcs=256, max_tasks=64)
    to = ta.TraceOracle(64)
    big = int(ids[0])
    for b in range(6):
        mixed = synth.gen_mixed(rng, 20_000, 40, ntask=8, nhosts=NHOSTS, nclients=500)
        mixed["svc_id"] = np.where(mixed["type"] != ge.EV_TASK, ids[mixed["svc_id"] % len(ids)], mixed["svc_id"])
        mixed["host_idx"] = np.where(mixed["type"] != ge.EV_TASK, mixed["svc_id"] % NHOSTS, mixed["host_idx"])
        rec = stream(rng, ids[:30], 3000, big=big if b in (1, 4) else None, nbig=20_000)
        ev = np.concatenate([mixed, events_of(rec)])
        if b == 2:
            ev = np.concatenate([ev, events_of(ta.api_tran(np.array([ids[35]], dtype=np.uint64), np.array([1234], dtype=np.uint64)))])
        feed(eng, orc, to, ev)
        check(eng, to)
        if b % 2:
            eng.flush(100 + 5 * b); orc.flush(100 + 5 * b); to.flush()
            check(eng, to)
    if hot:
        assert eng.hot_rows_in_use() > 0
    # the service state the RESP events feed is the oracle's, trace rows or not
    for id_ in ids[:30].tolist():
        for which in (ge.HIST_RESP_CUR, ge.HIST_RESP_ALL):
            a, b = eng.export_hist(id_, which), orc.export_hist(id_, which)
            assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]
        m, w, mn, mx = eng.export_tdigest(id_)
        om, ow = orc.export_tdigest(id_).centroids()
        assert m.tobytes() == om.tobytes() and np.array_equal(w, ow)


def test_long_segment_p99_accuracy():
    """a service with more than LONG_SEG trace samples per batch: the window digest's p99 within the t-digest's tolerance"""
    rng = np.random.default_rng(11)
    eng = ge.Engine(max_svcs=64, max_tasks=16, max_batch=1 << 20, max_trace_svcs=8)
    to = ta.TraceOracle(8)
    vals = []
    for _ in range(3):
        v = np.exp(rng.normal(9.0, 1.2, size=100_000)).astype(np.uint64)
        ev = ta.trace_events(ta.api_tran(np.full(len(v), 77, dtype=np.uint64), v), host_idx=host_of(77))
        eng.ingest_events(ev); eng.sync(); to.ingest(ev)
        vals.append(v)
    check(eng, to)
    allv = np.sort(np.concatenate(vals)).astype(np.float64)
    exact = allv[int(np.ceil(0.99 * len(allv))) - 1]
    p99 = eng.query_traces([77])[0].cur.p99_resp_us
    # compression 100 keeps half the clusters of the service digest's 200 the tolerance is stated for
    assert abs(p99 - exact) <= 2 * td_p99_tolerance(len(allv)) * exact, (p99, exact)


def test_wire_walk_stages_resp_and_trace():
    rng = np.random.default_rng(3)
    ids = np.arange(1, 9, dtype=np.uint64) + np.uint64(1 << 33)
    eng = ge.Engine(max_svcs=64, max_tasks=16, max_batch=1 << 16, max_trace_svcs=16)
    orc = po.OracleEngine(max_svcs=64, max_tasks=16)
    to = ta.TraceOracle(16)
    for b in range(3):
        rec = stream(rng, ids, 2000)
        eng.ingest_raw(ge.RAW_API_TRAN, rec, len(rec), host_idx=0)
        eng.sync()
        ev = np.empty(2 * len(rec), dtype=ge.EVENT_DTYPE)
        ev[0::2], ev[1::2] = ta.resp_events(rec), ta.trace_events(rec)
        orc.ingest(ev); to.ingest(ev)
        rows = eng.query_traces(ids)
        for id_, r in zip(ids.tolist(), rows):
            assert ta.row_bytes(r) == ta.row_bytes(to.row(id_, 0))
        for id_ in ids.tolist():
            a, o = eng.export_hist(id_, ge.HIST_RESP_CUR), orc.export_hist(id_, ge.HIST_RESP_CUR)
            assert np.array_equal(a[0], o[0]) and a[1:] == o[1:]
        eng.flush(10 + b); orc.flush(10 + b); to.flush()


def test_full_table_drops_then_eviction_recycles_rows():
    eng = ge.Engine(max_svcs=64, max_tasks=16, max_batch=1 << 16, max_trace_svcs=4, idle_evict_secs=10)
    to = ta.TraceOracle(4)
    rng = np.random.default_rng(5)

    def batch(ids, n=400):
        rec = stream(rng, np.asarray(ids, dtype=np.uint64), n)
        ev = events_of(rec)
        eng.ingest_events(ev); eng.sync(); to.ingest(ev)
        check(eng, to)

    def flush(t):
        eng.flush(t); to.flush()
        to.evict(eng.evicted_ids())
        check(eng, to)

    batch([11, 12, 13, 14])
    batch([11, 12, 15, 16])                 # table full: 15 and 16 dropped
    assert to.dropped > 0
    flush(100)
    batch([13, 14])
    flush(105)
    batch([13, 14])
    flush(125)                              # 11 and 12 idle since 100: evicted, their rows freed
    assert 11 not in to.in_use and 12 not in to.in_use and eng.trace_info()[0] == 2
    batch([15, 16, 13, 14])                 # the freed rows taken again
    batch([11])                             # table full again
    flush(130)


def test_grow_between_batches_of_a_window():
    rng = np.random.default_rng(9)
    ids = np.arange(1, 25, dtype=np.uint64) * np.uint64(1000003)
    eng = ge.Engine(max_svcs=32, max_tasks=16, max_batch=1 << 16, max_trace_svcs=24)
    to = ta.TraceOracle(24)
    for b in range(4):
        if b == 2:
            eng.grow(max_svcs=200)
        rec = stream(rng, ids[: 8 + 4 * b], 1500)
        ev = events_of(rec)
        eng.ingest_events(ev); eng.sync(); to.ingest(ev)
        check(eng, to)
    eng.flush(50); to.flush()
    check(eng, to)


def test_host_filter_and_active_only():
    rng = np.random.default_rng(13)
    ids = np.arange(100, 120, dtype=np.uint64)
    eng = ge.Engine(max_svcs=64, max_tasks=16, max_batch=1 << 16, max_trace_svcs=32)
    to = ta.TraceOracle(32)
    ev = events_of(stream(rng, ids, 2000))
    eng.ingest_events(ev); eng.sync(); to.ingest(ev)
    eng.flush(10); to.flush()
    ev = events_of(stream(rng, ids[:6], 500))               # the next window: only six of them
    eng.ingest_events(ev); eng.sync(); to.ingest(ev)
    eng.flush(15); to.flush()
    check(eng, to)
    for h in range(NHOSTS):
        for act in (False, True):
            rows, n = eng.query_trace_window(host_idx=h, active_only=act)
            want = sorted(i for i in to.in_use if host_of(i) == h and (not act or to.last[i]["nreq"]))
            assert n == len(want) and [r.glob_id for r in rows] == want
    rows, n = eng.query_trace_window(active_only=True, cap=2)
    assert n == 6 and len(rows) == 2 and [r.glob_id for r in rows] == sorted(ids[:6].tolist())[:2]


def test_trace_rows_without_trace_events_change_nothing():
    """an engine with trace rows fed no trace events answers every other read as one without them; without trace rows every trace call
    is GYSK_ERR_NOTSUP and a GYSK_EV_TRACE event is dropped"""
    rng = np.random.default_rng(1)
    ev = synth.gen_mixed(rng, 200_000, 300, ntask=32, nhosts=8, nclients=5000)
    a = ge.Engine(max_svcs=1024, max_tasks=64, max_batch=1 << 16, cms_log2_width=14)
    b = ge.Engine(max_svcs=1024, max_tasks=64, max_batch=1 << 16, cms_log2_width=14, max_trace_svcs=512)
    for eng in (a, b):
        for off in range(0, len(ev), 1 << 16):
            eng.ingest_events(ev[off: off + (1 << 16)])
            eng.sync()
        eng.flush(100)
        eng.ingest_events(ev[:5000]); eng.sync()
    ids = np.unique(ev["svc_id"][ev["type"] == ge.EV_RESP])
    wa, wb = a.query_window(), b.query_window()
    assert wa[1] == wb[1] and all(ta.row_bytes(x) == ta.row_bytes(y) for x, y in zip(wa[0], wb[0]))
    for id_ in ids[:50].tolist():
        for which in (ge.HIST_RESP_CUR, ge.HIST_RESP_LAST, ge.HIST_RESP_ALL):
            x, y = a.export_hist(id_, which), b.export_hist(id_, which)
            assert np.array_equal(x[0], y[0]) and x[1:] == y[1:]
        assert np.array_equal(a.export_hll(id_), b.export_hll(id_))
        x, y = a.export_tdigest(id_), b.export_tdigest(id_)
        assert x[0].tobytes() == y[0].tobytes() and np.array_equal(x[1], y[1]) and x[2:] == y[2:]
    assert np.array_equal(a.export_cms(), b.export_cms()) and np.array_equal(a.export_cms(True), b.export_cms(True))
    sa, sb = a.stats(), b.stats()
    sa.pop("kernel_launches"); sb.pop("kernel_launches")
    assert sa == sb
    assert b.trace_info() == (0, 0)
    # trace rows off: NOTSUP, and a trace event is dropped
    L = a.L
    n = C.c_uint32()
    assert L.gysk_query_traces(a.h, None, 0, None) == -95
    assert L.gysk_query_trace_window(a.h, -1, 0, None, 0, C.byref(n)) == -95
    assert L.gysk_trace_info(a.h, C.byref(n), C.byref(C.c_uint64())) == -95
    assert L.gysk_export_trace_tdigest_pgtext(a.h, 1, 0, C.create_string_buffer(64), 64) == -95
    before = a.stats()["events_dropped"]
    a.ingest_events(ta.trace_events(ta.api_tran(np.array([5], dtype=np.uint64), np.array([10], dtype=np.uint64)))); a.sync()
    assert a.stats()["events_dropped"] == before + 1
