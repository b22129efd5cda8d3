"""The reads over every merged logical service: gysk_query_logical_all, gysk_topn_logical and the digest / HLL exports of one logical
id, pinned against the restatement of test_gpu_merge_exact / test_gpu_merge_levels (one oracle engine per rank, the collectives
emulated) at world 1 ... 8, with and without GYSK_FLAG_MERGE_LEVELS, over late members, ghost ids, eviction and recycled slots.
Every answer must be the same on every rank, and none of the reads may change what the merge left behind."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import Shards, _dev_bytes, assert_summary, logical_map
from tests.test_gpu_merge_levels import KW, LevelRestatement, _events, _run_engines, _stream_ids
from tests.util import M32, MergeRestatement, same_double

INVAL, NOENT, NOTSUP = -22, -2, -95
QS = [0.5, 0.95, 0.99]
UNKNOWN = 123456789
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _code(fn):
    with pytest.raises(ge.GyskError) as ei:
        fn()
    return ei.value.code


def _raw_logical(e, ids):
    """the gysk_query_logical rows of ids, as bytes"""
    ids = np.ascontiguousarray(ids, dtype=np.uint64)
    out = (ge.SvcSummary * max(len(ids), 1))()
    e._chk(e.L.gysk_query_logical(e.h, ge._p(ids), len(ids), out))
    return [bytes(o) for o in out[: len(ids)]]


def _raw_topn(e, metric, n):
    out = (ge.TopnEntry * n)()
    k = C.c_uint32()
    e._chk(e.L.gysk_topn_logical(e.h, metric, n, out, C.byref(k)))
    return b"".join(bytes(o) for o in out[: k.value])


def host_td_compress(means, weights, delta=100):
    """the recompression of the Postgres export (host_td_compress, gysk_engine.cu): one fixed-grid K_1 pass over the centroids, cell j
    starting at weight (uint64)(q_j W)"""
    q = [0.5 * (math.sin(math.pi * (j / delta - 0.5)) + 1.0) for j in range(delta + 1)]
    q[0], q[delta] = 0.0, 1.0
    w = [int(x) for x in weights]
    W = sum(w)
    om, ow = [], []
    pref = cw = cur = 0
    csum = 0.0
    for i, (m, wi) in enumerate(zip(np.asarray(means, dtype=np.float64).tolist(), w)):
        lo = cur
        while lo + 1 < delta and int(q[lo + 1] * float(W)) <= pref:
            lo += 1
        if i and lo != cur:
            om.append(csum / float(cw)); ow.append(cw)
            cw, csum = 0, 0.0
        cur = lo
        csum += m * float(wi); cw += wi; pref += wi
    if w:
        om.append(csum / float(cw)); ow.append(cw)
    return np.array(om, dtype=np.float64), np.array(ow, dtype=np.uint64)


def pgtext(means, weights):
    """gysk_tdigest_to_pgtext of the host recompression of a digest's centroids"""
    om, ow = host_td_compress(means, weights)
    buf = C.create_string_buffer(8192)
    n = ge.load_library().gysk_tdigest_to_pgtext(ge._p(om), ge._p(ow), len(om), 100, buf, len(buf))
    assert n >= 0
    return buf.value.decode()


def _rel(a, b):
    if math.isnan(a) and math.isnan(b):
        return 0.0
    return abs(a - b) / abs(b) if b else abs(a - b)


def quantile_gap(e, rows, quantiles):
    """the largest relative gap between quantiles(id, {0.5, 0.95, 0.99}) and the row's td_p50_us / td_p95_us / td_p99_us"""
    gap = 0.0
    for r in rows:
        if r.td_count:
            for g, w in zip(quantiles(r.glob_id, QS), (r.td_p50_us, r.td_p95_us, r.td_p99_us)):
                gap = max(gap, _rel(float(g), float(w)))
    return gap


def check_reads(torch, sh, levels):
    """merge with the collectives emulated, then every new read on every rank against the restatement; returns the restated active
    logical ids"""
    _emulate_collectives(torch, sh.engines)
    rs = (LevelRestatement if levels else MergeRestatement)(sh.oracles, sh.glob, sh.logical, sh.delta, sh.hll_p)
    lib = ge.load_library()
    dense = list(dict.fromkeys(sh.logical.tolist()))        # dense logical index = order of first appearance
    lids = sorted(dense)
    cells = {lid: rs.cells(lid) for lid in lids}
    active = [lid for lid in lids if int(cells[lid]["last"]["count"].sum()) > 0 or cells[lid]["conn"][0] > 0]
    scores = {ge.TOPN_QPS: {l: min(int(c["last"]["count"].sum()), M32) for l, c in cells.items()},
              ge.TOPN_CONNS: {l: c["conn"][0] & M32 for l, c in cells.items()},
              ge.TOPN_NET: {l: c["conn"][1] & M32 for l, c in cells.items()}}
    if levels:
        scores[ge.TOPN_ACTIVE] = {l: rs.levels(l)["aux"][0] & M32 for l in lids}
    digests = {lid: rs.digest(lid) for lid in lids}
    want_rows = {lid: rs.summary(lid, lib) for lid in lids}
    tops = {}
    for r, e in enumerate(sh.engines):
        # every row, ascending logical id, each the by-id row of its id
        rows, n = e.query_logical_all()
        assert n == len(lids) and [x.glob_id for x in rows] == lids, r
        assert [bytes(x) for x in rows] == _raw_logical(e, lids), r
        for x in rows:
            assert_summary(x.asdict(), want_rows[x.glob_id], (r, x.glob_id))
        byid = {x.glob_id: bytes(x) for x in rows}
        arows, an = e.query_logical_all(active_only=True)
        assert an == len(active) and [x.glob_id for x in arows] == active, (r, [x.glob_id for x in arows], active)
        assert [bytes(x) for x in arows] == [byid[l] for l in active]
        # count-only and partial calls, as gysk_query_window's
        assert e.query_logical_all(cap=0) == ([], len(lids))
        assert e.query_logical_all(active_only=True, cap=0) == ([], len(active))
        for flag, want in ((False, lids), (True, active)):
            for cap in (1, max(1, len(want) // 3), len(want) + 5):
                part, pn = e.query_logical_all(active_only=flag, cap=cap)
                assert pn == len(want) and [bytes(x) for x in part] == [byid[l] for l in want[:cap]], (r, flag, cap)
        # rankings: the restated scores, best first, the later logical service first on equal scores, zero scores left out
        for metric, sc in scores.items():
            order = sorted(((s, dense.index(l), l) for l, s in sc.items() if s > 0), reverse=True)
            for k in (1, 7, 64):
                assert e.topn_logical(metric, k) == [(l, s, 0) for s, _, l in order[:k]], (r, metric, k)
                tops.setdefault((metric, k), set()).add(_raw_topn(e, metric, k))
        assert _code(lambda: e.topn_logical(ge.TOPN_ISSUE, 5)) == INVAL
        assert _code(lambda: e.topn(ge.TOPN_ACTIVE, 5)) == INVAL                # gysk_topn_svcs keeps rejecting it
        if not levels:
            assert _code(lambda: e.topn_logical(ge.TOPN_ACTIVE, 5)) == NOTSUP
        # exports of one logical id: the restated digest bit for bit, its Postgres text, the element-wise max of the registers
        for lid in lids:
            d = digests[lid]
            means, weights, mn, mx = e.export_logical_tdigest(lid)
            assert np.array_equal(weights, d.cent["weight"]) and means.tobytes() == d.cent["mean"].tobytes(), (r, lid)
            assert same_double(mn, d.minv) and same_double(mx, d.maxv), (r, lid, mn, d.minv, mx, d.maxv)
            assert e.export_logical_tdigest_pgtext(lid) == pgtext(means, weights), (r, lid)
            assert np.array_equal(e.export_logical_hll(lid), cells[lid]["regs"]), (r, lid)
        assert e.export_logical_tdigest(UNKNOWN) is None and e.export_logical_tdigest_pgtext(UNKNOWN) is None
        assert e.export_logical_hll(UNKNOWN) is None and _code(lambda: e.logical_quantiles(UNKNOWN, QS)) == NOENT
    assert all(len(v) == 1 for v in tops.values())                       # identical bytes on every rank
    # the quantiles of the exported digest agree with the row's t-digest fields as closely as the per-service pair does
    e = sh.engines[-1]
    logical_gap = quantile_gap(e, e.query_logical_all()[0], e.logical_quantiles)
    svc_gap = max(quantile_gap(x, x.query_window()[0], x.quantiles) for x in sh.engines)
    assert logical_gap <= max(svc_gap, 1e-12), (logical_gap, svc_gap)
    return active, scores


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_reads_equal_the_restatement(world, levels):
    """test_gpu_merge_exact's map (late members, ghost ids, connection-only members) plus two logical services of one
    connection-only member each, whose equal connection counts tie in the CONNS ranking; the last window leaves out every odd
    service, so their singletons drop out of the ACTIVE_ONLY read"""
    import torch
    rng = np.random.default_rng(1300 + 10 * world + levels)
    ids, conn_ids, ghost_ids = _stream_ids()
    sh = Shards(world, merge_levels=levels, **KW)
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    sh.set_map(np.append(glob, conn_ids[1:3]), np.append(logical, np.array([9006, 9005], dtype=np.uint64)))
    for w, t in enumerate((5, 10, 15)):
        ev = _events(rng, w, 20_000, ids, conn_ids)
        if w == 2:
            ev = ev[(ev["type"] == ge.EV_TASK) | ~np.isin(ev["svc_id"], ids[1::2])]
        sh.feed(ev, 1 << 16)
        sh.flush(t)
        if not w:
            continue
        active, scores = check_reads(torch, sh, levels)
        assert 9002 not in active and 9003 in active                       # ghosts only / connection events only
        c = scores[ge.TOPN_CONNS]
        assert c[9005] == c[9006] > 0                                        # the tie the ranking has to break
        if w == 2:
            odd, even = range(9117, 9148, 2), range(9116, 9148, 2)                  # the singletons of services 17, 19 ... / 16, 18 ...
            assert not any(l in active for l in odd) and any(l in active for l in even)
            if levels:
                assert sum(s > 0 for s in scores[ge.TOPN_ACTIVE].values()) > 2


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [False, True])
def test_reads_across_eviction_and_recycled_slots(levels):
    """test_gpu_merge_exact's eviction scenario: A (logical 7000 with B) is evicted, its slot goes to U outside the map, then A returns
    into another slot. One logical service, so every ranking asks for more than the map holds"""
    import torch
    sh = Shards(2, max_svcs=3, max_tasks=8, max_batch=1 << 14, cms_log2_width=10, idle_evict_secs=300, merge_levels=levels)
    A, B, U, F, G = (int(x) for x in synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 53)))
    host = {A: 0, F: 2, G: 4, U: 6, B: 1}
    sh.set_map(np.array([B, A], dtype=np.uint64), np.array([7000, 7000], dtype=np.uint64))
    rng = np.random.default_rng(46 + levels)

    def window(t, live, n=400):
        ev = np.zeros(n * len(live), dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = np.repeat(np.array(live, dtype=np.uint64), n)
        ev["host_idx"] = np.repeat(np.array([host[a] for a in live], dtype=np.uint32), n)
        ev["type"] = np.where(rng.random(len(ev)) < 0.8, ge.EV_RESP, ge.EV_ACCEPT)
        act = (ev["type"] == ge.EV_ACCEPT) & (rng.random(len(ev)) < 0.1)
        ev["type"][act] = ge.EV_ACTIVE
        ev["flags"][act] = rng.integers(1, 50, int(act.sum()))
        ev["value"] = np.minimum(np.exp(rng.normal(np.log(3000.0), 1.2, len(ev))), 9.0e8).astype(np.uint32)
        ev["flow_key"] = rng.integers(1, 1 << 62, len(ev), dtype=np.uint64)
        ev["tsec"] = t
        ev["tsec"][act] = (rng.random(int(act.sum())) * 300).astype(np.float32).view(np.uint32)
        sh.feed(ev[rng.permutation(len(ev))], 1 << 14)
        sh.flush(t)
        return set().union(*[set(int(i) for i in e.evicted_ids()) for e in sh.engines])

    for t in (5, 10, 200, 400):
        window(t, [A, B, F, G] if t < 100 else [B, F, G])
    assert window(606, [B, F]) == {A}
    check_reads(torch, sh, levels)
    window(620, [B, F, U])                                                  # U takes A's slot
    check_reads(torch, sh, levels)
    assert window(720, [B, F, U]) == {G}
    window(730, [A, B, F, U])                                               # A returns into G's slot
    active, scores = check_reads(torch, sh, levels)
    assert active == [7000] and scores[ge.TOPN_QPS][7000] > 0


@pytest.mark.gpu
def test_every_read_needs_a_finished_merge():
    """GYSK_ERR_INVAL without a map, with a map before a merge, and after gysk_merge_prepare before gysk_merge_finish"""
    rng = np.random.default_rng(5)
    ids, conn_ids, ghost_ids = _stream_ids()
    e = ge.Engine(merge_levels=True, **KW)
    calls = [lambda: e.query_logical_all(), lambda: e.query_logical_all(active_only=True, cap=0), lambda: e.topn_logical(ge.TOPN_QPS),
             lambda: e.topn_logical(ge.TOPN_ACTIVE, 64), lambda: e.export_logical_tdigest(9000), lambda: e.export_logical_tdigest_pgtext(9000),
             lambda: e.logical_quantiles(9000, QS), lambda: e.export_logical_hll(9000)]
    assert [_code(c) for c in calls] == [INVAL] * len(calls)
    e.set_logical_map(*logical_map(rng, ids, conn_ids, ghost_ids))
    assert [_code(c) for c in calls] == [INVAL] * len(calls)
    _run_engines([e], rng, ids, conn_ids, times=[5])
    e.merge_prepare()
    e.sync()
    assert [_code(c) for c in calls] == [INVAL] * len(calls)
    e.merge_finish()
    rows, n = e.query_logical_all()
    assert n == len(rows) > 0 and e.topn_logical(ge.TOPN_QPS) and e.export_logical_hll(9000) is not None
    e.close()


@pytest.mark.gpu
def test_reads_leave_the_merge_unchanged():
    """the new reads change nothing the merge left: the arena's region bytes and the by-id rows are the same after them, the next merge
    still takes six / five launches with / without the flag; the ranking takes as many launches as gysk_topn_svcs, the ACTIVE_ONLY read
    one select launch more than the plain one"""
    import torch
    rng = np.random.default_rng(77)
    ids, conn_ids, ghost_ids = _stream_ids()
    on, off = ge.Engine(merge_levels=True, **KW), ge.Engine(**KW)
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    lids = list(dict.fromkeys(logical.tolist()))
    for e in (on, off):
        e.set_logical_map(glob, logical)
    _run_engines([on, off], rng, ids, conn_ids, times=[5, 10, 15])

    def launches(e, fn):
        k0 = e.stats()["kernel_launches"]
        fn()
        return e.stats()["kernel_launches"] - k0

    for e, merge_launches in ((on, 6), (off, 5)):
        assert launches(e, lambda: _emulate_collectives(torch, [e])) == merge_launches
        regions = [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in e.merge_buffers()]
        rows = _raw_logical(e, lids)
        assert launches(e, lambda: e.query_logical_all(cap=len(lids))) == 1
        assert launches(e, lambda: e.query_logical_all(cap=0)) == 0
        assert launches(e, lambda: e.query_logical_all(active_only=True, cap=len(lids))) == 2
        assert launches(e, lambda: e.topn_logical(ge.TOPN_QPS, 64)) == launches(e, lambda: e.topn(ge.TOPN_QPS, 64))
        for lid in lids + [UNKNOWN]:
            for fn in (e.export_logical_tdigest, e.export_logical_tdigest_pgtext, e.export_logical_hll):
                assert launches(e, lambda: fn(lid)) == 0
        for m in (ge.TOPN_QPS, ge.TOPN_CONNS, ge.TOPN_NET) + ((ge.TOPN_ACTIVE,) if e is on else ()):
            e.topn_logical(m, 64)
        e.query_logical_all(active_only=True)
        assert [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in e.merge_buffers()] == regions
        assert _raw_logical(e, lids) == rows
        assert launches(e, lambda: _emulate_collectives(torch, [e])) == merge_launches
        assert _raw_logical(e, lids) == rows


def test_null_engine_and_header():
    """without an engine every new entry point is GYSK_ERR_INVAL (no device needed); the binding's GYSK_TOPN_ACTIVE is the header's"""
    L = ge.load_library()
    n, k = C.c_uint32(), C.c_uint32()
    out = (ge.TopnEntry * 4)()
    means, weights = np.zeros(4), np.zeros(4, dtype=np.uint64)
    buf = C.create_string_buffer(64)
    qs, q = np.array(QS), np.zeros(3)
    regs = np.zeros(1 << 16, dtype=np.uint8)
    assert L.gysk_query_logical_all(None, 0, None, 0, C.byref(n)) == INVAL
    assert L.gysk_topn_logical(None, ge.TOPN_QPS, 4, out, C.byref(k)) == INVAL
    assert L.gysk_export_logical_tdigest(None, 1, ge._p(means), ge._p(weights), 4, C.byref(n), None, None) == INVAL
    assert L.gysk_export_logical_tdigest_pgtext(None, 1, buf, len(buf)) == INVAL
    assert L.gysk_query_logical_quantiles(None, 1, ge._p(qs), 3, ge._p(q)) == INVAL
    assert L.gysk_export_logical_hll(None, 1, ge._p(regs)) == INVAL
    hdr = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert int(re.search(r"GYSK_TOPN_ACTIVE\s*=\s*(\d+)", hdr).group(1)) == ge.TOPN_ACTIVE == 4
