"""gysk_query_window / gysk_query_tasks / gysk_query_task_window against the CPU oracle (make_pair / feed_both), over several
flushes with idle eviction on: the rows are exactly the oracle's live ids, grouped by host and ordered by id; each service row is
byte-equal to gysk_query_svcs of its id and equals a restatement of the summary from the oracle's exports; each process row equals
the reference's percentile rule on the exported task histograms. gysk_query_svcs and gysk_query_tasks over several chunks of live,
unknown and zero ids; gysk_query_flows and gysk_register_ids over several chunks."""
import ctypes as C

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests.util import make_pair, feed_both

pytestmark = pytest.mark.gpu

M32 = 0xFFFFFFFF
HOSTS = 5


def _stream(rng, svc_ids, task_ids, n):
    """RESP (70 %), TCP (20 %) and TASK (10 %) events; a service always comes from host id % 5"""
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    kind = rng.random(n)
    resp, tcp = kind < 0.7, (kind >= 0.7) & (kind < 0.9)
    task = ~(resp | tcp)
    ev["svc_id"][resp | tcp] = rng.choice(svc_ids, int((resp | tcp).sum()))
    ev["svc_id"][task] = rng.choice(task_ids, int(task.sum())) if len(task_ids) else 0
    ev["type"][resp] = ge.EV_RESP
    ev["type"][tcp] = ge.EV_ACCEPT
    ev["type"][task] = ge.EV_TASK
    ev["value"][resp] = rng.lognormal(9.0, 1.5, int(resp.sum())).astype(np.uint32) + 1
    ev["value"][tcp] = rng.integers(0, 1 << 20, int(tcp.sum()))
    ev["value"][task] = rng.integers(0, 400, int(task.sum()))
    ev["flow_key"] = rng.integers(0, 1 << 62, n, dtype=np.uint64)
    ev["flow_key"][task] = (rng.integers(0, 70000, int(task.sum())).astype(np.uint64) << np.uint64(32)) | rng.integers(0, 70000, int(task.sum())).astype(np.uint64)
    ev["host_idx"] = (ev["svc_id"] % HOSTS).astype(np.uint32)
    return ev


def _live(orc, ids):
    return [int(i) for i in ids if orc.export_hist(int(i), ge.HIST_RESP_ALL) is not None]


def _order(ids):
    return sorted(ids, key=lambda i: (i % HOSTS, i))


def _svcs_rows(eng, ids):
    ids = np.ascontiguousarray(ids, dtype=np.uint64)
    out = (ge.SvcSummary * max(len(ids), 1))()
    assert eng.L.gysk_query_svcs(eng.h, ids.ctypes.data_as(C.c_void_p), len(ids), out) == 0
    return out[: len(ids)]


class _GyoSerial(C.Structure):
    _fields_ = [("count", C.c_uint64), ("sum", C.c_int64)]


class _GyoHist(C.Structure):
    """gyo_hist of oracle/gysk_oracle.h"""
    _fields_ = [("stats", _GyoSerial * 16), ("total_count", C.c_uint64), ("max_val", C.c_int64), ("cls", C.c_int32), ("tkind", C.c_int32)]


def _pct(cls, t_is_int, hist, pcts):
    """the oracle's get_percentiles (gyo_hist_percentiles) on an exported histogram {stats, total, max}"""
    O = po.lib()
    h = _GyoHist()
    O.gyo_hist_init(C.byref(h), C.c_int(cls), C.c_int(1 if t_is_int else 0))      # GYO_T_INT / GYO_T_INT64
    for i, (c, v) in enumerate(zip(hist[0]["count"].tolist(), hist[0]["sum"].tolist())):
        h.stats[i].count, h.stats[i].sum = c, v
    h.total_count, h.max_val = hist[1], hist[2]
    p = (C.c_float * len(pcts))(*pcts)
    out = (C.c_int64 * len(pcts))()
    O.gyo_hist_percentiles(C.byref(h), p, C.c_size_t(len(pcts)), out, None)
    return list(out)


def _restate(eng, orc, id_, row):
    """the service summary restated from the oracle's exports and its get_percentiles (gyo_hist_percentiles), and from the
    engine's sketch exports (HLL registers, centroids) through the host estimators"""
    L = eng.L
    last = orc.export_hist(id_, ge.HIST_RESP_LAST)
    assert row.nqrys_5s == last[1] and row.total_resp_5sec == int(last[0]["sum"].sum())
    assert [row.p95_5s_resp_ms, row.p99_5s_resp_ms, row.p25_5s_resp_ms] == _pct(0, 0, last, [95, 99, 25])
    h5m = orc.export_hist(id_, ge.HIST_RESP_5MIN)
    assert [row.p95_5min_resp_ms, row.p99_5min_resp_ms] == _pct(0, 0, h5m, [95, 99]) and row.nqrys_5min == h5m[1]
    h5d = orc.export_hist(id_, ge.HIST_RESP_5DAY)
    assert [row.p95_5day_resp_ms] == _pct(0, 0, h5d, [95]) and row.nqrys_5day == h5d[1]
    hall = orc.export_hist(id_, ge.HIST_RESP_ALL)
    assert [row.p95_all_resp_ms, row.p99_all_resp_ms] == _pct(0, 0, hall, [95, 99])
    assert row.nqrys_all == hall[1] and row.max_resp_ms == hall[2]
    _, clast, call_cnt, call_kb = orc.export_conn(id_)
    assert (row.nconns_5s, row.kbytes_5s, row.nconns_all, row.kbytes_all) == (clast & M32, clast >> 32, call_cnt, call_kb)
    aux = orc.export_aux(id_)
    assert (row.nconns_active, row.active_kbytes) == (aux["act_last"] & M32, aux["act_last"] >> 32)
    assert (row.cli_errors, row.ser_errors) == (aux["err_last"] & M32, aux["err_last"] >> 32)
    assert row.max_rtt_msec == aux["rtt_last"]
    st = orc.export_state(id_)
    assert (row.curr_state, row.curr_issue, row.issue_bit_hist, row.high_resp_bit_hist) == st[:4]
    regs = eng.export_hll(id_)
    assert row.distinct_clients == L.gysk_hll_estimate(regs.ctypes.data_as(C.c_void_p), eng.cfg.hll_p)
    means, w, mn, mx = eng.export_tdigest(id_)
    assert row.td_count == int(w.sum())
    for q, v in ((0.50, row.td_p50_us), (0.95, row.td_p95_us), (0.99, row.td_p99_us)):
        want = L.gysk_tdigest_quantile(means.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p), len(means), mn, mx, q)
        assert (np.isnan(v) and np.isnan(want)) or v == want, (hex(id_), q, v, want)


def _check_window(eng, orc, fed, active, restate=True):
    live = _live(orc, fed)
    rows, n = eng.query_window()
    got = [r.glob_id for r in rows]
    assert n == len(rows) and got == _order(live)
    assert all(r.found == 1 for r in rows)
    # byte-equal to the by-id read of the same ids (NaN quantiles included)
    by_id = _svcs_rows(eng, got)
    assert [bytes(a) for a in rows] == [bytes(b) for b in by_id]
    if restate:
        for r in rows:
            _restate(eng, orc, r.glob_id, r)
    # the same read with each row's host, in one call
    hrows, hosts, hn = eng.query_window_hosts()
    assert hn == n and [bytes(r) for r in hrows] == [bytes(r) for r in rows] and hosts.tolist() == [i % HOSTS for i in got]
    # host filters: each one is the slice of its host, and together they are the whole read
    union = []
    for h in range(HOSTS + 1):
        hr, hn = eng.query_window(host_idx=h)
        assert hn == len(hr) and [r.glob_id for r in hr] == [i for i in got if i % HOSTS == h]
        union += [bytes(r) for r in hr]
    assert union == [bytes(r) for r in rows]
    # only the ids with events in the closed window
    ar, an = eng.query_window(active_only=True)
    assert [r.glob_id for r in ar] == _order([i for i in live if i in active])
    assert [bytes(r) for r in ar] == [bytes(r) for r in rows if r.glob_id in active]
    return rows


def _check_tasks(eng, orc, task_ids):
    L = eng.L
    task_ids = [int(i) for i in task_ids]
    ids = task_ids + [0xDEAD0001, 0]
    rows = eng.query_tasks(ids)
    for id_, r in zip(ids, rows):
        hists = [eng.export_hist(id_, w) for w in (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY)]
        if hists[0] is None:
            assert bytes(r) == bytes(ge.TaskSummary(aggr_task_id=id_)), hex(id_)
            continue
        assert r.found == 1 and r.aggr_task_id == id_ and r.host_idx == id_ % HOSTS
        for k, (h, cls) in enumerate(zip(hists, (6, 3, 3))):
            o = orc.export_hist(id_, ge.HIST_TASK_CPU_PCT + k)
            assert np.array_equal(o[0], h[0]) and o[1] == h[1]
        p95 = [_pct(cls, 1, h, [95])[0] for h, cls in zip(hists, (6, 3, 3))]
        assert [r.p95_cpu_pct, r.p95_cpu_delay_ms, r.p95_blkio_delay_ms] == p95
        assert r.nsamples == hists[0][1]
        tl = orc.task_last(id_)
        assert list(r.last_count) == [int(tl[0]), int(tl[2]), int(tl[4])]
        assert list(r.last_sum) == [int(tl[k].view(np.int64)) for k in (1, 3, 5)]
    known = [i for i in task_ids if eng.export_hist(i, ge.HIST_TASK_CPU_PCT) is not None]
    wrows, wn = eng.query_task_window()
    assert wn == len(wrows) and [r.aggr_task_id for r in wrows] == _order(known)
    by_id = {r.aggr_task_id: bytes(r) for r in rows}
    assert [bytes(r) for r in wrows] == [by_id[r.aggr_task_id] for r in wrows]
    ar, _ = eng.query_task_window(active_only=True)
    assert [r.aggr_task_id for r in ar] == [r.aggr_task_id for r in wrows if sum(r.last_count)]
    for h in range(HOSTS):
        hr, _ = eng.query_task_window(host_idx=h)
        assert [bytes(r) for r in hr] == [bytes(r) for r in wrows if r.host_idx == h]


def _run(seed=1, nsvc=300, ntask=60, flushes=4, **kw):
    rng = np.random.default_rng(seed)
    eng, orc = make_pair(idle_evict_secs=10, **kw)
    svc_ids = rng.choice(1 << 40, nsvc, replace=False).astype(np.uint64) + 1
    task_ids = rng.choice(1 << 40, ntask, replace=False).astype(np.uint64) + (1 << 41)
    fed = set()
    # before any flush: every id is live, none had events in a closed window
    ev = _stream(rng, svc_ids[: nsvc // 2], task_ids, 4000)
    feed_both(eng, orc, ev, 1500)
    fed |= {int(i) for i in ev["svc_id"][ev["type"] != ge.EV_TASK]}
    _check_window(eng, orc, fed, set())
    for f in range(flushes):
        # later windows go quiet for a part of the services, so the 10-s idle rule evicts them, and new ones take their slots
        lo = (f * nsvc) // (2 * flushes)
        ev = _stream(rng, svc_ids[lo: lo + nsvc // 2], task_ids[: ntask - 10 * f], 6000)
        feed_both(eng, orc, ev, 2000)
        tsec = 5 * (f + 1) + (30 if f == flushes - 1 else 0)
        eng.flush(tsec)
        orc.flush(tsec)
        win = {int(i) for i in ev["svc_id"][ev["type"] != ge.EV_TASK]}
        fed |= win
        if f == flushes - 1 and f:
            assert len(eng.evicted_ids()) > 0
        _check_window(eng, orc, fed, win)
        _check_tasks(eng, orc, task_ids)
    return eng, orc


def test_window_read_equals_the_oracle_over_several_flushes():
    _run()


@pytest.mark.parametrize("cfg", [dict(hll_p=4), dict(hll_p=16), dict(td_compression=10), dict(td_compression=256)])
def test_window_read_at_the_edges_of_the_sketch_settings(cfg):
    _run(seed=2, flushes=2, **cfg)


@pytest.mark.parametrize("hot", ["off", "forced"])
def test_window_read_with_hot_rows(monkeypatch, hot):
    monkeypatch.setenv("GYSK_HOT_ROWS", "0" if hot == "off" else "2048")
    monkeypatch.setenv("GYSK_HOT_MIN", "4096" if hot == "off" else "1")
    _run(seed=3, flushes=2)


def test_capacity_count_only_and_errors():
    eng, orc = _run(seed=4, flushes=1)
    rows, n = eng.query_window()
    assert n > 40
    few, n2 = eng.query_window(cap=17)
    assert n2 == n and [bytes(r) for r in few] == [bytes(r) for r in rows[:17]]
    none, n3 = eng.query_window(cap=0)
    assert n3 == n and len(none) == 0
    trows, tn = eng.query_task_window()
    tfew, tn2 = eng.query_task_window(cap=3)
    assert tn2 == tn and [bytes(r) for r in tfew] == [bytes(r) for r in trows[:3]]
    k = C.c_uint32()
    assert eng.L.gysk_query_window(eng.h, -1, 2, None, 0, C.byref(k)) == -22        # unknown flag
    assert eng.L.gysk_query_window(eng.h, -1, 0, None, 5, C.byref(k)) == -22
    assert eng.L.gysk_query_task_window(eng.h, -1, 0, None, 0, None) == -22


def test_read_in_three_passes_and_recycled_slots():
    """more rows than two passes of the page-locked stage hold (8192 rows each); an evicted id is absent and the id that took
    its slot is read with its own host and values"""
    rng = np.random.default_rng(5)
    eng, orc = make_pair(max_svcs=1 << 15, idle_evict_secs=10)
    ids = (rng.choice(1 << 40, 20000, replace=False) + 1).astype(np.uint64)
    ev = np.zeros(len(ids) * 2, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = np.repeat(ids, 2)
    ev["type"] = ge.EV_RESP
    ev["value"] = rng.integers(1, 1 << 20, len(ev))
    ev["host_idx"] = (ev["svc_id"] % HOSTS).astype(np.uint32)
    feed_both(eng, orc, ev, 1 << 16)
    eng.flush(5); orc.flush(5)
    _check_window(eng, orc, ids, set(int(i) for i in ids), restate=False)
    # only the first 1000 stay busy: the rest is evicted at t = 40, and 500 new ids take recycled slots
    keep = ev[np.isin(ev["svc_id"], ids[:1000])]
    nevicted = 0
    for t in (10, 20, 30, 40):
        feed_both(eng, orc, keep, 1 << 16)
        eng.flush(t); orc.flush(t)
        nevicted += len(eng.evicted_ids())
    assert nevicted == 19000
    new = (rng.choice(1 << 40, 500, replace=False) + (1 << 42)).astype(np.uint64)
    ev2 = np.zeros(len(new), dtype=ge.EVENT_DTYPE)
    ev2["svc_id"] = new
    ev2["type"] = ge.EV_RESP
    ev2["value"] = 2500
    ev2["host_idx"] = (new % HOSTS).astype(np.uint32)
    feed_both(eng, orc, np.concatenate([keep, ev2]), 1 << 16)
    eng.flush(45); orc.flush(45)
    fed = [int(i) for i in ids] + [int(i) for i in new]
    rows = _check_window(eng, orc, fed, set(int(i) for i in ids[:1000]) | set(int(i) for i in new), restate=False)
    assert len(rows) == 1500 and {r.glob_id for r in rows} == set(int(i) for i in ids[:1000]) | set(int(i) for i in new)
    for r in rows[:: 50]:
        _restate(eng, orc, r.glob_id, r)


def test_by_id_read_across_chunks():
    """gysk_query_svcs of more than two 1024-id chunks, live ids shuffled among unknown ids and id 0: a live row is byte-equal to the
    window row of its id, every other row to the not-found row (the id, found = 0, every other byte zero, NaN quantiles)"""
    rng = np.random.default_rng(7)
    eng = ge.Engine(max_svcs=1 << 12)
    ids = (rng.choice(1 << 40, 1500, replace=False) + 1).astype(np.uint64)
    ev = _stream(rng, ids, np.zeros(0, dtype=np.uint64), 30000)
    eng.ingest_events(ev)
    eng.sync()
    eng.flush(5)
    rows, n = eng.query_window()
    win = {r.glob_id: bytes(r) for r in rows}
    assert n > 1000
    unknown = (rng.choice(1 << 40, 1200, replace=False) + (1 << 42)).astype(np.uint64)
    q = np.concatenate([np.array(list(win), dtype=np.uint64), unknown, np.zeros(300, dtype=np.uint64)])[rng.permutation(n + 1500)]
    assert len(q) > 2 * 1024
    nan = float("nan")
    for id_, r in zip(q.tolist(), _svcs_rows(eng, q)):
        want = win.get(id_) or bytes(ge.SvcSummary(glob_id=id_, td_p50_us=nan, td_p95_us=nan, td_p99_us=nan))
        assert bytes(r) == want, hex(id_)
    eng.close()


def test_task_flow_and_register_reads_across_chunks():
    """gysk_query_tasks, gysk_query_flows and gysk_register_ids over more than two 1024-entry chunks. Live process ids shuffled among
    unknown ids and id 0: a live row is byte-equal to the window row of its id, every other row to the zero row with only
    aggr_task_id set. Flow keys of the stream among random keys: each estimate is the min over the rows of the exported count-min
    table, in the current and in the last window. Registered ids are counted and read back as found."""
    from oracle import pyoracle as po
    rng = np.random.default_rng(8)
    eng = ge.Engine(max_svcs=1 << 12, max_tasks=1 << 12)
    svc_ids = (rng.choice(1 << 40, 300, replace=False) + 1).astype(np.uint64)
    task_ids = (rng.choice(1 << 40, 1500, replace=False) + (1 << 41)).astype(np.uint64)
    ev = _stream(rng, svc_ids, task_ids, 60000)
    eng.ingest_events(ev)
    eng.sync()
    eng.flush(5)
    ev2 = _stream(rng, svc_ids, task_ids, 20000)
    eng.ingest_events(ev2)
    eng.sync()

    rows, n = eng.query_task_window()
    win = {r.aggr_task_id: bytes(r) for r in rows}
    assert n > 1000
    unknown = (rng.choice(1 << 40, 1200, replace=False) + (1 << 42)).astype(np.uint64)
    q = np.concatenate([np.array(list(win), dtype=np.uint64), unknown, np.zeros(300, dtype=np.uint64)])[rng.permutation(n + 1500)]
    assert len(q) > 2 * 1024
    for id_, r in zip(q.tolist(), eng.query_tasks(q)):
        assert bytes(r) == (win.get(id_) or bytes(ge.TaskSummary(aggr_task_id=id_))), hex(id_)

    tcp = np.concatenate([ev, ev2])
    tcp = tcp[(tcp["type"] == ge.EV_ACCEPT)]
    keys = np.concatenate([np.unique(tcp["flow_key"])[:1500], rng.integers(0, 1 << 62, 1000, dtype=np.uint64)])[rng.permutation(2500)]
    O = po.lib()
    depth, log2w = eng.cfg.cms_depth, eng.cfg.cms_log2_width
    for lw in (False, True):
        tbl = eng.export_cms(last_window=lw).reshape(depth, -1)
        est = eng.query_flows(keys, last_window=lw)
        assert est["flow_key"].tolist() == keys.tolist()
        for k, e_ in zip(keys.tolist(), est):
            cells = [int(tbl[r, O.gyo_cms_index(k, r, log2w)]) for r in range(depth)]
            assert (e_["count"], e_["kbytes"]) == (min(c & M32 for c in cells), min(c >> 32 for c in cells)), (hex(k), lw)
    eng.close()

    eng = ge.Engine(max_svcs=1 << 12, max_tasks=1 << 12)
    for is_task, count in ((False, 2500), (True, 2100)):
        ids = (rng.choice(1 << 40, count, replace=False) + 1).astype(np.uint64)
        eng.register_ids(ids, is_task=is_task)
        assert eng.stats()["ntasks" if is_task else "nsvcs"] == count
        found = [r.found for r in eng.query_tasks(ids)] if is_task else [r.found for r in _svcs_rows(eng, ids)]
        assert found == [1] * count
    eng.close()


def test_same_stream_different_slots_gives_identical_bytes():
    """slot numbers follow insertion order (a race inside a batch); the rows do not. The second engine creates the services in the
    reverse order, in three batches of connection events, then both take the same response batches."""
    rng = np.random.default_rng(6)
    ids = (rng.choice(1 << 40, 3000, replace=False) + 1).astype(np.uint64)
    tcp = np.zeros(len(ids), dtype=ge.EVENT_DTYPE)
    tcp["svc_id"] = ids
    tcp["type"] = ge.EV_CONNECT
    tcp["value"] = 4096
    tcp["flow_key"] = rng.integers(0, 1 << 62, len(ids), dtype=np.uint64)
    tcp["host_idx"] = (ids % HOSTS).astype(np.uint32)
    resp = _stream(rng, ids, np.zeros(0, dtype=np.uint64), 60000)
    out = []
    for order, batch in ((slice(None), len(ids)), (slice(None, None, -1), 1000)):
        eng = ge.Engine()
        t = np.ascontiguousarray(tcp[order])
        for off in range(0, len(t), batch):
            eng.ingest_events(t[off: off + batch])
            eng.sync()
        for off in range(0, len(resp), 20000):
            eng.ingest_events(resp[off: off + 20000])
            eng.sync()
        eng.flush(5)
        rows, n = eng.query_window()
        out.append((b"".join(bytes(r) for r in rows), n))
        eng.close()
    assert out[0][1] == len(ids) and out[0] == out[1]
