"""The rest of the 5-s listener walk on the device: LISTENER_DAY_STATS rows (gysk_query_day_stats) and each host's listener counts
(gysk_query_host_listen), against a restatement built on the CPU oracle's own 5-day level, qps / active-connection histograms and listener
state (common/gy_socket_stat.cc:2101-2117, :4242-4277), and against the engine's own window read."""
import ctypes as C

import numpy as np
import pytest

from gyeeta_b200 import engine as ge, synth
from oracle import pyoracle as po
from tests.util import feed_both, make_pair

pytestmark = pytest.mark.gpu

M32 = 0xFFFFFFFF
AGE = 900                       # tcur > tstart + 15 * 60, gy_socket_stat.cc:2102


class _Hist(C.Structure):       # gyo_hist (oracle/gysk_oracle.h)
    _fields_ = [("stats", C.c_uint8 * 256), ("total_count", C.c_uint64), ("max_val", C.c_int64), ("cls", C.c_int32), ("tkind", C.c_int32)]


def _pct(h, cls, tkind):
    """gyo_hist_percentiles({95, 25}) of an exported (stats, total, max) triple"""
    ser, total, mx = h
    x = _Hist(total_count=total, max_val=mx, cls=cls, tkind=tkind)
    full = np.zeros(16, dtype=po.SERIAL_DTYPE)
    full[:15] = ser
    C.memmove(x.stats, full.ctypes.data, 256)
    L = po.lib()
    L.gyo_hist_percentiles.restype = None
    L.gyo_hist_percentiles.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    pcts, out = (C.c_float * 2)(95.0, 25.0), (C.c_int64 * 2)()
    L.gyo_hist_percentiles(C.byref(x), pcts, 2, out, None)
    return out[0], out[1]


def _i64(v):
    return ((int(v) + (1 << 63)) % (1 << 64)) - (1 << 63)


def oracle_day_stats(orc, id_):
    """gyo_day_stats: the LISTENER_DAY_STATS record of one service from the oracle's 5-day level (GY_HISTOGRAM percentiles, clamped at 0
    like TIME_HISTOGRAM::get_stats) and its qps / active-connection histograms, each value converted to uint32"""
    lvl = orc.export_hist(id_, ge.HIST_RESP_5DAY)
    p95, p25 = (max(v, 0) for v in _pct(lvl, 0, 0))
    q95, q25 = _pct(orc.export_hist(id_, ge.HIST_QPS), 2, 1)              # SEMI_LOG_HASH_LO, int
    a95, a25 = _pct(orc.export_hist(id_, ge.HIST_ACTIVE_CONN), 6, 1)      # HASH_1_3000, int
    tsum = _i64(sum(int(s) % (1 << 64) for s in lvl[0]["sum"].tolist()))
    return (int(id_), int(lvl[0]["count"].sum()), tsum, p95 & M32, p25 & M32, q95 & M32, q25 & M32, a95 & M32, a25 & M32)


def oracle_host_listen(orc, ids_by_host, evaluated):
    """gyo_host_listen: per host {nlisten, services evaluated at the last flush with issue bit 0 set, ... of them SEVERE or worse}"""
    out = []
    for h in sorted(ids_by_host):
        ni = ns = 0
        for id_ in ids_by_host[h]:
            st = orc.export_state(id_)
            if id_ in evaluated and st[2] & 1:
                ni += 1
                ns += st[0] >= ge.STATE_SEVERE
        out.append((h, len(ids_by_host[h]), ni, ns))
    return out


class Tracker:
    """what the test knows of its own stream: host of every id, tsec of the first flush that saw it, ids with events in the open window"""

    def __init__(self):
        self.host, self.first, self.pending, self.evaluated, self.last = {}, {}, set(), set(), 0

    def feed(self, ev):
        for id_, h in zip(ev["svc_id"].tolist(), ev["host_idx"].tolist()):
            self.host.setdefault(id_, h)
            self.pending.add(id_)

    def flush(self, tsec, evicted=()):
        for id_ in evicted:
            self.host.pop(id_, None); self.first.pop(id_, None)
        for id_ in self.host:
            self.first.setdefault(id_, tsec or 1)
        self.evaluated, self.pending, self.last = self.pending & set(self.host), set(), tsec

    def old(self):
        return {i for i, f in self.first.items() if self.last > f + AGE}

    def by_host(self):
        d = {}
        for i, h in self.host.items():
            d.setdefault(h, []).append(i)
        return d


def check_reads(eng, orc, tr):
    rows, hosts, n = eng.query_day_stats()
    got = [r.astuple() for r in rows]
    old = tr.old()
    want_ids = sorted(old, key=lambda i: (tr.host[i], i))
    assert n == len(old) and [g[0] for g in got] == want_ids and hosts.tolist() == [tr.host[i] for i in want_ids]
    assert got == [oracle_day_stats(orc, i) for i in want_ids]
    # ids / order / hosts = the window read restricted to the old enough, for every host filter
    for h in [-1] + sorted(set(tr.host.values())):
        w, wh, _ = eng.query_window_hosts(h)
        keep = [k for k, r in enumerate(w) if r.glob_id in old]
        r2, h2, n2 = eng.query_day_stats(h)
        assert [r.glob_id for r in r2] == [w[k].glob_id for k in keep] and h2.tolist() == [int(wh[k]) for k in keep] and n2 == len(keep)
    # per-host counts: the oracle, and the engine's own window reads
    hl, nh = eng.query_host_listen()
    got_hl = [(r.host_idx, r.nlisten, r.nlisten_issue, r.nlisten_severe) for r in hl]
    assert nh == len(got_hl) and got_hl == oracle_host_listen(orc, tr.by_host(), tr.evaluated)
    _w, wh, _ = eng.query_window_hosts(-1)
    a, ah, _ = eng.query_window_hosts(-1, active_only=True)
    for h, nl, ni, ns in got_hl:
        assert nl == int((wh == h).sum())
        assert ni == sum(1 for r, x in zip(a, ah) if x == h and r.issue_bit_hist & 1)
        assert ns == sum(1 for r, x in zip(a, ah) if x == h and r.issue_bit_hist & 1 and r.curr_state >= ge.STATE_SEVERE)
    return got_hl


# flush times: the first services are seen at 5; 905 is exactly 900 s later (no row), 906 the first second with rows
TIMES = [5 + 40 * w for w in range(22)] + [905, 906, 946, 986, 1026, 1066, 1106, 1146]


@pytest.mark.parametrize("kw,env", [
    (dict(), {}),
    (dict(), {"GYSK_HOT_ROWS": "2048", "GYSK_HOT_MIN": "8"}),                     # hot rows taken from the first batch on
    (dict(hll_p=4, td_compression=10), {}),
    (dict(hll_p=16, td_compression=256), {}),
], ids=["default", "hot_rows", "edges_low", "edges_high"])
def test_day_stats_and_host_counts_equal_the_oracle(monkeypatch, kw, env):
    """a stream that turns slow, error-prone and busy so that listeners reach BAD and SEVERE past the 100-s rule; after every flush the
    day-stats rows and host counts equal the restatement; services that stop sending keep their rows (stale); services that start late
    have none"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(7)
    nsvc = 48
    eng, orc = make_pair(max_svcs=256, max_tasks=16, max_batch=1 << 14, **kw)
    ids = synth.service_ids(nsvc)
    tr = Tracker()
    seen_issue = seen_severe = 0
    stale_rows = 0
    for w, t in enumerate(TIMES):
        n = 6000
        k = rng.integers(0, nsvc, n)
        k = k[(k < 36) | (w >= 10)]                                         # services 36.. start at window 10: young to the end
        k = k[~((k % 7 == 0) & (w >= 24))]                                   # every 7th service falls silent: stale, still a row
        ev = np.zeros(len(k), dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = ids[k]; ev["host_idx"] = k % 3; ev["type"] = ge.EV_RESP
        slow = (w >= 14) & (k % 4 == 0)
        ev["value"] = np.minimum(np.exp(rng.normal(np.log(20_000.0), 1.0, len(k))) * np.where(slow, 8.0, 1.0), 9e8).astype(np.uint32)
        ev["flow_key"] = rng.integers(0, 1 << 16, len(k))
        err = (w >= 10) & (k % 5 == 1) & (rng.random(len(k)) < (0.7 if w % 2 else 0.15))
        ev["flags"] = np.where(err, ge.EVF_SER_ERROR, 0)
        if w >= 18:
            ev = np.concatenate([ev] + [ev[(k % 4 == 2)]] * 5)
        if w % 3 == 0:
            act = np.zeros(36, dtype=ge.EVENT_DTYPE)
            act["svc_id"] = ids[:36]; act["host_idx"] = np.arange(36) % 3; act["type"] = ge.EV_ACTIVE; act["flow_key"] = 77
            act["flags"] = np.where((np.arange(36) % 8 == 3) & (w >= 20), 400, 3 + (np.arange(36) % 5))
            ev = np.concatenate([ev, act])
        tr.feed(ev)
        feed_both(eng, orc, ev, 1 << 14)
        eng.flush(t); orc.flush(t); tr.flush(t)
        hl = check_reads(eng, orc, tr)
        seen_issue += sum(ni - ns for _h, _n, ni, ns in hl)
        seen_severe += sum(ns for _h, _n, _ni, ns in hl)
        stale_rows += len(tr.old() - tr.evaluated)
        if t == 905:
            assert eng.query_day_stats(cap=0)[2] == 0
        if t == 906:
            assert eng.query_day_stats(cap=0)[2] == 36
    assert seen_issue > 0 and seen_severe > 0 and stale_rows > 0
    assert len(tr.host) == nsvc and len(tr.old()) == 36


def test_day_stats_boundary_recycled_slots_and_partial_reads():
    """900 s after the first flush gives no row, 901 s one; an evicted service's slot, taken by a new id, inherits nothing and gives no
    row until the new id's own 900 s; count-only and cap < n calls"""
    eng, orc = make_pair(max_svcs=64, max_tasks=16, max_batch=1 << 14, idle_evict_secs=300)
    keep, gone, fresh = (synth.service_ids(30)[a:b] for a, b in ((0, 10), (10, 20), (20, 30)))
    tr = Tracker()

    def window(t, ids, seed):
        rng = np.random.default_rng(seed)
        ev = np.zeros(600, dtype=ge.EVENT_DTYPE)
        k = rng.integers(0, len(ids), 600)
        ev["svc_id"] = ids[k]; ev["host_idx"] = (ids[k] % 4).astype(np.uint32); ev["type"] = ge.EV_RESP
        ev["value"] = rng.integers(100, 3_000_000, 600)
        tr.feed(ev)
        feed_both(eng, orc, ev, 1 << 14)
        eng.flush(t); orc.flush(t)
        ev_ids = eng.evicted_ids()
        assert sorted(ev_ids.tolist()) == sorted(orc.evicted_ids()[0].tolist())
        tr.flush(t, ev_ids.tolist())
        return ev_ids

    window(100, np.concatenate([keep, gone]), 1)
    window(1000, keep, 2)                                                  # 1000 = 100 + 900: no row; `gone` is evicted here
    assert sorted(tr.first) == sorted(keep.tolist())
    assert eng.query_day_stats(cap=0)[2] == 0
    check_reads(eng, orc, tr)
    window(1001, np.concatenate([keep, fresh]), 3)                         # `fresh` takes the recycled slots
    rows, hosts, n = eng.query_day_stats()
    assert n == len(keep) and sorted(r.glob_id for r in rows) == sorted(keep.tolist())
    check_reads(eng, orc, tr)
    # count-only and partial reads
    for cap in (0, 1, 3, n - 1):
        r2, h2, n2 = eng.query_day_stats(cap=cap)
        assert n2 == n and [r.astuple() for r in r2] == [r.astuple() for r in rows[:cap]] and h2.tolist() == hosts[:cap].tolist()
    hl, nh = eng.query_host_listen()
    for cap in (0, 1, nh - 1):
        h2, n2 = eng.query_host_listen(cap=cap)
        assert n2 == nh and [tuple(getattr(r, f) for f, _ in ge.HostListen._fields_) for r in h2] == \
            [tuple(getattr(r, f) for f, _ in ge.HostListen._fields_) for r in hl[:cap]]
    window(1900, np.concatenate([keep, fresh]), 4)                         # fresh first seen at 1001: 1900 < 1901
    assert {r.glob_id for r in eng.query_day_stats()[0]} == set(keep.tolist())
    window(1902, np.concatenate([keep, fresh]), 5)
    rows = eng.query_day_stats()[0]
    assert {r.glob_id for r in rows} == set(keep.tolist()) | set(fresh.tolist())
    check_reads(eng, orc, tr)
    # the recycled slots hold only the new ids' own samples: three windows of them
    for r in rows:
        if r.glob_id in set(fresh.tolist()):
            assert r.tcount_5d == int(orc.export_hist(r.glob_id, ge.HIST_RESP_ALL)[0]["count"].sum())


def test_day_stats_percentiles_equal_the_compiled_reference():
    """every p95 / p25 of the 5-day level equals the reference's own GY_HISTOGRAM::get_percentiles (oracle/_ref) run on
    gysk_export_hist(GYSK_HIST_RESP_5DAY): the engine's level rule is the GY_HISTOGRAM rule"""
    R = po.ref()
    if R is None:
        pytest.skip("oracle/_ref/libgyref.so was not built")
    rng = np.random.default_rng(11)
    eng = ge.Engine(max_svcs=256, max_tasks=16, max_batch=1 << 14)
    ids = synth.service_ids(64)
    for t in (10, 500, 950):
        k = rng.integers(0, 64, 8000)
        ev = np.zeros(8000, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = ids[k]; ev["type"] = ge.EV_RESP
        ev["value"] = np.minimum(np.exp(rng.normal(np.log(5_000.0 * (1 + k % 9)), 1.3)), 9e8).astype(np.uint32)
        eng.ingest_events(ev); eng.flush(t)
    rows = eng.query_day_stats()[0]
    assert len(rows) == 64
    for r in rows:
        ser, total, mx = eng.export_hist(r.glob_id, ge.HIST_RESP_5DAY)
        s = np.ascontiguousarray(ser)
        pcts = np.array([95.0, 25.0], dtype=np.float32)
        out, avg, nb = np.zeros(2, dtype=np.int64), C.c_float(), C.c_int()
        R.gyref_hist_pct_from_serial(0, 0, po._p(s), total, mx, po._p(pcts), 2, po._p(out), C.byref(avg))
        want = [max(int(v), 0) & M32 for v in out]                          # TIME_HISTOGRAM::get_stats clamps at 0 (gy_statistics.h:1352)
        assert [r.p95_5d_respms, r.p25_5d_respms] == want and r.tcount_5d == total, (r.glob_id, want, total)


def test_day_stats_follow_the_5day_ring_across_slots_and_expiry():
    """flushes in ten successive 43 200-s slots of the 5-day level, then two that skip slots: the oldest slots leave the level by the
    live mask alone (their planes still hold their samples) or by being cleared for reuse. Every row's count is the samples of the
    last ten slot epochs, and equals the restatement after every flush"""
    W = 43200
    times = [5, 905, 1000] + [W * k + 5 for k in range(1, 10)] + [11 * W + 5, 11 * W + 10, 13 * W + 5]
    eng, orc = make_pair(max_svcs=64, max_tasks=16, max_batch=1 << 14)
    ids = synth.service_ids(20)
    rng = np.random.default_rng(23)
    tr = Tracker()
    per_epoch = {}                                                          # (id, epoch) -> samples
    expired = 0
    for w, t in enumerate(times):
        n = 400 + 150 * w
        k = rng.integers(0, len(ids), n)
        ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = ids[k]; ev["host_idx"] = k % 2; ev["type"] = ge.EV_RESP
        ev["value"] = np.minimum(np.exp(rng.normal(np.log(3_000.0 * (1 + w % 4)), 1.2, n)), 9e8).astype(np.uint32)
        for id_, c in zip(*np.unique(ev["svc_id"], return_counts=True)):
            per_epoch[(int(id_), t // W)] = per_epoch.get((int(id_), t // W), 0) + int(c)
        tr.feed(ev)
        feed_both(eng, orc, ev, 1 << 14)
        eng.flush(t); orc.flush(t); tr.flush(t)
        check_reads(eng, orc, tr)
        now = t // W
        for r in eng.query_day_stats()[0]:
            want = sum(c for (i, ep), c in per_epoch.items() if i == r.glob_id and now - 10 < ep <= now)
            total = sum(c for (i, _ep), c in per_epoch.items() if i == r.glob_id)
            assert r.tcount_5d == want, (t, r.glob_id, r.tcount_5d, want)
            expired += want < total
    assert expired > 0
