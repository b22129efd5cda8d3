"""Every ingest path leaves the same state: the 32-byte records from pageable memory (whole or in pieces), from page-locked memory
and from device memory, and the packed record kinds bulk from pageable or page-locked memory or in pieces expanded on the calling
thread, all fed the same device batches. Also wide raw records, whose raw pieces hold fewer records than a device buffer, and many
threads mixing the bulk paths with the per-thread staging."""
import threading

import numpy as np
import pytest
import torch

from gyeeta_b200 import engine as ge, synth
from gyeeta_b200.wire import TCP_CONN, build_msg
from oracle import pyoracle as po
from tests.util import assert_hist_equal

pytestmark = pytest.mark.gpu

RAW_BULK_MIN = 16384
COUNTERS = ("events_in", "events_dropped", "events_resp", "events_tcp", "events_task", "nsvcs", "ntasks")
ORACLE_COUNTERS = dict(events_in="in", events_dropped="dropped", events_resp="resp", events_tcp="tcp", events_task="task")
CFG = dict(max_svcs=1024, max_tasks=128, cms_log2_width=14)


def _same(a, b):
    if isinstance(a, (tuple, list)):
        return isinstance(b, (tuple, list)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return np.asarray(a).dtype == np.asarray(b).dtype and np.asarray(a).tobytes() == np.asarray(b).tobytes()
    if isinstance(a, float):
        return np.float64(a).tobytes() == np.float64(b).tobytes()
    return a == b


def _state(eng, svcs, tasks):
    """counters, the count-min table, every service's histogram, t-digest, HLL registers and connection bitmap, and every process's
    three histograms"""
    st = eng.stats()
    out = {k: st[k] for k in COUNTERS}
    out["cms"] = eng.export_cms()
    for s in svcs:
        out["hist", s] = eng.export_hist(s, ge.HIST_RESP_CUR)
        out["td", s] = eng.export_tdigest(s)
        out["hll", s] = eng.export_hll(s)
        out["bm", s] = eng.export_conn_bitmap(s)
    for t in tasks:
        for w in (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY):
            out["task", t, w] = eng.export_hist(t, w)
    return out


def _assert_states_equal(name, want, got):
    assert want.keys() == got.keys()
    for k in want:
        assert _same(want[k], got[k]), (name, k)


def _pinned(arr):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).copy()).pin_memory()


def _packed(ev):
    resp, tcp, task = ev[ev["type"] == ge.EV_RESP], ev[(ev["type"] >= 1) & (ev["type"] <= 4)], ev[ev["type"] == ge.EV_TASK]
    r16 = np.zeros(len(resp), dtype=ge.RESP16_DTYPE)
    r16["svc_id"], r16["usec"], r16["host_idx"], r16["cli_port"] = resp["svc_id"], resp["value"], resp["host_idx"], resp["flow_key"]
    t24 = np.zeros(len(tcp), dtype=ge.TCP24_DTYPE)
    t24["svc_id"], t24["flow_key"], t24["bytes"], t24["host_idx"], t24["type"] = tcp["svc_id"], tcp["flow_key"], tcp["value"], tcp["host_idx"], tcp["type"]
    k24 = np.zeros(len(task), dtype=ge.TASK24_DTYPE)
    k24["aggr_task_id"], k24["cpu_pct"], k24["host_idx"] = task["svc_id"], task["value"], task["host_idx"]
    k24["cpu_delay_msec"], k24["blkio_delay_msec"] = task["flow_key"] & np.uint64(0xFFFFFFFF), task["flow_key"] >> np.uint64(32)
    return np.concatenate([resp, tcp, task]), [(ge.RAW_RESP16, r16), (ge.RAW_TCP24, t24), (ge.RAW_TASK24, k24)]


def test_every_ingest_path_leaves_the_same_state():
    rng = np.random.default_rng(21)
    ev = synth.gen_mixed(rng, 200_000, 400, ntask=32, nhosts=64, nclients=4000)
    ev["flow_key"][ev["type"] == ge.EV_RESP] &= np.uint64(0xFF)                 # the packed response record keeps 8 bits of the client port
    ev["tsec"] = 0
    order, packed = _packed(ev)
    assert all(len(a) >= RAW_BULK_MIN for _k, a in packed)
    batch = 4096                                                                 # bulk pieces straddle device buffers
    engines = {}

    def engine(name):
        engines[name] = ge.Engine(max_batch=batch, stage_batch=batch, **CFG)
        return engines[name]

    engine("event32 pageable").ingest_events(order)
    e = engine("event32 pieces")
    for off in range(0, len(order), 1000):
        e.ingest_events(order[off: off + 1000])
    keep = [_pinned(order)]
    engine("event32 pinned").ingest_pinned_ptr(keep[0].data_ptr(), len(order))
    keep.append(torch.from_numpy(order.view(np.uint8).copy()).cuda())
    torch.cuda.synchronize()
    engine("event32 device").ingest_device_ptr(keep[-1].data_ptr(), len(order))
    e = engine("packed pageable bulk")
    for kind, a in packed:
        e.ingest_raw(kind, a, len(a))
    e = engine("packed pinned bulk")
    for kind, a in packed:
        keep.append(_pinned(a))
        e.ingest_raw_ptr(kind, keep[-1].data_ptr(), len(a))
    e = engine("packed pieces")
    for kind, a in packed:
        for off in range(0, len(a), RAW_BULK_MIN - 1):
            piece = np.ascontiguousarray(a[off: off + RAW_BULK_MIN - 1])
            e.ingest_raw(kind, piece, len(piece))
    for e in engines.values():
        e.sync()
    del keep

    orc = po.OracleEngine(**CFG)
    for off in range(0, len(order), batch):
        orc.ingest(order[off: off + batch])
    svcs = [int(s) for s in np.unique(order["svc_id"][order["type"] != ge.EV_TASK])]
    tasks = [int(t) for t in np.unique(order["svc_id"][order["type"] == ge.EV_TASK])]
    states = {name: _state(e, svcs, tasks) for name, e in engines.items()}
    want = states["event32 pageable"]
    assert want["events_in"] == len(order) and want["events_task"] == len(packed[2][1])
    for name, got in states.items():
        _assert_states_equal(name, want, got)
    oc = orc.counters()
    for k, ok in ORACLE_COUNTERS.items():
        assert want[k] == oc[ok], k
    assert np.array_equal(want["cms"], orc.cms())
    e = engines["packed pinned bulk"]
    for s in svcs:
        assert_hist_equal(e, orc, s, ge.HIST_RESP_CUR)
        assert np.array_equal(want["hll", s], orc.export_hll(s)), hex(s)
        assert _same(want["bm", s], orc.export_conn_bitmap(s)), hex(s)
    for t in tasks:
        for w in (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY):
            assert_hist_equal(e, orc, t, w)


IPV6_EVENT = np.dtype(dict(names=["ts_ns", "bytes_received", "bytes_acked", "pid", "tid", "comm", "saddr", "daddr", "netns", "sport", "dport",
                                  "ipver", "type"],
                           formats=["<u8", "<u8", "<u8", "<u4", "<u4", "S16", ("<u4", 4), ("<u4", 4), "<u4", "<u2", "<u2", "u1", "u1"],
                           offsets=[0, 8, 16, 24, 28, 32, 48, 64, 80, 84, 86, 88, 89], itemsize=96))


def test_wide_raw_records_bulk_and_pieces():
    """tcp_ipv6_event_t (96 B): a raw piece holds a third of a device buffer. Bulk pads a dropped record, the pieces skip it, so only
    the two bulk paths share their batch boundaries."""
    rng = np.random.default_rng(22)
    n = 40_000
    rec = np.zeros(n, dtype=IPV6_EVENT)
    rec["saddr"][:, 0], rec["saddr"][:, 3] = 0x20010DB8, rng.integers(1, 9, n)        # 8 listener addresses
    # a connect-side record keys its service by the remote end: few remote addresses and ports, so every service fits the table
    rec["daddr"][:, 0], rec["daddr"][:, 3] = 0x20010DB9, rng.integers(1, 17, n)
    rec["netns"] = 4026531840
    rec["sport"] = rng.choice(np.array([80, 443, 8080], dtype=np.uint16).byteswap(), n)
    rec["dport"] = rng.choice(np.arange(40000, 40016, dtype=np.uint16).byteswap(), n)
    rec["type"] = rng.choice(np.array([0, 1, 2, 3, 4, 9], dtype=np.uint8), n, p=[0.05, 0.2, 0.3, 0.2, 0.2, 0.05])   # 0 and 9: dropped
    rec["bytes_received"], rec["bytes_acked"] = rng.integers(0, 1 << 33, n), rng.integers(0, 1 << 20, n)
    rec["ts_ns"] = rng.integers(0, 1 << 40, n)
    kw = dict(max_batch=4096, stage_batch=4096, **CFG)
    pageable, pinned, pieces = ge.Engine(**kw), ge.Engine(**kw), ge.Engine(**kw)
    pageable.ingest_raw(ge.RAW_TCP_IPV6_EVENT, rec, n)
    buf = _pinned(rec)
    pinned.ingest_raw_ptr(ge.RAW_TCP_IPV6_EVENT, buf.data_ptr(), n)
    for off in range(0, n, 5000):
        p = np.ascontiguousarray(rec[off: off + 5000])
        pieces.ingest_raw(ge.RAW_TCP_IPV6_EVENT, p, len(p))
    for e in (pageable, pinned, pieces):
        e.sync()
    del buf
    kept = int(((rec["type"] >= 1) & (rec["type"] <= 4)).sum())
    sa, sb, sc = pageable.stats(), pinned.stats(), pieces.stats()
    assert sa["events_tcp"] == kept and sa["events_in"] == kept
    for k in COUNTERS:
        assert sa[k] == sb[k] == sc[k], k
    assert np.array_equal(pageable.export_cms(), pinned.export_cms()) and np.array_equal(pageable.export_cms(), pieces.export_cms())
    (wa, na), (wb, nb) = pageable.query_window(), pinned.query_window()
    assert na == nb == sa["nsvcs"] and [bytes(r) for r in wa] == [bytes(r) for r in wb]
    svcs = [r.glob_id for r in wa]
    for s in svcs:
        assert _same(pageable.export_conn_bitmap(s), pinned.export_conn_bitmap(s)) and _same(pageable.export_hll(s), pinned.export_hll(s))


def test_concurrent_bulk_callers():
    """8 threads each mix pageable bulk RESP16, page-locked bulk TCP24, small raw pieces and wire messages on one engine with a
    small stage: the union is applied exactly once"""
    rng = np.random.default_rng(23)
    nthr = 8
    eng = ge.Engine(max_batch=1 << 16, stage_batch=1 << 12, **CFG)
    orc = po.OracleEngine(**CFG)
    work, evs = [], []
    for t in range(nthr):
        ev = synth.gen_mixed(rng, 60_000, 300, ntask=32, nhosts=64, nclients=4000)
        ev["flow_key"][ev["type"] == ge.EV_RESP] &= np.uint64(0xFF)
        ev["tsec"] = 0
        ev["host_idx"] = t
        _order, packed = _packed(ev)
        (_, r16), (_, t24), (_, k24) = packed
        bulk_resp, small_resp = r16[: RAW_BULK_MIN + 4000], r16[RAW_BULK_MIN + 4000:]
        t24 = np.concatenate([t24] * (RAW_BULK_MIN // len(t24) + 1))[: RAW_BULK_MIN + 1000]
        msgs, mev = [], []
        for _m in range(6):
            recs = []
            for _i in range(int(rng.integers(20, 200))):
                r = np.zeros(1, dtype=TCP_CONN)
                r["ser_glob_id"] = 1000 + int(rng.integers(0, 60)); r["cli_task_aggr_id"] = 5000 + int(rng.integers(0, 500))
                r["is_accept"] = 1; r["tusec_close"] = 9_000_000; r["tusec_start"] = 1_000_000
                r["bytes_sent"], r["bytes_rcvd"] = int(rng.integers(0, 1 << 20)), int(rng.integers(0, 1 << 20))
                recs.append((r, b"x" * int(rng.integers(0, 9))))
                e = np.zeros(1, dtype=ge.EVENT_DTYPE)
                e["svc_id"], e["flow_key"], e["type"], e["host_idx"] = r["ser_glob_id"], r["cli_task_aggr_id"], ge.EV_CLOSE_SER, t
                e["value"] = int(r["bytes_sent"][0]) + int(r["bytes_rcvd"][0])
                mev.append(e)
            msgs.append(build_msg(ge.NOTIFY_TCP_CONN, recs))
        pieces = [(ge.RAW_RESP16, small_resp[o: o + 700]) for o in range(0, len(small_resp), 700)] + \
                 [(ge.RAW_TASK24, k24[o: o + 900]) for o in range(0, len(k24), 900)]
        work.append(dict(host=t, bulk=bulk_resp, pinned=_pinned(t24), npinned=len(t24), pieces=pieces, msgs=msgs))
        te = np.zeros(len(t24), dtype=ge.EVENT_DTYPE)
        te["svc_id"], te["flow_key"], te["value"], te["host_idx"], te["type"] = t24["svc_id"], t24["flow_key"], t24["bytes"], t, t24["type"]
        evs += [ev[ev["type"] == ge.EV_RESP], ev[ev["type"] == ge.EV_TASK], te] + mev
    errs = []

    def run(w):
        try:
            eng.ingest_raw(ge.RAW_RESP16, w["bulk"], len(w["bulk"]))
            for i, m in enumerate(w["msgs"]):
                assert eng.ingest_msg(m, host_idx=w["host"]) == 0
                kind, p = w["pieces"][i % len(w["pieces"])]
                eng.ingest_raw(kind, np.ascontiguousarray(p), len(p))
            eng.ingest_raw_ptr(ge.RAW_TCP24, w["pinned"].data_ptr(), w["npinned"])
            for kind, p in w["pieces"][len(w["msgs"]):]:
                eng.ingest_raw(kind, np.ascontiguousarray(p), len(p))
        except Exception as ex:               # noqa: BLE001 - reported below
            errs.append(ex)

    ths = [threading.Thread(target=run, args=(w,)) for w in work]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errs, errs
    eng.sync()
    all_ev = np.concatenate(evs)
    orc.ingest(all_ev)
    st, oc = eng.stats(), orc.counters()
    for k, ok in ORACLE_COUNTERS.items():
        assert st[k] == oc[ok], k
    assert st["events_in"] == len(all_ev) and st["wire_msgs_ok"] == nthr * 6
    assert np.array_equal(eng.export_cms(), orc.cms())
    for s in np.unique(all_ev["svc_id"][all_ev["type"] != ge.EV_TASK]):
        assert_hist_equal(eng, orc, int(s), ge.HIST_RESP_CUR)
    for t in np.unique(all_ev["svc_id"][all_ev["type"] == ge.EV_TASK]):
        for w in (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY):
            assert_hist_equal(eng, orc, int(t), w)
