"""boundary rows of SURVEY.md §8 beyond the three original wire subtypes: ACTIVE_CONN_STATS (a11 / a12), the IPv6 eBPF structs
(a8 / a9), API_TRAN (a8b), device-side expansion of fixed-stride raw records and of the packed per-kind records (f2), concurrent
gysk_ingest callers on per-thread staging (§8b Threading), and the per-host top-N queues (a13 / a15 / f3)."""
import threading

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po
from tests.test_gpu_wire import COMM_EVENT_NOTIFY, HDR, PM_MAGIC, TASK, TCP_CONN, build_msg
from tests.util import assert_hist_equal

pytestmark = pytest.mark.gpu

ACTIVE = np.dtype([("listener_glob_id", "<u8"), ("cli_aggr_task_id", "<u8"), ("ser_comm", "S16"), ("cli_comm", "S16"), ("machid", "<u8", 2),
                   ("remote_madhava_id", "<u8"), ("bytes_sent", "<u8"), ("bytes_received", "<u8"), ("cli_delay_msec", "<u4"),
                   ("ser_delay_msec", "<u4"), ("max_rtt_msec", "<f4"), ("active_conns", "<u2"), ("flags", "u1"), ("pad", "u1")])
RESP4 = np.dtype([("saddr", "<u4"), ("daddr", "<u4"), ("netns", "<u4"), ("sport", "<u2"), ("dport", "<u2"), ("lsndtime", "<u4"), ("lrcvtime", "<u4")])
RESP6 = np.dtype([("saddr", "<u4", 4), ("daddr", "<u4", 4), ("netns", "<u4"), ("sport", "<u2"), ("dport", "<u2"), ("pad", "<u4", 2),
                  ("lsndtime", "<u4"), ("lrcvtime", "<u4"), ("tail", "<u4", 2)])
CONN6 = np.dtype([("ts_ns", "<u8"), ("bytes_received", "<u8"), ("bytes_acked", "<u8"), ("pid", "<u4"), ("tid", "<u4"), ("comm", "S16"),
                  ("saddr", "<u4", 4), ("daddr", "<u4", 4), ("netns", "<u4"), ("sport", "<u2"), ("dport", "<u2"), ("ipver", "u1"), ("type", "u1"),
                  ("pad", "u1", 6)])
assert ACTIVE.itemsize == 104 and RESP4.itemsize == 24 and RESP6.itemsize == 64 and CONN6.itemsize == 96


def fixed_msg(subtype, recs):
    hdr = np.zeros(1, dtype=HDR)
    body = recs.tobytes()
    hdr["magic"], hdr["data_type"] = PM_MAGIC, COMM_EVENT_NOTIFY
    hdr["total_sz"] = HDR.itemsize + len(body)
    hdr["subtype"], hdr["nevents"] = subtype, len(recs)
    return bytearray(hdr.tobytes() + body)


def test_active_conn_stats_message():
    """NOTIFY_ACTIVE_CONN_STATS (handle_partha_active_conns, gy_mconnhdlr.cc:7705): per {listener, client process} record the flow
    sketch takes connections + kbytes, the listener its window totals and max rtt; equal to the oracle fed the same records"""
    rng = np.random.default_rng(4)
    eng = ge.Engine(max_svcs=256, max_tasks=16, max_batch=1 << 14, cms_log2_width=12)
    orc = po.OracleEngine(max_svcs=256, max_tasks=16, cms_log2_width=12)
    n = 1500
    recs = np.zeros(n, dtype=ACTIVE)
    recs["listener_glob_id"] = 9000 + rng.integers(0, 40, n)
    recs["listener_glob_id"][::97] = 0                                             # skipped
    recs["cli_aggr_task_id"] = 100 + rng.integers(0, 300, n)
    recs["bytes_sent"] = rng.integers(0, 1 << 34, n); recs["bytes_received"] = rng.integers(0, 1 << 30, n)
    recs["max_rtt_msec"] = rng.random(n).astype(np.float32) * 200
    recs["active_conns"] = rng.integers(0, 50, n)
    assert eng.ingest_msg(fixed_msg(ge.NOTIFY_ACTIVE_CONN_STATS, recs), host_idx=2) == 0
    bad = fixed_msg(ge.NOTIFY_ACTIVE_CONN_STATS, recs[:5]); bad[20:24] = (3000).to_bytes(4, "little")          # nevents beyond MAX_NUM_CONNS / the body
    assert eng.ingest_msg(bad, host_idx=2) == -22
    ok = recs[recs["listener_glob_id"] != 0]
    ev = np.zeros(len(ok), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"] = ok["listener_glob_id"], ok["cli_aggr_task_id"]
    ev["value"] = np.minimum((ok["bytes_sent"] + ok["bytes_received"]) >> np.uint64(10), 0xFFFFFFFF)
    ev["tsec"] = ok["max_rtt_msec"].view(np.uint32); ev["type"] = ge.EV_ACTIVE; ev["flags"] = ok["active_conns"]; ev["host_idx"] = 2
    orc.ingest(ev)
    eng.sync()
    assert np.array_equal(eng.export_cms(), orc.cms())
    eng.flush(15); orc.flush(15)
    ids = np.unique(ok["listener_glob_id"])
    for s_, id_ in zip(eng.query_svcs(ids), ids):
        a = orc.export_aux(int(id_))
        assert s_["found"] == 1 and (s_["nconns_active"], s_["active_kbytes"]) == (a["act_last"] & 0xFFFFFFFF, a["act_last"] >> 32)
        assert s_["max_rtt_msec"] == a["rtt_last"] == float(ok["max_rtt_msec"][ok["listener_glob_id"] == id_].max())
        assert np.array_equal(eng.export_hll(int(id_)), orc.export_hll(int(id_)))
    st = eng.stats()
    assert st["events_tcp"] == len(ok) and st["wire_msgs_ok"] == 1 and st["wire_msgs_bad"] == 1
    # the summary encoder carries the active connections into LISTENER_STATE_NOTIFY::nconns_active_
    nrecs, raw = eng.listener_state_records(ids[:10])
    assert nrecs == 10 and int.from_bytes(raw[20:24], "little") == eng.query_svcs(ids[:1])[0]["nconns_active"]


def _resp_records(rng, n, v6):
    r = np.zeros(n, dtype=RESP6 if v6 else RESP4)
    if v6:
        r["saddr"] = [0x20010DB8, 0, 0x1234, 7]; r["daddr"] = rng.integers(1, 1 << 31, (n, 4))
    else:
        r["saddr"] = 0x0A000001; r["daddr"] = rng.integers(1, 1 << 31, n)
    r["netns"] = 4026531840
    r["sport"] = np.uint16(8443).byteswap()
    cport = rng.integers(16000, 60000, n).astype(np.uint16)
    r["dport"] = cport.byteswap()
    r["lrcvtime"] = rng.integers(0, 1 << 31, n)
    ms = rng.integers(0, 30000, n).astype(np.uint32); ms[::41] = 3_000_000
    r["lsndtime"] = r["lrcvtime"] + ms
    return r, ms, cport


@pytest.mark.parametrize("v6", [False, True])
def test_raw_resp_records_device_expansion_equals_host_expansion(v6):
    """tcp_ipv4_resp_event_t / tcp_ipv6_resp_event_t: a big batch is expanded by decode_raw_kernel on the device, the same records
    in small pieces by the calling thread — same listener, same histogram (= the reference's add_data over the msec values),
    same CONN_BITMAP"""
    rng = np.random.default_rng(6)
    n = 50_000
    r, ms, cport = _resp_records(rng, n, v6)
    kind = ge.RAW_TCP_IPV6_RESP if v6 else ge.RAW_TCP_IPV4_RESP
    big = ge.Engine(max_svcs=64, max_tasks=8, max_batch=1 << 16, cms_log2_width=10)
    small = ge.Engine(max_svcs=64, max_tasks=8, max_batch=1 << 16, cms_log2_width=10)
    big.ingest_raw(kind, r, n); big.sync()
    for off in range(0, n, 1000):
        small.ingest_raw(kind, r[off: off + 1000], min(1000, n - off))
    small.sync()
    kept = ms <= 1_000_000
    want = po.hist_run(po.lib(), "gyo_hist_run", 0, 0, ms[kept].astype(np.int64))
    for e_ in (big, small):
        st = e_.stats()
        assert st["events_resp"] == int(kept.sum()) and st["nsvcs"] == 1 and st["events_dropped"] == 0
    # the listener id is an internal fold of {ip, netns, port}: find it through the evicted-id-free route — top-N of the window
    big.flush(5); small.flush(5)
    (sid, score, _h), = big.topn(0, 1)
    assert small.topn(0, 1)[0][0] == sid and score == int(kept.sum())
    for e_ in (big, small):
        h = e_.export_hist(sid, ge.HIST_RESP_LAST)
        assert np.array_equal(h[0]["count"], want["stats"]["count"][:15]) and np.array_equal(h[0]["sum"], want["stats"]["sum"][:15])
        assert h[1] == want["total"] and h[2] == want["max"]
    mb, ms_ = big.export_conn_bitmap(sid, True), small.export_conn_bitmap(sid, True)
    assert np.array_equal(mb[0], ms_[0])
    want_masks = np.zeros(15, dtype=np.uint32)
    for m_, p_ in zip(ms[kept], cport[kept]):
        want_masks[po.lib().gyo_bucket(0, int(m_))] |= np.uint32(1 << (int(p_) & 31))
    assert np.array_equal(mb[0], want_masks)


def test_raw_ipv6_conn_events():
    """tcp_ipv6_event_t (handle_ipv6_conn_event, gy_socket_stat.cc:269): accept / close on the server side key the listener by the
    local address, connect / close on the client side by the remote one; bulk (device) and piecewise (host) expansion agree"""
    rng = np.random.default_rng(8)
    n = 20_000
    c = np.zeros(n, dtype=CONN6)
    srv = np.array([0x20010DB8, 0, 0, 0x50], dtype=np.uint32)
    typ = rng.integers(1, 5, n).astype(np.uint8); typ[::333] = 9
    ser_side = (typ == 2) | (typ == 4)
    cli = rng.integers(1, 1 << 31, (n, 4)).astype(np.uint32)
    c["saddr"] = np.where(ser_side[:, None], srv[None, :], cli); c["daddr"] = np.where(ser_side[:, None], cli, srv[None, :])
    sp, cp = np.uint16(443).byteswap(), rng.integers(20000, 60000, n).astype(np.uint16).byteswap()
    c["sport"] = np.where(ser_side, sp, cp); c["dport"] = np.where(ser_side, cp, sp)
    c["netns"], c["type"], c["ipver"] = 4026531999, typ, 6
    c["bytes_acked"] = rng.integers(0, 1 << 22, n); c["bytes_received"] = rng.integers(0, 1 << 22, n)
    big = ge.Engine(max_svcs=64, max_tasks=8, max_batch=1 << 16, cms_log2_width=12)
    small = ge.Engine(max_svcs=64, max_tasks=8, max_batch=1 << 16, cms_log2_width=12)
    big.ingest_raw(ge.RAW_TCP_IPV6_EVENT, c, n); big.sync()
    for off in range(0, n, 2000):
        small.ingest_raw(ge.RAW_TCP_IPV6_EVENT, c[off: off + 2000], 2000)
    small.sync()
    good = int((typ <= 4).sum())
    for e_ in (big, small):
        st = e_.stats()
        assert st["events_tcp"] == good and st["nsvcs"] == 1
    assert np.array_equal(big.export_cms(), small.export_cms())
    cms = big.export_cms().reshape(4, -1)
    kb = int(((c["bytes_acked"] + c["bytes_received"])[typ <= 4] >> np.uint64(10)).sum())
    for row in cms:
        assert int((row & np.uint64(0xFFFFFFFF)).sum()) == good and int((row >> np.uint64(32)).sum()) == kb


def test_api_tran_records():
    """API_TRAN (common/gy_proto_common.h:140-204, variable stride) through SVC_INFO_CAP::upd_stats_on_req semantics
    (gy_proto_parser.cc:2678-2694): response_usec_ / 1000 into the response histogram, error counters per listener"""
    rng = np.random.default_rng(10)
    eng = ge.Engine(max_svcs=64, max_tasks=8, max_batch=1 << 14, cms_log2_width=10)
    orc = po.OracleEngine(max_svcs=64, max_tasks=8, cms_log2_width=10)
    n = 3000
    buf = bytearray()
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    for i in range(n):
        rec = bytearray(176)
        usec = int(rng.integers(50, 40_000_000))
        gid = 700 + int(rng.integers(0, 12))
        err = int(rng.choice([0, 0, 0, 404, 500, 503]))
        cport = int(rng.integers(1024, 65535))
        reqlen, extlen = int(rng.integers(0, 60)), int(rng.integers(0, 20))
        pad = (-(176 + reqlen + extlen)) % 8
        rec[16:24] = (1_700_000_000_000_000 + i).to_bytes(8, "little")            # tupd_usec_
        rec[48:56] = usec.to_bytes(8, "little"); rec[120:128] = gid.to_bytes(8, "little")
        rec[152:156] = err.to_bytes(4, "little"); rec[166:168] = cport.to_bytes(2, "little")
        rec[170:172] = reqlen.to_bytes(2, "little"); rec[172:174] = extlen.to_bytes(2, "little"); rec[174] = pad
        buf += rec + bytes(rng.integers(32, 120, reqlen + extlen, dtype=np.uint8)) + b"\0" * pad
        ev[i] = (gid, cport, usec, 1, 0, ge.EV_RESP, 0 if not err else (ge.EVF_SER_ERROR if err >= 500 else ge.EVF_CLI_ERROR))
    raw = np.frombuffer(bytes(buf), dtype=np.uint8)
    eng.ingest_raw(ge.RAW_API_TRAN, raw, n, host_idx=1)
    eng.sync(); orc.ingest(ev)
    eng.flush(5); orc.flush(5)
    ids = np.unique(ev["svc_id"])
    for s_, id_ in zip(eng.query_svcs(ids), ids):
        assert_hist_equal(eng, orc, int(id_), ge.HIST_RESP_LAST)
        a = orc.export_aux(int(id_))
        m = ev["svc_id"] == id_
        assert (s_["cli_errors"], s_["ser_errors"]) == (a["err_last"] & 0xFFFFFFFF, a["err_last"] >> 32) == \
            (int((ev["flags"][m] == 1).sum()), int((ev["flags"][m] == 2).sum()))
        g, o = eng.export_conn_bitmap(int(id_), True), orc.export_conn_bitmap(int(id_), True)
        assert np.array_equal(g[0], o[0])


def test_packed_kinds_equal_the_canonical_records():
    """gysk_resp16 / gysk_tcp24 / gysk_task24 batches (expanded on the device) leave the same state as the 32-byte records"""
    rng = np.random.default_rng(14)
    ev = synth.gen_mixed(rng, 120_000, 400, ntask=32, nhosts=64, nclients=4000)
    ev["flow_key"][ev["type"] == ge.EV_RESP] &= np.uint64(0xFF)                 # the packed response record keeps 8 bits of the client port
    ev["tsec"] = 0
    a = ge.Engine(max_svcs=1024, max_tasks=128, max_batch=1 << 18, cms_log2_width=14)
    b = ge.Engine(max_svcs=1024, max_tasks=128, max_batch=1 << 18, cms_log2_width=14)
    orc = po.OracleEngine(max_svcs=1024, max_tasks=128, cms_log2_width=14)
    resp, tcp, task = ev[ev["type"] == ge.EV_RESP], ev[(ev["type"] >= 1) & (ev["type"] <= 4)], ev[ev["type"] == ge.EV_TASK]
    order = np.concatenate([resp, tcp, task])
    a.ingest_events(order); a.sync(); orc.ingest(order)
    r16 = np.zeros(len(resp), dtype=ge.RESP16_DTYPE)
    r16["svc_id"], r16["usec"], r16["host_idx"], r16["cli_port"] = resp["svc_id"], resp["value"], resp["host_idx"], resp["flow_key"]
    t24 = np.zeros(len(tcp), dtype=ge.TCP24_DTYPE)
    t24["svc_id"], t24["flow_key"], t24["bytes"], t24["host_idx"], t24["type"] = tcp["svc_id"], tcp["flow_key"], tcp["value"], tcp["host_idx"], tcp["type"]
    k24 = np.zeros(len(task), dtype=ge.TASK24_DTYPE)
    k24["aggr_task_id"], k24["cpu_pct"], k24["host_idx"] = task["svc_id"], task["value"], task["host_idx"]
    k24["cpu_delay_msec"], k24["blkio_delay_msec"] = task["flow_key"] & np.uint64(0xFFFFFFFF), task["flow_key"] >> np.uint64(32)
    b.ingest_raw(ge.RAW_RESP16, r16, len(r16)); b.ingest_raw(ge.RAW_TCP24, t24, len(t24)); b.ingest_raw(ge.RAW_TASK24, k24, len(k24)); b.sync()
    sa, sb = a.stats(), b.stats()
    for k in ("events_in", "events_resp", "events_tcp", "events_task", "events_dropped", "nsvcs", "ntasks"):
        assert sa[k] == sb[k], k
    assert np.array_equal(a.export_cms(), b.export_cms()) and np.array_equal(a.export_cms(), orc.cms())
    for id_ in np.unique(resp["svc_id"])[:80]:
        for e_ in (a, b):
            assert_hist_equal(e_, orc, int(id_), ge.HIST_RESP_CUR)
        ta, tb, to = a.export_tdigest(int(id_)), b.export_tdigest(int(id_)), orc.export_tdigest(int(id_))
        om, ow = to.centroids()
        assert np.array_equal(ta[0], tb[0]) and np.array_equal(ta[1], tb[1]) and np.array_equal(ta[0], om) and np.array_equal(ta[1], ow)
        assert np.array_equal(a.export_hll(int(id_)), b.export_hll(int(id_)))
    for id_ in np.unique(task["svc_id"])[:20]:
        assert_hist_equal(b, orc, int(id_), ge.HIST_TASK_CPU_DELAY)


def test_concurrent_callers_on_per_thread_staging():
    """16 threads call gysk_ingest_msg at once (the handle_l2_misc fan-in, gy_mconnhdlr.cc:16252): the union is applied exactly once"""
    rng = np.random.default_rng(16)
    eng = ge.Engine(max_svcs=512, max_tasks=64, max_batch=1 << 16, stage_batch=1 << 12, cms_log2_width=12)
    orc = po.OracleEngine(max_svcs=512, max_tasks=64, cms_log2_width=12)
    nthr, per = 16, 30
    msgs, evs = [[] for _ in range(nthr)], []
    for t in range(nthr):
        for _ in range(per):
            recs = []
            for _i in range(int(rng.integers(20, 200))):
                r = np.zeros(1, dtype=TCP_CONN)
                r["ser_glob_id"] = 1000 + int(rng.integers(0, 60)); r["cli_task_aggr_id"] = 5000 + int(rng.integers(0, 500))
                r["is_accept"] = 1; r["tusec_close"] = 9_000_000; r["tusec_start"] = 1_000_000
                r["bytes_sent"], r["bytes_rcvd"] = int(rng.integers(0, 1 << 20)), int(rng.integers(0, 1 << 20))
                recs.append((r, b"x" * int(rng.integers(0, 9))))
                e = np.zeros(1, dtype=ge.EVENT_DTYPE)
                e["svc_id"], e["flow_key"], e["type"] = r["ser_glob_id"], r["cli_task_aggr_id"], 4
                e["value"] = int(r["bytes_sent"][0]) + int(r["bytes_rcvd"][0])
                evs.append(e)
            msgs[t].append(build_msg(ge.NOTIFY_TCP_CONN, recs))
    errs = []

    def run(t):
        for m in msgs[t]:
            if eng.ingest_msg(m, host_idx=t) != 0:
                errs.append(t)
    th = [threading.Thread(target=run, args=(t,)) for t in range(nthr)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errs
    eng.sync()
    orc.ingest(np.concatenate(evs))
    st = eng.stats()
    assert st["events_tcp"] == len(evs) and st["wire_msgs_ok"] == nthr * per
    assert np.array_equal(eng.export_cms(), orc.cms())
    for id_ in range(1000, 1060, 7):
        assert np.array_equal(eng.export_hll(id_), orc.export_hll(id_))


def test_per_host_topn_queues():
    """the four listener rankings of partha_listener_state (gy_mconnhdlr.cc:11262-11304) and the seven process rankings of
    partha_aggr_task_state (:10012-10079): entry conditions, comparators, 10 entries per host"""
    from tests.test_gpu_wire import build_msg as bm
    LSN = np.dtype([("glob_id", "<u8"), ("nqrys_5s", "<u4"), ("total_resp_5sec", "<u4"), ("nconns", "<u4"), ("nconns_active", "<u4"),
                    ("ntasks", "<u4"), ("p95_5s", "<u4"), ("p95_5min", "<u4"), ("kb_in", "<u4"), ("kb_out", "<u4"), ("ser_errors", "<u4"),
                    ("cli_errors", "<u4"), ("tasks_delay_usec", "<u4"), ("t2", "<u4"), ("t3", "<u4"), ("t4", "<u4"), ("t5", "<u4"), ("t6", "<u4"),
                    ("ntasks_issue", "<u2"), ("is_http", "u1"), ("curr_state", "u1"), ("curr_issue", "u1"), ("issue_bit_hist", "u1"),
                    ("high_resp_bit_hist", "u1"), ("last_issue_subsrc", "u1"), ("query_flags", "u1"), ("issue_string_len", "u1"),
                    ("padding_len", "u1"), ("pad", "u1")])
    rng = np.random.default_rng(18)
    eng = ge.Engine(max_svcs=64, max_tasks=16, max_batch=2048, cms_log2_width=10)
    lrecs, rows = [], []
    for i in range(120):
        r = np.zeros(1, dtype=LSN)
        r["glob_id"] = 100 + i
        r["nqrys_5s"] = int(rng.integers(0, 4000)); r["nconns_active"] = int(rng.integers(0, 30))
        r["kb_in"], r["kb_out"] = int(rng.integers(0, 900)), int(rng.integers(0, 900))
        r["curr_state"] = int(rng.integers(0, 6)); r["tasks_delay_usec"] = int(rng.integers(0, 1 << 20))
        lrecs.append((r, b"")); rows.append(r[0])
    assert eng.ingest_msg(bm(ge.NOTIFY_LISTENER_STATE, lrecs), host_idx=4) == 0
    rows = np.array(rows)

    def top(score, cond):
        s = [(int(sc), int(g)) for sc, g, c in zip(score, rows["glob_id"], cond) if c]
        return [x[0] for x in sorted(s, key=lambda x: (-x[0], x[1]))[:10]]
    got = eng.topn_host(ge.HOSTTOP_SVC_QPS, 10, host_idx=4)
    assert [s for _, s, _ in got] == top(rows["nqrys_5s"], rows["nqrys_5s"] >= 5) and all(h == 4 for *_x, h in got)
    assert [s for _, s, _ in eng.topn_host(ge.HOSTTOP_SVC_CONNS, 10, host_idx=4)] == top(rows["nconns_active"], rows["nconns_active"] >= 1)
    net = rows["kb_in"].astype(np.int64) + rows["kb_out"]
    assert [s for _, s, _ in eng.topn_host(ge.HOSTTOP_SVC_NET, 10)] == top(net, net > 0)
    issue = (rows["curr_state"].astype(np.int64) << 32) | rows["tasks_delay_usec"]
    assert [s for _, s, _ in eng.topn_host(ge.HOSTTOP_SVC_ISSUE, 10, host_idx=4)] == top(issue, rows["curr_state"] > 2)
    assert eng.topn_host(ge.HOSTTOP_SVC_QPS, 10, host_idx=5) == []

    trecs, trows = [], []
    for i in range(80):
        r = np.zeros(1, dtype=TASK)
        r["aggr_task_id"] = 7000 + i
        r["tcp_kbytes"] = int(rng.integers(0, 3)) * int(rng.integers(1, 5000)); r["total_cpu_pct"] = float(rng.random() * 50) if i % 3 else 0.05
        r["rss_mb"] = int(rng.integers(0, 2000)); r["cpu_delay_msec"] = int(rng.integers(0, 3)) * int(rng.integers(1, 900))
        r["vm_delay_msec"] = int(rng.integers(0, 2)) * int(rng.integers(1, 90)); r["blkio_delay_msec"] = int(rng.integers(0, 400))
        r["curr_state"] = int(rng.integers(0, 6)); r["ntasks_issue"] = int(rng.integers(0, 5)); r["severe_issue_bit_hist"] = int(rng.integers(0, 2))
        trecs.append((r, b"")); trows.append(r[0])
    assert eng.ingest_msg(bm(ge.NOTIFY_AGGR_TASK_STATE, trecs), host_idx=4) == 0
    trows = np.array(trows)

    def ttop(score, cond):
        s = [(int(sc), int(g)) for sc, g, c in zip(score, trows["aggr_task_id"], cond) if c]
        return [x[0] for x in sorted(s, key=lambda x: (-x[0], x[1]))[:10]]
    assert [s for _, s, _ in eng.topn_host(ge.HOSTTOP_TASK_NET, 10, 4)] == ttop(trows["tcp_kbytes"], trows["tcp_kbytes"] > 0)
    cpu_bits = trows["total_cpu_pct"].view(np.uint32)
    assert [s for _, s, _ in eng.topn_host(ge.HOSTTOP_TASK_CPU, 10, 4)] == ttop(cpu_bits, trows["total_cpu_pct"] >= np.float32(0.1))
    assert [s for _, s, _ in eng.topn_host(ge.HOSTTOP_TASK_RSS, 10, 4)] == ttop(trows["rss_mb"], trows["rss_mb"] >= 5)
    for what, col in ((ge.HOSTTOP_TASK_CPU_DELAY, "cpu_delay_msec"), (ge.HOSTTOP_TASK_VM_DELAY, "vm_delay_msec"), (ge.HOSTTOP_TASK_BLKIO_DELAY, "blkio_delay_msec")):
        assert [s for _, s, _ in eng.topn_host(what, 10, 4)] == ttop(trows[col], trows[col] > 0)
    sev = ((trows["severe_issue_bit_hist"] & 1).astype(np.int64) * (trows["ntasks_issue"] > 0)) << 32
    assert [s for _, s, _ in eng.topn_host(ge.HOSTTOP_TASK_ISSUE, 10, 4)] == ttop(sev | (trows["ntasks_issue"].astype(np.int64) + 1), trows["curr_state"] > 2)


def _proc_samples(rng, n, ngroups):
    s = np.zeros(n, dtype=ge.PROC_SAMPLE_DTYPE)
    s["aggr_task_id"] = synth.splitmix64(rng.integers(1, ngroups + 1, n).astype(np.uint64) + np.uint64(1 << 41))
    s["pid"] = rng.integers(2, 1 << 22, n)
    # cpu percentages whose float sum depends on the order of the additions
    s["cpu_pct"] = (rng.random(n) ** 6 * 3000.0 + rng.random(n) * 1e-3).astype(np.float32)
    s["rss_mb"] = rng.integers(0, 1 << 14, n)
    for f in ("cpu_delay_msec", "vm_delay_msec", "blkio_delay_msec"):
        s[f] = np.minimum(np.exp(rng.normal(2.0, 2.5, n)), 1e6).astype(np.uint32)
    net = rng.random(n) < 0.3
    s["tcp_kbytes"] = np.where(net, rng.integers(0, 1 << 20, n), 0); s["tcp_conns"] = np.where(net, rng.integers(0, 500, n), 0)
    s["state"] = rng.integers(0, 5, n); s["issue"] = rng.integers(0, 12, n)
    s["is_issue"] = rng.random(n) < 0.15
    s["issue_bit_hist"] = rng.integers(0, 256, n); s["severe_issue_bit_hist"] = rng.integers(0, 256, n)
    s["comm"] = [b"proc%d" % (i % 97) for i in range(n)]
    return s


def test_task_groupby_equals_the_walk_of_the_reference():
    """row a15b: per-process samples folded by aggr_task_id in arrival order (common/gy_task_handler.cc:752-880) on the device; every
    field of every AGGR_TASK_STATE_NOTIFY record — incl. the order-dependent float cpu sum and the pid slots — equals the CPU statement
    of the walk, groups in order of first appearance; the records are a valid NOTIFY_AGGR_TASK_STATE body for gysk_ingest"""
    from gyeeta_b200 import wire
    rng = np.random.default_rng(41)
    eng = ge.Engine(max_svcs=64, max_tasks=1 << 14, max_batch=1 << 18)
    for n, ngroups in ((1, 1), (37, 5), (5000, 1200), (200_000, 9000)):
        s = _proc_samples(rng, n, ngroups)
        want = po.task_groupby(s, wire.TASK)
        got, ng = eng.task_groupby(s)
        assert ng == len(want) == len(np.unique(s["aggr_task_id"]))
        assert got.tobytes() == want.tobytes(), (n, ngroups)
        # the float sum really is order-dependent on this data: a sorted-order sum differs somewhere
        if n >= 5000:
            resum = np.array([np.sum(np.sort(s["cpu_pct"][s["aggr_task_id"] == g]), dtype=np.float32) for g in want["aggr_task_id"][:300]])
            assert (resum != want["total_cpu_pct"][:300]).any()
    # cap smaller than the number of groups: the first `cap` groups, the count still complete
    part, ng = eng.task_groupby(s, cap=100)
    assert ng == len(want) and part.tobytes() == want[:100].tobytes()
    # feed the first 1200 records (MAX_NUM_TASKS per message) to the engine as partha would send them
    recs = want[:1200]
    msg = wire.build_msg_fixed(ge.NOTIFY_AGGR_TASK_STATE, recs)
    assert eng.ingest_msg(msg, host_idx=1) == 0
    eng.sync()
    st = eng.stats()
    assert st["events_task"] == int((recs["aggr_task_id"] != 0).sum()) and st["wire_msgs_ok"] == 1


def test_task_groupby_at_the_sort_edges():
    """the group-by's two sorts on a field of ceil(log2 n) bits at new plan shapes: 65 537 samples (17 bits: a 9-bit pass with its
    carry, then 8), 262 145 (19 bits: 8, 8, 3); and 4097 groups, so the sort of the groups' first arrivals ends one key into a tile"""
    from gyeeta_b200 import wire
    rng = np.random.default_rng(43)
    eng = ge.Engine(max_svcs=64, max_tasks=1 << 14, max_batch=1 << 19)
    for n, ngroups in ((65_537, 3000), (262_145, 40_000), (12_000, 4097), (65_537, 4097)):
        s = _proc_samples(rng, n, ngroups)
        if ngroups == 4097:         # every group present
            s["aggr_task_id"] = synth.splitmix64(rng.permutation(np.arange(n) % ngroups).astype(np.uint64) + np.uint64(1 << 42))
        want = po.task_groupby(s, wire.TASK)
        got, ng = eng.task_groupby(s)
        assert ng == len(want) == len(np.unique(s["aggr_task_id"]))
        assert ngroups != 4097 or ng == 4097
        assert got.tobytes() == want.tobytes(), (n, ngroups)
