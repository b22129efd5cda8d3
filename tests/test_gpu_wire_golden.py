"""Records the reference itself wrote (tests/golden/wire_ref_golden.npz, from oracle/ref_wire.cc) through every ingest entry that takes
them, against an oracle engine fed events expanded in Python from the golden's named field values, never from the bytes.

The expansion follows the decoders' rules: partha_tcp_conn_info (gy_mconnhdlr.cc:9130), partha_aggr_task_state (:9959),
handle_partha_active_conns (:7705), TCP_SOCK_HANDLER::handle_ipv4/ipv6_conn_event (gy_socket_stat.cc:241-294) and
handle_ipv4/ipv6_resp_event (:1517-1552), SVC_INFO_CAP::upd_stats_on_req for API_TRAN. Entries:
  - gysk_ingest_msg with the whole COMM_HEADER + EVENT_NOTIFY message, and gysk_ingest with the same body (host decode_wire);
  - gysk_ingest_raw with the eBPF records: a few records on the host, and the bulk path (decode_raw_kernel) from pageable and from
    page-locked memory, in one piece and split across calls and across device buffers;
  - gysk_ingest_raw(GYSK_RAW_API_TRAN) with and without trace rows.
After each batch and each flush: the count-min table, every service's and process's histograms, HLL registers and CONN_BITMAP, the
active-connection and RTT fields of gysk_query_svcs, the host summary of the listener states and the trace rows. Records the
decoders skip (zero ids, eBPF type 0 and 5, response times over the limit, neither connect nor accept) must leave nothing behind."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests import trace_agg as ta
from tests.util import assert_hist_equal

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wire_ref_golden.npz")
M32 = 0xFFFFFFFF
GY_SEED = 0xCEEDFEAD
CFG = dict(max_svcs=1 << 12, max_tasks=256, cms_log2_width=12)
RAW_BULK_MIN = 16384                    # gysk_engine.h: from this many records on, raw records are expanded on the device


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def vals(g, name):
    return {str(f): g[f"{name}.{f}"] for f in g[f"{name}__fields"]}


def msg(g, name):
    body = g[f"{name}__bytes"]
    m = np.zeros(int(g[f"{name}__msg_len"]), dtype=np.uint8)
    m[:24] = g[f"{name}__msg_head"]
    m[24: 24 + len(body)] = body
    return m


def pair(**kw):
    c = dict(CFG, **kw)
    eng = ge.Engine(max_batch=1 << 16, **c)
    orc = po.OracleEngine(max_svcs=c["max_svcs"], max_tasks=c["max_tasks"], cms_log2_width=c["cms_log2_width"])
    return eng, orc


def events(n):
    return np.zeros(n, dtype=ge.EVENT_DTYPE)


# ---- expansions from the named values ----------------------------------------------------------------------------------------------

def exp_tcp_conn(v, host):
    keep = (v["ser_glob_id_"] != 0) & (v["cli_task_aggr_id_"] != 0) & ((v["is_tcp_accept_event_"] != 0) | (v["is_tcp_connect_event_"] != 0))
    ev = events(int(keep.sum()))
    acc = v["is_tcp_accept_event_"][keep] != 0                         # accept is tested first when both are set
    closed = v["tusec_close_"][keep] != 0
    ev["type"] = np.where(acc, np.where(closed, ge.EV_CLOSE_SER, ge.EV_ACCEPT), np.where(closed, ge.EV_CLOSE_CLI, ge.EV_CONNECT))
    ev["svc_id"], ev["flow_key"] = v["ser_glob_id_"][keep], v["cli_task_aggr_id_"][keep]
    tot = [min(int(a) + int(b), M32) for a, b in zip(v["bytes_sent_"][keep], v["bytes_rcvd_"][keep])]
    ev["value"] = np.where(closed, np.array(tot, dtype=np.uint64), 0)
    t = np.where(closed, v["tusec_close_"][keep], v["tusec_start_"][keep]) // np.uint64(1_000_000)
    ev["tsec"] = (t & np.uint64(M32)).astype(np.uint32)
    ev["host_idx"] = host
    return ev


def exp_task(v, host):
    keep = v["aggr_task_id_"] != 0
    ev = events(int(keep.sum()))
    ev["svc_id"] = v["aggr_task_id_"][keep]
    ev["flow_key"] = v["cpu_delay_msec_"][keep].astype(np.uint64) | (v["blkio_delay_msec_"][keep].astype(np.uint64) << np.uint64(32))
    ev["value"] = v["total_cpu_pct_"][keep].astype(np.int32).astype(np.uint32)      # (int)total_cpu_pct_, gy_msocket.h:1014
    ev["type"], ev["host_idx"] = ge.EV_TASK, host
    return ev


def exp_active(v, host):
    keep = v["listener_glob_id_"] != 0
    ev = events(int(keep.sum()))
    ev["svc_id"], ev["flow_key"] = v["listener_glob_id_"][keep], v["cli_aggr_task_id_"][keep]
    ev["value"] = [min((int(a) + int(b)) >> 10, M32) for a, b in zip(v["bytes_sent_"][keep], v["bytes_received_"][keep])]
    rtt = v["max_rtt_msec_"][keep]
    ev["tsec"] = np.where(rtt > 0, rtt, np.float32(0)).astype(np.float32).view(np.uint32)
    ev["type"], ev["flags"], ev["host_idx"] = ge.EV_ACTIVE, v["active_conns_"][keep], host
    return ev


def jh(a, b, iv):
    return po.lib().gyo_jhash_2words(int(a) & M32, int(b) & M32, int(iv) & M32)


def raw_svc_id(ip, netns, port):
    id_ = (jh(ip, netns, GY_SEED) << 32) | jh(port, netns, GY_SEED ^ int(ip))
    return id_ or 1


def fold(a):
    if a.ndim == 1:
        return a.astype(np.uint64)
    w = a.view(np.uint32).reshape(len(a), 4)
    return np.array([jh(x[2], x[3], jh(x[0], x[1], GY_SEED)) for x in w], dtype=np.uint64)


def bswap16(a):
    return a.astype(np.uint16).byteswap().astype(np.uint64)


def exp_conn(v, host):
    t = v["type"]
    keep = (t >= ge.EV_CONNECT) & (t <= ge.EV_CLOSE_SER)
    s, d = fold(v["saddr"])[keep], fold(v["daddr"])[keep]
    hs, hd, ns, ty = bswap16(v["sport"][keep]), bswap16(v["dport"][keep]), v["netns"][keep], t[keep]
    ser = (ty == ge.EV_ACCEPT) | (ty == ge.EV_CLOSE_SER)
    sip, sport = np.where(ser, s, d), np.where(ser, hs, hd)
    cip, cport = np.where(ser, d, s), np.where(ser, hd, hs)
    ev = events(int(keep.sum()))
    ev["svc_id"] = [raw_svc_id(a, b, c) for a, b, c in zip(sip, ns, sport)]
    ev["flow_key"] = (cip << np.uint64(32)) | cport
    ev["value"] = [min(int(a) + int(b), M32) for a, b in zip(v["bytes_received"][keep], v["bytes_acked"][keep])]
    ev["tsec"] = ((v["ts_ns"][keep] // np.uint64(10 ** 9)) & np.uint64(M32)).astype(np.uint32)
    ev["type"], ev["host_idx"] = ty, host
    return ev


def exp_resp(v, host):
    tresp = (v["lsndtime"].astype(np.int64) - v["lrcvtime"].astype(np.int64)) & M32
    keep = tresp <= 1_000_000
    sip, cip = fold(v["tup.saddr"])[keep], fold(v["tup.daddr"])[keep]
    ev = events(int(keep.sum()))
    ev["svc_id"] = [raw_svc_id(a, b, c) for a, b, c in zip(sip, v["tup.netns"][keep], bswap16(v["tup.sport"][keep]))]
    ev["flow_key"] = (cip << np.uint64(32)) | bswap16(v["tup.dport"][keep])
    ev["value"] = tresp[keep] * 1000
    ev["type"], ev["host_idx"] = ge.EV_RESP, host
    return ev


def exp_api_tran(v, host, trace):
    n = len(v["glob_id_"])
    err = v["errorcode_"]
    rs = events(n)
    rs["svc_id"], rs["flow_key"] = v["glob_id_"], v["cliport_"]
    rs["value"] = np.minimum(v["response_usec_"], M32)
    rs["tsec"] = ((v["tupd_usec_"] // np.uint64(1_000_000)) & np.uint64(M32)).astype(np.uint32)
    rs["type"], rs["host_idx"] = ge.EV_RESP, host
    rs["flags"] = np.where(err == 0, 0, np.where(err >= 500, ge.EVF_SER_ERROR, ge.EVF_CLI_ERROR))
    if not trace:
        return rs
    tr = events(n)
    tr["svc_id"] = v["glob_id_"]
    tr["flow_key"] = np.minimum(v["reqlen_"], M32) | (np.minimum(v["reslen_"], M32) << np.uint64(32))
    tr["value"], tr["tsec"], tr["host_idx"], tr["type"] = rs["value"], rs["tsec"], host, ge.EV_TRACE
    tr["flags"] = np.where(err != 0, ge.EVF_TRACE_ERROR, 0) | np.where(v["reqnum_"] == 0, ge.EVF_TRACE_NEWCONN, 0)
    ev = events(2 * n)
    ev[0::2], ev[1::2] = rs, tr
    return ev


# ---- comparisons ---------------------------------------------------------------------------------------------------------------------

def compare(eng, orc, ev, flushed=False):
    eng.sync()
    assert np.array_equal(eng.export_cms(), orc.cms()), "count-min table"
    if flushed:
        assert np.array_equal(eng.export_cms(last_window=True), orc.cms(last_window=True)), "last window's count-min table"
    st, oc = eng.stats(), orc.counters()
    assert (st["nsvcs"], st["events_tcp"], st["events_task"]) == (oc["nsvcs"], oc["tcp"], oc["task"])
    svc = np.unique(ev["svc_id"][ev["type"] != ge.EV_TASK])
    for id_ in svc.tolist():
        for w in (ge.HIST_RESP_CUR, ge.HIST_RESP_LAST, ge.HIST_RESP_ALL):
            assert_hist_equal(eng, orc, id_, w)
        assert np.array_equal(eng.export_hll(id_), orc.export_hll(id_)), hex(id_)
        for last in (False, True):
            a, b = eng.export_conn_bitmap(id_, last), orc.export_conn_bitmap(id_, last)
            z = (np.zeros(15, np.uint32), np.zeros(15, np.uint8))
            a, b = a if a is not None else z, b if b is not None else z
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), hex(id_)
    if flushed and len(svc):
        for s_, id_ in zip(eng.query_svcs(svc), svc.tolist()):
            a = orc.export_aux(id_)
            assert s_["found"] == 1 and (s_["nconns_active"], s_["active_kbytes"]) == (a["act_last"] & M32, a["act_last"] >> 32), hex(id_)
            assert s_["max_rtt_msec"] == a["rtt_last"], hex(id_)
    for id_ in np.unique(ev["svc_id"][ev["type"] == ge.EV_TASK]).tolist():
        for w in (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY):
            assert_hist_equal(eng, orc, id_, w)


def skipped_leave_nothing(eng, ids):
    """ids the decoders must have skipped: no service behind them"""
    for id_ in ids:
        assert eng.query_svcs(np.array([id_], dtype=np.uint64))[0]["found"] == 0


def ingest_records(eng, subtype, body, nevents, host):
    """gysk_ingest: one message body, the arguments handle_l2_misc hands to partha_<kind>()"""
    buf = np.ascontiguousarray(body, dtype=np.uint8).copy()
    p = buf.ctypes.data
    return eng.L.gysk_ingest(eng.h, eng._host_id, host, subtype, C.c_void_p(p), nevents, C.c_void_p(p + len(buf)))


# ---- tests ---------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("entry", ["msg", "records"])
def test_notify_messages(g, entry):
    eng, orc = pair()
    allev = []
    for b, (name, exp) in enumerate((("tcp_conn", exp_tcp_conn), ("task", exp_task), ("active", exp_active))):
        v = vals(g, name)
        n = len(next(iter(v.values())))
        host = 3 + b
        if entry == "msg":
            assert eng.ingest_msg(bytearray(msg(g, name).tobytes()), host_idx=host) == 0, name
        else:
            assert ingest_records(eng, int(g[f"{name}__subtype"]), g[f"{name}__bytes"], n, host) == 0, name
        ev = exp(v, host)
        orc.ingest(ev)
        allev.append(ev)
        compare(eng, orc, np.concatenate(allev))
    ev = np.concatenate(allev)
    eng.flush(20); orc.flush(20)
    compare(eng, orc, ev, flushed=True)
    # the message walks again into the next window: the last window is the first one's
    for b, name in enumerate(("tcp_conn", "task", "active")):
        assert eng.ingest_msg(bytearray(msg(g, name).tobytes()), host_idx=3 + b) == 0
    orc.ingest(ev)
    compare(eng, orc, ev)
    eng.flush(25); orc.flush(25)
    compare(eng, orc, ev, flushed=True)
    st = eng.stats()
    assert st["wire_msgs_bad"] == 0
    v = vals(g, "tcp_conn")
    skipped = set(v["ser_glob_id_"][(v["cli_task_aggr_id_"] == 0) | ((v["is_tcp_accept_event_"] == 0) & (v["is_tcp_connect_event_"] == 0))].tolist())
    skipped -= set(ev["svc_id"].tolist())
    skipped_leave_nothing(eng, sorted(skipped - {0}))


def test_listener_state_host_summary(g):
    """LISTENER_STATE_NOTIFY rolled up per host like LISTEN_SUMM_STATS::update inside partha_listener_state (gy_mconnhdlr.cc:11251)"""
    eng = ge.Engine(max_svcs=64, max_tasks=16, max_batch=2048, cms_log2_width=10)
    v = vals(g, "listener")
    want = dict(nstates=[0] * 8, tot_qps=0, tot_act_conn=0, tot_kb_inbound=0, tot_kb_outbound=0, tot_ser_errors=0, nlisteners=0, nactive=0)
    for i in range(len(v["glob_id_"])):
        if int(v["query_flags_"][i]) == 0xC0 or int(v["curr_state_"][i]) > 5:
            continue
        want["nstates"][int(v["curr_state_"][i])] += 1
        want["tot_qps"] += int(v["nqrys_5s_"][i]) // 5
        want["tot_act_conn"] += int(v["nconns_active_"][i])
        want["tot_kb_inbound"] += int(v["curr_kbytes_inbound_"][i])
        want["tot_kb_outbound"] += int(v["curr_kbytes_outbound_"][i])
        want["tot_ser_errors"] += int(v["ser_errors_"][i])
        want["nlisteners"] += 1
        want["nactive"] += int(v["nqrys_5s_"][i] != 0)
    # LISTEN_SUMM_STATS<int>: the sums wrap in int32, as they do in the reference; the golden set's counters make them wrap
    i32 = lambda x: (x + (1 << 31)) % (1 << 32) - (1 << 31)       # noqa: E731
    assert any(i32(x) != x for x in want.values() if isinstance(x, int))
    want = {k: [i32(x) for x in w] if isinstance(w, list) else i32(w) for k, w in want.items()}
    assert eng.ingest_msg(bytearray(msg(g, "listener").tobytes()), host_idx=9) == 0
    got = eng.host_summary(9)
    assert got == want
    eng2 = ge.Engine(max_svcs=64, max_tasks=16, max_batch=2048, cms_log2_width=10)
    assert ingest_records(eng2, int(g["listener__subtype"]), g["listener__bytes"], len(v["glob_id_"]), 9) == 0
    assert eng2.host_summary(9) == got


@pytest.mark.parametrize("name", ["ipv4_event", "ipv6_event", "ipv4_resp", "ipv6_resp"])
def test_raw_ebpf_records(g, name):
    kind = dict(ipv4_event=ge.RAW_TCP_IPV4_EVENT, ipv6_event=ge.RAW_TCP_IPV6_EVENT, ipv4_resp=ge.RAW_TCP_IPV4_RESP,
                ipv6_resp=ge.RAW_TCP_IPV6_RESP)[name]
    exp = exp_conn if name.endswith("event") else exp_resp
    v = vals(g, name)
    raw = g[f"{name}__bytes"]
    n = len(next(iter(v.values())))
    stride = len(raw) // n
    ev1 = exp(v, 5)
    assert len(ev1) < n                                                 # some records are skipped
    reps = (2 * RAW_BULK_MIN + 1500) // n + 1                           # the reference's records repeated past twice the bulk threshold
    bulk = np.tile(raw, reps)
    evb = np.concatenate([ev1] * reps)
    # a few records on the host, then the bulk path from pageable memory, page-locked memory, and in pieces across calls; each engine's
    # device buffer holds 1 << 13 events, so the bulk batches straddle device buffers
    eng, orc = pair()
    small = ge.Engine(max_batch=1 << 13, **CFG)
    pinned = ge.Engine(max_batch=1 << 13, **CFG)
    buf = torch.from_numpy(bulk.copy()).pin_memory()
    for e in (eng, small, pinned):
        e.ingest_raw(kind, raw, n, host_idx=5)
    orc.ingest(ev1)
    compare(eng, orc, ev1)
    eng.ingest_raw(kind, bulk, n * reps, host_idx=5)
    pinned.ingest_raw_ptr(kind, buf.data_ptr(), n * reps, host_idx=5)
    cut = [0, RAW_BULK_MIN + 3, RAW_BULK_MIN + 3 + 700, n * reps]       # bulk, a few on the host, bulk again
    assert n * reps - cut[2] >= RAW_BULK_MIN
    for a, b in zip(cut[:-1], cut[1:]):
        small.ingest_raw(kind, bulk[a * stride: b * stride], b - a, host_idx=5)
    orc.ingest(evb)
    ev = np.concatenate([ev1, evb])
    for e in (eng, small, pinned):
        compare(e, orc, ev)
    for e in (eng, small, pinned):
        e.flush(30)
    orc.flush(30)
    for e in (eng, small, pinned):
        compare(e, orc, ev, flushed=True)
    del buf


@pytest.mark.parametrize("trace", [False, True])
def test_api_tran(g, trace):
    v = vals(g, "api_tran")
    raw = g["api_tran__bytes"]
    n = len(v["glob_id_"])
    eng = ge.Engine(max_batch=1 << 16, max_trace_svcs=64 if trace else 0, **CFG)
    orc = po.OracleEngine(max_svcs=CFG["max_svcs"], max_tasks=CFG["max_tasks"], cms_log2_width=CFG["cms_log2_width"])
    to = ta.TraceOracle(64) if trace else None
    ids = np.unique(v["glob_id_"])
    for b in range(3):
        host = 0
        eng.ingest_raw(ge.RAW_API_TRAN, raw, n, host_idx=host)
        ev = exp_api_tran(v, host, trace)
        orc.ingest(ev)
        if trace:
            to.ingest(ev)
        compare(eng, orc, ev)
        # response times over the validity rule count nowhere in the histograms
        big = v["response_usec_"] > 1_000_000_999
        assert big.any() and sum(eng.export_hist(int(i), ge.HIST_RESP_CUR)[1] for i in ids) == int((~big).sum())
        if trace:
            for id_, r in zip(ids.tolist(), eng.query_traces(ids)):
                assert ta.row_bytes(r) == ta.row_bytes(to.row(id_, host)), hex(id_)
        eng.flush(40 + b); orc.flush(40 + b)
        if trace:
            to.flush()
        compare(eng, orc, ev, flushed=True)
        if trace:
            for id_, r in zip(ids.tolist(), eng.query_traces(ids)):
                assert ta.row_bytes(r) == ta.row_bytes(to.row(id_, host)), hex(id_)
