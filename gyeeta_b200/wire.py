"""numpy mirrors of the wire records of the hot path (common/gy_comm_proto.h:1665-1742 TCP_CONN_NOTIFY, :2114-2254 AGGR_TASK_STATE_NOTIFY /
LISTENER_STATE_NOTIFY, COMM_HEADER + EVENT_NOTIFY :300-420) and of the eBPF structs (common/gy_ebpf_kernel.h:20-130), plus builders of
whole COMM_HEADER messages — what a feeder or a test hands to gysk_ingest_msg / gysk_ingest_raw. Every dtype and encoder is pinned to the
reference's own compiled structs and the records they build by tests/test_wire_layout_host.py."""
import numpy as np

HDR = np.dtype([("magic", "<u4"), ("total_sz", "<u4"), ("data_type", "<u4"), ("padding_sz", "<u4"), ("subtype", "<u4"), ("nevents", "<u4")])
IP_PORT = np.dtype([("ip128", "u1", 16), ("ip32", "<u4"), ("aftype", "<i2"), ("ipflags", "<u2"), ("port", "<u2"), ("pad", "u1", 6)])
TCP_CONN = np.dtype([("cli", IP_PORT), ("ser", IP_PORT), ("nat_cli", IP_PORT), ("nat_ser", IP_PORT), ("tusec_start", "<u8"),
                     ("tusec_close", "<u8"), ("cli_task_aggr_id", "<u8"), ("cli_related_listen_id", "<u8"), ("cli_madhava_id", "<u8"),
                     ("machid", "<u8", 2), ("ser_related_listen_id", "<u8"), ("ser_glob_id", "<u8"), ("ser_madhava_id", "<u8"),
                     ("bytes_sent", "<u8"), ("bytes_rcvd", "<u8"), ("cli_pid", "<i4"), ("ser_pid", "<i4"), ("ser_conn_hash", "<u4"),
                     ("ser_sock_inode", "<u4"), ("cli_comm", "S16"), ("ser_comm", "S16"), ("cli_cmdline_len", "<u2"),
                     ("is_connect", "u1"), ("is_accept", "u1"), ("is_loopback", "u1"), ("is_pre_existing", "u1"), ("notified_before", "u1"),
                     ("padding_len", "u1")])
TASK = np.dtype([("aggr_task_id", "<u8"), ("onecomm", "S16"), ("pid_arr", "<i4", 2), ("tcp_kbytes", "<u4"), ("tcp_conns", "<u4"),
                 ("total_cpu_pct", "<f4"), ("rss_mb", "<u4"), ("cpu_delay_msec", "<u4"), ("vm_delay_msec", "<u4"), ("blkio_delay_msec", "<u4"),
                 ("ntasks_total", "<u2"), ("ntasks_issue", "<u2"), ("curr_state", "u1"), ("curr_issue", "u1"), ("issue_bit_hist", "u1"),
                 ("severe_issue_bit_hist", "u1"), ("issue_string_len", "u1"), ("padding_len", "u1"), ("pad", "u1", 2)])
# AGGR_TASK_HIST_STATS, common/gy_comm_proto.h:2966-2977 (the records of handle_aggr_task_hist_stats)
AGGR_TASK_HIST_STATS = np.dtype([("aggr_task_id", "<u8"), ("starttimeusec", "<u8"), ("p95_cpu_pct", "<u4"), ("p95_cpu_delay_ms", "<u4"),
                                 ("p95_blkio_delay_ms", "<u4"), ("nprocs", "<u4"), ("nthreads", "<u4"), ("max_cores_allowed", "<u2"),
                                 ("cpu_cg_pct_limit", "u1"), ("max_mem_cg_pct_rss", "u1")])
assert AGGR_TASK_HIST_STATS.itemsize == 40
# ACTIVE_CONN_STATS, common/gy_comm_proto.h:2766-2810 (fixed stride); flags holds the three bit-fields cli_listener_proc_ : 1,
# is_remote_listen_ : 1, is_remote_cli_ : 1
ACTIVE = np.dtype([("listener_glob_id", "<u8"), ("cli_aggr_task_id", "<u8"), ("ser_comm", "S16"), ("cli_comm", "S16"), ("machid", "<u8", 2),
                   ("remote_madhava_id", "<u8"), ("bytes_sent", "<u8"), ("bytes_received", "<u8"), ("cli_delay_msec", "<u4"),
                   ("ser_delay_msec", "<u4"), ("max_rtt_msec", "<f4"), ("active_conns", "<u2"), ("flags", "u1"), ("pad", "u1")])
# API_TRAN, common/gy_proto_common.h:140-204 (the fixed part; request_len bytes of request and lenext bytes of extension fields
# follow, then padlen zero bytes to the next multiple of 8)
API_TRAN = np.dtype([("treq_usec", "<u8"), ("tres_usec", "<u8"), ("tupd_usec", "<u8"), ("reqlen", "<u8"), ("reslen", "<u8"),
                     ("reqnum", "<u8"), ("response_usec", "<u8"), ("reaction_usec", "<u8"), ("tconnect_usec", "<u8"), ("cliip", "V24"),
                     ("serip", "V24"), ("glob_id", "<u8"), ("conn_id", "<u8"), ("comm", "S16"), ("errorcode", "<i4"), ("app_sleep_ms", "<u4"),
                     ("tran_type", "<u4"), ("proto", "<u2"), ("cliport", "<u2"), ("serport", "<u2"), ("request_len", "<u2"),
                     ("lenext", "<u2"), ("padlen", "u1"), ("_pad", "V1")])
# raw eBPF records, common/gy_ebpf_kernel.h:37-68,106-118 over gy_ebpf_bpf_common.h:23-39; ports in network byte order
CONN4 = np.dtype([("ts_ns", "<u8"), ("bytes_received", "<u8"), ("bytes_acked", "<u8"), ("pid", "<u4"), ("tid", "<u4"), ("comm", "S16"),
                  ("saddr", "<u4"), ("daddr", "<u4"), ("netns", "<u4"), ("sport", "<u2"), ("dport", "<u2"), ("ipver", "u1"), ("type", "u1")],
                 align=True)
CONN6 = np.dtype(dict(names=["ts_ns", "bytes_received", "bytes_acked", "pid", "tid", "comm", "saddr", "daddr", "netns", "sport", "dport",
                             "ipver", "type"],
                      formats=["<u8", "<u8", "<u8", "<u4", "<u4", "S16", ("<u4", 4), ("<u4", 4), "<u4", "<u2", "<u2", "u1", "u1"],
                      offsets=[0, 8, 16, 24, 28, 32, 48, 64, 80, 84, 86, 88, 89], itemsize=96))
RESP4 = np.dtype([("saddr", "<u4"), ("daddr", "<u4"), ("netns", "<u4"), ("sport", "<u2"), ("dport", "<u2"), ("lsndtime", "<u4"), ("lrcvtime", "<u4")])
RESP6 = np.dtype(dict(names=["saddr", "daddr", "netns", "sport", "dport", "lsndtime", "lrcvtime"],
                      formats=[("<u4", 4), ("<u4", 4), "<u4", "<u2", "<u2", "<u4", "<u4"],
                      offsets=[0, 16, 32, 36, 38, 48, 52], itemsize=64))
assert TCP_CONN.itemsize == 280 and TASK.itemsize == 72 and HDR.itemsize == 24 and RESP4.itemsize == 24
assert ACTIVE.itemsize == 104 and API_TRAN.itemsize == 176 and CONN4.itemsize == 72 and CONN6.itemsize == 96 and RESP6.itemsize == 64
PM_MAGIC, COMM_EVENT_NOTIFY = 0x05666605, 14
MAX_NUM_CONNS, MAX_NUM_TASKS = 2048, 2048          # per-message record caps of the validators (gy_comm_proto.h:1742, :2254)


def header(subtype, nevents, body_len):
    hdr = np.zeros(1, dtype=HDR)
    hdr["magic"], hdr["data_type"] = PM_MAGIC, COMM_EVENT_NOTIFY
    hdr["total_sz"] = HDR.itemsize + body_len
    hdr["subtype"], hdr["nevents"] = subtype, nevents
    return hdr


def build_msg(subtype, recs_with_tail):
    """recs_with_tail: list of (record 1-elem array, tail bytes). Sets padding so every element is 8-byte aligned."""
    body = bytearray()
    for rec, tail in recs_with_tail:
        rec = rec.copy()
        sz = rec.dtype.itemsize + len(tail)
        pad = (-sz) % 8
        if "cli_cmdline_len" in rec.dtype.names:
            rec["cli_cmdline_len"] = len(tail)
        else:
            rec["issue_string_len"] = len(tail)
        rec["padding_len"] = pad
        body += rec.tobytes() + tail + b"\0" * pad
    return bytearray(header(subtype, len(recs_with_tail), len(body)).tobytes() + bytes(body))


def pack_api_tran(recs, tails):
    """API_TRAN records (a structured array of API_TRAN) each followed by its request string and lenext zero bytes, request_len set to
    the string's length and padlen to the next multiple of 8 (API_TRAN::set_padding_len): what gysk_ingest_raw(GYSK_RAW_API_TRAN) reads"""
    out = bytearray()
    for rec, tail in zip(recs, tails):
        rec = rec.copy()
        rec["request_len"] = len(tail)
        act = API_TRAN.itemsize + len(tail) + int(rec["lenext"])
        rec["padlen"] = (-act) % 8
        out += rec.tobytes() + tail + b"\0" * (int(rec["lenext"]) + int(rec["padlen"]))
    return out


def build_msg_fixed(subtype, recs):
    """one message of tail-less records (a structured array, itemsize a multiple of 8): header + the array's bytes"""
    assert recs.dtype.itemsize % 8 == 0
    out = np.empty(HDR.itemsize + recs.nbytes, dtype=np.uint8)
    out[: HDR.itemsize] = header(subtype, len(recs), recs.nbytes).view(np.uint8)
    out[HDR.itemsize:] = recs.view(np.uint8).reshape(-1)
    return out
