"""Generates tests/golden/wire_ref_golden.npz by RUNNING THE REFERENCE's own record types (oracle/_ref/libgyrefwire.so, compiled
from the reference tree by oracle/Makefile from oracle/ref_wire.cc). Run only where that tree exists:
    python tests/golden/make_wire_golden.py
The fixture holds
  - the layout table: sizeof / alignof of every wire, eBPF and API_TRAN record type and the offset and size of every field the
    decoders, gyeeta_b200/wire.py or the shim touch (layout_*);
  - seeded record sets: the field values by name (<set>.<field>), each record's trailing string (<set>__tail, <set>__toff), the
    bytes the reference wrote from them (<set>__bytes) and, for the message kinds, the whole COMM_HEADER + EVENT_NOTIFY message
    its COMM_HEADER constructor made (<set>__msg_head: the 24 header bytes; <set>__msg_len: the message length).
tests/test_wire_layout_host.py holds the library's mirrors and encoders to it and rebuilds it when the library is present;
tests/test_gpu_wire_golden.py feeds its bytes through every ingest entry."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pyoracle as po  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "wire_ref_golden.npz")

NOW_US = 1_760_000_000_000_000          # about 2025-10-09 in Unix-epoch microseconds
MAX_US32 = (1 << 32) * 1_000_000 - 1     # the largest time in usec whose / 1e6 still fits uint32
PORTS = np.array([0, 1, 255, 256, 65535, 80, 443, 8080], dtype=np.uint16)


def be16(p):
    """a port as the kernel stores it: network byte order"""
    return np.asarray(p, dtype=np.uint16).byteswap()


def tails_of(rng, n, maxlen):
    """trailing strings of lengths 0..9 (every padding length 0..7 over any fixed part) and the maximum"""
    lens = np.array([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, maxlen])[np.arange(n) % 11]
    return [bytes(rng.integers(0x21, 0x7F, int(k), dtype=np.uint8)) for k in lens]


def times_us(rng, n):
    t = NOW_US + rng.integers(0, 600_000_000, n, dtype=np.int64).astype(np.uint64)
    t[3::17] = MAX_US32
    t[5::29] = MAX_US32 + 1
    return t


def bytes_pair(rng, n):
    """two byte counters whose sum sometimes crosses 2^32"""
    a = rng.integers(0, 1 << 34, n, dtype=np.int64).astype(np.uint64)
    b = rng.integers(0, 1 << 20, n, dtype=np.int64).astype(np.uint64)
    a[::7] = (1 << 32) - 10; b[::7] = 5
    a[1::7] = (1 << 32) - 10; b[1::7] = 10
    a[2::7] = (1 << 32) - 10; b[2::7] = 20
    return a, b


# Fields no decoder reads take values from small pools, so that the fixture stays small; they still fill every byte of the field.
def pool(rng, n, rows):
    return rows[rng.integers(0, len(rows), n)]


def other(rng, n, lo, hi, dtype):
    """n values of a field no decoder reads, from 16 drawn in [lo, hi)"""
    return pool(rng, n, rng.integers(lo, hi, 16, dtype=np.int64).astype(dtype))


def ids64(rng, n):
    return pool(rng, n, rng.integers(0, 1 << 63, 16, dtype=np.int64).astype(np.uint64) | np.uint64(1 << 63))


def machid(rng, n):
    return pool(rng, n, rng.integers(0, 256, (8, 16), dtype=np.int64).astype(np.uint8))


def comm(rng, n):
    c = np.zeros((16, 16), dtype=np.uint8)
    c[:, :15] = rng.integers(0x61, 0x7B, (16, 15))
    c[::3, 5:] = 0
    return pool(rng, n, c)


def ip_port(rng, n):
    """IP_PORT: GY_IP_ADDR {ip128_be_, ip32_be_, aftype_, ipflags_} + port_, as 32 raw bytes"""
    b = np.zeros((16, 32), dtype=np.uint8)
    b[:, :16] = rng.integers(0, 256, (16, 16))
    b[:, 16:20] = rng.integers(0, 256, (16, 4))
    b[:, 20:22] = np.array([2, 0], dtype=np.uint8)
    b[:, 24:26] = PORTS[np.arange(16) % len(PORTS)].view(np.uint8).reshape(-1, 2)
    return pool(rng, n, b)


def set_tcp_conn(rng, n):
    v = {}
    v["cli_"], v["ser_"], v["nat_cli_"], v["nat_ser_"] = ip_port(rng, n), ip_port(rng, n), ip_port(rng, n), ip_port(rng, n)
    v["tusec_start_"] = times_us(rng, n)
    close = times_us(rng, n) + np.uint64(1000)
    close[::2] = 0                                                       # open connections
    v["tusec_close_"] = close
    v["cli_task_aggr_id_"] = rng.integers(1, 300, n, dtype=np.int64).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    v["cli_task_aggr_id_"][11::41] = 0                                   # skipped by the :9143 guard
    v["ser_glob_id_"] = rng.integers(1, 40, n, dtype=np.int64).astype(np.uint64) * np.uint64(0xC2B2AE3D27D4EB4F)
    v["ser_glob_id_"][13::37] = 0
    v["cli_related_listen_id_"] = ids64(rng, n)
    v["cli_madhava_id_"] = ids64(rng, n)
    v["cli_ser_machine_id_"] = machid(rng, n)
    v["ser_related_listen_id_"] = ids64(rng, n)
    v["ser_madhava_id_"] = ids64(rng, n)
    v["bytes_sent_"], v["bytes_rcvd_"] = bytes_pair(rng, n)
    v["cli_pid_"] = other(rng, n, -5, 1 << 22, np.int32)
    v["ser_pid_"] = other(rng, n, -5, 1 << 22, np.int32)
    v["ser_conn_hash_"] = other(rng, n, 0, 1 << 32, np.uint32)
    v["ser_sock_inode_"] = other(rng, n, 0, 1 << 32, np.uint32)
    v["cli_comm_"], v["ser_comm_"] = comm(rng, n), comm(rng, n)
    kind = np.arange(n) % 5                                              # accept, connect, both, neither, accept
    v["is_tcp_connect_event_"] = np.isin(kind, [1, 2]).astype(np.uint8)
    v["is_tcp_accept_event_"] = np.isin(kind, [0, 2, 4]).astype(np.uint8)
    v["is_loopback_conn_"] = (np.arange(n) % 3 == 0).astype(np.uint8)
    v["is_pre_existing_"] = (np.arange(n) % 4 == 0).astype(np.uint8)
    v["notified_before_"] = (np.arange(n) % 6 == 0).astype(np.uint8)
    return "TCP_CONN_NOTIFY", v, tails_of(rng, n, 256), "NOTIFY_TCP_CONN"


def set_task(rng, n):
    v = {}
    v["aggr_task_id_"] = rng.integers(1, 60, n, dtype=np.int64).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    v["aggr_task_id_"][7::31] = 0
    v["onecomm_"] = comm(rng, n)
    v["pid_arr_"] = np.stack([other(rng, n, 0, 1 << 31, np.int32), other(rng, n, 0, 1 << 31, np.int32)], axis=1)
    v["tcp_kbytes_"] = other(rng, n, 0, 1 << 32, np.uint32)
    v["tcp_conns_"] = other(rng, n, 0, 1 << 20, np.uint32)
    edges = np.array([0, 0.25, 0.999, 1, 1.001, 1.5, 2, 4.999, 5, 9.999, 10, 10.5, 20, 49.99, 50, 99.9, 100, 100.01, 199.5, 200,
                      250.75, 400, 799.99, 1000, 3199.5], dtype=np.float32)
    cpu = (rng.random(n) * 900).astype(np.float32)
    cpu[::2] = edges[np.arange(0, n, 2) // 2 % len(edges)]
    v["total_cpu_pct_"] = cpu
    v["rss_mb_"] = other(rng, n, 0, 1 << 20, np.uint32)
    cd = rng.integers(0, 70000, n, dtype=np.int64).astype(np.uint32)
    cd[::9] = 0xFFFFFFFF
    v["cpu_delay_msec_"] = cd
    v["vm_delay_msec_"] = other(rng, n, 0, 1 << 16, np.uint32)
    bd = rng.integers(0, 1 << 32, n, dtype=np.int64).astype(np.uint32)
    bd[::5] = 0
    v["blkio_delay_msec_"] = bd
    v["ntasks_total_"] = other(rng, n, 0, 1 << 16, np.uint16)
    v["ntasks_issue_"] = other(rng, n, 0, 1 << 16, np.uint16)
    v["curr_state_"] = (np.arange(n) % 6).astype(np.uint8)
    v["curr_issue_"] = other(rng, n, 0, 16, np.uint8)
    v["issue_bit_hist_"] = other(rng, n, 0, 256, np.uint8)
    v["severe_issue_bit_hist_"] = other(rng, n, 0, 256, np.uint8)
    return "AGGR_TASK_STATE_NOTIFY", v, tails_of(rng, n, 255), "NOTIFY_AGGR_TASK_STATE"


def set_listener(rng, n):
    v = {}
    v["glob_id_"] = np.arange(1, n + 1, dtype=np.uint64) * np.uint64(0xC2B2AE3D27D4EB4F)
    u32 = lambda hi=1 << 32: rng.integers(0, hi, n, dtype=np.int64).astype(np.uint32)   # noqa: E731
    q = u32(1 << 20)
    q[::4] = 0
    q[1::23] = 0xFFFFFFFF
    v["nqrys_5s_"] = q
    for k in ("total_resp_5sec_", "nconns_", "ntasks_", "p95_5s_resp_ms_", "p95_5min_resp_ms_", "cli_errors_", "tasks_delay_usec_",
              "tasks_cpudelay_usec_", "tasks_blkiodelay_usec_", "tasks_user_cpu_", "tasks_sys_cpu_", "tasks_rss_mb_"):
        v[k] = other(rng, n, 0, 1 << 32, np.uint32)
    for k in ("nconns_active_", "curr_kbytes_inbound_", "curr_kbytes_outbound_", "ser_errors_"):
        v[k] = u32(1 << 24)
        v[k][::19] = 0xFFFFFFFF >> 2                                     # sums of several stay below 2^32
    v["ntasks_issue_"] = other(rng, n, 0, 1 << 16, np.uint16)
    v["is_http_svc_"] = (np.arange(n) % 2).astype(np.uint8)
    v["curr_state_"] = (np.arange(n) % 8).astype(np.uint8)               # 6 and 7 lie beyond STATE_DOWN
    v["curr_issue_"] = other(rng, n, 0, 16, np.uint8)
    v["issue_bit_hist_"] = other(rng, n, 0, 256, np.uint8)
    v["high_resp_bit_hist_"] = other(rng, n, 0, 256, np.uint8)
    v["last_issue_subsrc_"] = other(rng, n, 0, 16, np.uint8)
    v["query_flags_"] = np.array([0, 0, 1, 0xC0, 0, 0x40, 0x80], dtype=np.uint8)[np.arange(n) % 7]
    return "LISTENER_STATE_NOTIFY", v, tails_of(rng, n, 255), "NOTIFY_LISTENER_STATE"


def set_host(rng, n):
    v = {"curr_time_usec_": np.array([NOW_US], dtype=np.uint64)}
    for k in ("ntasks_issue_", "ntasks_severe_", "ntasks_", "nlisten_issue_", "nlisten_severe_", "nlisten_", "total_cpu_delayms_",
              "total_vm_delayms_", "total_io_delayms_"):
        v[k] = rng.integers(1, 1 << 32, n, dtype=np.int64).astype(np.uint32)
    v["curr_state_"], v["issue_bit_hist_"] = np.array([3], np.uint8), np.array([0xA5], np.uint8)
    v["cpu_issue_"], v["mem_issue_"], v["severe_cpu_issue_"], v["severe_mem_issue_"] = (np.array([x], np.uint8) for x in (1, 0, 1, 1))
    return "HOST_STATE_NOTIFY", v, None, "NOTIFY_HOST_STATE"


def set_active(rng, n):
    v = {}
    v["listener_glob_id_"] = rng.integers(1, 40, n, dtype=np.int64).astype(np.uint64) * np.uint64(0xC2B2AE3D27D4EB4F)
    v["listener_glob_id_"][17::43] = 0
    v["cli_aggr_task_id_"] = rng.integers(1, 300, n, dtype=np.int64).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    v["ser_comm_"], v["cli_comm_"] = comm(rng, n), comm(rng, n)
    v["remote_machine_id_"] = machid(rng, n)
    v["remote_madhava_id_"] = ids64(rng, n)
    a = rng.integers(0, 1 << 45, n, dtype=np.int64).astype(np.uint64)
    b = rng.integers(0, 1 << 30, n, dtype=np.int64).astype(np.uint64)
    a[::5], b[::5] = (1 << 42) - 2048, 1023                             # >> 10 = 2^32 - 2
    a[1::5], b[1::5] = (1 << 42) - 2048, 1024                           # >> 10 = 2^32 - 1
    a[2::5], b[2::5] = (1 << 42) - 1, 1                                 # >> 10 = 2^32: clamped
    a[3::11], b[3::11] = (1 << 32) - 10, 20                             # the sum crosses 2^32 before the shift
    v["bytes_sent_"], v["bytes_received_"] = a, b
    v["cli_delay_msec_"] = other(rng, n, 0, 1 << 32, np.uint32)
    v["ser_delay_msec_"] = other(rng, n, 0, 1 << 32, np.uint32)
    rtt = (rng.random(n) * 300).astype(np.float32)
    rtt[::6] = np.array([-3.5, -0.0, 0.0, 0.25, 1e-3, 123.875], dtype=np.float32)[np.arange(0, n, 6) // 6 % 6]
    v["max_rtt_msec_"] = rtt
    ac = rng.integers(0, 1 << 16, n, dtype=np.int64).astype(np.uint16)
    ac[::13] = 0
    ac[1::13] = 65535
    v["active_conns_"] = ac
    v["cli_listener_proc_"] = (np.arange(n) % 2).astype(np.uint8)
    v["is_remote_listen_"] = (np.arange(n) % 3 == 0).astype(np.uint8)
    v["is_remote_cli_"] = (np.arange(n) % 5 == 0).astype(np.uint8)
    return "ACTIVE_CONN_STATS", v, None, "NOTIFY_ACTIVE_CONN_STATS"


def set_api_tran(rng, n):
    v = {}
    v["treq_usec_"] = pool(rng, n, times_us(rng, 16))
    v["tres_usec_"] = pool(rng, n, times_us(rng, 16))
    v["tupd_usec_"] = times_us(rng, n)
    v["reqlen_"], v["reslen_"] = bytes_pair(rng, n)
    v["reslen_"][4::9] = (1 << 32) + 5
    rq = rng.integers(1, 1000, n, dtype=np.int64).astype(np.uint64)
    rq[::3] = 0                                                          # a new connection
    v["reqnum_"] = rq
    r = rng.integers(0, 30_000_000, n, dtype=np.int64).astype(np.uint64)
    r[::8] = np.array([0, 999, 1_000_000_999, 1_000_001_000, 1_000_001_001, 1 << 32, (1 << 32) + 7, 300_000],
                      dtype=np.uint64)[np.arange(0, n, 8) // 8 % 8]
    v["response_usec_"] = r
    v["reaction_usec_"] = other(rng, n, 0, 1 << 40, np.uint64)
    v["tconnect_usec_"] = pool(rng, n, times_us(rng, 16))
    v["cliip_"] = ip_port(rng, n)[:, :24]
    v["serip_"] = ip_port(rng, n)[:, :24]
    v["glob_id_"] = rng.integers(1, 24, n, dtype=np.int64).astype(np.uint64) * np.uint64(0xC2B2AE3D27D4EB4F)
    v["conn_id_"] = ids64(rng, n)
    v["comm_"] = comm(rng, n)
    v["errorcode_"] = np.array([0, 1, 499, 500, 0, 200, 503, -1, 0], dtype=np.int32)[np.arange(n) % 9]
    v["app_sleep_ms_"] = other(rng, n, 0, 1 << 32, np.uint32)
    v["tran_type_"] = other(rng, n, 0, 1 << 32, np.uint32)
    v["proto_"] = (np.arange(n) % 10).astype(np.uint16)
    v["cliport_"] = PORTS[np.arange(n) % len(PORTS)]
    v["serport_"] = PORTS[(np.arange(n) + 3) % len(PORTS)]
    v["lenext_"] = np.array([0, 0, 3, 0, 13, 0, 0], dtype=np.uint16)[np.arange(n) % 7]
    return "API_TRAN", v, tails_of(rng, n, 300), None


def conn_common(rng, n, v6):
    v = {}
    ts = (NOW_US * 1000 + rng.integers(0, 600_000_000_000, n, dtype=np.int64)).astype(np.uint64)
    ts[3::17] = ((1 << 32) * 10 ** 9) - 1
    v["ts_ns"] = ts
    v["bytes_received"], v["bytes_acked"] = bytes_pair(rng, n)
    v["pid"] = other(rng, n, 0, 1 << 22, np.uint32)
    v["tid"] = other(rng, n, 0, 1 << 22, np.uint32)
    v["comm"] = comm(rng, n)
    nsrv = 24
    srv = rng.integers(1, 1 << 32, nsrv, dtype=np.int64).astype(np.uint32)
    sel = rng.integers(0, nsrv, n)
    cli = rng.integers(1, 1 << 32, n, dtype=np.int64).astype(np.uint32)
    if v6:
        def addr(a32, mapped):
            w = np.zeros((len(a32), 4), dtype=np.uint32)
            w[:, 3] = a32
            w[mapped, 2] = np.uint32(0xFFFF0000).byteswap()             # ::ffff:a.b.c.d
            full = ~mapped
            w[full, 0] = np.uint32(0x20010DB8).byteswap()
            w[full, 1] = rng.integers(0, 1 << 32, int(full.sum()), dtype=np.int64).astype(np.uint32)
            w[full, 2] = rng.integers(0, 1 << 32, int(full.sum()), dtype=np.int64).astype(np.uint32)
            return w
        smapped = (np.arange(nsrv) % 2 == 0)
        srv_w = addr(srv, smapped)
        v["saddr"], v["daddr"] = srv_w[sel], addr(cli, np.arange(n) % 3 == 0)
    else:
        v["saddr"], v["daddr"] = srv[sel], cli
    v["netns"] = np.array([4026531840, 4026532000], dtype=np.uint32)[sel % 2]
    v["sport"] = be16(PORTS[sel % len(PORTS)])
    v["dport"] = be16(np.where(np.arange(n) % 4 == 0, PORTS[np.arange(n) % len(PORTS)], rng.integers(16000, 60000, n)).astype(np.uint16))
    v["ipver"] = np.full(n, 6 if v6 else 4, dtype=np.uint8)
    v["type"] = (np.arange(n) % 6).astype(np.uint8)                      # 0 and 5 are skipped
    return v


def set_ipv4_event(rng, n):
    return "tcp_ipv4_event_t", conn_common(rng, n, False), None, None


def set_ipv6_event(rng, n):
    return "tcp_ipv6_event_t", conn_common(rng, n, True), None, None


def resp_common(rng, n, v6):
    c = conn_common(rng, n, v6)
    # server side of the tuple: saddr / sport the listener, daddr / dport the client
    v = {"tup.saddr": c["saddr"], "tup.daddr": c["daddr"], "tup.netns": c["netns"], "tup.sport": c["sport"], "tup.dport": c["dport"]}
    rcv = rng.integers(0, 1 << 32, n, dtype=np.int64).astype(np.uint32)
    d = rng.integers(0, 30000, n, dtype=np.int64).astype(np.uint32)
    d[::7] = 1_000_000
    d[1::7] = 1_000_001
    d[2::11] = np.uint32(0xFFFFFFFF)                                     # lsndtime just below lrcvtime: wraps below zero
    d[3::13] = 0
    v["lrcvtime"] = rcv
    v["lsndtime"] = (rcv.astype(np.uint64) + d).astype(np.uint32)        # modulo 2^32 like the kernel's jiffies
    return v


def set_ipv4_resp(rng, n):
    return "tcp_ipv4_resp_event_t", resp_common(rng, n, False), None, None


def set_ipv6_resp(rng, n):
    return "tcp_ipv6_resp_event_t", resp_common(rng, n, True), None, None


# name: (builder, distinct records, records in the set). A set of the message kinds holds each kind's per-message maximum
# (TCP_CONN_NOTIFY::MAX_NUM_CONNS 2048, AGGR_TASK_STATE_NOTIFY::MAX_NUM_TASKS 1200, LISTENER_STATE_NOTIFY::MAX_NUM_LISTENERS 512,
# ACTIVE_CONN_STATS::MAX_NUM_CONNS 2048, API_TRAN::MAX_NUM_REQS 256). Its records repeat a block of distinct ones that reaches
# every edge; each block stays under the 32 KB window of the fixture's compression, so the repeats cost almost nothing.
SETS = dict(tcp_conn=(set_tcp_conn, 64, 2048), task=(set_task, 96, 1200), listener=(set_listener, 96, 512), host=(set_host, 1, 1),
            active=(set_active, 96, 2048), api_tran=(set_api_tran, 72, 256), ipv4_event=(set_ipv4_event, 128, 128),
            ipv6_event=(set_ipv6_event, 128, 128), ipv4_resp=(set_ipv4_resp, 128, 128), ipv6_resp=(set_ipv6_resp, 128, 128))


def repeat(a, n):
    """the first n rows of a repeated"""
    return np.concatenate([a] * (-(-n // len(a))))[:n]


def generate(R):
    """the fixture's arrays, built with the reference library R"""
    structs, fields = po.wire_layout(R)
    out = {
        "layout_struct_name": np.array(list(structs)), "layout_struct_size": np.array([s for s, _ in structs.values()], dtype=np.uint32),
        "layout_struct_align": np.array([a for _, a in structs.values()], dtype=np.uint32),
        "layout_field_struct": np.array([f[0] for f in fields]), "layout_field_name": np.array([f[1] for f in fields]),
        "layout_field_off": np.array([f[2] for f in fields], dtype=np.uint32), "layout_field_size": np.array([f[3] for f in fields], dtype=np.uint32),
    }
    for i, (name, (fn, k, n)) in enumerate(SETS.items()):
        rng = np.random.default_rng(20261017 + i)
        strct, vals, tails, subtype = fn(rng, k)
        vals = {f: repeat(a, n) for f, a in vals.items()}
        tails = None if tails is None else [tails[j % k] for j in range(n)]
        out[f"{name}__struct"] = np.array(strct)
        out[f"{name}__fields"] = np.array(list(vals))
        for k, a in vals.items():
            out[f"{name}.{k}"] = a
        if tails is not None:
            out[f"{name}__tail"] = np.frombuffer(b"".join(tails), dtype=np.uint8).copy()
            out[f"{name}__toff"] = np.concatenate([[0], np.cumsum([len(t) for t in tails])]).astype(np.uint64)
        body = po.wire_build(R, strct, vals, tails)
        out[f"{name}__bytes"] = body
        if subtype:
            st = R.gyref_wire_const(subtype.encode())
            out[f"{name}__subtype"] = np.uint32(st)
            msg = po.wire_msg(R, st, n, body)
            # the message is the header the reference's COMM_HEADER / EVENT_NOTIFY wrote, the body above, then the header's padding
            out[f"{name}__msg_head"] = msg[:24].copy()
            out[f"{name}__msg_len"] = np.uint64(len(msg))
    return out


def main():
    R = po.refwire()
    assert R is not None, "reference wire library not built (make -C oracle)"
    np.savez_compressed(PATH, **generate(R))
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
