"""ctypes binding of libgysketch.so (the C ABI of include/gysketch.h). Fails loudly when the CUDA library is missing."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libgysketch.so")

EVENT_DTYPE = np.dtype([("svc_id", "<u8"), ("flow_key", "<u8"), ("value", "<u4"), ("host_idx", "<u4"),
                        ("tsec", "<u4"), ("type", "<u2"), ("flags", "<u2")], align=True)
assert EVENT_DTYPE.itemsize == 32
SERIAL_DTYPE = np.dtype([("count", "<u8"), ("sum", "<i8")])
FLOW_EST_DTYPE = np.dtype([("flow_key", "<u8"), ("count", "<u4"), ("kbytes", "<u4")])
FLOW_QRY_EST_DTYPE = np.dtype([("flow_key", "<u8"), ("queries", "<u4"), ("resp_ms", "<u4")])     # gysk_flow_qry_est
FLOW_RESP_EST_DTYPE = np.dtype([("flow_key", "<u8"), ("counts", "<u4", (15,)), ("total", "<u4"), ("p25_ms", "<i8"), ("p95_ms", "<i8"),
                                ("p99_ms", "<i8")])                                                   # gysk_flow_resp_est
RESP_HIST_WORDS = 8     # u64 words of one flow response histogram cell
# gysk_svc_top_clients (GYSK_FLAG_SVC_TOP_CLIENTS): a service's heaviest clients, best first, and the bound delta
TOPC_K = 16
TOPC_ENTRY_DTYPE = np.dtype([("flow_key", "<u8"), ("kbytes", "<u4"), ("conns", "<u4")])
SVC_TOP_CLIENTS_DTYPE = np.dtype([("glob_id", "<u8"), ("found", "<i4"), ("n", "<u4"), ("delta", "<u8"), ("entries", TOPC_ENTRY_DTYPE, (TOPC_K,))])
assert SVC_TOP_CLIENTS_DTYPE.itemsize == 280
TOPC_OPEN, TOPC_LAST, TOPC_5MIN = 0, 1, 2
FLOW_ERR_EST_DTYPE = np.dtype([("flow_key", "<u8"), ("queries", "<u4"), ("cli_errors", "<u4"), ("ser_errors", "<u4"),
                               ("pad", "<u4")])                                                       # gysk_flow_err_est

EV_CONNECT, EV_ACCEPT, EV_CLOSE_CLI, EV_CLOSE_SER, EV_RESP, EV_TASK, EV_ACTIVE = 1, 2, 3, 4, 5, 6, 7
EVF_CLI_ERROR, EVF_SER_ERROR = 1, 2
HIST_RESP_CUR, HIST_RESP_LAST, HIST_RESP_ALL, HIST_TASK_CPU_PCT, HIST_TASK_CPU_DELAY, HIST_TASK_BLKIO_DELAY, HIST_RESP_5MIN, HIST_RESP_5DAY, HIST_QPS, HIST_ACTIVE_CONN = range(10)
STATE_IDLE, STATE_GOOD, STATE_OK, STATE_BAD, STATE_SEVERE, STATE_DOWN = range(6)
ISSUE_NONE, ISSUE_LISTENER_TASKS, ISSUE_QPS_HIGH, ISSUE_ACTIVE_CONN_HIGH, ISSUE_SERVER_ERRORS, ISSUE_OS_CPU, ISSUE_OS_MEMORY, ISSUE_DEPENDENT, ISSUE_UNKNOWN = range(9)
TOPN_QPS, TOPN_CONNS, TOPN_NET, TOPN_ISSUE, TOPN_ACTIVE = range(5)
RAW_EVENT32, RAW_TCP_IPV4_EVENT, RAW_TCP_IPV4_RESP, RAW_TCP_IPV6_EVENT, RAW_TCP_IPV6_RESP, RAW_API_TRAN, RAW_RESP16, RAW_TCP24, RAW_TASK24 = range(9)
RESP16_DTYPE = np.dtype([("svc_id", "<u8"), ("usec", "<u4"), ("host_idx", "<u2"), ("cli_port", "u1"), ("flags", "u1")])
TCP24_DTYPE = np.dtype([("svc_id", "<u8"), ("flow_key", "<u8"), ("bytes", "<u4"), ("host_idx", "<u2"), ("type", "u1"), ("pad", "u1")])
TASK24_DTYPE = np.dtype([("aggr_task_id", "<u8"), ("cpu_pct", "<u4"), ("cpu_delay_msec", "<u4"), ("blkio_delay_msec", "<u4"), ("host_idx", "<u2"), ("pad", "<u2")])
PROC_SAMPLE_DTYPE = np.dtype([("aggr_task_id", "<u8"), ("pid", "<i4"), ("cpu_pct", "<f4"), ("rss_mb", "<u4"), ("cpu_delay_msec", "<u4"),
                              ("vm_delay_msec", "<u4"), ("blkio_delay_msec", "<u4"), ("tcp_kbytes", "<u4"), ("tcp_conns", "<u4"), ("state", "u1"),
                              ("issue", "u1"), ("issue_bit_hist", "u1"), ("severe_issue_bit_hist", "u1"), ("is_issue", "u1"), ("pad", "u1", 3),
                              ("comm", "S16")])
assert PROC_SAMPLE_DTYPE.itemsize == 64
assert RESP16_DTYPE.itemsize == 16 and TCP24_DTYPE.itemsize == 24 and TASK24_DTYPE.itemsize == 24
NOTIFY_LISTENER_STATE, NOTIFY_TCP_CONN, NOTIFY_AGGR_TASK_STATE, NOTIFY_ACTIVE_CONN_STATS = 0x309, 0x30C, 0x310, 0x312
(HOSTTOP_SVC_ISSUE, HOSTTOP_SVC_QPS, HOSTTOP_SVC_CONNS, HOSTTOP_SVC_NET, HOSTTOP_TASK_ISSUE, HOSTTOP_TASK_NET, HOSTTOP_TASK_CPU, HOSTTOP_TASK_RSS,
 HOSTTOP_TASK_CPU_DELAY, HOSTTOP_TASK_VM_DELAY, HOSTTOP_TASK_BLKIO_DELAY) = range(11)
FLAG_AUTO_REGISTER, FLAG_MERGE_LEVELS, FLAG_MERGE_STATES, FLAG_MERGE_CLUSTERS, FLAG_MERGE_TOPN, FLAG_FLOW_LEVEL = 1, 2, 4, 8, 16, 32
FLAG_MERGE_TRACES = 64
FLAG_FLOW_QUERIES = 128
FLAG_FLOW_QUERY_LEVEL = 0x100
FLAG_FLOW_RESP_HIST = 0x200
FLAG_FLOW_TOPK = 0x400
FLAG_FLOW_TOPK_5MIN = 0x800
FLAG_FLOW_TOPK_SLOW = 0x1000
FLAG_CLIENT_LEVELS = 0x2000
FLAG_FLOW_ERRORS = 0x4000
FLAG_SVC_TOP_CLIENTS = 0x8000
HLL_WINDOW_P = 8
CLIENTS_LAST, CLIENTS_5MIN = 0, 1
FLOW_TOPK_CAP = 4096
TOPN_TASK_CPU, TOPN_TASK_CPU_DELAY, TOPN_TASK_BLKIO_DELAY = range(3)
TD_CAP = 256


class GyskError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"gysketch error {code}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("max_svcs", C.c_uint32), ("max_tasks", C.c_uint32),
                ("cms_depth", C.c_uint32), ("cms_log2_width", C.c_uint32), ("hll_p", C.c_uint32),
                ("td_compression", C.c_uint32), ("max_batch", C.c_uint32), ("flags", C.c_uint32), ("rank", C.c_uint32),
                ("world", C.c_uint32), ("stage_batch", C.c_uint32), ("idle_evict_secs", C.c_uint32),
                ("task_idle_evict_secs", C.c_uint32), ("max_trace_svcs", C.c_uint32)]


class SvcSummary(C.Structure):
    _fields_ = [("glob_id", C.c_uint64), ("found", C.c_int32), ("nqrys_5s", C.c_uint32), ("total_resp_5sec", C.c_uint64),
                ("p95_5s_resp_ms", C.c_int64), ("p99_5s_resp_ms", C.c_int64), ("p25_5s_resp_ms", C.c_int64),
                ("p95_5min_resp_ms", C.c_int64), ("p99_5min_resp_ms", C.c_int64), ("nqrys_5min", C.c_uint64),
                ("p95_5day_resp_ms", C.c_int64), ("nqrys_5day", C.c_uint64),
                ("p95_all_resp_ms", C.c_int64), ("p99_all_resp_ms", C.c_int64), ("nqrys_all", C.c_uint64),
                ("max_resp_ms", C.c_int64), ("nconns_5s", C.c_uint32), ("kbytes_5s", C.c_uint32), ("nconns_all", C.c_uint64),
                ("kbytes_all", C.c_uint64), ("distinct_clients", C.c_double), ("td_p50_us", C.c_double),
                ("td_p95_us", C.c_double), ("td_p99_us", C.c_double), ("td_count", C.c_uint64),
                ("nconns_active", C.c_uint32), ("active_kbytes", C.c_uint32), ("max_rtt_msec", C.c_float),
                ("cli_errors", C.c_uint32), ("ser_errors", C.c_uint32), ("curr_state", C.c_uint8), ("curr_issue", C.c_uint8),
                ("issue_bit_hist", C.c_uint8), ("high_resp_bit_hist", C.c_uint8)]

    def asdict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


WINDOW_ACTIVE_ONLY = 1


class TaskSummary(C.Structure):
    _fields_ = [("aggr_task_id", C.c_uint64), ("found", C.c_int32), ("host_idx", C.c_uint32), ("p95_cpu_pct", C.c_int32),
                ("p95_cpu_delay_ms", C.c_int32), ("p95_blkio_delay_ms", C.c_int32), ("pad", C.c_uint32), ("nsamples", C.c_uint64),
                ("last_count", C.c_uint64 * 3), ("last_sum", C.c_int64 * 3)]

    def asdict(self):
        d = {f: getattr(self, f) for f, _ in self._fields_ if f != "pad"}
        d["last_count"], d["last_sum"] = list(self.last_count), list(self.last_sum)
        return d


class ListenerStateIn(C.Structure):
    """gysk_listener_state_in: the inputs of TCP_LISTENER::get_curr_state (include/gysketch.h)"""
    _fields_ = [(n, C.c_int64) for n in ("r5p95", "r5p99", "r300p95", "r300p99", "r5dp95", "r5dp99", "r5dp25", "rallp95", "rallp99")] + \
               [(n, C.c_uint64) for n in ("nqrys_5s", "total_resp_msec", "tcount_5d")] + \
               [(n, C.c_double) for n in ("mean5", "mean300", "mean5d", "meanall")] + \
               [(n, C.c_int64) for n in ("qps_p95", "qps_p25", "act_p95", "act_p25", "secs_5d")] + \
               [("last_qps_count", C.c_int32), ("nconn", C.c_int32), ("curr_active_conn", C.c_int32), ("ser_errors", C.c_uint32),
                ("nactive_conn_arr", C.c_uint8 * 16), ("task_issue", C.c_uint8), ("task_severe", C.c_uint8), ("task_delay", C.c_uint8),
                ("cpu_issue", C.c_uint8), ("mem_issue", C.c_uint8), ("pad0", C.c_uint8 * 3), ("ntasks_issue", C.c_int32),
                ("ntasks_noissue", C.c_int32), ("tasks_delay_msec", C.c_uint64), ("nserdepends", C.c_uint32), ("pad1", C.c_uint32)]


def classify_listener(inp, high_resp_bit_hist=0):
    """gysk_classify_listener: -> (state, issue, new high_resp_bit_hist)"""
    L = load_library()
    hb, st, iss = C.c_uint8(high_resp_bit_hist), C.c_uint8(), C.c_uint8()
    rc = L.gysk_classify_listener(C.byref(inp), C.byref(hb), C.byref(st), C.byref(iss))
    if rc:
        raise GyskError(rc, "gysk_classify_listener")
    return st.value, iss.value, hb.value


class ListenerDayStats(C.Structure):
    """gysk_listener_day_stats: byte-compatible with LISTENER_DAY_STATS (48 bytes)"""
    _fields_ = [("glob_id", C.c_uint64), ("tcount_5d", C.c_int64), ("tsum_5d", C.c_int64)] + \
               [(n, C.c_uint32) for n in ("p95_5d_respms", "p25_5d_respms", "p95_qps", "p25_qps", "p95_nactive", "p25_nactive")]

    def astuple(self):
        return tuple(getattr(self, f) for f, _ in self._fields_)


class HostListen(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("host_idx", "nlisten", "nlisten_issue", "nlisten_severe")]


class HostStateIn(C.Structure):
    """gysk_host_state_in: the inputs of host_status_update's state rule"""
    _fields_ = [(n, C.c_uint8) for n in ("cpu_issue", "mem_issue", "severe_cpu_issue", "severe_mem_issue", "cpu_idle")] + \
               [("pad", C.c_uint8 * 3)] + [(n, C.c_uint32) for n in ("ntasks_issue", "ntasks_severe", "nlisten_issue", "nlisten_severe")]


def classify_host(**kw):
    """gysk_classify_host on the named fields of HostStateIn (missing ones 0) -> GYSK_STATE_*"""
    L = load_library()
    st = C.c_uint8()
    rc = L.gysk_classify_host(C.byref(HostStateIn(**kw)), C.byref(st))
    if rc:
        raise GyskError(rc, "gysk_classify_host")
    return st.value


class HostSummary(C.Structure):
    _fields_ = [("nstates", C.c_int32 * 8)] + [(n, C.c_int32) for n in ("tot_qps", "tot_act_conn", "tot_kb_inbound", "tot_kb_outbound",
                                                                         "tot_ser_errors", "nlisteners", "nactive", "pad")]


class LogicalState(C.Structure):
    """gysk_logical_state: the member listeners' LISTEN_SUMM_STATS of one logical service (GYSK_FLAG_MERGE_STATES)"""
    _fields_ = [("logical_id", C.c_uint64), ("found", C.c_int32), ("nsvc_issue", C.c_uint32), ("summ", HostSummary)]


assert C.sizeof(LogicalState) == 80


class SvcClients(C.Structure):
    """gysk_svc_clients: distinct clients of a service (or logical service) in the last window and the rolling 300 s
    (GYSK_FLAG_CLIENT_LEVELS)"""
    _fields_ = [("glob_id", C.c_uint64), ("found", C.c_int32), ("pad", C.c_uint32), ("last_5s", C.c_double), ("last_5min", C.c_double)]


assert C.sizeof(SvcClients) == 32


class ClusterState(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("nhosts", "nsvc_issue", "nsvcissue_hosts", "nsvc", "total_qps", "svc_net_mb")] + [("pad", C.c_uint32 * 2)]


class ClusterRow(C.Structure):
    """gysk_cluster_row: the service half of MS_CLUSTER_STATE of one host cluster over every rank (GYSK_FLAG_MERGE_CLUSTERS)"""
    _fields_ = [("cluster_id", C.c_uint64), ("found", C.c_int32), ("pad", C.c_uint32), ("st", ClusterState)]


assert C.sizeof(ClusterRow) == 48


class TopnEntry(C.Structure):
    _fields_ = [("glob_id", C.c_uint64), ("score", C.c_uint64), ("host_idx", C.c_uint32), ("pad", C.c_uint32)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("events_in", "events_dropped", "events_resp", "events_tcp", "events_task", "nsvcs",
                                          "ntasks", "batches", "kernel_launches", "wire_msgs_ok", "wire_msgs_bad", "svcs_evicted")]

    def asdict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


class Capacity(C.Structure):
    """gysk_capacity: current capacities, slots in use, growths so far and the device bytes the engine holds"""
    _fields_ = [(n, C.c_uint32) for n in ("max_svcs", "max_tasks", "svcs_in_use", "tasks_in_use", "ngrows", "pad")] + \
               [("device_bytes", C.c_uint64)]

    def asdict(self):
        return {f: getattr(self, f) for f, _ in self._fields_ if f != "pad"}


assert C.sizeof(Capacity) == 32


def slot_bytes(hll_p=12, task_idle_evict_secs=0):
    """gysk_slot_bytes (no device needed): (device bytes of one service slot, of one process slot) at this hll_p, with or without
    process eviction"""
    L = load_library()
    cfg = Config()
    L.gysk_config_default(C.byref(cfg))
    cfg.hll_p = hll_p
    cfg.task_idle_evict_secs = task_idle_evict_secs
    s, t = C.c_uint64(), C.c_uint64()
    rc = L.gysk_slot_bytes(C.byref(cfg), C.byref(s), C.byref(t))
    if rc:
        raise GyskError(rc, "gysk_slot_bytes")
    return s.value, t.value


class BufferDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("dptr", C.c_void_p), ("nbytes", C.c_uint64), ("redop", C.c_int32), ("pad", C.c_int32)]


_lib = None


def load_library(path=None):
    """dlopen libgysketch.so. Raises when it has not been built: there is no fallback implementation."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise GyskError(-19, f"{path} is missing: build it with `python -m gyeeta_b200.build` "
                             "(CUDA library is the product; no CPU fallback exists)")
    L = C.CDLL(path)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    sig = {
        "gysk_abi_version": (i32, []),
        "gysk_config_default": (None, [vp]),
        "gysk_create": (i32, [vp, vp]),
        "gysk_destroy": (None, [vp]),
        "gysk_last_error": (C.c_char_p, [vp]),
        "gysk_get_stats": (i32, [vp, vp]),
        "gysk_hot_rows_in_use": (C.c_int64, [vp]),
        "gysk_last_batch_keys": (C.c_int64, [vp]),
        "gysk_last_batch_flow_direct": (C.c_int64, [vp]),
        "gysk_flow_table_used": (C.c_int64, [vp]),
        "gysk_register_ids": (i32, [vp, vp, u32, i32]),
        "gysk_ingest": (i32, [vp, vp, u32, u32, vp, u32, vp]),
        "gysk_ingest_msg": (i32, [vp, vp, u32, vp, u32]),
        "gysk_ingest_raw": (i32, [vp, vp, u32, u32, vp, u32]),
        "gysk_ingest_pinned": (i32, [vp, vp, u64]),
        "gysk_ingest_device": (i32, [vp, vp, u64]),
        "gysk_sync": (i32, [vp]),
        "gysk_flush": (i32, [vp, u32]),
        "gysk_evicted_ids": (i32, [vp, vp, u32, vp]),
        "gysk_evicted_task_ids": (i32, [vp, vp, u32, vp]),
        "gysk_task_evict_count": (i32, [vp, vp]),
        "gysk_query_svcs": (i32, [vp, vp, u32, vp]),
        "gysk_query_traces": (i32, [vp, vp, u32, vp]),
        "gysk_query_trace_window": (i32, [vp, i32, u32, vp, u32, vp]),
        "gysk_export_trace_tdigest": (i32, [vp, u64, i32, vp, vp, u32, vp, vp, vp]),
        "gysk_export_trace_tdigest_pgtext": (i32, [vp, u64, i32, vp, u32]),
        "gysk_trace_info": (i32, [vp, vp, vp]),
        "gysk_query_flows": (i32, [vp, vp, u32, i32, vp]),
        "gysk_query_window": (i32, [vp, C.c_int32, u32, vp, u32, vp]),
        "gysk_query_window_hosts": (i32, [vp, C.c_int32, u32, vp, vp, u32, vp]),
        "gysk_query_tasks": (i32, [vp, vp, u32, vp]),
        "gysk_query_task_window": (i32, [vp, C.c_int32, u32, vp, u32, vp]),
        "gysk_query_host_summary": (i32, [vp, u32, vp]),
        "gysk_topn_svcs": (i32, [vp, i32, C.c_int32, u32, vp, vp]),
        "gysk_topn_tasks": (i32, [vp, i32, u32, vp, vp]),
        "gysk_topn_host": (i32, [vp, i32, C.c_int32, u32, vp, vp]),
        "gysk_query_cluster_state": (i32, [vp, vp, u32, vp]),
        "gysk_export_hist": (i32, [vp, u64, i32, vp, vp, vp]),
        "gysk_export_task_hist": (i32, [vp, u64, i32, vp, vp, vp]),
        "gysk_export_hll": (i32, [vp, u64, vp]),
        "gysk_export_conn_bitmap": (i32, [vp, u64, i32, vp, vp]),
        "gysk_export_tdigest": (i32, [vp, u64, vp, vp, u32, vp, vp, vp]),
        "gysk_query_quantiles": (i32, [vp, u64, vp, u32, vp]),
        "gysk_tdigest_to_pgtext": (i32, [vp, vp, u32, u32, vp, u32]),
        "gysk_encode_listener_state": (i32, [vp, u32, vp, u32, vp, vp]),
        "gysk_export_tdigest_pgtext": (i32, [vp, u64, vp, u32]),
        "gysk_export_cms": (i32, [vp, i32, vp]),
        "gysk_hist_nbuckets": (i32, [i32]),
        "gysk_hist_bucket": (i32, [i32, C.c_int64]),
        "gysk_hist_percentiles": (i32, [i32, i32, vp, u64, vp, u32, vp]),
        "gysk_classify_listener": (i32, [vp, vp, vp, vp]),
        "gysk_query_day_stats": (i32, [vp, C.c_int32, vp, vp, u32, vp]),
        "gysk_query_host_listen": (i32, [vp, vp, u32, vp]),
        "gysk_classify_host": (i32, [vp, vp]),
        "gysk_task_groupby": (i32, [vp, vp, u32, vp, u32, vp]),
        "gysk_hll_estimate": (C.c_double, [vp, u32]),
        "gysk_tdigest_quantile": (C.c_double, [vp, vp, u32, C.c_double, C.c_double, C.c_double]),
        "gysk_uint64_hash": (u32, [u64]),
        "gysk_set_logical_map": (i32, [vp, vp, vp, u32]),
        "gysk_merge_prepare": (i32, [vp]),
        "gysk_merge_buffers": (i32, [vp, vp, u32, vp]),
        "gysk_merge_tdigest_slab": (i32, [vp, vp, vp]),
        "gysk_merge_finish": (i32, [vp, vp, u32]),
        "gysk_query_logical": (i32, [vp, vp, u32, vp]),
        "gysk_export_logical_hist": (i32, [vp, u64, i32, vp, vp, vp]),
        "gysk_merge_flush_range": (i32, [vp, vp, vp]),
        "gysk_query_logical_all": (i32, [vp, u32, vp, u32, vp]),
        "gysk_topn_logical": (i32, [vp, i32, u32, vp, vp]),
        "gysk_export_logical_tdigest": (i32, [vp, u64, vp, vp, u32, vp, vp, vp]),
        "gysk_export_logical_tdigest_pgtext": (i32, [vp, u64, vp, u32]),
        "gysk_query_logical_quantiles": (i32, [vp, u64, vp, u32, vp]),
        "gysk_export_logical_hll": (i32, [vp, u64, vp]),
        "gysk_query_logical_states": (i32, [vp, vp, u32, vp]),
        "gysk_query_logical_states_all": (i32, [vp, u32, vp, u32, vp]),
        "gysk_query_logical_traces": (i32, [vp, vp, u32, vp]),
        "gysk_query_logical_traces_all": (i32, [vp, u32, vp, u32, vp]),
        "gysk_export_logical_trace_tdigest": (i32, [vp, u64, vp, vp, u32, vp, vp, vp]),
        "gysk_export_logical_trace_tdigest_pgtext": (i32, [vp, u64, vp, u32]),
        "gysk_set_cluster_map": (i32, [vp, vp, vp, u32]),
        "gysk_query_cluster_states": (i32, [vp, vp, u32, vp]),
        "gysk_query_cluster_states_all": (i32, [vp, u32, vp, u32, vp]),
        "gysk_topn_global": (i32, [vp, i32, u32, vp, vp, vp]),
        "gysk_topn_global_tasks": (i32, [vp, i32, u32, vp, vp, vp]),
        "gysk_query_flows_global": (i32, [vp, vp, u32, i32, vp]),
        "gysk_query_flows_5min": (i32, [vp, vp, u32, vp]),
        "gysk_export_cms_5min": (i32, [vp, vp]),
        "gysk_query_flows_global_5min": (i32, [vp, vp, u32, vp]),
        "gysk_query_flow_queries": (i32, [vp, vp, u32, i32, vp]),
        "gysk_export_cms_queries": (i32, [vp, i32, vp]),
        "gysk_query_flow_queries_global": (i32, [vp, vp, u32, i32, vp]),
        "gysk_query_flow_queries_5min": (i32, [vp, vp, u32, vp]),
        "gysk_export_cms_queries_5min": (i32, [vp, vp]),
        "gysk_query_flow_queries_global_5min": (i32, [vp, vp, u32, vp]),
        "gysk_last_batch_flow_query_direct": (C.c_int64, [vp]),
        "gysk_query_flow_resp": (i32, [vp, vp, u32, i32, vp]),
        "gysk_export_cms_resp": (i32, [vp, i32, vp]),
        "gysk_query_flow_resp_global": (i32, [vp, vp, u32, i32, vp]),
        "gysk_query_flow_resp_5min": (i32, [vp, vp, u32, vp]),
        "gysk_export_cms_resp_5min": (i32, [vp, vp]),
        "gysk_query_flow_resp_global_5min": (i32, [vp, vp, u32, vp]),
        "gysk_last_batch_flow_resp_direct": (C.c_int64, [vp]),
        "gysk_topk_flows": (i32, [vp, i32, u32, vp, vp]),
        "gysk_topk_flow_queries": (i32, [vp, i32, u32, vp, vp]),
        "gysk_topk_flows_global": (i32, [vp, u32, vp, vp]),
        "gysk_topk_flow_queries_global": (i32, [vp, u32, vp, vp]),
        "gysk_topk_flows_5min": (i32, [vp, u32, vp, vp, vp]),
        "gysk_topk_flow_queries_5min": (i32, [vp, u32, vp, vp, vp]),
        "gysk_topk_flows_global_5min": (i32, [vp, u32, vp, vp, vp]),
        "gysk_topk_flow_queries_global_5min": (i32, [vp, u32, vp, vp, vp]),
        "gysk_set_flow_slow": (i32, [vp, u32]),
        "gysk_topk_flow_slow": (i32, [vp, i32, u32, vp, vp]),
        "gysk_topk_flow_slow_global": (i32, [vp, u32, vp, vp]),
        "gysk_topk_flow_slow_5min": (i32, [vp, u32, vp, vp, vp]),
        "gysk_topk_flow_slow_global_5min": (i32, [vp, u32, vp, vp, vp]),
        "gysk_query_flow_errors": (i32, [vp, vp, u32, i32, vp]),
        "gysk_query_flow_errors_5min": (i32, [vp, vp, u32, vp]),
        "gysk_query_flow_errors_global": (i32, [vp, vp, u32, i32, vp]),
        "gysk_query_flow_errors_global_5min": (i32, [vp, vp, u32, vp]),
        "gysk_export_cms_errors": (i32, [vp, i32, vp]),
        "gysk_export_cms_errors_5min": (i32, [vp, vp]),
        "gysk_last_batch_flow_err_direct": (C.c_int64, [vp]),
        "gysk_topk_flow_errors": (i32, [vp, i32, u32, vp, vp]),
        "gysk_topk_flow_errors_global": (i32, [vp, u32, vp, vp]),
        "gysk_topk_flow_errors_5min": (i32, [vp, u32, vp, vp, vp]),
        "gysk_topk_flow_errors_global_5min": (i32, [vp, u32, vp, vp, vp]),
        "gysk_query_svc_clients": (i32, [vp, vp, u32, vp]),
        "gysk_query_svc_top_clients": (i32, [vp, vp, u32, i32, vp]),
        "gysk_query_top_clients_window": (i32, [vp, C.c_int32, u32, i32, vp, vp, u32, vp]),
        "gysk_query_logical_top_clients": (i32, [vp, vp, u32, i32, vp]),
        "gysk_query_logical_top_clients_all": (i32, [vp, u32, i32, vp, u32, vp]),
        "gysk_query_clients_window": (i32, [vp, C.c_int32, u32, vp, vp, u32, vp]),
        "gysk_export_hll_window": (i32, [vp, u64, i32, vp]),
        "gysk_query_logical_clients": (i32, [vp, vp, u32, vp]),
        "gysk_export_logical_hll_window": (i32, [vp, u64, i32, vp]),
        "gysk_nccl_unique_id": (i32, [vp]),
        "gysk_nccl_comm_init": (i32, [vp, vp, u32, u32]),
        "gysk_merge_global": (i32, [vp, vp]),
        "gysk_stream": (vp, [vp]),
        "gysk_profile_enable": (i32, [vp, i32]),
        "gysk_profile_read": (i32, [vp, vp, vp, vp]),
        "gysk_grow": (i32, [vp, u32, u32]),
        "gysk_set_auto_grow": (i32, [vp, u32, u32]),
        "gysk_capacity_info": (i32, [vp, vp]),
        "gysk_slot_bytes": (i32, [vp, vp, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)          # AttributeError here = the library does not export what the header declares
        fn.restype = res
        fn.argtypes = args
    if path == LIB_PATH:
        _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class TraceWindow(C.Structure):
    """gysk_trace_window: one 5-s window of a service's request traces (the trace view's columns)"""
    _fields_ = [(n, C.c_uint64) for n in ("nreq", "nerr", "nconns", "sum_resp_us", "max_resp_us", "bytes_in", "bytes_out",
                                          "max_bytes_in", "max_bytes_out")] + \
               [("resp_buckets", C.c_uint64 * 8), ("td_count", C.c_uint64), ("p99_resp_us", C.c_double)]

    def asdict(self):
        d = {f: getattr(self, f) for f, _ in self._fields_}
        d["resp_buckets"] = list(self.resp_buckets)
        return d


class TraceRow(C.Structure):
    _fields_ = [("glob_id", C.c_uint64), ("found", C.c_int32), ("host_idx", C.c_uint32), ("cur", TraceWindow), ("last", TraceWindow)]

    def asdict(self):
        return {"glob_id": self.glob_id, "found": self.found, "host_idx": self.host_idx, "cur": self.cur.asdict(), "last": self.last.asdict()}




class LogicalTrace(C.Structure):
    """gysk_logical_trace: the members' last closed trace windows of one logical service, merged over every rank (GYSK_FLAG_MERGE_TRACES)"""
    _fields_ = [("logical_id", C.c_uint64), ("found", C.c_int32), ("ntraced", C.c_uint32), ("last", TraceWindow)]

    def asdict(self):
        return {"logical_id": self.logical_id, "found": self.found, "ntraced": self.ntraced, "last": self.last.asdict()}


assert C.sizeof(TraceWindow) == 152 and C.sizeof(TraceRow) == 320 and C.sizeof(LogicalTrace) == 168
TRACE_TD_CAP = 100
EV_TRACE = 8
EVF_TRACE_ERROR, EVF_TRACE_NEWCONN = 0x1, 0x2


class Engine:
    """One engine = one GPU. Mirrors the C ABI one to one."""

    def __init__(self, device=0, max_svcs=1 << 14, max_tasks=1 << 12, cms_depth=4, cms_log2_width=20, hll_p=12,
                 td_compression=200, max_batch=1 << 20, auto_register=True, rank=0, world=1, stage_batch=0, idle_evict_secs=0,
                 merge_levels=False, merge_states=False, merge_clusters=False, merge_topn=False, flow_level=False, task_idle_evict_secs=0,
                 max_trace_svcs=0, merge_traces=False, flow_queries=False, flow_query_level=False, flow_resp_hist=False,
                 flow_topk=False, flow_topk_5min=False, flow_topk_slow=False, client_levels=False, flow_errors=False,
                 svc_top_clients=False):
        self.L = load_library()
        cfg = Config()
        self.L.gysk_config_default(C.byref(cfg))
        cfg.device, cfg.max_svcs, cfg.max_tasks = device, max_svcs, max_tasks
        cfg.cms_depth, cfg.cms_log2_width, cfg.hll_p, cfg.td_compression = cms_depth, cms_log2_width, hll_p, td_compression
        cfg.max_batch = max_batch
        cfg.stage_batch = stage_batch
        cfg.idle_evict_secs = idle_evict_secs
        cfg.task_idle_evict_secs = task_idle_evict_secs
        cfg.max_trace_svcs = max_trace_svcs
        cfg.flags = (FLAG_AUTO_REGISTER if auto_register else 0) | (FLAG_MERGE_LEVELS if merge_levels else 0) | \
                    (FLAG_MERGE_STATES if merge_states else 0) | (FLAG_MERGE_CLUSTERS if merge_clusters else 0) | \
                    (FLAG_MERGE_TOPN if merge_topn else 0) | (FLAG_FLOW_LEVEL if flow_level else 0) | (FLAG_MERGE_TRACES if merge_traces else 0) | \
                    (FLAG_FLOW_QUERIES if flow_queries else 0) | (FLAG_FLOW_QUERY_LEVEL if flow_query_level else 0) | \
                    (FLAG_FLOW_RESP_HIST if flow_resp_hist else 0) | (FLAG_FLOW_TOPK if flow_topk else 0) | \
                    (FLAG_FLOW_TOPK_5MIN if flow_topk_5min else 0) | (FLAG_FLOW_TOPK_SLOW if flow_topk_slow else 0) | \
                    (FLAG_CLIENT_LEVELS if client_levels else 0) | (FLAG_FLOW_ERRORS if flow_errors else 0) | \
                    (FLAG_SVC_TOP_CLIENTS if svc_top_clients else 0)
        cfg.rank, cfg.world = rank, world
        self.cfg = cfg
        self.h = C.c_void_p()
        rc = self.L.gysk_create(C.byref(cfg), C.byref(self.h))
        if rc:
            raise GyskError(rc, (self.L.gysk_last_error(None) or b"").decode())
        self._host_id = (C.c_uint8 * 16)()

    def _chk(self, rc):
        if rc:
            raise GyskError(rc, (self.L.gysk_last_error(self.h) or b"").decode())

    def close(self):
        if getattr(self, "h", None):
            self.L.gysk_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- ingest ----
    def register_ids(self, ids, is_task=False):
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        self._chk(self.L.gysk_register_ids(self.h, _p(ids), len(ids), int(is_task)))

    def ingest_events(self, ev, host_idx=0):
        assert ev.dtype == EVENT_DTYPE
        ev = np.ascontiguousarray(ev)
        self._chk(self.L.gysk_ingest_raw(self.h, self._host_id, host_idx, RAW_EVENT32, _p(ev), len(ev)))

    def ingest_raw(self, kind, buf, n, host_idx=0):
        self._chk(self.L.gysk_ingest_raw(self.h, self._host_id, host_idx, kind, _p(buf), n))

    def ingest_raw_ptr(self, kind, ptr, n, host_idx=0):
        """ingest_raw on a raw host address (e.g. a page-locked torch tensor's data_ptr())"""
        self._chk(self.L.gysk_ingest_raw(self.h, self._host_id, host_idx, kind, C.c_void_p(ptr), n))

    def ingest_pinned_ptr(self, ptr, n):
        self._chk(self.L.gysk_ingest_pinned(self.h, C.c_void_p(ptr), n))

    def ingest_device_ptr(self, dptr, n):
        self._chk(self.L.gysk_ingest_device(self.h, C.c_void_p(dptr), n))

    def ingest_msg(self, msg, host_idx=0):
        """msg: writable bytes-like holding COMM_HEADER + EVENT_NOTIFY + records"""
        buf = np.frombuffer(msg, dtype=np.uint8)
        return self.L.gysk_ingest_msg(self.h, self._host_id, host_idx, _p(buf), len(buf))

    def sync(self):
        self._chk(self.L.gysk_sync(self.h))

    def flush(self, tsec=0):
        self._chk(self.L.gysk_flush(self.h, tsec))

    def evicted_ids(self, cap=1 << 16):
        """ids evicted by the most recent flush (LISTEN_FLAG_DELETE notifications)"""
        out = np.zeros(cap, dtype=np.uint64)
        n = C.c_uint32()
        self._chk(self.L.gysk_evicted_ids(self.h, _p(out), cap, C.byref(n)))
        return out[:min(n.value, cap)].copy()

    def evicted_task_ids(self, cap=1 << 16):
        """aggregated-process ids evicted by the most recent flush (task_idle_evict_secs), ascending"""
        out = np.zeros(cap, dtype=np.uint64)
        n = C.c_uint32()
        self._chk(self.L.gysk_evicted_task_ids(self.h, _p(out), cap, C.byref(n)))
        return out[:min(n.value, cap)].copy()

    def query_traces(self, ids):
        """gysk_query_traces: one TraceRow per id"""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (TraceRow * max(len(ids), 1))()
        self._chk(self.L.gysk_query_traces(self.h, _p(ids), len(ids), out))
        return out[:len(ids)]

    def query_trace_window(self, host_idx=-1, active_only=False, cap=None):
        """gysk_query_trace_window: (TraceRow rows in ascending glob_id, number of matching rows); cap None = all rows"""
        flags = WINDOW_ACTIVE_ONLY if active_only else 0
        n = C.c_uint32()
        if cap is None:
            self._chk(self.L.gysk_query_trace_window(self.h, host_idx, flags, None, 0, C.byref(n)))
            cap = n.value
        out = (TraceRow * max(cap, 1))()
        self._chk(self.L.gysk_query_trace_window(self.h, host_idx, flags, out if cap else None, cap, C.byref(n)))
        return out[:min(cap, n.value)], n.value

    def export_trace_tdigest(self, id_, last_window=False):
        """gysk_export_trace_tdigest: (means, weights, min, max) of one window's digest, None for an id without a trace row"""
        means = np.zeros(TRACE_TD_CAP, dtype=np.float64)
        weights = np.zeros(TRACE_TD_CAP, dtype=np.uint64)
        n, mn, mx = C.c_uint32(), C.c_double(), C.c_double()
        rc = self.L.gysk_export_trace_tdigest(self.h, int(id_), int(bool(last_window)), _p(means), _p(weights), TRACE_TD_CAP, C.byref(n),
                                              C.byref(mn), C.byref(mx))
        if rc == -2:
            return None
        self._chk(rc)
        return means[: n.value].copy(), weights[: n.value].copy(), mn.value, mx.value

    def export_trace_tdigest_pgtext(self, id_, last_window=False):
        buf = C.create_string_buffer(8192)
        rc = self.L.gysk_export_trace_tdigest_pgtext(self.h, int(id_), int(bool(last_window)), buf, len(buf))
        if rc == -2:
            return None
        if rc < 0:
            self._chk(rc)
        return buf.value.decode()

    def trace_info(self):
        """gysk_trace_info: (rows in use, trace events dropped for want of a row)"""
        rows, dropped = C.c_uint32(), C.c_uint64()
        self._chk(self.L.gysk_trace_info(self.h, C.byref(rows), C.byref(dropped)))
        return rows.value, dropped.value

    def task_evict_count(self):
        """aggregated processes evicted so far"""
        t = C.c_uint64()
        self._chk(self.L.gysk_task_evict_count(self.h, C.byref(t)))
        return t.value

    def stream(self):
        return self.L.gysk_stream(self.h)

    def profile_enable(self, on=True):
        self._chk(self.L.gysk_profile_enable(self.h, int(on)))

    def profile_read(self):
        a, b, n = C.c_double(), C.c_double(), C.c_uint64()
        self._chk(self.L.gysk_profile_read(self.h, C.byref(a), C.byref(b), C.byref(n)))
        return a.value, b.value, n.value

    # ---- capacity ----
    def grow(self, max_svcs=None, max_tasks=None):
        """gysk_grow: raise the service / process capacity (None: keep that one). Every answer stays as an engine created at the
        new capacity would give it."""
        cap = self.capacity()
        ms = cap["max_svcs"] if max_svcs is None else max_svcs
        mt = cap["max_tasks"] if max_tasks is None else max_tasks
        self._chk(self.L.gysk_grow(self.h, ms, mt))
        self.cfg.max_svcs, self.cfg.max_tasks = ms, mt

    def set_auto_grow(self, max_svcs_limit=0, max_tasks_limit=0):
        """gysk_set_auto_grow: at each flush, double a table that was half full at the previous flush, up to its limit (0 = never)"""
        self._chk(self.L.gysk_set_auto_grow(self.h, max_svcs_limit, max_tasks_limit))

    def capacity(self):
        """gysk_capacity_info as a dict; also brings self.cfg's capacities up to date after automatic growth"""
        c = Capacity()
        self._chk(self.L.gysk_capacity_info(self.h, C.byref(c)))
        self.cfg.max_svcs, self.cfg.max_tasks = c.max_svcs, c.max_tasks
        return c.asdict()

    # ---- queries ----
    def stats(self):
        s = Stats()
        self._chk(self.L.gysk_get_stats(self.h, C.byref(s)))
        return s.asdict()

    def _counter(self, fn):
        """one int64 diagnostic of fn (a negative value is an error code)"""
        n = fn(self.h)
        if n < 0:
            self._chk(int(n))
        return int(n)

    def hot_rows_in_use(self):
        """rows of dense value bins handed out to hot services so far (diagnostic; results never depend on it)"""
        return self._counter(self.L.gysk_hot_rows_in_use)

    def last_batch_keys(self):
        """response samples of the last device batch that travelled as sort keys (diagnostic)"""
        return self._counter(self.L.gysk_last_batch_keys)

    def last_batch_flow_direct(self):
        """connection records of the last device batch whose count-min update bypassed the flow table (diagnostic)"""
        return self._counter(self.L.gysk_last_batch_flow_direct)

    def last_batch_flow_query_direct(self):
        """response samples of the last device batch whose flow query update bypassed the query flow table (flow_queries=True)"""
        return self._counter(self.L.gysk_last_batch_flow_query_direct)

    def last_batch_flow_resp_direct(self):
        """response samples of the last device batch whose flow response histogram update bypassed its flow table (flow_resp_hist=True)"""
        return self._counter(self.L.gysk_last_batch_flow_resp_direct)

    def last_batch_flow_err_direct(self):
        """error samples of the last device batch whose flow error update bypassed the error flow table (flow_errors=True)"""
        return self._counter(self.L.gysk_last_batch_flow_err_direct)

    def flow_table_used(self):
        """non-zero entries of the batch flow tables (the query one too with flow_queries=True, the response one with
        flow_resp_hist=True, the error one with flow_errors=True): 0 whenever no batch is in flight (diagnostic)"""
        n = self.L.gysk_flow_table_used(self.h)
        if n < 0:
            self._chk(int(n))
        return int(n)

    def query_svcs(self, ids):
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (SvcSummary * len(ids))()
        self._chk(self.L.gysk_query_svcs(self.h, _p(ids), len(ids), out))
        return [o.asdict() for o in out]

    def listener_state_records(self, ids):
        """query_svcs + gysk_encode_listener_state: the LISTENER_STATE_NOTIFY records (bytes) of the known ids, <= 512"""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (SvcSummary * len(ids))()
        self._chk(self.L.gysk_query_svcs(self.h, _p(ids), len(ids), out))
        buf = C.create_string_buffer(88 * 512)
        nrecs, nbytes = C.c_uint32(), C.c_uint32()
        self._chk(self.L.gysk_encode_listener_state(out, len(ids), buf, len(buf), C.byref(nrecs), C.byref(nbytes)))
        return nrecs.value, buf.raw[: nbytes.value]

    def _window(self, fn, row_type, args, active_only, cap):
        """fn(h, *args, flags, out, cap, &n): (rows, number of matching rows); cap None = a count call first, then every row"""
        flags = WINDOW_ACTIVE_ONLY if active_only else 0
        n = C.c_uint32()
        if cap is None:
            self._chk(fn(self.h, *args, flags, None, 0, C.byref(n)))
            cap = n.value
        out = (row_type * max(cap, 1))()
        self._chk(fn(self.h, *args, flags, out if cap else None, cap, C.byref(n)))
        return out[: min(cap, n.value)], n.value

    def query_window(self, host_idx=-1, active_only=False, cap=None):
        """gysk_query_window: (SvcSummary rows grouped by host, ids ascending within a host; number of matching rows).
        cap None = all rows (a count call first); 0 = the count only"""
        return self._window(self.L.gysk_query_window, SvcSummary, (host_idx,), active_only, cap)

    def query_window_hosts(self, host_idx=-1, active_only=False, cap=None):
        """gysk_query_window_hosts: (rows, host_idx of each row as a uint32 array, number of matching rows)"""
        flags = WINDOW_ACTIVE_ONLY if active_only else 0
        n = C.c_uint32()
        if cap is None:
            self._chk(self.L.gysk_query_window_hosts(self.h, host_idx, flags, None, None, 0, C.byref(n)))
            cap = n.value
        out = (SvcSummary * max(cap, 1))()
        hosts = np.zeros(max(cap, 1), dtype=np.uint32)
        self._chk(self.L.gysk_query_window_hosts(self.h, host_idx, flags, out if cap else None, _p(hosts) if cap else None, cap, C.byref(n)))
        k = min(cap, n.value)
        return out[:k], hosts[:k].copy(), n.value

    def query_day_stats(self, host_idx=-1, cap=None):
        """gysk_query_day_stats: (ListenerDayStats rows in the order of query_window_hosts, host_idx of each row, number of rows).
        cap None = all rows (a count call first); 0 = the count only"""
        n = C.c_uint32()
        if cap is None:
            self._chk(self.L.gysk_query_day_stats(self.h, host_idx, None, None, 0, C.byref(n)))
            cap = n.value
        out = (ListenerDayStats * max(cap, 1))()
        hosts = np.zeros(max(cap, 1), dtype=np.uint32)
        self._chk(self.L.gysk_query_day_stats(self.h, host_idx, out if cap else None, _p(hosts) if cap else None, cap, C.byref(n)))
        k = min(cap, n.value)
        return out[:k], hosts[:k].copy(), n.value

    def query_host_listen(self, cap=None):
        """gysk_query_host_listen: (HostListen rows by ascending host, number of hosts). cap None = all rows; 0 = the count only"""
        n = C.c_uint32()
        if cap is None:
            self._chk(self.L.gysk_query_host_listen(self.h, None, 0, C.byref(n)))
            cap = n.value
        out = (HostListen * max(cap, 1))()
        self._chk(self.L.gysk_query_host_listen(self.h, out if cap else None, cap, C.byref(n)))
        return out[: min(cap, n.value)], n.value

    def query_tasks(self, ids):
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (TaskSummary * max(len(ids), 1))()
        self._chk(self.L.gysk_query_tasks(self.h, _p(ids), len(ids), out))
        return out[: len(ids)]

    def query_task_window(self, host_idx=-1, active_only=False, cap=None):
        """gysk_query_task_window: (TaskSummary rows in the order of query_window, number of matching rows)"""
        return self._window(self.L.gysk_query_task_window, TaskSummary, (host_idx,), active_only, cap)

    def _point_query(self, fn, dtype, keys, *window):
        """a count-min point query fn(h, keys, n, [last_window,] out): one row of dtype per key"""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        out = np.zeros(len(keys), dtype=dtype)
        self._chk(fn(self.h, _p(keys), len(keys), *window, _p(out)))
        return out

    def _export_cells(self, fn, *window, words=1):
        """the cells of a count-min table, fn(h, [last_window,] cells); words > 1: shape (cells, words)"""
        out = np.zeros((self.cfg.cms_depth << self.cfg.cms_log2_width) * words, dtype=np.uint64)
        self._chk(fn(self.h, *window, _p(out)))
        return out if words == 1 else out.reshape(-1, words)

    def query_flows(self, keys, last_window=False):
        return self._point_query(self.L.gysk_query_flows, FLOW_EST_DTYPE, keys, int(last_window))

    def query_flows_5min(self, keys):
        """gysk_query_flows_5min: the point query on the rolling 300-s count-min level (flow_level=True)"""
        return self._point_query(self.L.gysk_query_flows_5min, FLOW_EST_DTYPE, keys)

    def query_flow_queries(self, keys, last_window=False):
        """gysk_query_flow_queries: requests and response msec per flow key, min over rows (flow_queries=True)"""
        return self._point_query(self.L.gysk_query_flow_queries, FLOW_QRY_EST_DTYPE, keys, int(last_window))

    def query_flow_queries_5min(self, keys):
        """gysk_query_flow_queries_5min: the point query on the rolling 300-s flow query level (flow_query_level=True)"""
        return self._point_query(self.L.gysk_query_flow_queries_5min, FLOW_QRY_EST_DTYPE, keys)

    def _topk(self, fn, dtype, n, *window):
        """a heaviest-flow read fn(h, [last_window,] n, out, nout): the rows, best first"""
        out = np.zeros(n, dtype=dtype)
        k = C.c_uint32()
        self._chk(fn(self.h, *window, n, _p(out), C.byref(k)))
        return out[: k.value]

    def topk_flows(self, n=FLOW_TOPK_CAP, last_window=False):
        """gysk_topk_flows: the n heaviest flows by kbytes of the open or last window, with their estimates (flow_topk=True)"""
        return self._topk(self.L.gysk_topk_flows, FLOW_EST_DTYPE, n, int(last_window))

    def topk_flow_queries(self, n=FLOW_TOPK_CAP, last_window=False):
        """gysk_topk_flow_queries: the n heaviest flows by queries of the open or last window (flow_topk=True, flow_queries=True)"""
        return self._topk(self.L.gysk_topk_flow_queries, FLOW_QRY_EST_DTYPE, n, int(last_window))

    def topk_flows_global(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flows_global: the n heaviest flows by kbytes over every rank, from the last finished merge (flow_topk=True)"""
        return self._topk(self.L.gysk_topk_flows_global, FLOW_EST_DTYPE, n)

    def topk_flow_queries_global(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flow_queries_global: the n heaviest flows by queries over every rank, from the last finished merge"""
        return self._topk(self.L.gysk_topk_flow_queries_global, FLOW_QRY_EST_DTYPE, n)

    def _topk_5min(self, fn, dtype, n):
        """a 300-s heaviest-flow read fn(h, n, out, nout, bound): the rows, best first, and the bound on every flow left out"""
        out = np.zeros(n, dtype=dtype)
        k, b = C.c_uint32(), C.c_uint64()
        self._chk(fn(self.h, n, _p(out), C.byref(k), C.byref(b)))
        return out[: k.value], b.value

    def topk_flows_5min(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flows_5min: (rows, bound): the n heaviest flows by kbytes of the rolling 300-s connection level, with their
        estimates, and B_L: every flow left out scores at most that over the 300 s (flow_topk_5min=True, flow_level=True)"""
        return self._topk_5min(self.L.gysk_topk_flows_5min, FLOW_EST_DTYPE, n)

    def topk_flow_queries_5min(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flow_queries_5min: (rows, bound) of the rolling 300-s flow query level by queries (flow_topk_5min=True,
        flow_query_level=True)"""
        return self._topk_5min(self.L.gysk_topk_flow_queries_5min, FLOW_QRY_EST_DTYPE, n)

    def topk_flows_global_5min(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flows_global_5min: (rows, bound) over every rank's connection level, from the last finished merge"""
        return self._topk_5min(self.L.gysk_topk_flows_global_5min, FLOW_EST_DTYPE, n)

    def topk_flow_queries_global_5min(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flow_queries_global_5min: (rows, bound) over every rank's flow query level, from the last finished merge"""
        return self._topk_5min(self.L.gysk_topk_flow_queries_global_5min, FLOW_QRY_EST_DTYPE, n)

    def set_flow_slow(self, above_ms):
        """gysk_set_flow_slow: a counted response sample above above_ms msec (one of the 13 RESP_TIME_HASH thresholds) is slow; before
        the first event or flush (flow_topk_slow=True; the default is 300)"""
        self._chk(self.L.gysk_set_flow_slow(self.h, above_ms))

    def topk_flow_slow(self, n=FLOW_TOPK_CAP, last_window=False):
        """gysk_topk_flow_slow: the n flows with the most slow responses of the open or last window, each row its
        query_flow_resp row (flow_topk_slow=True)"""
        return self._topk(self.L.gysk_topk_flow_slow, FLOW_RESP_EST_DTYPE, n, int(last_window))

    def topk_flow_slow_global(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flow_slow_global: the n flows with the most slow responses over every rank, from the last finished merge"""
        return self._topk(self.L.gysk_topk_flow_slow_global, FLOW_RESP_EST_DTYPE, n)

    def topk_flow_slow_5min(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flow_slow_5min: (rows, bound) of the rolling 300-s response level by slow responses (flow_topk_slow=True,
        flow_topk_5min=True, flow_query_level=True)"""
        return self._topk_5min(self.L.gysk_topk_flow_slow_5min, FLOW_RESP_EST_DTYPE, n)

    def topk_flow_slow_global_5min(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flow_slow_global_5min: (rows, bound) over every rank's response level, from the last finished merge"""
        return self._topk_5min(self.L.gysk_topk_flow_slow_global_5min, FLOW_RESP_EST_DTYPE, n)

    def topn(self, metric, n=10, host_idx=-1):
        out = (TopnEntry * n)()
        k = C.c_uint32()
        self._chk(self.L.gysk_topn_svcs(self.h, metric, host_idx, n, out, C.byref(k)))
        return [(o.glob_id, o.score, o.host_idx) for o in out[: k.value]]

    def topn_tasks(self, metric, n=10):
        out = (TopnEntry * n)()
        k = C.c_uint32()
        self._chk(self.L.gysk_topn_tasks(self.h, metric, n, out, C.byref(k)))
        return [(o.glob_id, o.score) for o in out[: k.value]]

    def task_groupby(self, samples, cap=None):
        """gysk_task_groupby: PROC_SAMPLE_DTYPE array -> (wire.TASK records of the groups in order of first appearance, number of groups)"""
        from .wire import TASK
        samples = np.ascontiguousarray(samples, dtype=PROC_SAMPLE_DTYPE)
        cap = len(samples) if cap is None else cap
        out = np.zeros(max(cap, 1), dtype=TASK)
        ng = C.c_uint32()
        self._chk(self.L.gysk_task_groupby(self.h, _p(samples), len(samples), _p(out), cap, C.byref(ng)))
        return out[: min(ng.value, cap)].copy(), ng.value

    def topn_host(self, what, n=10, host_idx=-1):
        out = (TopnEntry * n)()
        k = C.c_uint32()
        self._chk(self.L.gysk_topn_host(self.h, what, host_idx, n, out, C.byref(k)))
        return [(o.glob_id, o.score, o.host_idx) for o in out[: k.value]]

    def cluster_state(self, host_idxs=None):
        cs = ClusterState()
        if host_idxs is None:
            self._chk(self.L.gysk_query_cluster_state(self.h, None, 0, C.byref(cs)))
        else:
            h = np.ascontiguousarray(host_idxs, dtype=np.uint32)
            self._chk(self.L.gysk_query_cluster_state(self.h, _p(h), len(h), C.byref(cs)))
        return {f: getattr(cs, f) for f, _ in cs._fields_ if f != "pad"}

    def host_summary(self, host_idx):
        hs = HostSummary()
        rc = self.L.gysk_query_host_summary(self.h, host_idx, C.byref(hs))
        if rc == -2:
            return None
        self._chk(rc)
        d = {f: getattr(hs, f) for f, _ in hs._fields_ if f not in ("nstates", "pad")}
        d["nstates"] = list(hs.nstates)
        return d

    def export_hist(self, id_, which):
        out = np.zeros(15, dtype=SERIAL_DTYPE)
        total, mx = C.c_uint64(), C.c_int64()
        rc = self.L.gysk_export_hist(self.h, int(id_), which, _p(out), C.byref(total), C.byref(mx))
        if rc == -2:
            return None
        self._chk(rc)
        return out, total.value, mx.value

    def export_hll(self, id_):
        return self._hll(self.L.gysk_export_hll, id_)

    def query_svc_clients(self, ids):
        """gysk_query_svc_clients: SvcClients rows of service ids as of the last flush (client_levels=True)"""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (SvcClients * max(len(ids), 1))()
        self._chk(self.L.gysk_query_svc_clients(self.h, _p(ids), len(ids), out))
        return out[: len(ids)]

    def query_clients_window(self, host_idx=-1, active_only=False, cap=None):
        """gysk_query_clients_window: (SvcClients rows in the order of query_window_hosts, host_idx of each row, number of rows).
        cap None = all rows (a count call first); 0 = the count only"""
        flags = WINDOW_ACTIVE_ONLY if active_only else 0
        n = C.c_uint32()
        if cap is None:
            self._chk(self.L.gysk_query_clients_window(self.h, host_idx, flags, None, None, 0, C.byref(n)))
            cap = n.value
        out = (SvcClients * max(cap, 1))()
        hosts = np.zeros(max(cap, 1), dtype=np.uint32)
        self._chk(self.L.gysk_query_clients_window(self.h, host_idx, flags, out if cap else None, _p(hosts) if cap else None, cap, C.byref(n)))
        k = min(cap, n.value)
        return out[:k], hosts[:k].copy(), n.value

    def query_svc_top_clients(self, ids, which=TOPC_LAST):
        """gysk_query_svc_top_clients: SVC_TOP_CLIENTS_DTYPE rows of service ids, summary TOPC_OPEN, TOPC_LAST or TOPC_5MIN
        (svc_top_clients=True)"""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = np.zeros(max(len(ids), 1), dtype=SVC_TOP_CLIENTS_DTYPE)
        self._chk(self.L.gysk_query_svc_top_clients(self.h, _p(ids), len(ids), which, _p(out)))
        return out[: len(ids)]

    def query_top_clients_window(self, which=TOPC_LAST, host_idx=-1, active_only=False, cap=None):
        """gysk_query_top_clients_window: (SVC_TOP_CLIENTS_DTYPE rows in the order of query_window_hosts, host_idx of each row, number
        of rows). cap None = all rows (a count call first); 0 = the count only"""
        flags = WINDOW_ACTIVE_ONLY if active_only else 0
        n = C.c_uint32()
        if cap is None:
            self._chk(self.L.gysk_query_top_clients_window(self.h, host_idx, flags, which, None, None, 0, C.byref(n)))
            cap = n.value
        out = np.zeros(max(cap, 1), dtype=SVC_TOP_CLIENTS_DTYPE)
        hosts = np.zeros(max(cap, 1), dtype=np.uint32)
        self._chk(self.L.gysk_query_top_clients_window(self.h, host_idx, flags, which, _p(out) if cap else None, _p(hosts) if cap else None, cap,
                                                       C.byref(n)))
        k = min(cap, n.value)
        return out[:k], hosts[:k].copy(), n.value

    def export_hll_window(self, id_, which=CLIENTS_LAST):
        """gysk_export_hll_window: the 256 client registers of CLIENTS_LAST or CLIENTS_5MIN, None for an unknown id"""
        return self._hll_window(self.L.gysk_export_hll_window, id_, which)

    def _hll_window(self, fn, id_, which):
        regs = np.zeros(1 << HLL_WINDOW_P, dtype=np.uint8)
        rc = fn(self.h, int(id_), which, _p(regs))
        if rc == -2:
            return None
        self._chk(rc)
        return regs

    def _hll(self, fn, id_):
        regs = np.zeros(1 << self.cfg.hll_p, dtype=np.uint8)
        rc = fn(self.h, int(id_), _p(regs))
        if rc == -2:
            return None
        self._chk(rc)
        return regs

    def export_conn_bitmap(self, id_, last_window=False):
        masks = np.zeros(15, dtype=np.uint32)
        cnt = np.zeros(15, dtype=np.uint8)
        rc = self.L.gysk_export_conn_bitmap(self.h, int(id_), int(last_window), _p(masks), _p(cnt))
        if rc == -2:
            return None
        self._chk(rc)
        return masks, cnt

    def export_tdigest(self, id_):
        return self._tdigest(self.L.gysk_export_tdigest, id_)

    def _tdigest(self, fn, id_):
        means = np.zeros(TD_CAP, dtype=np.float64)
        weights = np.zeros(TD_CAP, dtype=np.uint64)
        n, mn, mx = C.c_uint32(), C.c_double(), C.c_double()
        rc = fn(self.h, int(id_), _p(means), _p(weights), TD_CAP, C.byref(n), C.byref(mn), C.byref(mx))
        if rc == -2:
            return None
        self._chk(rc)
        return means[: n.value].copy(), weights[: n.value].copy(), mn.value, mx.value

    def export_tdigest_pgtext(self, id_):
        return self._pgtext(self.L.gysk_export_tdigest_pgtext, id_)

    def _pgtext(self, fn, id_):
        buf = C.create_string_buffer(8192)
        rc = fn(self.h, int(id_), buf, len(buf))
        if rc == -2:
            return None
        if rc < 0:
            self._chk(rc)
        return buf.value.decode()

    def quantiles(self, id_, qs):
        return self._quantiles(self.L.gysk_query_quantiles, id_, qs)

    def _quantiles(self, fn, id_, qs):
        qs = np.ascontiguousarray(qs, dtype=np.float64)
        out = np.zeros(len(qs), dtype=np.float64)
        self._chk(fn(self.h, int(id_), _p(qs), len(qs), _p(out)))
        return out

    # ---- multi-GPU merge ----
    def set_logical_map(self, glob_ids, logical_ids):
        g = np.ascontiguousarray(glob_ids, dtype=np.uint64)
        l = np.ascontiguousarray(logical_ids, dtype=np.uint64)
        assert len(g) == len(l)
        self._chk(self.L.gysk_set_logical_map(self.h, _p(g), _p(l), len(g)))

    def set_cluster_map(self, host_idxs, cluster_ids):
        """gysk_set_cluster_map: host_idxs[i] belongs to cluster cluster_ids[i] (merge_clusters=True)"""
        h = np.ascontiguousarray(host_idxs, dtype=np.uint32)
        c = np.ascontiguousarray(cluster_ids, dtype=np.uint64)
        assert len(h) == len(c)
        self._chk(self.L.gysk_set_cluster_map(self.h, _p(h), _p(c), len(h)))

    def merge_prepare(self):
        self._chk(self.L.gysk_merge_prepare(self.h))

    def merge_buffers(self):
        descs = (BufferDesc * 8)()
        n = C.c_uint32()
        self._chk(self.L.gysk_merge_buffers(self.h, descs, 8, C.byref(n)))
        return [(d.name.decode(), d.dptr, d.nbytes, d.redop) for d in descs[: n.value]]

    def merge_tdigest_slab(self):
        p, nb = C.c_void_p(), C.c_uint64()
        self._chk(self.L.gysk_merge_tdigest_slab(self.h, C.byref(p), C.byref(nb)))
        return p.value, nb.value

    def merge_finish(self, gathered_ptr=None, world=1):
        self._chk(self.L.gysk_merge_finish(self.h, C.c_void_p(gathered_ptr), world))

    def nccl_unique_id(self):
        buf = (C.c_uint8 * 128)()
        self._chk(self.L.gysk_nccl_unique_id(buf))
        return bytes(buf)

    def nccl_comm_init(self, uid, nranks, rank):
        buf = (C.c_uint8 * 128).from_buffer_copy(uid)
        self._chk(self.L.gysk_nccl_comm_init(self.h, buf, nranks, rank))

    def merge_global(self, comm=None):
        """fold + one grouped NCCL launch + merge-compress, all inside the library (gysk_merge_global)"""
        self._chk(self.L.gysk_merge_global(self.h, C.c_void_p(comm)))

    def query_logical(self, ids):
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (SvcSummary * len(ids))()
        self._chk(self.L.gysk_query_logical(self.h, _p(ids), len(ids), out))
        return [o.asdict() for o in out]

    def export_logical_hist(self, logical_id, which):
        """gysk_export_logical_hist: (SERIAL_DTYPE[15], total, max) of a logical service from the last merge; None for an id
        the map does not have"""
        out = np.zeros(15, dtype=SERIAL_DTYPE)
        total, mx = C.c_uint64(), C.c_int64()
        rc = self.L.gysk_export_logical_hist(self.h, int(logical_id), which, _p(out), C.byref(total), C.byref(mx))
        if rc == -2:
            return None
        self._chk(rc)
        return out, total.value, mx.value

    def query_logical_all(self, active_only=False, cap=None):
        """gysk_query_logical_all: (SvcSummary rows of the merged logical services in ascending logical id, number of matching rows).
        cap None = all rows (a count call first); 0 = the count only"""
        return self._window(self.L.gysk_query_logical_all, SvcSummary, (), active_only, cap)

    def topn_logical(self, metric, n=10):
        """gysk_topn_logical: [(logical id, score, 0)] of the n best logical services of the last merge, best first"""
        out = (TopnEntry * n)()
        k = C.c_uint32()
        self._chk(self.L.gysk_topn_logical(self.h, metric, n, out, C.byref(k)))
        return [(o.glob_id, o.score, o.host_idx) for o in out[: k.value]]

    def export_logical_tdigest(self, logical_id):
        """(means, weights, min, max) of a logical service's merged digest; None for an id the map does not have"""
        return self._tdigest(self.L.gysk_export_logical_tdigest, logical_id)

    def export_logical_tdigest_pgtext(self, logical_id):
        return self._pgtext(self.L.gysk_export_logical_tdigest_pgtext, logical_id)

    def logical_quantiles(self, logical_id, qs):
        return self._quantiles(self.L.gysk_query_logical_quantiles, logical_id, qs)

    def export_logical_hll(self, logical_id):
        return self._hll(self.L.gysk_export_logical_hll, logical_id)

    def query_logical_clients(self, ids):
        """gysk_query_logical_clients: SvcClients rows of logical ids from the last merge (client_levels=True)"""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (SvcClients * max(len(ids), 1))()
        self._chk(self.L.gysk_query_logical_clients(self.h, _p(ids), len(ids), out))
        return out[: len(ids)]

    def query_logical_top_clients(self, ids, which=TOPC_LAST):
        """gysk_query_logical_top_clients: SVC_TOP_CLIENTS_DTYPE rows of logical ids from the last merge, summary TOPC_LAST or TOPC_5MIN
        (svc_top_clients=True)"""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = np.zeros(max(len(ids), 1), dtype=SVC_TOP_CLIENTS_DTYPE)
        self._chk(self.L.gysk_query_logical_top_clients(self.h, _p(ids), len(ids), which, _p(out)))
        return out[: len(ids)]

    def query_logical_top_clients_all(self, which=TOPC_LAST, active_only=False, cap=None):
        """gysk_query_logical_top_clients_all: (SVC_TOP_CLIENTS_DTYPE rows in the order of query_logical_all, number of matching rows).
        cap None = all rows (a count call first); 0 = the count only"""
        flags = WINDOW_ACTIVE_ONLY if active_only else 0
        n = C.c_uint32()
        if cap is None:
            self._chk(self.L.gysk_query_logical_top_clients_all(self.h, flags, which, None, 0, C.byref(n)))
            cap = n.value
        out = np.zeros(max(cap, 1), dtype=SVC_TOP_CLIENTS_DTYPE)
        self._chk(self.L.gysk_query_logical_top_clients_all(self.h, flags, which, _p(out) if cap else None, cap, C.byref(n)))
        return out[: min(cap, n.value)], n.value

    def export_logical_hll_window(self, logical_id, which=CLIENTS_LAST):
        """gysk_export_logical_hll_window: the merged 256 client registers of one logical service, None outside the map"""
        return self._hll_window(self.L.gysk_export_logical_hll_window, logical_id, which)

    def query_logical_states(self, ids):
        """gysk_query_logical_states: LogicalState rows of logical ids from the last merge (merge_states=True)"""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (LogicalState * max(len(ids), 1))()
        self._chk(self.L.gysk_query_logical_states(self.h, _p(ids), len(ids), out))
        return out[: len(ids)]

    def query_logical_states_all(self, active_only=False, cap=None):
        """gysk_query_logical_states_all: (LogicalState rows in ascending logical id, number of matching rows); cap as query_logical_all"""
        return self._window(self.L.gysk_query_logical_states_all, LogicalState, (), active_only, cap)

    def query_logical_traces(self, ids):
        """gysk_query_logical_traces: LogicalTrace rows of logical ids from the last merge (merge_traces=True)"""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (LogicalTrace * max(len(ids), 1))()
        self._chk(self.L.gysk_query_logical_traces(self.h, _p(ids), len(ids), out))
        return out[: len(ids)]

    def query_logical_traces_all(self, active_only=False, cap=None):
        """gysk_query_logical_traces_all: (LogicalTrace rows in ascending logical id, number of matching rows); cap as query_logical_all"""
        return self._window(self.L.gysk_query_logical_traces_all, LogicalTrace, (), active_only, cap)

    def export_logical_trace_tdigest(self, logical_id):
        """(means, weights, min, max) of a logical service's merged trace digest; None for an id the map does not have"""
        means = np.zeros(TRACE_TD_CAP, dtype=np.float64)
        weights = np.zeros(TRACE_TD_CAP, dtype=np.uint64)
        n, mn, mx = C.c_uint32(), C.c_double(), C.c_double()
        rc = self.L.gysk_export_logical_trace_tdigest(self.h, int(logical_id), _p(means), _p(weights), TRACE_TD_CAP, C.byref(n), C.byref(mn),
                                                      C.byref(mx))
        if rc == -2:
            return None
        self._chk(rc)
        return means[: n.value].copy(), weights[: n.value].copy(), mn.value, mx.value

    def export_logical_trace_tdigest_pgtext(self, logical_id):
        return self._pgtext(self.L.gysk_export_logical_trace_tdigest_pgtext, logical_id)

    def query_cluster_states(self, ids):
        """gysk_query_cluster_states: ClusterRow rows of cluster ids from the last merge (merge_clusters=True)"""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = (ClusterRow * max(len(ids), 1))()
        self._chk(self.L.gysk_query_cluster_states(self.h, _p(ids), len(ids), out))
        return out[: len(ids)]

    def query_cluster_states_all(self, active_only=False, cap=None):
        """gysk_query_cluster_states_all: (ClusterRow rows in ascending cluster id, number of matching rows); cap as query_logical_all"""
        return self._window(self.L.gysk_query_cluster_states_all, ClusterRow, (), active_only, cap)

    def _topn_global(self, fn, row_type, metric, n, rows):
        out = (TopnEntry * max(n, 1))()
        rws = (row_type * max(n, 1))() if rows else None
        k = C.c_uint32()
        self._chk(fn(self.h, metric, n, out, rws, C.byref(k)))
        return out[: k.value], (rws[: k.value] if rows else None)

    def topn_global(self, metric, n=10, rows=True):
        """gysk_topn_global: (TopnEntry list, SvcSummary rows or None) of the n best services over every rank, best first, from the last
        merge (merge_topn=True)"""
        return self._topn_global(self.L.gysk_topn_global, SvcSummary, metric, n, rows)

    def topn_global_tasks(self, metric, n=10, rows=True):
        """gysk_topn_global_tasks: (TopnEntry list, TaskSummary rows or None) of the n best processes over every rank (merge_topn=True)"""
        return self._topn_global(self.L.gysk_topn_global_tasks, TaskSummary, metric, n, rows)

    def merge_flush_range(self):
        """gysk_merge_flush_range: (earliest, latest) tsec of the ranks' last flush, as the last merge all-reduced them"""
        lo, hi = C.c_uint32(), C.c_uint32()
        self._chk(self.L.gysk_merge_flush_range(self.h, C.byref(lo), C.byref(hi)))
        return lo.value, hi.value

    def query_flows_global(self, keys, last_window=False):
        return self._point_query(self.L.gysk_query_flows_global, FLOW_EST_DTYPE, keys, int(last_window))

    def query_flows_global_5min(self, keys):
        """gysk_query_flows_global_5min: the point query on the 300-s count-min level summed over the ranks by the last merge"""
        return self._point_query(self.L.gysk_query_flows_global_5min, FLOW_EST_DTYPE, keys)

    def export_cms(self, last_window=False):
        return self._export_cells(self.L.gysk_export_cms, int(last_window))

    def export_cms_queries(self, last_window=False):
        """gysk_export_cms_queries: the cells {queries | resp msec << 32} of the flow query table (flow_queries=True)"""
        return self._export_cells(self.L.gysk_export_cms_queries, int(last_window))

    def query_flow_queries_global(self, keys, last_window=False):
        """gysk_query_flow_queries_global: the point query on the flow query tables summed over the ranks by the last merge"""
        return self._point_query(self.L.gysk_query_flow_queries_global, FLOW_QRY_EST_DTYPE, keys, int(last_window))

    def query_flow_resp(self, keys, last_window=False):
        """gysk_query_flow_resp: per flow key the response-time bucket counts (min over rows), their total and p25 / p95 / p99 msec
        (flow_resp_hist=True)"""
        return self._point_query(self.L.gysk_query_flow_resp, FLOW_RESP_EST_DTYPE, keys, int(last_window))

    def export_cms_resp(self, last_window=False):
        """gysk_export_cms_resp: the flow response histogram cells, shape (depth << log2_width, 8) (flow_resp_hist=True)"""
        return self._export_cells(self.L.gysk_export_cms_resp, int(last_window), words=RESP_HIST_WORDS)

    def query_flow_resp_global(self, keys, last_window=False):
        """gysk_query_flow_resp_global: the point query on the flow response histograms summed over the ranks by the last merge"""
        return self._point_query(self.L.gysk_query_flow_resp_global, FLOW_RESP_EST_DTYPE, keys, int(last_window))

    def query_flow_resp_5min(self, keys):
        """gysk_query_flow_resp_5min: the point query on the rolling 300-s level of the flow response histograms
        (flow_resp_hist=True, flow_query_level=True)"""
        return self._point_query(self.L.gysk_query_flow_resp_5min, FLOW_RESP_EST_DTYPE, keys)

    def export_cms_resp_5min(self):
        """gysk_export_cms_resp_5min: the cells of that level, shape (depth << log2_width, 8)"""
        return self._export_cells(self.L.gysk_export_cms_resp_5min, words=RESP_HIST_WORDS)

    def query_flow_resp_global_5min(self, keys):
        """gysk_query_flow_resp_global_5min: the point query on that level summed over the ranks by the last merge"""
        return self._point_query(self.L.gysk_query_flow_resp_global_5min, FLOW_RESP_EST_DTYPE, keys)

    def query_flow_errors(self, keys, last_window=False):
        """gysk_query_flow_errors: per flow key its queries (as query_flow_queries) and client / server errors, min over rows
        (flow_errors=True)"""
        return self._point_query(self.L.gysk_query_flow_errors, FLOW_ERR_EST_DTYPE, keys, int(last_window))

    def export_cms_errors(self, last_window=False):
        """gysk_export_cms_errors: the cells {cli_errors | ser_errors << 32} of the flow error table (flow_errors=True)"""
        return self._export_cells(self.L.gysk_export_cms_errors, int(last_window))

    def query_flow_errors_global(self, keys, last_window=False):
        """gysk_query_flow_errors_global: the point query on the flow error and query tables summed over the ranks by the last merge"""
        return self._point_query(self.L.gysk_query_flow_errors_global, FLOW_ERR_EST_DTYPE, keys, int(last_window))

    def query_flow_errors_5min(self, keys):
        """gysk_query_flow_errors_5min: the point query on the rolling 300-s level of the flow error tables
        (flow_errors=True, flow_query_level=True)"""
        return self._point_query(self.L.gysk_query_flow_errors_5min, FLOW_ERR_EST_DTYPE, keys)

    def export_cms_errors_5min(self):
        """gysk_export_cms_errors_5min: the cells of that level"""
        return self._export_cells(self.L.gysk_export_cms_errors_5min)

    def query_flow_errors_global_5min(self, keys):
        """gysk_query_flow_errors_global_5min: the point query on that level summed over the ranks by the last merge"""
        return self._point_query(self.L.gysk_query_flow_errors_global_5min, FLOW_ERR_EST_DTYPE, keys)

    def topk_flow_errors(self, n=FLOW_TOPK_CAP, last_window=False):
        """gysk_topk_flow_errors: the n flows with the most server errors of the open or last window, each row its
        query_flow_errors row (flow_errors=True, flow_topk=True)"""
        return self._topk(self.L.gysk_topk_flow_errors, FLOW_ERR_EST_DTYPE, n, int(last_window))

    def topk_flow_errors_global(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flow_errors_global: the n flows with the most server errors over every rank, from the last finished merge"""
        return self._topk(self.L.gysk_topk_flow_errors_global, FLOW_ERR_EST_DTYPE, n)

    def topk_flow_errors_5min(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flow_errors_5min: (rows, bound) of the rolling 300-s error level by server errors (flow_errors=True,
        flow_topk_5min=True, flow_query_level=True)"""
        return self._topk_5min(self.L.gysk_topk_flow_errors_5min, FLOW_ERR_EST_DTYPE, n)

    def topk_flow_errors_global_5min(self, n=FLOW_TOPK_CAP):
        """gysk_topk_flow_errors_global_5min: (rows, bound) over every rank's error level, from the last finished merge"""
        return self._topk_5min(self.L.gysk_topk_flow_errors_global_5min, FLOW_ERR_EST_DTYPE, n)

    def export_cms_queries_5min(self):
        """gysk_export_cms_queries_5min: the cells of the rolling 300-s flow query level (flow_query_level=True)"""
        return self._export_cells(self.L.gysk_export_cms_queries_5min)

    def query_flow_queries_global_5min(self, keys):
        """gysk_query_flow_queries_global_5min: the point query on the 300-s flow query level summed over the ranks by the last merge"""
        return self._point_query(self.L.gysk_query_flow_queries_global_5min, FLOW_QRY_EST_DTYPE, keys)

    def export_cms_5min(self):
        """gysk_export_cms_5min: the cells of the rolling 300-s count-min level (flow_level=True)"""
        return self._export_cells(self.L.gysk_export_cms_5min)
