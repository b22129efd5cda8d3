/*
 * gysketch.h — C ABI of libgysketch.so, the H100-native streaming-sketch aggregation engine that sits
 * behind Gyeeta's madhava ingest path.
 *
 * Every entry point replaces (or is what a cgo/ctypes/C++ shim would bind for) a named piece of the
 * reference; citations are relative to the reference tree:
 *
 *   gysk_ingest()         the per-message dispatch of MCONN_HANDLER::handle_l2_misc  server/gy_mconnhdlr.cc:4745-4800
 *                         (phdr/pevtnot/recs/nevents/pendptr arithmetic) and the record walks of
 *                         partha_tcp_conn_info :9052/:9130, partha_listener_state :10993/:11175,
 *                         partha_aggr_task_state :9959, incl. the L1 validators common/gy_comm_proto.cc:840-996
 *   gysk_ingest_raw()     the per-sample reduction lifted off partha: TCP_SOCK_HANDLER::handle_ipv4_resp_event /
 *                         handle_tcp_resp_event  common/gy_socket_stat.cc:1517-1677, handle_ipv4_conn_event :241,
 *                         SVC_INFO_CAP::upd_stats_on_req  common/gy_proto_parser.cc:2678-2694
 *   gysk_ingest_device()  same reduction for event batches already resident in HBM (bench / device generators)
 *   gysk_flush()          the 5-second reducer TCP_SOCK_HANDLER::listener_stats_update  common/gy_socket_stat.cc:3898-4445
 *   gysk_query_svcs()     readers of MTCP_LISTENER::state_ (server/gy_msocket.h:1304) through SvcStateFields
 *                         (server/gy_mfields.h:1383-1412): qps5s, nqry5s, resp5s, p95resp5s ...
 *   gysk_export_hist()    GY_HISTOGRAM::get_serialized  common/gy_statistics.h:656-673 (HIST_SERIAL byte-compatible)
 *   gysk_hist_percentiles GY_HISTOGRAM::get_percentiles common/gy_statistics.h:707-791
 *   gysk_query_flows()    new capability: count-min point query replacing the exact two-level group-by of
 *                         partha_tcp_conn_info  server/gy_mconnhdlr.cc:9245-9311
 *   gysk_export_hll()     new capability: distinct clients per service, replacing the exact client sets
 *                         (cli_aggr_task_tbl_, server/gy_msocket.h:1335)
 *   gysk_export_tdigest() new capability: response-time quantile sketch; the reference's only t-digest user is the
 *   gysk_query_quantiles  Postgres extension with compression 100 (common/gy_query_common.cc:1805-1858)
 *   gysk_merge_*          additive roll-up  MS_CLUSTER_STATE::STATE_ONE::add_stats common/gy_comm_proto.h:3199-3214 /
 *                         SHCONN_HANDLER::aggregate_cluster_state server/gy_shconnhdlr.cc:4583
 *
 * Conventions: plain pointers and sizes, no exceptions cross the boundary, 0 = ok, negative = -errno style
 * (mirrors the reference handlers' bool/int returns wrapped in GY_CATCH_EXCEPTION, gy_mconnhdlr.cc:4763-4774).
 * CUDA errors are sticky: once a call fails with GYSK_ERR_CUDA every later call fails too; gysk_last_error()
 * returns the text. There is NO CPU fallback: gysk_create() fails when no sm_90 device is usable.
 */
#ifndef GYSKETCH_H
#define GYSKETCH_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GYSK_ABI_VERSION		2

/* ---- error codes ---- */
#define GYSK_OK				0
#define GYSK_ERR_INVAL			(-22)	/* EINVAL  : bad argument / failed wire validation */
#define GYSK_ERR_NOMEM			(-12)	/* ENOMEM  */
#define GYSK_ERR_NOENT			(-2)	/* ENOENT  : unknown service / task id */
#define GYSK_ERR_NOSPC			(-28)	/* ENOSPC  : service table full */
#define GYSK_ERR_NODEV			(-19)	/* ENODEV  : no usable CUDA device (no CPU fallback exists) */
#define GYSK_ERR_CUDA			(-5)	/* EIO     : CUDA runtime error (sticky) */
#define GYSK_ERR_NOTSUP			(-95)	/* EOPNOTSUPP */

/* ---- canonical 32-byte event record (SURVEY.md §8d) ---- */
enum {
	GYSK_EV_CONNECT		= 1,	/* TCP_EVENT_TYPE_CONNECT    common/gy_ebpf_kernel.h:24 */
	GYSK_EV_ACCEPT		= 2,	/* TCP_EVENT_TYPE_ACCEPT */
	GYSK_EV_CLOSE_CLI	= 3,	/* TCP_EVENT_TYPE_CLOSE_CLI */
	GYSK_EV_CLOSE_SER	= 4,	/* TCP_EVENT_TYPE_CLOSE_SER */
	GYSK_EV_RESP		= 5,	/* service response-time sample (tcp_ipv4_resp_event_t / API_TRAN) */
	GYSK_EV_TASK		= 6,	/* per-process 5-s sample (AGGR_TASK_STATE_NOTIFY) */
	GYSK_EV_ACTIVE		= 7,	/* one ACTIVE_CONN_STATS record (common/gy_comm_proto.h:2766): the 15-s inet_diag group-by
					   {ser_glob_id, cli_task_aggr_id} of upd_conn_from_diag (common/gy_socket_stat.cc:6156-6194) */
	GYSK_EV_TRACE		= 8,	/* one request trace (an API_TRAN, the row handle_trace_requests writes to tracereqtbl,
					   server/gy_mconnhdlr.cc:5883-6060), kept only by an engine with trace rows
					   (gysk_config.max_trace_svcs; dropped without). Fields reused as by ACTIVE:
					     svc_id   = glob_id_
					     flow_key = min(reqlen_, 2^32 - 1) | min(reslen_, 2^32 - 1) << 32   (bytes in | bytes out)
					     value    = response_usec_ clamped to 32 bits
					     flags    = GYSK_EVF_TRACE_ERROR (errorcode_ != 0) | GYSK_EVF_TRACE_NEWCONN (reqnum_ == 0)
					   gysk_ingest_raw(GYSK_RAW_API_TRAN) stages one next to the record's GYSK_EV_RESP */
};

/* gysk_event.flags of a GYSK_EV_RESP event that came from an API_TRAN (SVC_INFO_CAP::upd_stats_on_req, gy_proto_parser.cc:2678-2694) */
#define GYSK_EVF_CLI_ERROR		0x1u	/* stats_.ncli_errors_++ */
#define GYSK_EVF_SER_ERROR		0x2u	/* stats_.nser_errors_++ */
/* gysk_event.flags of a GYSK_EV_TRACE event */
#define GYSK_EVF_TRACE_ERROR		0x1u	/* errorcode_ != 0: counted in nerr */
#define GYSK_EVF_TRACE_NEWCONN		0x2u	/* reqnum_ == 0: counted in nconns */

typedef struct gysk_event
{
	uint64_t	svc_id;		/* ser_glob_id_ ; for GYSK_EV_TASK: aggr_task_id_. 0 is invalid (dropped) */
	uint64_t	flow_key;	/* TCP/RESP: cli_task_aggr_id_ or a 64-bit fold of the 5-tuple.
					   TASK: low 32 = cpu_delay_msec_, high 32 = blkio_delay_msec_ */
	uint32_t	value;		/* RESP: response time in usec; TCP: bytes; TASK: (int)total_cpu_pct_; ACTIVE: kbytes sent + received */
	uint32_t	host_idx;	/* dense index of the sending partha (shard key: host_idx % world) */
	uint32_t	tsec;		/* event time, seconds — informational: a sample lands in the window that is open when it ARRIVES,
					   as in the reference (handle_tcp_resp_event stamps samples with time(nullptr) of their
					   processing, common/gy_socket_stat.cc:1560-1579). ACTIVE: IEEE-754 bits of max_rtt_msec_ */
	uint16_t	type;		/* GYSK_EV_* */
	uint16_t	flags;		/* RESP: GYSK_EVF_*; ACTIVE: active_conns_; else 0 */
} gysk_event;

/* ---- histogram classes (bucket thresholds of common/gy_statistics.h:1674-2063) ---- */
enum {
	GYSK_CLS_RESP_TIME	= 0,	/* RESP_TIME_HASH	:1674  (msec) */
	GYSK_CLS_SEMI_LOG	= 1,	/* SEMI_LOG_HASH	:1729 */
	GYSK_CLS_SEMI_LOG_LO	= 2,	/* SEMI_LOG_HASH_LO	:1782 */
	GYSK_CLS_DURATION	= 3,	/* DURATION_HASH	:1835 */
	GYSK_CLS_HASH_10_5000	= 4,	/* HASH_10_5000		:1908 */
	GYSK_CLS_HASH_5_250	= 5,	/* HASH_5_250		:1960 */
	GYSK_CLS_HASH_1_3000	= 6,	/* HASH_1_3000		:2013 */
	GYSK_CLS_PERCENT	= 7,	/* PERCENT_HASH		:1624 */
};

#define GYSK_HIST_MAX_BUCKETS		15	/* largest max_buckets among the classes above */

/* byte-compatible with HIST_SERIAL, common/gy_statistics.h:458-468 */
typedef struct gysk_hist_serial
{
	uint64_t	count;
	int64_t		sum;
} gysk_hist_serial;

/* which histogram of an id */
enum {
	GYSK_HIST_RESP_CUR	= 0,	/* service: response msec, window being filled		(RESP_TIME_HASH, T=int64) */
	GYSK_HIST_RESP_LAST	= 1,	/* service: last closed 5-s window */
	GYSK_HIST_RESP_ALL	= 2,	/* service: since start ("Since Process start" level, gy_statistics.h:1548) */
	GYSK_HIST_TASK_CPU_PCT	= 3,	/* task: MTASK_HIST::cpu_pct_histogram_		(HASH_1_3000, T=int)  server/gy_msocket.h:707 */
	GYSK_HIST_TASK_CPU_DELAY= 4,	/* task: cpu_delay_histogram_			(DURATION_HASH, T=int) */
	GYSK_HIST_TASK_BLKIO_DELAY = 5,	/* task: blkio_delay_histogram_			(DURATION_HASH, T=int) */
	GYSK_HIST_RESP_5MIN	= 6,	/* service: 300-s level    (Level_5s_5min_5days_all, gy_statistics.h:1545-1551; 10 slots, :1105) */
	GYSK_HIST_RESP_5DAY	= 7,	/* service: 432000-s level */
	GYSK_HIST_QPS		= 8,	/* service: TCP_LISTENER::qps_hist_		(SEMI_LOG_HASH_LO, T=int) common/gy_socket_stat.h:548,633: one
					   sample per closed window = queries / 5, common/gy_socket_stat.cc:4111-4121 */
	GYSK_HIST_ACTIVE_CONN	= 9,	/* service: active_conn_hist_			(HASH_1_3000, T=int) :549,635: one sample per closed window =
					   the listener's active connections, :4124-4130 */
};

/* ---- listener state (OBJ_STATE_E, common/gy_json_field_maps.h:242-250) and issue source (LISTENER_ISSUE_SRC, :419-435) ---- */
enum { GYSK_STATE_IDLE = 0, GYSK_STATE_GOOD = 1, GYSK_STATE_OK = 2, GYSK_STATE_BAD = 3, GYSK_STATE_SEVERE = 4, GYSK_STATE_DOWN = 5 };
enum { GYSK_ISSUE_NONE = 0, GYSK_ISSUE_LISTENER_TASKS = 1, GYSK_ISSUE_QPS_HIGH = 2, GYSK_ISSUE_ACTIVE_CONN_HIGH = 3, GYSK_ISSUE_SERVER_ERRORS = 4,
       GYSK_ISSUE_OS_CPU = 5, GYSK_ISSUE_OS_MEMORY = 6, GYSK_ISSUE_DEPENDENT_SERVER_LISTENER = 7, GYSK_ISSUE_SRC_UNKNOWN = 8 };

/* Inputs of TCP_LISTENER::get_curr_state (common/gy_socket_stat.cc:2020-2875), the once-per-window state decision of a listener.
 * gysk_flush() evaluates it on the device for every service from the engine's own state, with the block "outside the path" zero;
 * gysk_classify_listener() is the same code for a caller that has those inputs. Response values in msec. */
typedef struct gysk_listener_state_in
{
	int64_t		r5p95, r5p99;			/* last 5-s window: p95 / p99 bucket thresholds		(:2082-2083) */
	int64_t		r300p95, r300p99;		/* 300-s level						(:2084-2085) */
	int64_t		r5dp95, r5dp99, r5dp25;		/* 5-day level						(:2086-2088) */
	int64_t		rallp95, rallp99;		/* all-time level					(:2089-2090) */
	uint64_t	nqrys_5s;			/* histstat_[n5].tcount_ */
	uint64_t	total_resp_msec;		/* histstat_[n5].tsum_ */
	uint64_t	tcount_5d;			/* histstat_[n5days].tcount_ */
	double		mean5, mean300, mean5d, meanall;	/* tsum / max(tcount, 1), common/gy_statistics.h:1358 */
	int64_t		qps_p95, qps_p25;		/* qps_hist_ percentiles				(:2097) */
	int64_t		act_p95, act_p25;		/* active_conn_hist_ percentiles			(:2098) */
	int64_t		secs_5d;			/* seconds the 5-day level covers so far: min(432000, age)	(:2067-2074) */
	int32_t		last_qps_count;			/* last_qps_count_: queries per second of the window	(:4121) */
	int32_t		nconn;				/* last_chk_nconn_					(:2036) */
	int32_t		curr_active_conn;		/* (:4158-4170) max of nconn_recent_active_ and the CONN_BITMAP bucket counts */
	uint32_t	ser_errors;
	uint8_t		nactive_conn_arr[16];		/* CONN_BITMAP::get_conn_breakup of the window, per response bucket (:4160-4163) */
	/* outside the path: the engine passes zeros */
	uint8_t		task_issue, task_severe, task_delay;	/* TCP_LISTENER::is_task_issue (:1914) verdicts */
	uint8_t		cpu_issue, mem_issue;		/* host state */
	uint8_t		pad0[3];
	int32_t		ntasks_issue, ntasks_noissue;
	uint64_t	tasks_delay_msec;
	uint32_t	nserdepends;			/* related_listen_->id_depends_ count (:2820-2823) */
	uint32_t	pad1;
} gysk_listener_state_in;

/* ---- raw record kinds for gysk_ingest_raw ---- */
enum {
	GYSK_RAW_EVENT32	= 0,	/* gysk_event[] */
	GYSK_RAW_TCP_IPV4_EVENT	= 1,	/* tcp_ipv4_event_t[]      72 B  common/gy_ebpf_kernel.h:37  */
	GYSK_RAW_TCP_IPV4_RESP	= 2,	/* tcp_ipv4_resp_event_t[] 24 B  common/gy_ebpf_kernel.h:106 */
	GYSK_RAW_TCP_IPV6_EVENT	= 3,	/* tcp_ipv6_event_t[]      96 B  common/gy_ebpf_kernel.h:54  (handle_ipv6_conn_event, gy_socket_stat.cc:269) */
	GYSK_RAW_TCP_IPV6_RESP	= 4,	/* tcp_ipv6_resp_event_t[] 64 B  common/gy_ebpf_kernel.h:113 (handle_ipv6_resp_event, gy_socket_stat.cc:1535) */
	GYSK_RAW_API_TRAN	= 5,	/* API_TRAN records, variable stride (common/gy_proto_common.h:140-204; nevents records walked with
					   get_elem_size()); `events` must stay readable for nevents strides */
	GYSK_RAW_RESP16		= 6,	/* gysk_resp16[]  packed response samples */
	GYSK_RAW_TCP24		= 7,	/* gysk_tcp24[]   packed conn events */
	GYSK_RAW_TASK24		= 8,	/* gysk_task24[]  packed process samples */
};

/* Packed per-kind records: what a feeder that already knows the kind of a batch ships instead of the 32-byte canonical record
 * (18.4 bytes per event on the 70 / 20 / 10 mix instead of 32 — the host link is the end-to-end limit). Decoded ON THE DEVICE
 * into the canonical record, as are the fixed-stride eBPF structs above: gysk_ingest_raw copies the raw bytes, a kernel expands them. */
typedef struct gysk_resp16 { uint64_t svc_id; uint32_t usec; uint16_t host_idx; uint8_t cli_port; uint8_t flags; } gysk_resp16;
typedef struct gysk_tcp24 { uint64_t svc_id; uint64_t flow_key; uint32_t bytes; uint16_t host_idx; uint8_t type; uint8_t pad; } gysk_tcp24;
typedef struct gysk_task24 { uint64_t aggr_task_id; uint32_t cpu_pct; uint32_t cpu_delay_msec; uint32_t blkio_delay_msec; uint16_t host_idx; uint16_t pad; } gysk_task24;

/* ---- wire subtypes accepted by gysk_ingest (NOTIFY_TYPE_E, common/gy_comm_proto.h:155-200) ---- */
#define GYSK_NOTIFY_LISTENER_STATE	0x309u
#define GYSK_NOTIFY_TCP_CONN		0x30Cu
#define GYSK_NOTIFY_AGGR_TASK_STATE	0x310u
#define GYSK_NOTIFY_ACTIVE_CONN_STATS	0x312u	/* handle_partha_active_conns, server/gy_mconnhdlr.cc:7705 (dispatched at :5250) */

/* ---- configuration ---- */
#define GYSK_FLAG_AUTO_REGISTER		0x1u	/* unknown svc/task ids are inserted on first sight (device side);
						   without it unknown ids are skipped like a failed
						   listen_tbl_.lookup_single_elem_locked, gy_mconnhdlr.cc:11183 */
#define GYSK_FLAG_MERGE_LEVELS		0x2u	/* the merge step also folds the 300-s / 5-day levels, active connections, errors
						   and max rtt of the member services into each logical service (see
						   gysk_query_logical); without it the merge arena and its collectives are as before */
#define GYSK_FLAG_MERGE_STATES		0x4u	/* the merge step also rolls up the listener states of the member services into each
						   logical service (LISTEN_SUMM_STATS per logical service: gysk_query_logical_states,
						   GYSK_TOPN_ISSUE of gysk_topn_logical); with or without GYSK_FLAG_MERGE_LEVELS, the
						   same flags on every rank. Without it the merge arena and its collectives are as before */
#define GYSK_FLAG_MERGE_CLUSTERS	0x8u	/* the merge step also rolls up the service state of each host cluster (gysk_set_cluster_map,
						   gysk_query_cluster_states); combines freely with the two flags above, the same flags on
						   every rank. Without it the merge arena and its collectives are as before */
#define GYSK_FLAG_MERGE_TOPN		0x10u	/* the merge step also ranks the services and processes of every rank (gysk_topn_global,
						   gysk_topn_global_tasks); combines freely with the three flags above, the same flags on
						   every rank. Its candidates travel in the t-digest slab: gysk_merge_tdigest_slab reports
						   the larger size, the collectives stay the same. A merge needs no gysk_set_logical_map.
						   Without it the merge slab, arena and collectives are as before */
#define GYSK_FLAG_FLOW_LEVEL		0x20u	/* a rolling 300-s count-min level beside the current and last windows' tables
						   (gysk_query_flows_5min, gysk_export_cms_5min); with it the merge step also sums the
						   level across ranks (gysk_query_flows_global_5min; the same flags on every rank).
						   Costs NSLOTS + 1 = 11 more tables of depth << log2_width cells. Without it nothing is
						   allocated, every other call answers as before and the three calls are GYSK_ERR_NOTSUP */
#define GYSK_FLAG_MERGE_TRACES		0x40u	/* the merge step also merges the members' last closed trace windows into each logical
						   service (gysk_query_logical_traces, "request traces of logical services" below); combines
						   freely with the flags above, the same flags on every rank. Needs trace rows: gysk_create
						   refuses it with max_trace_svcs == 0. Without it the merge arena, slab and collectives are
						   as before */
#define GYSK_FLAG_FLOW_QUERIES		0x80u	/* a count-min of response samples per flow beside the connection count-min: requests and
						   response msec of a client in the open and the last window (gysk_query_flow_queries,
						   "flow queries" below); with it the merge step also sums those tables across ranks (the
						   same flags on every rank). Costs 2 more tables of depth << log2_width cells and a second
						   batch flow table. Without it nothing is allocated, every other call answers as before and
						   the flow query calls are GYSK_ERR_NOTSUP */
#define GYSK_FLAG_FLOW_QUERY_LEVEL	0x100u	/* a rolling 300-s level of the flow query tables (gysk_query_flow_queries_5min,
						   gysk_export_cms_queries_5min); with it the merge step also sums the level across ranks
						   (gysk_query_flow_queries_global_5min; the same flags on every rank). Needs
						   GYSK_FLAG_FLOW_QUERIES: gysk_create refuses it without; combines freely with every other
						   flag. Costs NSLOTS + 1 = 11 more tables of depth << log2_width cells. Without it nothing is
						   allocated, every other call answers as before and the three calls are GYSK_ERR_NOTSUP */
#define GYSK_FLAG_FLOW_RESP_HIST	0x200u	/* a count-min of the flow query samples by response-time bucket: each client flow's
						   response histogram and its p25 / p95 / p99 in the open and the last window
						   (gysk_query_flow_resp, "flow response histograms" below), with GYSK_FLAG_FLOW_QUERY_LEVEL
						   also over the rolling 300 s; with it the merge step also sums those tables across ranks
						   (the same flags on every rank). Needs GYSK_FLAG_FLOW_QUERIES: gysk_create refuses it
						   without. Costs 8x the words of a query table: 2 tables of depth << log2_width 64-byte
						   cells (512 MiB at 4 x 2^20), 11 more with GYSK_FLAG_FLOW_QUERY_LEVEL (2.75 GiB), and a
						   third batch flow table; gysk_merge_prepare's arena holds one more copy of each held
						   table (512 MiB more, 768 MiB with the level). Measured on one H100 80GB HBM3 at 700 W with the bench workload
						   (100 M-event batches, against GYSK_FLAG_FLOW_QUERIES alone): the TCP drain pass 6.4 ->
						   24.5 ms and the TASK pass 0.9 -> 1.2 ms per batch (its flows x cell words overflow the
						   batch table, so 10 M samples a batch update the cells directly), gysk_flush 0.51 -> 0.63
						   ms (1.92 ms with the level), gysk_merge_prepare +0.41 ms (+0.56 ms with the level). Without it nothing is allocated, every other
						   call answers as before and the flow response calls are GYSK_ERR_NOTSUP */
#define GYSK_FLAG_FLOW_TOPK		0x400u	/* the GYSK_FLOW_TOPK_CAP heaviest client flows of each window beside the connection
						   count-min (by kbytes) and, with GYSK_FLAG_FLOW_QUERIES, the flow query tables (by
						   queries), ranked on each rank and across ranks (gysk_topk_flows, "heaviest flows"
						   below). Needs no other flag. Without it nothing is allocated, every other call answers
						   as before and the four calls are GYSK_ERR_NOTSUP */
#define GYSK_FLOW_TOPK_CAP		4096u	/* K: the flows each heaviest-flow set holds (fixed: gysk_config has no word for it) */
#define GYSK_FLAG_FLOW_TOPK_5MIN	0x800u	/* the GYSK_FLOW_TOPK_CAP heaviest client flows of each held rolling 300-s flow level,
						   with a bound on every flow they leave out (gysk_topk_flows_5min, "heaviest flows of the
						   300-s levels" below), on each rank and across ranks. Needs GYSK_FLAG_FLOW_TOPK and
						   GYSK_FLAG_FLOW_LEVEL or GYSK_FLAG_FLOW_QUERY_LEVEL: gysk_create refuses it without.
						   Without it nothing is allocated, every other call answers as before and the four calls
						   are GYSK_ERR_NOTSUP */
#define GYSK_FLAG_FLOW_TOPK_SLOW	0x1000u	/* the GYSK_FLOW_TOPK_CAP client flows with the most slow responses of each window and,
						   with GYSK_FLAG_FLOW_TOPK_5MIN and GYSK_FLAG_FLOW_QUERY_LEVEL, of the rolling 300-s
						   level, on each rank and across ranks (gysk_topk_flow_slow, "flows with the most slow
						   responses" below). Needs GYSK_FLAG_FLOW_TOPK and GYSK_FLAG_FLOW_RESP_HIST: gysk_create
						   refuses it without. Without it nothing is allocated, every other call answers as before
						   and the five calls are GYSK_ERR_NOTSUP */
#define GYSK_FLAG_CLIENT_LEVELS		0x2000u	/* each service's distinct clients in the last window and the rolling 300 s, on each rank
						   and merged across ranks (gysk_query_svc_clients, "distinct clients per window" below).
						   Needs no other flag. Without it nothing is allocated, every other call answers as
						   before and the five calls are GYSK_ERR_NOTSUP */
#define GYSK_FLAG_FLOW_ERRORS		0x4000u	/* a count-min of each client flow's client and server errors beside the flow query
						   tables, in the open and last window and with GYSK_FLAG_FLOW_QUERY_LEVEL the rolling
						   300 s (gysk_query_flow_errors, "flow errors" below); with GYSK_FLAG_FLOW_TOPK also the
						   flows with the most server errors; the merge step sums the tables and ranks the sets
						   across ranks. Needs GYSK_FLAG_FLOW_QUERIES: gysk_create refuses it without; combines
						   freely with every other flag. Costs 2 more tables of depth << log2_width cells (13 with
						   the level), a fourth batch flow table and, with GYSK_FLAG_FLOW_TOPK, a candidate list
						   of K + max_batch keys (device_bytes +1.24 GB at the bench's sizes). Measured on one H100
						   80GB HBM3 at 700 W with the bench workload (100 M-event batches) at 1 % error samples:
						   the TCP drain pass 6.57 -> 6.75 ms and the TASK pass 1.40 -> 1.58 ms per batch; at 100 %
						   the TCP pass 17.2 ms. Without it nothing is allocated, every other call answers as
						   before and the flow error calls are GYSK_ERR_NOTSUP */
#define GYSK_FLAG_SVC_TOP_CLIENTS	0x8000u	/* each service's GYSK_SVC_TOPC_K heaviest clients by kbytes, in the open window, the
						   last one and the rolling 300 s, with a stated error bound (gysk_query_svc_top_clients,
						   "each service's heaviest clients" below). Needs no other flag. Without it nothing is
						   allocated, every other call answers as before and the two calls are GYSK_ERR_NOTSUP */
#define GYSK_HLL_WINDOW_P		8u	/* precision of the windowed client registers: 256 one-byte registers per set (fixed:
						   gysk_config has no word for it) */

typedef struct gysk_config
{
	uint32_t	struct_size;		/* sizeof(gysk_config) */
	int32_t		device;			/* CUDA device ordinal */
	uint32_t	max_svcs;		/* service (listener) capacity */
	uint32_t	max_tasks;		/* aggregated-process capacity */
	uint32_t	cms_depth;		/* rows, 1..8 (default 4) */
	uint32_t	cms_log2_width;		/* columns = 1 << this (default 20) */
	uint32_t	hll_p;			/* registers per service = 1 << p, 4..16 (default 12) */
	uint32_t	td_compression;		/* t-digest delta, 10..256 (default 200: up to 256 centroids kept; exports for Postgres are
						   recompressed to public.tdigest(x, 100), gy_query_common.cc:1855) */
	uint32_t	max_batch;		/* max events per device batch = one ingest + merge pass, < 2^27 (default 1 << 22) */
	uint32_t	flags;			/* GYSK_FLAG_* */
	uint32_t	rank, world;		/* this engine owns events with host_idx % world == rank; world 0/1 = all */
	uint32_t	stage_batch;		/* events per host staging buffer / H2D chunk; 0 = min(max_batch, 1 << 22) */
	uint32_t	idle_evict_secs;	/* a service without events for this long (and older than twice that) is evicted at
						   gysk_flush: TIMEOUT_INET_DIAG_SECS 300, common/gy_socket_stat.h:997, rule of
						   common/gy_socket_stat.cc:3968-3982. 0 (default) = never */
	uint32_t	task_idle_evict_secs;	/* an aggregated process whose last sample arrived in a window closed more than this many
						   seconds before the tsec of a gysk_flush is evicted by that flush: the rule of
						   MCONN_HANDLER::cleanup_partha_unused_aggr_tasks (server/gy_mconnhdlr.cc:16492-16541), whose
						   value is 1800 (last_tusec_ older than 30 min). 0 (default) = never; "process eviction" below */
	uint32_t	max_trace_svcs;		/* trace rows: services whose request traces (GYSK_EV_TRACE) are summed per 5-s window on the
					   device ("request traces" below). 0 (default) = off: GYSK_EV_TRACE events are dropped, nothing
					   is allocated and the trace calls are GYSK_ERR_NOTSUP. max_svcs + 1 + max_trace_svcs <= 1 << 24
					   (gysk_create and gysk_grow refuse more). This was the last spare word of the struct: a new
					   setting needs a new ABI version */
} gysk_config;

typedef struct gysk_engine gysk_engine;

/* ---- per-service summary: the fields SvcStateFields exposes + the new sketch answers ---- */
typedef struct gysk_svc_summary
{
	uint64_t	glob_id;
	int32_t		found;			/* 0 if the id is unknown */
	uint32_t	nqrys_5s;		/* LISTENER_STATE_NOTIFY::nqrys_5s_       (last closed window) */
	uint64_t	total_resp_5sec;	/* ::total_resp_5sec_ (msec sum, last closed window) */
	int64_t		p95_5s_resp_ms;		/* ::p95_5s_resp_ms_   = get_percentile(95) of the last window */
	int64_t		p99_5s_resp_ms;
	int64_t		p25_5s_resp_ms;		/* the three percentiles listener_stats_update reads, gy_socket_stat.h:459 */
	int64_t		p95_5min_resp_ms;	/* ::p95_5min_resp_ms_ = get_percentile(95) of the 300-s level */
	int64_t		p99_5min_resp_ms;
	uint64_t	nqrys_5min;
	int64_t		p95_5day_resp_ms;
	uint64_t	nqrys_5day;
	int64_t		p95_all_resp_ms;
	int64_t		p99_all_resp_ms;
	uint64_t	nqrys_all;
	int64_t		max_resp_ms;		/* max_val_seen_ of the all-time histogram */
	uint32_t	nconns_5s;		/* TCP events of the last window */
	uint32_t	kbytes_5s;
	uint64_t	nconns_all;
	uint64_t	kbytes_all;
	double		distinct_clients;	/* HLL estimate */
	double		td_p50_us, td_p95_us, td_p99_us;	/* t-digest quantiles (usec); NaN when empty */
	uint64_t	td_count;
	uint32_t	nconns_active;		/* ACTIVE_CONN_STATS of the last window: sum of active_conns_ (-> LISTENER_STATE_NOTIFY::nconns_active_) */
	uint32_t	active_kbytes;		/* ... sum of (bytes_sent_ + bytes_received_) >> 10 */
	float		max_rtt_msec;		/* ... max of max_rtt_msec_ */
	uint32_t	cli_errors, ser_errors;	/* API_TRAN error counters of the last window (-> ::cli_errors_, ::ser_errors_) */
	uint8_t		curr_state;		/* GYSK_STATE_*: get_curr_state of the last closed window (-> ::curr_state_) */
	uint8_t		curr_issue;		/* GYSK_ISSUE_* (-> ::curr_issue_) */
	uint8_t		issue_bit_hist;		/* one bit per window, 1 = state >= BAD (-> ::issue_bit_hist_, gy_socket_stat.cc:4242-4249) */
	uint8_t		high_resp_bit_hist;	/* one bit per window, 1 = response above the 5-day level (-> ::high_resp_bit_hist_) */
} gysk_svc_summary;

/* per-host roll-up of the listener states of one 5-s tick: LISTEN_SUMM_STATS<int>, server/gy_msocket.h:840-866 */
typedef struct gysk_host_summary
{
	int32_t		nstates[8];		/* per OBJ_STATE_E value (STATE_IDLE .. STATE_DOWN) */
	int32_t		tot_qps;		/* += nqrys_5s_ / 5 */
	int32_t		tot_act_conn;		/* += nconns_active_ */
	int32_t		tot_kb_inbound;
	int32_t		tot_kb_outbound;
	int32_t		tot_ser_errors;
	int32_t		nlisteners;
	int32_t		nactive;		/* += !!nqrys_5s_ */
	int32_t		pad;
} gysk_host_summary;

/* cluster roll-up of the host summaries: the service part of MS_CLUSTER_STATE::STATE_ONE (common/gy_comm_proto.h:3183-3214) as
 * CLUSTER_STATE_ONE::update_from_state fills it from PARTHA_INFO::summstats_ (server/gy_mconnhdlr.cc:16036-16046). The task / cpu /
 * memory issue counters come from the host agent's HOST_STATE_NOTIFY and stay zero here. */
typedef struct gysk_cluster_state
{
	uint32_t	nhosts;			/* hosts with a listener-state summary (gysk_cluster_row: hosts with a live service) */
	uint32_t	nsvc_issue;		/* listeners in STATE_BAD / STATE_SEVERE / STATE_DOWN */
	uint32_t	nsvcissue_hosts;	/* hosts with at least one such listener */
	uint32_t	nsvc;			/* += nlisteners */
	uint32_t	total_qps;		/* += tot_qps_ */
	uint32_t	svc_net_mb;		/* += (tot_kb_inbound_ + tot_kb_outbound_) / 1024 */
	uint32_t	pad[2];
} gysk_cluster_state;

/* top-N services of the last closed window (BOUNDED_PRIO_QUEUE users of partha_listener_state, gy_mconnhdlr.cc:11262-11304) */
enum { GYSK_TOPN_QPS = 0, GYSK_TOPN_CONNS = 1, GYSK_TOPN_NET = 2, GYSK_TOPN_ISSUE = 3 /* curr_state > OK, worst first: LISTEN_TOPN::is_comp_issue, server/gy_msocket.h:745 */,
       GYSK_TOPN_ACTIVE = 4 /* gysk_topn_logical and gysk_topn_global only: active connections (top_active_conn_listen_, server/gy_mconnhdlr.cc:11284-11291) */ };
/* top-N aggregated processes of the last closed window: atask_top_cpu_ / atask_top_cpu_delay_ / atask_top_io_delay_ of
 * partha_aggr_task_state (server/gy_mconnhdlr.cc:10020-10065; a task whose metric is zero never enters a queue).
 * score = the window's sum of cpu_pct / cpu_delay msec / blkio_delay msec samples */
enum { GYSK_TOPN_TASK_CPU = 0, GYSK_TOPN_TASK_CPU_DELAY = 1, GYSK_TOPN_TASK_BLKIO_DELAY = 2 };
typedef struct gysk_topn_entry
{
	uint64_t	glob_id;
	uint64_t	score;			/* nqrys_5s / conn events / kbytes of the last window */
	uint32_t	host_idx;
	uint32_t	pad;
} gysk_topn_entry;

/* per-host rankings of gysk_topn_host: the four listener queues of partha_listener_state (server/gy_mconnhdlr.cc:11262-11304) and the
 * seven process queues of partha_aggr_task_state (:10012-10079), as of the host's last message of that kind (10 entries each,
 * BOUNDED_PRIO_QUEUE::try_emplace_locked semantics). score: SVC_ISSUE = curr_state_ << 32 | tasks_delay_usec_; TASK_ISSUE = severe << 32 |
 * ntasks_issue_ + 1; TASK_CPU = IEEE bits of total_cpu_pct_ (orders like the float); else the raw field */
enum {
	GYSK_HOSTTOP_SVC_ISSUE = 0, GYSK_HOSTTOP_SVC_QPS, GYSK_HOSTTOP_SVC_CONNS, GYSK_HOSTTOP_SVC_NET,
	GYSK_HOSTTOP_TASK_ISSUE, GYSK_HOSTTOP_TASK_NET, GYSK_HOSTTOP_TASK_CPU, GYSK_HOSTTOP_TASK_RSS, GYSK_HOSTTOP_TASK_CPU_DELAY,
	GYSK_HOSTTOP_TASK_VM_DELAY, GYSK_HOSTTOP_TASK_BLKIO_DELAY,
};

typedef struct gysk_flow_est
{
	uint64_t	flow_key;
	uint32_t	count;			/* min over rows of the count halves */
	uint32_t	kbytes;			/* min over rows of the kbytes halves */
} gysk_flow_est;

/* a point query on the flow query tables (GYSK_FLAG_FLOW_QUERIES): the layout of gysk_flow_est */
typedef struct gysk_flow_qry_est
{
	uint64_t	flow_key;
	uint32_t	queries;		/* min over rows of the query halves */
	uint32_t	resp_ms;		/* min over rows of the response msec halves */
} gysk_flow_qry_est;

/* a point query on the flow response histograms (GYSK_FLAG_FLOW_RESP_HIST), 96 bytes */
typedef struct gysk_flow_resp_est
{
	uint64_t	flow_key;
	uint32_t	counts[15];		/* per RESP_TIME_HASH bucket the minimum over rows */
	uint32_t	total;			/* the sum of counts (mod 2^32) */
	int64_t		p25_ms, p95_ms, p99_ms;	/* GY_HISTOGRAM::get_percentiles of RESP_TIME_HASH on counts (the full sum as the
						   total): the rule of gysk_svc_summary::p95_5s_resp_ms, so gysk_hist_percentiles(GYSK_CLS_RESP_TIME,
						   0, ...) on the same counts; -1 when the cut-off falls in bucket 0 (an empty histogram) */
} gysk_flow_resp_est;

/* a point query on the flow error tables (GYSK_FLAG_FLOW_ERRORS), 24 bytes */
typedef struct gysk_flow_err_est
{
	uint64_t	flow_key;
	uint32_t	queries;		/* the flow query tables' count for the same window (gysk_query_flow_queries) */
	uint32_t	cli_errors;		/* min over rows of the client-error halves */
	uint32_t	ser_errors;		/* min over rows of the server-error halves */
	uint32_t	pad;
} gysk_flow_err_est;

typedef struct gysk_stats
{
	uint64_t	events_in;		/* events handed to the device */
	uint64_t	events_dropped;		/* svc_id 0, bad type, table full, unknown id without AUTO_REGISTER */
	uint64_t	events_resp, events_tcp, events_task;
	uint64_t	nsvcs, ntasks;
	uint64_t	batches;
	uint64_t	kernel_launches;	/* launches of this library's own kernels so far */
	uint64_t	wire_msgs_ok, wire_msgs_bad;
	uint64_t	svcs_evicted;		/* idle services evicted so far (their slots are recycled) */
} gysk_stats;

/* mergeable device buffers (for the multi-GPU merge step) */
enum { GYSK_RED_SUM_U64 = 0, GYSK_RED_MAX_U8 = 1, GYSK_RED_MAX_I64 = 2 };
typedef struct gysk_buffer_desc
{
	const char	*name;			/* name and dptr stay valid until the next gysk_set_logical_map */
	void		*dptr;			/* device pointer */
	uint64_t	nbytes;
	int32_t		redop;			/* GYSK_RED_* */
	int32_t		pad;
} gysk_buffer_desc;

/* ---- lifecycle ---- */
int		gysk_abi_version(void);
void		gysk_config_default(gysk_config *cfg);
int		gysk_create(const gysk_config *cfg, gysk_engine **out);
void		gysk_destroy(gysk_engine *e);
const char *	gysk_last_error(gysk_engine *e);		/* e may be NULL: error of the last failed gysk_create */
int		gysk_get_stats(gysk_engine *e, gysk_stats *out);	/* synchronises the ingest stream */
/* diagnostic: rows of dense value bins handed out so far to "hot" services — services that brought GYSK_HOT_MIN (environment, default
 * 4096) response samples in one device batch take their later samples as direct updates of an L2-resident row instead of sort keys
 * (GYSK_HOT_ROWS rows, default 2048, 0 = off). Routing only: no result depends on it. Negative = GYSK_ERR_*. */
int64_t		gysk_hot_rows_in_use(gysk_engine *e);
/* introspection (host only, no device needed): the 64-bit word of value bin `bin` (0 .. 847) inside a hot row's first half
 * {samples | sub-msec remainders}; the bin's usec sum lies GYSK_HOT_ROW_BINS words further on. Neighbouring bins are two 128-byte
 * lines apart (DESIGN.md §3). ~0 for a bin the engine does not have. */
#define GYSK_HOT_ROW_BINS	1024u
uint32_t	gysk_hot_row_word(uint32_t bin);
/* diagnostic: response samples of the last device batch that travelled as sort keys (the rest updated hot rows). Negative = GYSK_ERR_*. */
int64_t		gysk_last_batch_keys(gysk_engine *e);
/* diagnostic: connection records of the last device batch whose count-min update did not go through the batch's flow table (its probe
 * limit reached: more flows than the table holds). Routing only, as above. Negative = GYSK_ERR_*. */
int64_t		gysk_last_batch_flow_direct(gysk_engine *e);
/* diagnostic: entries of the batch flow table left non-zero; 0 whenever no batch is in flight. Copies the table (up to 32 MB) to the
 * host. Negative = GYSK_ERR_*. */
int64_t		gysk_flow_table_used(gysk_engine *e);
/* diagnostic (GYSK_FLAG_FLOW_QUERIES): response samples of the last device batch whose flow query update did not go through the batch's
 * query flow table (its probe limit reached). Routing only. GYSK_ERR_NOTSUP without the flag; negative = GYSK_ERR_*. */
int64_t		gysk_last_batch_flow_query_direct(gysk_engine *e);
/* diagnostic (GYSK_FLAG_FLOW_RESP_HIST): response samples of the last device batch whose flow response histogram update did not go
 * through the batch's response flow table (its probe limit reached). Routing only. GYSK_ERR_NOTSUP without the flag. */
int64_t		gysk_last_batch_flow_resp_direct(gysk_engine *e);
/* diagnostic (GYSK_FLAG_FLOW_ERRORS): error samples of the last device batch whose flow error update did not go through the batch's
 * error flow table (its probe limit reached). Routing only. GYSK_ERR_NOTSUP without the flag. */
int64_t		gysk_last_batch_flow_err_direct(gysk_engine *e);

/* ---- capacity: growing the service / process tables of a live engine ---- */
/* Raise the service / process capacity of a live engine (either may equal the current value; neither may shrink, both <= 1 << 24).
 * Slot numbers, every per-slot state, the free stack of recycled slots, the hot rows, the last flush's evicted ids, the maps of
 * gysk_set_logical_map / gysk_set_cluster_map and the last finished merge's results are kept: every read answers afterwards exactly as an
 * engine created with the new capacity and given the same calls would. Serialised with the ingest threads like a reader (their stages
 * are drained first). Between gysk_merge_prepare and gysk_merge_finish it is allowed: the prepared buffers do not depend on the
 * capacity. GYSK_ERR_INVAL: shrink or beyond 1 << 24, or max_svcs + 1 + max_trace_svcs beyond 1 << 24 (the engine unchanged). GYSK_ERR_NOMEM: the new arrays do not fit the device's free memory; this is
 * checked before anything is allocated, and the engine is unchanged. Arrays move one at a time, so the device holds at most the new
 * footprint plus the largest old array while it runs. Should an allocation still fail after the check (another user of the device
 * took the memory meanwhile), the result is GYSK_ERR_NOMEM too: the engine keeps its capacity and answers every read as before, the
 * arrays already moved keep their larger size (device_bytes shows it), and a later gysk_grow reuses them. */
int		gysk_grow(gysk_engine *e, uint32_t max_svcs, uint32_t max_tasks);

/* Auto-grow: at gysk_flush, a table whose slots in use (handed out minus the free stack) reached half its capacity is doubled, up to the
 * limit (0 = never grow that table; the default). The decision uses the counts as of the PREVIOUS gysk_flush (copied to page-locked
 * memory there, read after an event wait on work that is one window old), so neither the ingest path nor gysk_flush gains a
 * synchronisation, and growth points depend only on the sequence of calls. A growth the device's free memory refuses leaves the table
 * as it is (the flush goes on). GYSK_ERR_INVAL: a limit beyond 1 << 24. */
int		gysk_set_auto_grow(gysk_engine *e, uint32_t max_svcs_limit, uint32_t max_tasks_limit);

typedef struct gysk_capacity
{
	uint32_t	max_svcs, max_tasks;		/* current capacities */
	uint32_t	svcs_in_use, tasks_in_use;	/* handed out minus the free stack */
	uint32_t	ngrows, pad;			/* gysk_grow calls that changed something, explicit or automatic */
	uint64_t	device_bytes;			/* device memory the engine holds */
} gysk_capacity;
int		gysk_capacity_info(gysk_engine *e, gysk_capacity *out);	/* synchronises the ingest stream */

/* host only, no device needed: the device bytes one service slot (its rolling-level rows included) and one process slot take in an
 * engine of this configuration (NULL: the defaults); they depend on hll_p and on whether task_idle_evict_secs is set. An engine's footprint is about
 * max_svcs x svc_slot_bytes + max_tasks x task_slot_bytes, plus the id tables (16 B x the power of two >= 2 x slots each), the sort
 * buffers and the count-min tables: 2 tables of cms_depth << cms_log2_width 8-byte cells, 11 more with GYSK_FLAG_FLOW_LEVEL (its 10 ring
 * slots and the level: 352 MiB more at the default 4 x 2^20), 2 more with GYSK_FLAG_FLOW_QUERIES (64 MiB at 4 x 2^20, plus a second
 * batch flow table of up to 32 MiB), 11 more with GYSK_FLAG_FLOW_QUERY_LEVEL (352 MiB at 4 x 2^20, 2.8 GiB at 8 x 2^22), 2 tables of
 * 64-byte cells with GYSK_FLAG_FLOW_RESP_HIST (512 MiB at 4 x 2^20, plus a third batch flow table) and 11 more with it and
 * GYSK_FLAG_FLOW_QUERY_LEVEL (2.75 GiB at 4 x 2^20). The count-min tables do not depend on capacity, so gysk_grow and eviction leave
 * them; gysk_capacity.device_bytes counts them. The merge arena (gysk_merge_prepare, in device_bytes) holds one more copy of every
 * count-min table the engine holds.
 * Trace rows (max_trace_svcs) are not per service slot and not counted here: 3784 bytes each, in gysk_capacity.device_bytes. */
int		gysk_slot_bytes(const gysk_config *cfg, uint64_t *svc_slot_bytes, uint64_t *task_slot_bytes);

/* ---- registration (control path; mirrors partha_listener_info registering listeners before state arrives) ---- */
int		gysk_register_ids(gysk_engine *e, const uint64_t *ids, uint32_t n, int is_task);

/* ---- ingest ---- */
int		gysk_ingest(gysk_engine *e, const uint8_t host_id[16], uint32_t host_idx, uint32_t subtype,
				void *recs, uint32_t nevents, const void *endptr);
int		gysk_ingest_msg(gysk_engine *e, const uint8_t host_id[16], uint32_t host_idx, void *comm_header_msg, uint32_t msglen);
int		gysk_ingest_raw(gysk_engine *e, const uint8_t host_id[16], uint32_t host_idx, uint32_t kind,
				const void *events, uint32_t nevents);
/* zero-copy variant for GYSK_RAW_EVENT32 in page-locked host memory: the buffer is read asynchronously and must stay
 * valid and unmodified until the next gysk_sync() returns */
int		gysk_ingest_pinned(gysk_engine *e, const gysk_event *pinned_events, uint64_t nevents);
int		gysk_ingest_device(gysk_engine *e, const gysk_event *d_events, uint64_t nevents);
int		gysk_export_task_hist(gysk_engine *e, uint64_t aggr_task_id, int which, gysk_hist_serial out[GYSK_HIST_MAX_BUCKETS],
				uint64_t *total_count, int64_t *max_val);
int		gysk_sync(gysk_engine *e);
int		gysk_flush(gysk_engine *e, uint32_t tsec);
/* ids evicted by the most recent gysk_flush (the LISTEN_FLAG_DELETE notifications of common/gy_socket_stat.cc:4023-4033);
 * synchronises the ingest stream. *n = number of ids (may exceed cap: then only cap are written) */
int		gysk_evicted_ids(gysk_engine *e, uint64_t *out, uint32_t cap, uint32_t *n);

/* ---- process eviction (gysk_config.task_idle_evict_secs != 0) ----
 * Arrival is known to the window: a process's last-activity time is the tsec of the last gysk_flush whose closed window held one of its
 * samples, or of the first flush that saw it when no flush has yet closed a window with its samples (a process registered by
 * gysk_register_ids counts from that flush on, as a MAGGR_TASK's last_tusec_ counts from its creation). gysk_flush(tsec) evicts every
 * process whose time t has t + task_idle_evict_secs < tsec (strict): the decision uses the window that flush closes, so samples that
 * arrive in it keep the process. The rule applies to each process on its own, whatever its host. An evicted process's table entry
 * becomes a tombstone, its slot gets the state of a never-used one and goes on the process table's free stack; the next unknown id takes
 * it. So, from that flush on:
 *  - gysk_query_tasks gives found = 0 for the id, gysk_export_task_hist GYSK_ERR_NOENT, gysk_query_task_window no row;
 *  - gysk_topn_tasks never returns it, nor does gysk_topn_global_tasks as of the first merge after the flush;
 *  - the same id seen again takes a slot with three empty histograms and an empty last window;
 *  - gysk_capacity_info.tasks_in_use (and gysk_stats.ntasks) no longer count it, and auto-grow decides on that count;
 *  - gysk_grow keeps the free stack.
 * The per-host queues of gysk_topn_host are what the hosts sent and are not touched; gysk_task_groupby keeps no state and is not affected.
 * The setting adds 20 bytes to each process slot (gysk_slot_bytes counts them only when it is set). */
/* ids evicted by the most recent gysk_flush, in ascending id order: where madhava deletes the MAGGR_TASK of each and its row. The
 * contract of gysk_evicted_ids: synchronises the ingest stream, *n = number of ids (may exceed cap: then only cap are written) */
int		gysk_evicted_task_ids(gysk_engine *e, uint64_t *out, uint32_t cap, uint32_t *n);
/* processes evicted so far */
int		gysk_task_evict_count(gysk_engine *e, uint64_t *total);

/* ---- queries ---- */
int		gysk_query_svcs(gysk_engine *e, const uint64_t *glob_ids, uint32_t n, gysk_svc_summary *out);

/* ---- window reads: every live id of the engine in one device pass, summarised on the device ----
 * Rows are grouped by ascending host_idx and, within a host, ordered by ascending id. The host_idx of an id is the host of the
 * event that created its slot (what gysk_topn_svcs reports); ids created by gysk_register_ids have host 0.
 * host_idx < 0 reads every host. *n = number of matching rows; at most cap rows are written (out may be NULL when cap is 0). */
#define GYSK_WINDOW_ACTIVE_ONLY		0x1u	/* only ids whose closed window held events (the last gysk_flush) */
/* A service row equals the gysk_query_svcs row of its id, byte for byte: what madhava's 5-s tick reads for every listener
 * (partha_listener_state, server/gy_mconnhdlr.cc:10993-11410) once the reduction runs in the engine */
int		gysk_query_window(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_svc_summary *out, uint32_t cap, uint32_t *n);
/* the same read with the host_idx of every written row in hosts[] (cap entries, or NULL): rows and hosts come from one
 * snapshot, so a caller that splits the rows by host (the shim's window_listener_states) needs one call, not one per host */
int		gysk_query_window_hosts(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_svc_summary *out, uint32_t *hosts, uint32_t cap,
				uint32_t *n);

/* ---- the rest of the 5-s listener walk (TCP_SOCK_HANDLER::listener_stats_update, common/gy_socket_stat.cc:3898-4445) ---- */

/* byte-compatible with LISTENER_DAY_STATS, common/gy_comm_proto.h:1620-1653 (48 bytes, at most 2048 per NOTIFY_LISTENER_DAY_STATS
 * message): what madhava's handle_listener_day_stats (server/gy_mconnhdlr.cc:12805-12836) turns into the svcinfo fields p95resp5d,
 * avgresp5d, p95qps and p95aconn */
typedef struct gysk_listener_day_stats
{
	uint64_t	glob_id;
	int64_t		tcount_5d;		/* histstat_[n5days].tcount_ */
	int64_t		tsum_5d;		/* histstat_[n5days].tsum_ (msec) */
	uint32_t	p95_5d_respms, p25_5d_respms;	/* r5daysp95 / r5daysp25 */
	uint32_t	p95_qps, p25_qps;	/* qps_hist_ percentiles */
	uint32_t	p95_nactive, p25_nactive;	/* active_conn_hist_ percentiles */
} gysk_listener_day_stats;

/* The LISTENER_DAY_STATS records of get_curr_state (common/gy_socket_stat.cc:2101-2117), as of the last gysk_flush:
 *  - rows, their order (grouped by ascending host_idx, ascending id within a host), hosts[] and the count / capacity rules are those of
 *    gysk_query_window_hosts (cap 0 counts; *n may exceed cap), restricted to the services old enough for a row;
 *  - a service has a row only when last flush tsec > tsec of the first flush that saw its slot + 900: the reference's
 *    tcur > tstart + 15 * 60 (:2102), under which a young listener sends nothing (statn.glob_id_ == 0, :4367). A slot recycled after an
 *    eviction starts over. A stale service (no events in the closed window) has a row: the reference evaluates it too;
 *  - tcount_5d / tsum_5d / p95_5d_respms / p25_5d_respms: the 5-day level (GYSK_HIST_RESP_5DAY) with the GY_HISTOGRAM percentile rule,
 *    the values gysk_flush hands the state classifier; p95_qps / p25_qps / p95_nactive / p25_nactive: the percentiles of qps_hist_ and
 *    active_conn_hist_ (GYSK_HIST_QPS / GYSK_HIST_ACTIVE_CONN) as they stand after the flush: for a service evaluated at that flush the
 *    classifier's values, for a stale one what the reference computes without an add_data (:4099-4112). Every value is stored into its
 *    field by the reference's int64 -> uint32 conversion (an empty qps histogram's -1 becomes 0xFFFFFFFF);
 *  - the reference sends these every 5 minutes (next_listen_stat_tsec_, :4420): the cadence is the caller's, the engine keeps no timer. */
int		gysk_query_day_stats(gysk_engine *e, int32_t host_idx, gysk_listener_day_stats *out, uint32_t *hosts, uint32_t cap, uint32_t *n);

/* the listener half of the tuple listener_stats_update returns to host_status_update (common/gy_socket_stat.cc:173-175) */
typedef struct gysk_host_listen
{
	uint32_t	host_idx;
	uint32_t	nlisten;		/* nlist++ (:4277): the host's rows of gysk_query_window_hosts(-1, 0) */
	uint32_t	nlisten_issue;		/* nissue++ (:4242-4249): services evaluated at the last flush whose issue bit 0 was set there */
	uint32_t	nlisten_severe;		/* nsevere++ (:4250-4252): ... of those, the ones in GYSK_STATE_SEVERE or worse */
} gysk_host_listen;
/* One row per host with live services, ascending host_idx; *n = number of such hosts, at most cap rows are written (out may be NULL
 * when cap is 0). Only these rows travel to the host, not one per service. nlisten_issue / nlisten_severe are those of the last
 * gysk_flush; nlisten is the row count of gysk_query_window_hosts(-1, 0) at the time of the call, so it also counts services whose first
 * events arrived after the last flush (and a host with only such services has a row). The reference's walk skips a listener younger
 * than 1 s (:4040-4062); here arrival granularity is the window. Every call lists and sorts every live service: a caller with one
 * message per host and window (HOST_STATE_NOTIFY) reads all hosts once per flush and answers the messages from those rows, as the
 * shim's host_state does. */
int		gysk_query_host_listen(gysk_engine *e, gysk_host_listen *out, uint32_t cap, uint32_t *n);

/* inputs of host_status_update's state rule (common/gy_socket_stat.cc:4455-4528) */
typedef struct gysk_host_state_in
{
	uint8_t		cpu_issue, mem_issue, severe_cpu_issue, severe_mem_issue, cpu_idle, pad[3];
	uint32_t	ntasks_issue, ntasks_severe, nlisten_issue, nlisten_severe;
} gysk_host_state_in;
/* host_status_update's state rule: writes the GYSK_STATE_* of HOST_STATE_NOTIFY::curr_state_. Pure, no engine, like gysk_classify_listener */
int		gysk_classify_host(const gysk_host_state_in *in, uint8_t *state);

/* per aggregated process: the p95 fields of AGGR_TASK_HIST_STATS (common/gy_comm_proto.h:2966-2977) as
 * handle_aggr_task_hist_stats fills them (server/gy_mconnhdlr.cc:14648-14706: get_percentiles({95}) of the three MTASK_HIST
 * histograms, T = int, -1 for an empty histogram) and the last closed window of each histogram, the window the top-N lists rank */
typedef struct gysk_task_summary
{
	uint64_t	aggr_task_id;
	int32_t		found;			/* 0 if the id is unknown (the other fields are then zero) */
	uint32_t	host_idx;		/* host of the event that created the slot */
	int32_t		p95_cpu_pct;		/* cpu_pct_histogram_		(HASH_1_3000) */
	int32_t		p95_cpu_delay_ms;	/* cpu_delay_histogram_		(DURATION_HASH) */
	int32_t		p95_blkio_delay_ms;	/* blkio_delay_histogram_	(DURATION_HASH) */
	uint32_t	pad;
	uint64_t	nsamples;		/* samples since start (count of the cpu % histogram) */
	uint64_t	last_count[3];		/* last closed window per histogram {cpu %, cpu delay, blkio delay}: samples */
	int64_t		last_sum[3];		/* ... and their sum */
} gysk_task_summary;
int		gysk_query_tasks(gysk_engine *e, const uint64_t *ids, uint32_t n, gysk_task_summary *out);
/* the task rows of every live aggregated process, in the order and with the count / capacity rules of gysk_query_window */
int		gysk_query_task_window(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_task_summary *out, uint32_t cap, uint32_t *n);
int		gysk_query_flows(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_est *out);
/* LISTEN_SUMM_STATS of the last NOTIFY_LISTENER_STATE message of a host (partha_listener_state, gy_mconnhdlr.cc:11251) */
/* host_idx < 0: over all hosts of this engine; n <= 64 */
int		gysk_topn_svcs(gysk_engine *e, int metric, int32_t host_idx, uint32_t n, gysk_topn_entry *out, uint32_t *nout);
int		gysk_topn_tasks(gysk_engine *e, int metric, uint32_t n, gysk_topn_entry *out, uint32_t *nout);
int		gysk_topn_host(gysk_engine *e, int what /* GYSK_HOSTTOP_* */, int32_t host_idx /* < 0: all hosts */, uint32_t n, gysk_topn_entry *out, uint32_t *nout);
/* roll-up over the given hosts (the hosts of one cluster_name_; host_idxs NULL = every host of this engine): what
 * MCONN_HANDLER::send_cluster_state (server/gy_mconnhdlr.cc:16052) sends to shyama per cluster */
int		gysk_query_cluster_state(gysk_engine *e, const uint32_t *host_idxs, uint32_t n, gysk_cluster_state *out);	/* n <= 64; glob_id = aggr_task_id */
int		gysk_query_host_summary(gysk_engine *e, uint32_t host_idx, gysk_host_summary *out);
int		gysk_export_hist(gysk_engine *e, uint64_t id, int which, gysk_hist_serial out[GYSK_HIST_MAX_BUCKETS],
				uint64_t *total_count, int64_t *max_val);
int		gysk_export_hll(gysk_engine *e, uint64_t glob_id, uint8_t *regs /* 1 << hll_p bytes */);
/* TCP_LISTENER::CONN_BITMAP (common/gy_socket_stat.h:390-455): per response bucket a 32-bit mask over (client port & 0x1F) and its
 * popcount = get_conn_breakup(); bit index = flow_key & 0x1F */
int		gysk_export_conn_bitmap(gysk_engine *e, uint64_t glob_id, int last_window, uint32_t masks[GYSK_HIST_MAX_BUCKETS],
				uint8_t nconn_arr[GYSK_HIST_MAX_BUCKETS]);
int		gysk_export_tdigest(gysk_engine *e, uint64_t glob_id, double *means, uint64_t *weights, uint32_t cap, uint32_t *n,
				double *min_val, double *max_val);
int		gysk_query_quantiles(gysk_engine *e, uint64_t glob_id, const double *qs, uint32_t nq, double *out);
int		gysk_export_cms(gysk_engine *e, int last_window, uint64_t *cells /* depth << log2_width entries */);

/* ---- the rolling 300-s flow level (GYSK_FLAG_FLOW_LEVEL): connections and kbytes of a flow in the last five minutes ----
 * The level holds every flow update, from any ingest route, of the windows closed by the flushes the 300-s response level holds:
 * those whose tsec / 30 lies within the last 10 epochs of the last gysk_flush's tsec / 30 (ring slot (tsec / 30) % 10, a slot
 * holding an older epoch cleared first). It follows that level's rule over gaps and repeated tsec exactly, and is empty before the
 * first flush. The open window is not in it. Because the count-min is linear, the level is the cell-wise sum of those windows'
 * gysk_export_cms(last_window = 1) tables, each packed {count | kbytes << 32} cell mod 2^64 like the table itself.
 * gysk_query_flows_5min: the point query of gysk_query_flows on the level, the minimum over rows of each half.
 * gysk_export_cms_5min: the level's cells (depth << log2_width entries).
 * gysk_query_flows_global_5min: the point query on the level summed over the ranks by the last merge (GYSK_ERR_INVAL before
 * gysk_merge_prepare). A rank's level is relative to its own last flush: gysk_merge_flush_range shows whether the ranks had closed
 * the same window.
 * All three are GYSK_ERR_NOTSUP without the flag. */
int		gysk_query_flows_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_est *out);
int		gysk_export_cms_5min(gysk_engine *e, uint64_t *cells /* depth << log2_width entries */);
int		gysk_query_flows_global_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_est *out);

/* ---- flow queries (GYSK_FLAG_FLOW_QUERIES): requests and response time per client flow ----
 * The connection count-min counts connections and kbytes; a pooled keep-alive client opens one connection and sends thousands of
 * requests. These tables count the requests. They have the depth, width and row hashes of the connection count-min (gysk_export_cms), so
 * a key lands in the same columns of both. Each cell is one u64 {queries : low 32 | response msec sum : high 32}, mod 2^64 like the
 * connection cells; msec = usec / 1000, the step the response histogram takes.
 * A response sample counts iff it reaches its service's response histogram: a known service (a slot) and a value within the RESP
 * validity rule (<= 1 000 000 msec), on every route. Unknown ids, dropped events and GYSK_EV_TRACE events do not count; an API_TRAN
 * counts through the GYSK_EV_RESP it stages. So for every row the low halves of the open window's cells sum to the nqrys of every
 * service's open window (mod 2^32). The window rule is the count-min's: gysk_flush closes the open table and opens an empty one.
 * The key of a sample is its event's flow_key, which each route sets as follows:
 *   GYSK_RAW_TCP_IPV4_RESP / _IPV6_RESP : (client ip << 32) | client port (an IPv6 address folded to 32 bits), the key the same
 *                                         client's connection events carry, so one key answers both sketches
 *   GYSK_RAW_EVENT32, gysk_ingest_device : the feeder's flow_key
 *   GYSK_RAW_RESP16, GYSK_RAW_API_TRAN   : the client port alone: their samples count under the port, not under a client
 * gysk_query_flow_queries: per key the minimum over rows of each half (a count-min estimate: never below the exact count).
 * gysk_export_cms_queries: the open (last_window = 0) or last closed table, depth << log2_width cells.
 * gysk_query_flow_queries_global: the point query on the tables summed over the ranks by the last merge (GYSK_ERR_INVAL before
 * gysk_merge_prepare). gysk_grow and eviction leave the tables alone: they do not depend on the service table.
 * All three are GYSK_ERR_NOTSUP without the flag. */
int		gysk_query_flow_queries(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_qry_est *out);
int		gysk_export_cms_queries(gysk_engine *e, int last_window, uint64_t *cells /* depth << log2_width entries */);
int		gysk_query_flow_queries_global(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_qry_est *out);

/* ---- the rolling 300-s flow query level (GYSK_FLAG_FLOW_QUERY_LEVEL): requests and response time of a flow in the last five minutes ----
 * The level holds the flow query tables of the windows closed by the flushes the 300-s response level holds, by the rule of the
 * connection count-min's level (GYSK_FLAG_FLOW_LEVEL): ring slot (tsec / 30) % 10, a slot holding an older epoch replaced, the same
 * behaviour over gaps, repeated tsec and a step back, empty before the first flush. The open window is not in it. Each cell is the
 * cell-wise sum mod 2^64 of those windows' gysk_export_cms_queries(last_window = 1) tables: the table one window fed all their samples
 * would hold, {queries | response msec << 32} with the carry of the table itself.
 * gysk_query_flow_queries_5min: the point query of gysk_query_flow_queries on the level, the minimum over rows of each half.
 * gysk_export_cms_queries_5min: the level's cells (depth << log2_width entries).
 * gysk_query_flow_queries_global_5min: the point query on the level summed over the ranks by the last merge (GYSK_ERR_INVAL before
 * gysk_merge_prepare). A rank's level is relative to its own last flush: gysk_merge_flush_range shows whether the ranks had closed
 * the same window.
 * All three are GYSK_ERR_NOTSUP without the flag. */
int		gysk_query_flow_queries_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_qry_est *out);
int		gysk_export_cms_queries_5min(gysk_engine *e, uint64_t *cells /* depth << log2_width entries */);
int		gysk_query_flow_queries_global_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_qry_est *out);

/* ---- flow response histograms (GYSK_FLAG_FLOW_RESP_HIST): how slow a client's slow requests were ----
 * The flow query tables give a client's mean response time; these give its response histogram, so its p95 / p99. They count exactly
 * the samples the flow query tables count, under the same keys (RESP16 and API_TRAN samples under the client port alone), with the
 * depth, width and row hashes of the connection count-min: a key lands in the same columns of all three table families. A cell is 8 u64
 * words (64 bytes): the count of RESP_TIME_HASH bucket b (0 .. 14, of msec = usec / 1000) sits in half b & 1 (low 32 bits: 0) of word
 * b >> 1, word 7's high half is always 0. Every word is summed mod 2^64 like every other count-min cell; a known edge: a bucket count
 * past 2^32 in one cell carries into its neighbour bucket, as the query half of a flow query cell carries into its msec half. So for
 * every row and column the 15 counts of a cell sum to the query half of the same flow query cell (mod 2^32), and for every row and
 * bucket the column sum equals that bucket summed over every service's response histogram of the same window.
 * The windows: the open table and the last closed one, by the count-min's flush rule; with GYSK_FLAG_FLOW_QUERY_LEVEL also the rolling
 * 300-s level by the rule of gysk_query_flow_queries_5min: the cell-wise sum of the held windows' gysk_export_cms_resp(last_window = 1)
 * tables.
 * gysk_query_flow_resp: per key and bucket the minimum over rows (a count-min estimate: never below the key's exact count), their sum and
 *   the percentiles of those counts (gysk_flow_resp_est). A key alone in its columns gets its exact histogram and percentiles.
 * gysk_export_cms_resp: the open (last_window = 0) or last closed table, (depth << log2_width) x 8 words, cell-major.
 * gysk_query_flow_resp_global: the point query on the tables summed over the ranks by the last merge (GYSK_ERR_INVAL before
 *   gysk_merge_prepare). The _5min triple: the same on the level (GYSK_ERR_NOTSUP without GYSK_FLAG_FLOW_QUERY_LEVEL).
 * gysk_grow and eviction leave the tables alone. Every call is GYSK_ERR_NOTSUP without the flag. */
int		gysk_query_flow_resp(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_resp_est *out);
int		gysk_export_cms_resp(gysk_engine *e, int last_window, uint64_t *words /* (depth << log2_width) x 8 entries */);
int		gysk_query_flow_resp_global(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_resp_est *out);
int		gysk_query_flow_resp_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_resp_est *out);
int		gysk_export_cms_resp_5min(gysk_engine *e, uint64_t *words /* (depth << log2_width) x 8 entries */);
int		gysk_query_flow_resp_global_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_resp_est *out);

/* ---- heaviest flows (GYSK_FLAG_FLOW_TOPK): which clients to ask the flow tables about ----
 * Every flow table answers a point query on a key the caller already has; these sets name the keys. There is one set per held windowed
 * table: the connection count-min, scored by the kbytes half, and with GYSK_FLAG_FLOW_QUERIES the flow query table, scored by the queries
 * half. A flow's score is the point estimate of that half: the minimum over rows, what gysk_query_flows / gysk_query_flow_queries return.
 * The rule, after each device batch, once all of the batch's increments are in the open table: let B be the distinct flow keys whose
 * records reached that table in the batch (connection records of services that hold a slot, from every route including
 * NOTIFY_ACTIVE_CONN_STATS; counted response samples for the query table; dropped events, unknown ids and GYSK_EV_TRACE events never
 * enter B). The open set C becomes the K = GYSK_FLOW_TOPK_CAP best of C u B by (score descending, flow key ascending), scored on the
 * table as it is after the batch. gysk_flush moves the open set to the last window's set and starts the open set empty, as it swaps the
 * tables. Two keys whose two lookup2 hashes both agree are one flow to every count-min: the set may name either.
 * Guarantee: if no cell half wraps during the window, every flow whose exact score in the window exceeds the smallest score of a full set
 * (K members) is in that set; a window of at most K flows has every one of them in its set. (Scores never fall within a window, so the
 * K-th score of the set never falls; a flow that leaves the set, or is never admitted, scores at most the K-th at that batch, and its
 * exact score is at most its estimate.)
 * Across ranks: gysk_merge_prepare carries each rank's last-window sets in the t-digest slab (no logical map needed); gysk_merge_finish
 * scores the union U of every rank's sets on the summed last-window tables and keeps the K best by the same order. A flow whose exact
 * global score exceeds sum over ranks of thr_r is in U (thr_r: the smallest score of rank r's set when it is full, else 0).
 * Cost: per held table a candidate list of K + max_batch flow keys and a key per batch flow-table entry (8 B each); each batch sorts its
 * candidates by key, scores the distinct ones and sorts them by score. DESIGN.md section 7 has the measured times.
 * gysk_topk_flows: the first min(n, K) of the open (last_window = 0) or last set, best first, with their current estimates; entries with
 *   a zero score are left out, so *nout may be below n. gysk_topk_flow_queries: the same for the query table (GYSK_ERR_NOTSUP without
 *   GYSK_FLAG_FLOW_QUERIES). The _global pair: the merged lists of the last gysk_merge_finish, with their estimates on the summed tables
 *   (GYSK_ERR_INVAL before the first one). Every call is GYSK_ERR_NOTSUP without the flag.
 * Not covered: per-(service, client) pairs, a configurable K. */
int		gysk_topk_flows(gysk_engine *e, int last_window, uint32_t n, gysk_flow_est *out, uint32_t *nout);
int		gysk_topk_flow_queries(gysk_engine *e, int last_window, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout);
int		gysk_topk_flows_global(gysk_engine *e, uint32_t n, gysk_flow_est *out, uint32_t *nout);
int		gysk_topk_flow_queries_global(gysk_engine *e, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout);

/* ---- heaviest flows of the 300-s levels (GYSK_FLAG_FLOW_TOPK_5MIN): the top talkers and requesters of the last five minutes ----
 * A client that sends steadily for five minutes may never be among one window's K heaviest, yet be the heaviest of the five minutes.
 * One set per held level: the connection level (GYSK_FLAG_FLOW_LEVEL), scored by its kbytes half, and the flow query level
 * (GYSK_FLAG_FLOW_QUERY_LEVEL), scored by its queries half. A score is the level's point estimate (gysk_query_flows_5min /
 * gysk_query_flow_queries_5min); the order is the window sets' (score descending, flow key ascending); K = GYSK_FLOW_TOPK_CAP.
 * The rule follows the level's own ring: at every gysk_flush, once the closing window is in ring slot s = (tsec / 30) % 10, and before
 * the window sets swap, per held level:
 *   1. slot fold: if the flush cleared slot s, its set S_s and bound B_s are cleared first. S_s becomes the K best of S_s u W scored on
 *      ring slot s, W the closing window's heaviest-flow set; B_s = max(thr(S_s), B_s + thr(W));
 *   2. level set: L becomes the K best of the union of the live slots' sets scored on the level; B_L = max(thr(L), sum of the live B_s).
 * thr(X) is the smallest score of X when it holds K flows, else 0. Before the first flush L is empty and B_L = 0; the open window is
 * not in the level, so not in L either.
 * Guarantee: if no cell half wraps, every flow that L does not hold has an exact 5-minute score of at most B_L; every flow whose exact
 * score exceeds B_L is in L. (A flow outside W scores at most thr(W) in that window; a flow cut at a fold scores at most that fold's
 * threshold; a slot's scores never fall within its epoch. DESIGN.md section 2 has the proof.) A steady client that no window ranks can
 * leave B_L large: the bound says how much of the five minutes the list can have missed.
 * Across ranks: gysk_merge_prepare carries each rank's L sets and B_L after the window sets in the t-digest slab (no logical map
 * needed); gysk_merge_finish keeps the K best of the union of every rank's set scored on the summed levels, with B_G = max(thr(G), sum
 * over ranks of B_L). Each rank's level is relative to its own last flush: gysk_merge_flush_range shows whether they closed the same one.
 * gysk_topk_flows_5min / gysk_topk_flow_queries_5min: the first min(n, K) flows of L, best first, each row what the _5min point query
 *   answers for its key; entries with a zero score are left out, so *nout may be below n. *bound (may be NULL) = B_L. GYSK_ERR_NOTSUP
 *   without the flag or without the level the call reads. The _global pair: the same of the last gysk_merge_finish, each row what the
 *   _global_5min point query answers, *bound = B_G (GYSK_ERR_INVAL before the first one). */
int		gysk_topk_flows_5min(gysk_engine *e, uint32_t n, gysk_flow_est *out, uint32_t *nout, uint64_t *bound);
int		gysk_topk_flow_queries_5min(gysk_engine *e, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout, uint64_t *bound);
int		gysk_topk_flows_global_5min(gysk_engine *e, uint32_t n, gysk_flow_est *out, uint32_t *nout, uint64_t *bound);
int		gysk_topk_flow_queries_global_5min(gysk_engine *e, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout, uint64_t *bound);

/* ---- flows with the most slow responses (GYSK_FLAG_FLOW_TOPK_SLOW): which clients get the slow answers ----
 * The heaviest-flow sets rank by volume, so a client with few requests, many of them slow, is never listed there; the flow response
 * histograms answer only for a key the caller has. These sets name the clients behind a bad p99.
 * A counted response sample (one the flow response histograms count) is slow when its msec is above the threshold T, one of the 13
 * RESP_TIME_HASH thresholds (1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000): exactly when its bucket
 * gysk_hist_bucket(GYSK_CLS_RESP_TIME, msec) >= b_slow = 2 + the index of T. T defaults to 300 ms (b_slow = 9), a choice of this
 * library: the reference has no per-client rule. gysk_set_flow_slow sets it before the engine takes its first event or gysk_flush;
 * every rank of a merge must use the same T, as with the flags (a set or slot folded under two thresholds has no guarantee).
 * Score of a flow on a response table (open, last, ring slot, level or merged sum): S = sum over b >= b_slow of counts[b], the
 * per-bucket minimum over rows that gysk_query_flow_resp returns, saturated at 2^32 - 1. S is never below the flow's exact slow count,
 * never above the minimum over rows of the row sums, and never falls within a window, so the guarantees below are those of the sets
 * above, word for word (DESIGN.md section 2).
 * Window sets: one open and one last set of K = GYSK_FLOW_TOPK_CAP keys on the response tables. After each device batch the open set
 * becomes the K best of C u B_slow by (score descending, flow key ascending), scored on the table after the batch; B_slow is the
 * distinct flow keys with at least one slow counted sample in the batch (GYSK_EV_TRACE samples never enter). gysk_flush moves the open
 * set to the last one. Guarantee: if no cell half wraps, a flow whose exact slow count exceeds the smallest score of a full set is in
 * it; a window of at most K slow flows has every one of them. A flow with only fast samples is never listed.
 * 300-s level (with GYSK_FLAG_FLOW_TOPK_5MIN and GYSK_FLAG_FLOW_QUERY_LEVEL): slot sets, L, B_s and B_L by the rule of the 300-s heaviest-
 * flow sets above, on the response ring slots and level, scored by S; every flow outside L has an exact 5-minute slow count of at most B_L.
 * Across ranks: gysk_merge_prepare carries the last-window slow set, and with the level L and B_L, after the other heaviest-flow sets
 * in the t-digest slab; gysk_merge_finish keeps the K best of the union on the summed response tables, with B_G = max(thr(G), sum over
 * ranks of B_L) for the level. A flow whose exact global slow count exceeds the sum of the ranks' thresholds is in the window union.
 * Cost: a candidate list of K + max_batch keys (8 B each) and the sets; each batch appends one key per slow sample in the TCP drain pass,
 * then sorts, scores (each candidate reads its depth 64-byte cells) and ranks the candidates after the other sets' selections, in the
 * same sort buffers. Measured on one H100 80GB HBM3 at 700 W, bench workload (100 M-event batches, few slow samples): about 0.2 ms more
 * in the TCP pass and 0.2 ms of selection per batch, gysk_merge_finish +0.15 ms, gysk_flush unchanged, device_bytes +1.07 GB (the list
 * at max_batch = 2^27). DESIGN.md section 7 has the measurements.
 * gysk_set_flow_slow: GYSK_ERR_NOTSUP without the flag; GYSK_ERR_INVAL when above_ms is not one of the 13 thresholds, or once the
 *   engine has taken an event or a gysk_flush (the engine is left unchanged).
 * gysk_topk_flow_slow: the first min(n, K) flows of the open (last_window = 0) or last set, best first, each row byte-equal to what
 *   gysk_query_flow_resp(last_window) answers for its key (so score == sum of out.counts[b] from b_slow on, saturated); entries with a
 *   zero score are left out, so *nout may be below n. gysk_topk_flow_slow_5min: the same of L with *bound (may be NULL) = B_L, rows as
 *   gysk_query_flow_resp_5min (GYSK_ERR_NOTSUP without the level). The _global pair: the same of the last gysk_merge_finish, rows as
 *   gysk_query_flow_resp_global(1) / _global_5min, *bound = B_G (GYSK_ERR_INVAL before the first one). */
int		gysk_set_flow_slow(gysk_engine *e, uint32_t above_ms);
int		gysk_topk_flow_slow(gysk_engine *e, int last_window, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout);
int		gysk_topk_flow_slow_global(gysk_engine *e, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout);
int		gysk_topk_flow_slow_5min(gysk_engine *e, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout, uint64_t *bound);
int		gysk_topk_flow_slow_global_5min(gysk_engine *e, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout, uint64_t *bound);

/* ---- flow errors (GYSK_FLAG_FLOW_ERRORS): which clients get the errors ----
 * gysk_svc_summary.cli_errors / ser_errors count a service's errors, and ser_errors can turn a listener BAD, but no other answer names
 * the clients that got them: the heaviest-flow sets rank by volume, the query tables count every request whatever its outcome, and a
 * failing request is often fast. These tables count each client flow's errors.
 * Counting rule: a response sample counts iff it counts in the flow query tables (gysk_query_flow_queries) and its event carries
 * GYSK_EVF_CLI_ERROR and/or GYSK_EVF_SER_ERROR. It adds 1 to each half whose bit is set, exactly as the service's error counts take it.
 * The key is the flow query tables' key, and the tables have their depth, width and row hashes, so a key lands in the same columns of
 * every flow table family. Each cell is one u64 {cli_errors : low 32 | ser_errors : high 32}, summed mod 2^64. Hot-row and key routes
 * count alike; GYSK_EV_TRACE events, samples beyond the validity rule, unknown ids and dropped events never count. Two limits follow
 * from the routes: a GYSK_RAW_API_TRAN sample counts under the client port alone (as in the query tables), and the raw eBPF response
 * events (GYSK_RAW_TCP_IPV4_RESP / _IPV6_RESP) carry no error bits, so they never count.
 * Invariants: for every row the error halves of the open table sum to the open-window cli_errors / ser_errors of every service
 * (mod 2^32); cell by cell each error half is at most the query half of the same flow query cell.
 * Windows: the open table and the last closed one, by the count-min's flush rule; with GYSK_FLAG_FLOW_QUERY_LEVEL also the rolling 300-s
 * level by the rule of gysk_query_flow_queries_5min.
 * gysk_query_flow_errors: per key queries as gysk_query_flow_queries answers it for the same window, and each error half's minimum over
 *   rows (a count-min estimate: never below the exact count). gysk_export_cms_errors: the open (last_window = 0) or last closed table,
 *   depth << log2_width cells. The _global pair: the same on the tables summed over the ranks by the last merge (GYSK_ERR_INVAL before
 *   gysk_merge_prepare). The _5min calls: the same on the level (GYSK_ERR_NOTSUP without GYSK_FLAG_FLOW_QUERY_LEVEL).
 * Flows with the most server errors (with GYSK_FLAG_FLOW_TOPK; GYSK_ERR_NOTSUP without): one open and one last set of K =
 *   GYSK_FLOW_TOPK_CAP keys on the error tables, scored by the ser_errors half, by the rule and guarantee of the heaviest-flow sets; the
 *   candidates are the distinct flow keys with a server-error sample in the batch. A flow with no server error (a client-error-only
 *   flow) is never listed. With GYSK_FLAG_FLOW_TOPK_5MIN and GYSK_FLAG_FLOW_QUERY_LEVEL the 300-s sets, L and B_L by the rule of the
 *   heaviest flows of the 300-s levels, on the error ring and level. gysk_merge_prepare carries the last-window set, and with the level
 *   L and B_L, after the slow sets in the t-digest slab; gysk_merge_finish keeps the K best of the union on the summed error tables, with
 *   B_G = max(thr(G), sum over ranks of B_L).
 * gysk_topk_flow_errors(_5min / _global / _global_5min): the first min(n, K) flows of the set, best first, each row byte-equal to what the
 *   matching point query answers for its key; entries with zero ser_errors are left out, so *nout may be below n; *bound (may be NULL)
 *   = B_L or B_G.
 * Cost: each counted sample with an error bit adds a third batch flow-table update in the TCP drain pass, each server-error sample a
 * candidate key, and the TASK pass sweeps one more table. Measured on one H100 80GB HBM3 at 700 W, bench workload (100 M-event batches,
 * against GYSK_FLAG_FLOW_QUERIES and GYSK_FLAG_FLOW_TOPK alone): with no error samples the TASK pass +0.08 ms; at 1 % error samples the
 * TCP pass 6.57 -> 6.75 ms, the TASK pass 1.40 -> 1.58 ms and the selection +0.3 ms per batch; at 100 % the TCP pass 6.6 -> 17.2 ms and the
 * selection +4.9 ms; gysk_flush +0.02 ms, gysk_merge_prepare +0.06 ms, gysk_merge_finish up to +0.14 ms, device_bytes +1.24 GB (the
 * candidate list at max_batch = 2^27). DESIGN.md section 7 has the measurements. */
int		gysk_query_flow_errors(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_err_est *out);
int		gysk_query_flow_errors_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_err_est *out);
int		gysk_query_flow_errors_global(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_err_est *out);
int		gysk_query_flow_errors_global_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_err_est *out);
int		gysk_export_cms_errors(gysk_engine *e, int last_window, uint64_t *cells /* depth << log2_width entries */);
int		gysk_export_cms_errors_5min(gysk_engine *e, uint64_t *cells /* depth << log2_width entries */);
int		gysk_topk_flow_errors(gysk_engine *e, int last_window, uint32_t n, gysk_flow_err_est *out, uint32_t *nout);
int		gysk_topk_flow_errors_global(gysk_engine *e, uint32_t n, gysk_flow_err_est *out, uint32_t *nout);
int		gysk_topk_flow_errors_5min(gysk_engine *e, uint32_t n, gysk_flow_err_est *out, uint32_t *nout, uint64_t *bound);
int		gysk_topk_flow_errors_global_5min(gysk_engine *e, uint32_t n, gysk_flow_err_est *out, uint32_t *nout, uint64_t *bound);

/* ---- distinct clients per window (GYSK_FLAG_CLIENT_LEVELS): how many clients a service has now ----
 * gysk_svc_summary.distinct_clients is an all-time estimate: its registers are never cleared, so it cannot show a new caller fleet, a
 * client pool that drained away, or a scan. The reference answers with the set of a listener's current client processes
 * (MTCP_LISTENER::cli_aggr_task_tbl_). These calls answer with HyperLogLog registers per window:
 *  - each service holds register sets at the fixed precision GYSK_HLL_WINDOW_P = 8 (256 one-byte registers), raised from the hash of
 *    the all-time registers (fmix64 of the flow key's two lookup2 words): standard error 1.04 / 16 = 6.5 % in the raw range, linear
 *    counting below 2.5 x 256 = 640 distinct clients;
 *  - a record raises the open set's register exactly when it raises the service's all-time registers: the connection events of every
 *    route (event32 CONNECT / ACCEPT / CLOSE, TCP24, raw connection records, NOTIFY_TCP_CONN) and NOTIFY_ACTIVE_CONN_STATS records.
 *    Response samples, API_TRAN and trace events never count;
 *  - at each gysk_flush the closing open set is max-merged into ring slot (tsec / 30) % 10 (a slot holding an older epoch is replaced),
 *    the 300-s level becomes the registerwise maximum of the live ring slots, and the open set becomes the last one while a cleared set
 *    opens. The level covers exactly the windows of the other 300-s levels (p95_5min_resp_ms, gysk_query_flows_5min);
 *  - an evicted service's sets are cleared with its slot; gysk_grow keeps them.
 * Every read answers as of the last gysk_flush. The estimates are gysk_hll_estimate(regs, GYSK_HLL_WINDOW_P) of the exported registers.
 * Cost: (2 + 10 + 1) x 256 = 3 328 device bytes per service slot (gysk_slot_bytes: 14 904 -> 18 232 at the defaults; 3.3 GB at 1 M
 * services, 0.87 GB at 2^18), and 512 B per logical service in the merge arena. Measured on one H100 80GB HBM3 at 700 W, bench workload
 * (100 M-event batches): the TCP drain pass +0.4 to 0.6 ms per batch, gysk_flush +0.06 ms at 2^17 and +0.55 ms at 2^20 service slots,
 * gysk_merge_prepare +0.09 ms for 100 000 logical services (DESIGN.md section 7).
 * gysk_query_svc_clients: one row per id; found = 0 and zero estimates for an unknown id.
 * gysk_query_clients_window: the rows of gysk_query_window_hosts' services, in its order, with its host filter, GYSK_WINDOW_ACTIVE_ONLY
 *   and count / capacity rules; each row byte-equal to gysk_query_svc_clients' row of its id.
 * gysk_export_hll_window: the 256 registers of GYSK_CLIENTS_LAST or GYSK_CLIENTS_5MIN, with the contract of gysk_export_hll
 *   (GYSK_ERR_NOENT for an unknown id).
 * Across ranks (the flag on every rank): gysk_merge_prepare folds each logical service's members' last and 300-s sets by registerwise
 *   maximum into the u8 MAX region after the all-time registers, the HLL of the union of their clients (512 bytes per logical service).
 *   gysk_query_logical_clients (found = 0 for an id outside the map) and gysk_export_logical_hll_window read them; both are
 *   GYSK_ERR_INVAL before a finished merge. Each rank's sets are relative to its own last flush: gysk_merge_flush_range shows whether
 *   the ranks closed the same window.
 * Every call is GYSK_ERR_NOTSUP without the flag. */
#define GYSK_CLIENTS_LAST		0	/* gysk_export_hll_window: the window the last gysk_flush closed */
#define GYSK_CLIENTS_5MIN		1	/* ... the rolling 300-s level */
typedef struct gysk_svc_clients
{
	uint64_t	glob_id;		/* the queried id (logical reads: the logical id) */
	int32_t		found;
	uint32_t	pad;
	double		last_5s;		/* distinct clients of the last closed window */
	double		last_5min;		/* distinct clients of the rolling 300-s level */
} gysk_svc_clients;
int		gysk_query_svc_clients(gysk_engine *e, const uint64_t *ids, uint32_t n, gysk_svc_clients *out);
int		gysk_query_clients_window(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_svc_clients *out, uint32_t *hosts, uint32_t cap,
				uint32_t *n);
int		gysk_export_hll_window(gysk_engine *e, uint64_t glob_id, int which, uint8_t regs[256]);
int		gysk_query_logical_clients(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_svc_clients *out);
int		gysk_export_logical_hll_window(gysk_engine *e, uint64_t logical_id, int which, uint8_t regs[256]);

/* ---- each service's heaviest clients (GYSK_FLAG_SVC_TOP_CLIENTS): who loads a listener ----
 * The reference answers "who is loading this listener" from a per-listener map of client processes and their bytes, cleared every
 * interval (connlistenmap_, written to activeconntbl). Here each service slot holds bounded summaries of K = GYSK_SVC_TOPC_K entries
 * {flow_key, kbytes, conns} and one bound delta:
 *  - what counts: exactly the records that feed the service's exact {count, kbytes} cell (nconns_5s / kbytes_5s): event32 CONNECT /
 *    ACCEPT / CLOSE_CLI / CLOSE_SER, TCP24, raw IPv4 / IPv6 connection records and NOTIFY_TCP_CONN (flow_key = cli_task_aggr_id_).
 *    Each adds conns += 1 and kbytes += bytes >> 10 to the pair (service, flow_key). Response samples, API_TRAN, trace events,
 *    NOTIFY_ACTIVE_CONN_STATS, process records, unknown ids and dropped events never count;
 *  - the rule is weighted Misra-Gries in its mergeable form (Agarwal et al., Mergeable Summaries, 2012). A merge of summaries, or of a
 *    summary with exact per-client sums: group the union by flow_key and sum kbytes and conns, dropping a group with 0 kbytes; c = the
 *    (K + 1)-th largest kbytes of the groups (0 with at most K groups); keep the groups with kbytes > c as kbytes - c with their conns;
 *    delta = the sum of the inputs' deltas + c. Entries are ordered by kbytes descending, then flow_key ascending; kbytes and conns
 *    saturate at 2^32 - 1. The result depends on neither record order nor route;
 *  - guarantees, for every client f of the service over the records the summary covers (est = 0 for an unlisted client):
 *    est(f) <= exact(f) <= est(f) + delta; sum(est) + (K + 1) x delta <= the service's kbytes over the same records; a service with at
 *    most K clients of positive kbytes lists them all exactly with delta = 0; a listed client's conns is at most its exact count;
 *  - after each device batch the open summary is merged with the batch's exact per-client sums. At gysk_flush the open summary is merged
 *    into ring slot (tsec / 30) % 10 (it replaces a slot holding an older epoch), the 300-s level becomes the merge of the live ring
 *    slots (the windows of p95_5min_resp_ms), and the open summary becomes the last one while a cleared one opens;
 *  - an evicted service's summaries are cleared with its slot; gysk_grow keeps them.
 * Cost: 13 summaries of 264 bytes per service slot (3 432 B; gysk_slot_bytes counts them), and a batch pair table of 32 bytes x
 * next_pow2(2 x max_batch) entries plus the piece lists of the long segments (about 260 MiB at the default max_batch = 2^22; 8 GiB at 2^27).
 * gysk_query_svc_top_clients: one row per id of the summary `which`; found = 0, n = 0 and zero entries for an unknown id. GYSK_TOPC_OPEN
 *   answers as of the events handed in so far, the other two as of the last gysk_flush.
 * gysk_query_top_clients_window: the rows of gysk_query_window_hosts' services, in its order, with its host filter,
 *   GYSK_WINDOW_ACTIVE_ONLY and count / capacity rules; each row byte-equal to gysk_query_svc_top_clients' row of its id.
 * Both are GYSK_ERR_NOTSUP without the flag and GYSK_ERR_INVAL for another `which`. K is fixed: gysk_config has no word for it.
 * Across ranks (the flag on every rank): gysk_merge_prepare and gysk_merge_finish build two summaries per logical service of
 *   gysk_set_logical_map, GYSK_TOPC_LAST from the members' last-window summaries and GYSK_TOPC_5MIN from their 300-s levels (the open
 *   window is never merged), each by the merge above as a sequential fold acc = merge(acc, s) from the empty summary: on each rank the
 *   members in map order (a member without a slot on the rank, being unmapped, evicted or never seen there, is skipped: merging with an
 *   empty summary is the identity), then the ranks' results in ascending rank order. The result is bit-exact at any launch shape. The
 *   guarantees above hold for every client over the records of every member summary on every rank, with the logical service's kbytes
 *   N_L = the sum of its members' (for GYSK_TOPC_LAST: gysk_query_logical's kbytes_5s); a client of members on several ranks is summed
 *   across them. Each rank's summaries are relative to its own last flush: gysk_merge_flush_range shows whether the ranks closed the same
 *   window.
 *   Cost: 528 bytes per logical service in each rank's slab (one all-gather; 52.8 MB at 100 000 logical services, 422 MB gathered at
 *   world 8) and 528 bytes of merged summaries. Measured on one H100 80GB HBM3 at 700 W, logical services of 16 members, world 1:
 *   gysk_merge_prepare +0.34 ms at 6 250 logical services and +2.80 ms at 62 500 (0.32 -> 0.67 ms, 2.42 -> 5.22 ms), gysk_merge_finish
 *   +0.02 / +0.20 ms; the all-gather of the larger slab across GPUs was not measured (DESIGN.md section 7).
 * gysk_query_logical_top_clients: one row per logical id of the merged summary `which` (glob_id = the logical id); found = 0, n = 0 and
 *   zero entries for an id outside the map.
 * gysk_query_logical_top_clients_all: every logical service's row, with the ids, order, GYSK_WINDOW_ACTIVE_ONLY set and count / capacity
 *   rules of gysk_query_logical_all; each row byte-equal to gysk_query_logical_top_clients' row of its id.
 * Both are GYSK_ERR_NOTSUP without the flag, and GYSK_ERR_INVAL for GYSK_TOPC_OPEN or another `which` and before a finished merge. */
#define GYSK_SVC_TOPC_K			16u
#define GYSK_TOPC_OPEN			0	/* the open window */
#define GYSK_TOPC_LAST			1	/* the window the last gysk_flush closed */
#define GYSK_TOPC_5MIN			2	/* the rolling 300-s level */
typedef struct gysk_topc_entry
{
	uint64_t	flow_key;		/* the client: the connection's flow key (NOTIFY_TCP_CONN: cli_task_aggr_id_) */
	uint32_t	kbytes;			/* the estimate est(f), at most the client's exact kbytes */
	uint32_t	conns;			/* records counted since the entry last entered the summary */
} gysk_topc_entry;
typedef struct gysk_svc_top_clients
{
	uint64_t	glob_id;		/* the queried id (logical reads: the logical id) */
	int32_t		found;
	uint32_t	n;			/* entries held, best first; entries[n ..] are zero */
	uint64_t	delta;			/* the bound: exact(f) <= est(f) + delta for every client */
	gysk_topc_entry	entries[GYSK_SVC_TOPC_K];
} gysk_svc_top_clients;
int		gysk_query_svc_top_clients(gysk_engine *e, const uint64_t *ids, uint32_t n, int which, gysk_svc_top_clients *out);
int		gysk_query_top_clients_window(gysk_engine *e, int32_t host_idx, uint32_t flags, int which, gysk_svc_top_clients *out, uint32_t *hosts,
				uint32_t cap, uint32_t *n);
int		gysk_query_logical_top_clients(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, int which, gysk_svc_top_clients *out);
int		gysk_query_logical_top_clients_all(gysk_engine *e, uint32_t flags, int which, gysk_svc_top_clients *out, uint32_t cap, uint32_t *n);

/* ---- request traces (gysk_config.max_trace_svcs != 0): the trace view per service and 5-s window ----
 * madhava writes every API_TRAN as one row of tracereqtbl (handle_trace_requests, server/gy_mconnhdlr.cc:5883-6060) and the trace view
 * aggregates those rows per service and time bucket in SQL (tracereq_aggr_info, common/gy_json_field_maps.h:2628-2664). Here each traced
 * service holds a trace row on the device, and each window of it carries that aggregate's columns, so one row per service and window
 * reaches the database instead of one per request:
 *  - a service takes a row with its first GYSK_EV_TRACE event, from the rows an evicted service freed first, else the next fresh one.
 *    With every row taken, the events of services without one are dropped (gysk_trace_info's dropped, and gysk_stats.events_dropped).
 *    An evicted service's row is zeroed and freed; the same id seen again starts from empty windows;
 *  - a sample lands in the window open when it arrives, as every other sample; gysk_flush closes it into `last` and opens an empty one;
 *  - every sample counts in every counter. A response beyond the GYSK_EV_RESP validity rule (1 000 000 msec) stays out of the digest,
 *    as it stays out of the service's;
 *  - the digest is a merging t-digest at compression 100, the public.tdigest(response, 100) of the trace view's p99respus: its
 *    pgtext export is stored as it is, and Postgres merges a range of windows with public.tdigest(col). p99_resp_us is its 0.99
 *    quantile (the rule of gysk_tdigest_quantile), NaN while it is empty. */
typedef struct gysk_trace_window
{
	uint64_t	nreq;			/* count(*) */
	uint64_t	nerr;			/* errorcode != 0 */
	uint64_t	nconns;			/* reqnum = 0 */
	uint64_t	sum_resp_us;		/* avgrespus = sum_resp_us / nreq */
	uint64_t	max_resp_us;		/* maxrespus */
	uint64_t	bytes_in, bytes_out;	/* sum(bytesin), sum(bytesout) */
	uint64_t	max_bytes_in, max_bytes_out;
	uint64_t	resp_buckets[8];	/* resplt300us, resplt1ms, resplt10ms, resplt30ms, resplt100ms, resplt300ms, resplt1sec, respgt1sec:
						   [0, 300), [300, 1000), [1000, 10000), [10000, 30000), [30000, 100000), [100000, 300000),
						   [300000, 1000000), [1000000, inf) usec */
	uint64_t	td_count;		/* samples in the digest (nreq less those beyond the validity rule) */
	double		p99_resp_us;		/* p99respus; NaN when the digest is empty */
} gysk_trace_window;			/* 152 bytes */

typedef struct gysk_trace_row
{
	uint64_t		glob_id;
	int32_t			found;		/* 0: unknown id, or a service without a trace row (the windows are then zero) */
	uint32_t		host_idx;	/* host of the event that created the service's slot */
	gysk_trace_window	cur, last;	/* the window being filled and the last closed one */
} gysk_trace_row;			/* 320 bytes */

/* the rows of n ids. GYSK_ERR_NOTSUP without trace rows */
int		gysk_query_traces(gysk_engine *e, const uint64_t *glob_ids, uint32_t n, gysk_trace_row *out);
/* one row per service holding a trace row, in ascending glob_id; each equals the gysk_query_traces row of its id. host_idx < 0 reads
 * every host; GYSK_WINDOW_ACTIVE_ONLY keeps the rows whose last window holds requests. Count and capacity as gysk_query_window */
int		gysk_query_trace_window(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_trace_row *out, uint32_t cap, uint32_t *n);
/* the digest of a service's open (last_window = 0) or last closed window: the contract of gysk_export_tdigest (min / max: the extremes
 * of the digested samples, +inf / -inf while empty). GYSK_ERR_NOENT for an id without a trace row */
int		gysk_export_trace_tdigest(gysk_engine *e, uint64_t glob_id, int last_window, double *means, uint64_t *weights, uint32_t cap,
				uint32_t *n, double *min_val, double *max_val);
/* the same digest as Postgres tdigest text (gysk_tdigest_to_pgtext at compression 100, no recompress); the string length or GYSK_ERR_* */
int		gysk_export_trace_tdigest_pgtext(gysk_engine *e, uint64_t glob_id, int last_window, char *buf, uint32_t cap);
/* rows in use (handed out less the freed ones) and the trace events dropped so far for want of a row */
int		gysk_trace_info(gysk_engine *e, uint32_t *rows_in_use, uint64_t *dropped);

/* ---- row a15b: the per-process -> per-aggregate-process group-by in front of partha_aggr_task_state ----
 * One record per process and 5-s tick, holding what TASK_HANDLER's walk has at hand when it folds the process into
 * aggrnotmap.try_emplace(aggr_task_id) (common/gy_task_handler.cc:752-880). */
typedef struct gysk_proc_sample
{
	uint64_t	aggr_task_id;		/* ptask->aggr_task_id_ */
	int32_t		pid;			/* ptask->task_pid */
	float		cpu_pct;		/* avg_cpu_pct / npct: this tick's cpu % averaged with the ticks the server missed (:826-839) */
	uint32_t	rss_mb;
	uint32_t	cpu_delay_msec, vm_delay_msec, blkio_delay_msec;	/* last_*_delay_nsec / GY_NSEC_PER_MSEC (:858-860) */
	uint32_t	tcp_kbytes, tcp_conns;	/* last_sent_tcp_kbytes_ / _conns_: non-zero in the 15-s network ticks only (:791-813) */
	uint8_t		state;			/* pext->issue_hist_[0].state (OBJ_STATE_E) */
	uint8_t		issue;			/* pext->issue_hist_[0].issue */
	uint8_t		issue_bit_hist, severe_issue_bit_hist;
	uint8_t		is_issue;
	uint8_t		pad[3];
	char		comm[16];		/* ptask->task_comm */
} gysk_proc_sample;
/* Folds the samples by aggr_task_id IN ARRAY ORDER with the reference's statement order (the float cpu sum sees the same sequence of
 * additions) and writes one AGGR_TASK_STATE_NOTIFY record (72 bytes, common/gy_comm_proto.h:2114-2170, no issue string) per group,
 * groups in order of first appearance: the body of a NOTIFY_AGGR_TASK_STATE message, ready for gysk_ingest(). *ngroups = number of
 * groups found; at most `cap` records are written. n <= gysk_config.max_batch. */
int		gysk_task_groupby(gysk_engine *e, const gysk_proc_sample *samples, uint32_t n, void *out_records, uint32_t cap, uint32_t *ngroups);

/* ---- pure helpers (host side, no engine): the reference's percentile rule and the sketch estimators ---- */
int		gysk_hist_nbuckets(int cls);
int		gysk_hist_bucket(int cls, int64_t value);	/* RESP_TIME_HASH::get_bucket_from_data & siblings */
int		gysk_hist_percentiles(int cls, int t_is_int, const gysk_hist_serial *stats, uint64_t total_count,
				const float *pcts, uint32_t npct, int64_t *out);
double		gysk_hll_estimate(const uint8_t *regs, uint32_t p);
/* TCP_LISTENER::get_curr_state (common/gy_socket_stat.cc:2020-2875): shifts / sets *high_resp_bit_hist, writes GYSK_STATE_* / GYSK_ISSUE_* */
int		gysk_classify_listener(const gysk_listener_state_in *in, uint8_t *high_resp_bit_hist, uint8_t *state, uint8_t *issue);
/* per-service summaries -> LISTENER_STATE_NOTIFY records (common/gy_comm_proto.h:2183-2254), the body of one
 * NOTIFY_LISTENER_STATE message (<= 512 records, 88 bytes each) that MTCP_LISTENER::set_state / partha_listener_state consume
 * (server/gy_mconnhdlr.cc:11175-11251). Entries with found == 0 are skipped. No engine needed. */
int		gysk_encode_listener_state(const gysk_svc_summary *sums, uint32_t n, void *buf, uint32_t cap, uint32_t *nrecs, uint32_t *nbytes);
/* a digest in the text form of the Postgres `tdigest` type the reference stores and queries (public.tdigest(expr, 100) /
 * tdigest_percentile, common/gy_query_common.cc:1805-1858): "flags 1 count N compression C centroids K (mean, count) ...".
 * Both return the string length, or a negative GYSK_ERR_* */
int		gysk_tdigest_to_pgtext(const double *means, const uint64_t *weights, uint32_t n, uint32_t compression, char *buf, uint32_t cap);
int		gysk_export_tdigest_pgtext(gysk_engine *e, uint64_t glob_id, char *buf, uint32_t cap);
double		gysk_tdigest_quantile(const double *means, const uint64_t *weights, uint32_t n, double min_val, double max_val, double q);
uint32_t	gysk_uint64_hash(uint64_t key);		/* get_uint64_hash, common/gy_common_inc.h:1120 */

/* ---- multi-GPU merge (SURVEY.md §8e) ---- */
/* Which services form a logical service (the reference's svc-mesh cluster id). The same list on every rank; dense logical indices
 * follow first appearance. Ids need not be registered (or owned by this rank): the map keeps every pair and looks the slots up at
 * every gysk_merge_prepare / gysk_merge_global. */
int		gysk_set_logical_map(gysk_engine *e, const uint64_t *glob_ids, const uint64_t *logical_ids, uint32_t n);
int		gysk_merge_prepare(gysk_engine *e);		/* fold per-service sketches into per-logical-service arrays; asynchronous on
							   gysk_stream(e): enqueue the collectives on that stream, or gysk_sync() first */
int		gysk_merge_buffers(gysk_engine *e, gysk_buffer_desc *out, uint32_t cap, uint32_t *n);
int		gysk_merge_tdigest_slab(gysk_engine *e, void **dptr, uint64_t *nbytes);	/* fixed slab to all-gather */
int		gysk_merge_finish(gysk_engine *e, const void *d_gathered_slabs, uint32_t world);
/* The same step with NCCL inside the library (a C++ madhava has no torch.distributed): fold, then ONE grouped NCCL launch — an
 * all-reduce per reduction kind (u64 SUM, i64 MAX, u8 MAX) and the all-gather of the t-digest slabs — then the merge-compress,
 * all enqueued on the engine's stream. libnccl.so.2 is loaded on first use (dlopen; GYSK_ERR_NOTSUP when absent).
 * comm: an ncclComm_t created by the caller over the engines' devices (ncclCommInitAll / ncclCommInitRank), or NULL to use the one
 * gysk_nccl_comm_init() made: rank 0 calls gysk_nccl_unique_id(), ships the 128 bytes to its peers, every rank calls
 * gysk_nccl_comm_init(engine, uid, nranks, rank). */
#define GYSK_NCCL_UNIQUE_ID_BYTES	128
int		gysk_nccl_unique_id(uint8_t out[GYSK_NCCL_UNIQUE_ID_BYTES]);
int		gysk_nccl_comm_init(gysk_engine *e, const uint8_t uid[GYSK_NCCL_UNIQUE_ID_BYTES], uint32_t nranks, uint32_t rank);
int		gysk_merge_global(gysk_engine *e, void *nccl_comm);
/* One gysk_svc_summary per logical id from the last finished merge: glob_id = the logical id, found = 0 for an id not in the map.
 * The merge always folds the last closed window, the all-time histogram, the connection counters, the HLL registers and the
 * t-digest. curr_state, curr_issue, issue_bit_hist and high_resp_bit_hist are always 0: a logical service is not classified (its
 * members' states are counted by gysk_query_logical_states with GYSK_FLAG_MERGE_STATES).
 * Without GYSK_FLAG_MERGE_LEVELS nqrys_5min, nqrys_5day, nconns_active, active_kbytes, max_rtt_msec, cli_errors and ser_errors
 * are 0, and p95_5min_resp_ms, p99_5min_resp_ms and p95_5day_resp_ms -1 (the percentiles of an empty histogram).
 * With it those fields are the member services' own, merged exactly at any GPU count:
 *   nqrys_5min / nqrys_5day and the three level percentiles: the live ring slots of every member (the lvl its gysk_query_svcs row
 *     shows) summed cell by cell over members and ranks, through the GY_HISTOGRAM percentile rule;
 *   nconns_active, active_kbytes, cli_errors, ser_errors: sums over the members' last closed window, truncated to 32 bits;
 *   max_rtt_msec: the largest of the members' values.
 * A rank's levels are relative to its own last gysk_flush: see gysk_merge_flush_range. */
int		gysk_query_logical(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_svc_summary *out);
/* The merged histogram of one logical service from the last finished merge, with the contract of gysk_export_hist (HIST_SERIAL
 * byte-compatible, for GY_HISTOGRAM::update_from_serialized): which = GYSK_HIST_RESP_LAST, _RESP_ALL, _RESP_5MIN or _RESP_5DAY.
 * GYSK_ERR_NOENT for an id the map does not have, GYSK_ERR_NOTSUP for the two levels without GYSK_FLAG_MERGE_LEVELS,
 * GYSK_ERR_INVAL before a finished merge or for another `which`. */
int		gysk_export_logical_hist(gysk_engine *e, uint64_t logical_id, int which, gysk_hist_serial out[GYSK_HIST_MAX_BUCKETS],
				uint64_t *total_count, int64_t *max_val);
/* The earliest and latest tsec of the ranks' last gysk_flush, as all-reduced by the last finished merge (GYSK_FLAG_MERGE_LEVELS,
 * GYSK_FLAG_FLOW_LEVEL, GYSK_FLAG_FLOW_QUERY_LEVEL or GYSK_FLAG_MERGE_TRACES; GYSK_ERR_NOTSUP without all four, GYSK_ERR_INVAL before a
 * finished merge). Each rank's
 * level slots and last trace window are relative to its own last flush, so *min_tsec != *max_tsec means the ranks had closed different
 * windows and the merged levels or trace windows mix them. That is not an
 * error: the collectives cannot fail on one rank alone, so the caller decides what to do with such an answer. */
int		gysk_merge_flush_range(gysk_engine *e, uint32_t *min_tsec, uint32_t *max_tsec);

/* ---- reads over every merged logical service (SURVEY.md §8e, §8f): the global dashboard and the global digests ----
 * Each needs a finished merge (GYSK_ERR_INVAL before one, as gysk_query_logical) and reads only what the merge left on the device,
 * so every rank returns the same answer. */
/* One gysk_svc_summary per logical service of the map, in ascending logical id; each row equals the gysk_query_logical row of its id,
 * byte for byte. GYSK_WINDOW_ACTIVE_ONLY keeps the logical services whose merged last window holds response samples or connection
 * events. Count and capacity as gysk_query_window: *n = number of matching rows; at most cap rows are written (out may be NULL when cap
 * is 0, which only counts). */
int		gysk_query_logical_all(gysk_engine *e, uint32_t flags, gysk_svc_summary *out, uint32_t cap, uint32_t *n);
/* The n <= 64 best logical services of the last finished merge, best first: the global half of the per-host listener rankings
 * (SURVEY.md §8f row 3). Scores as gysk_topn_svcs scores a service, from the merged arrays: GYSK_TOPN_QPS the last window's response
 * samples, GYSK_TOPN_CONNS / GYSK_TOPN_NET its connection events / kbytes (nconns_5s / kbytes_5s of the row), GYSK_TOPN_ACTIVE the
 * merged active connections (nconns_active; GYSK_FLAG_MERGE_LEVELS, GYSK_ERR_NOTSUP without it). GYSK_TOPN_ISSUE ranks by the member
 * listeners in BAD / SEVERE / DOWN (nsvc_issue of gysk_query_logical_states) with GYSK_FLAG_MERGE_STATES, and is GYSK_ERR_INVAL without
 * it. Equal scores rank the later logical service of the map (first appearance) first. As in
 * gysk_topn_svcs, entries with a zero score are left out, so *nout may be below n. glob_id = the logical id, host_idx = 0.
 * GYSK_ERR_NOSPC for a map of more logical services than max(max_batch, max(max_svcs, max_tasks) + 1). */
int		gysk_topn_logical(gysk_engine *e, int metric, uint32_t n, gysk_topn_entry *out, uint32_t *nout);
/* The merged t-digest, its Postgres text (recompressed to compression 100), its quantiles and the merged HLL registers of one
 * logical service (SURVEY.md §8e items 4 and 5, §8f row 4): the contracts of gysk_export_tdigest, gysk_export_tdigest_pgtext,
 * gysk_query_quantiles and gysk_export_hll, with GYSK_ERR_NOENT for an id the map does not have. The digest is the one the row's
 * td_p50_us / td_p95_us / td_p99_us come from; the registers give its distinct_clients. */
int		gysk_export_logical_tdigest(gysk_engine *e, uint64_t logical_id, double *means, uint64_t *weights, uint32_t cap, uint32_t *n,
				double *min_val, double *max_val);
int		gysk_export_logical_tdigest_pgtext(gysk_engine *e, uint64_t logical_id, char *buf, uint32_t cap);
int		gysk_query_logical_quantiles(gysk_engine *e, uint64_t logical_id, const double *qs, uint32_t nq, double *out);
int		gysk_export_logical_hll(gysk_engine *e, uint64_t logical_id, uint8_t *regs /* 1 << hll_p bytes */);

/* ---- listener states of logical services (GYSK_FLAG_MERGE_STATES): how many instances of a service are in trouble ----
 * Each member service that holds a slot on a rank adds LISTEN_SUMM_STATS::update (server/gy_msocket.h:853-864) of the
 * LISTENER_STATE_NOTIFY record gysk_encode_listener_state writes from its own gysk_query_svcs row: nstates[curr_state] += 1,
 * tot_qps += nqrys_5s / 5, tot_act_conn += nconns_active, tot_kb_inbound += kbytes_5s, tot_kb_outbound += 0, tot_ser_errors += ser_errors,
 * nlisteners += 1, nactive += !!nqrys_5s; summed over members and ranks with LISTEN_SUMM_STATS<int>'s wrap-around, so exact at any GPU
 * count. The states are those of each member's last gysk_flush on its rank. A logical service itself is not classified. */
typedef struct gysk_logical_state
{
	uint64_t		logical_id;
	int32_t			found;		/* 0: not in the map (summ all zero) */
	uint32_t		nsvc_issue;	/* summ.nstates[BAD] + [SEVERE] + [DOWN], as MS_CLUSTER_STATE counts it */
	gysk_host_summary	summ;		/* LISTEN_SUMM_STATS over the member listeners, every rank */
} gysk_logical_state;			/* 80 bytes */
/* by id, from the last finished merge. GYSK_ERR_NOTSUP without GYSK_FLAG_MERGE_STATES, GYSK_ERR_INVAL before a finished merge */
int		gysk_query_logical_states(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_logical_state *out);
/* one row per logical service: the ids, order, GYSK_WINDOW_ACTIVE_ONLY set and count / capacity rules of gysk_query_logical_all */
int		gysk_query_logical_states_all(gysk_engine *e, uint32_t flags, gysk_logical_state *out, uint32_t cap, uint32_t *n);

/* ---- request traces of logical services (GYSK_FLAG_MERGE_TRACES): the trace view of each logical service's last window ----
 * Each member service that holds a slot and a trace row on a rank adds the last closed window of its row (the `last` of its
 * gysk_query_traces row); members without a row add nothing. Over members and ranks:
 *   nreq, nerr, nconns, sum_resp_us, bytes_in, bytes_out, resp_buckets[8] and td_count are sums;
 *   max_resp_us, max_bytes_in and max_bytes_out are maxima;
 *   the digest is the members' window digests merged in map order on each rank, then the ranks' in ascending rank, at compression 100;
 *   p99_resp_us is its 0.99 quantile (the rule of gysk_tdigest_quantile), NaN when it is empty.
 * Integer fields are exact at any GPU count. Each rank folds its own last closed window: gysk_merge_flush_range tells whether every rank
 * had closed the same one. The layout of the merge buffers depends only on the flags and the logical map, not on max_trace_svcs. */
typedef struct gysk_logical_trace
{
	uint64_t		logical_id;
	int32_t			found;		/* 1 for a mapped logical id, as gysk_query_logical_states; 0: not in the map (all zero) */
	uint32_t		ntraced;	/* member services holding a trace row, summed over the ranks */
	gysk_trace_window	last;		/* the members' last closed windows merged */
} gysk_logical_trace;			/* 168 bytes */
/* by id, from the last finished merge. GYSK_ERR_NOTSUP without GYSK_FLAG_MERGE_TRACES, GYSK_ERR_INVAL before a finished merge */
int		gysk_query_logical_traces(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_logical_trace *out);
/* one row per logical service in the order of gysk_query_logical_all; GYSK_WINDOW_ACTIVE_ONLY keeps the rows whose merged window has
 * nreq != 0. Count and capacity as gysk_query_logical_all */
int		gysk_query_logical_traces_all(gysk_engine *e, uint32_t flags, gysk_logical_trace *out, uint32_t cap, uint32_t *n);
/* the merged trace digest of one logical service: the contract of gysk_export_logical_tdigest (min / max: the extremes of the digested
 * samples, +inf / -inf while empty; GYSK_ERR_NOENT for an id the map does not have) */
int		gysk_export_logical_trace_tdigest(gysk_engine *e, uint64_t logical_id, double *means, uint64_t *weights, uint32_t cap,
				uint32_t *n, double *min_val, double *max_val);
/* the same digest as Postgres tdigest text (gysk_tdigest_to_pgtext at compression 100, no recompress): what a per-logical-service
 * trace table stores for public.tdigest(col) to merge over a time range. The string length or GYSK_ERR_* */
int		gysk_export_logical_trace_tdigest_pgtext(gysk_engine *e, uint64_t logical_id, char *buf, uint32_t cap);

/* ---- host clusters (GYSK_FLAG_MERGE_CLUSTERS): MS_CLUSTER_STATE across every rank ----
 * Which host belongs to which cluster: host_idxs[i] -> cluster_ids[i] (the caller hashes PARTHA_INFO::cluster_name_ into the id). The same
 * list on every rank; dense cluster indices follow first appearance. A host that is not in the list belongs to no cluster; a host listed
 * twice is GYSK_ERR_INVAL, as is a host_idx >= 2^24. GYSK_ERR_NOTSUP without the flag. The call may come before or after
 * gysk_set_logical_map: either one lays out the merge arena again (the last merge's results are gone), and each keeps the other's map. A
 * merge of clusters alone needs no gysk_set_logical_map: this call also sets up an empty logical map when the engine has none. */
int		gysk_set_cluster_map(gysk_engine *e, const uint32_t *host_idxs, const uint64_t *cluster_ids, uint32_t n);
/* One cluster's row. st is the service half of CLUSTER_STATE_ONE::update_from_state (server/gy_mconnhdlr.cc:16032-16050), summed over
 * every host of the cluster on every rank; each uint32 wraps, as the reference's counters do. For each host with at least one live
 * service (a row of gysk_query_window_hosts(-1, 0)), with nlisten / nlisten_issue its gysk_query_host_listen row:
 *   nhosts += 1, nsvc += nlisten, nsvc_issue += nlisten_issue, nsvcissue_hosts += !!nlisten_issue,
 * and with LISTEN_SUMM_STATS<int> over the host's gysk_query_window_hosts(-1, 0) rows (each the record gysk_encode_listener_state writes,
 * LISTEN_SUMM_STATS::update, server/gy_msocket.h:853-864):
 *   total_qps += tot_qps, svc_net_mb += (tot_kb_inbound + tot_kb_outbound) / 1024, divided per host in int32 before the cluster sum (:16045).
 * nsvc_issue counts the services evaluated at the last gysk_flush with issue bit 0 set there, the HOST_STATE_NOTIFY::nlisten_issue_ the
 * reference sums; gysk_query_cluster_state counts the host summaries' BAD / SEVERE / DOWN listeners instead. The two differ by the services
 * that had no events in the window the last flush closed: such a service is not evaluated there, so it is no issue here, but its row
 * keeps the state of its last evaluation, which gysk_query_cluster_state counts when that is BAD or worse.
 * Left to the caller (HOST_STATE_NOTIFY): ntasks_issue, ntaskissue_hosts, ntasks, ncpu_issue, nmem_issue, and the hosts without listeners,
 * which the reference's nhosts also counts (gy_gysk_shim.h: cluster_state_one). The states are those of each rank's last gysk_flush. */
typedef struct gysk_cluster_row
{
	uint64_t		cluster_id;
	int32_t			found;		/* 0: not in the map (st all zero) */
	uint32_t		pad;
	gysk_cluster_state	st;
} gysk_cluster_row;			/* 48 bytes */
/* by id, from the last finished merge. GYSK_ERR_NOTSUP without GYSK_FLAG_MERGE_CLUSTERS, GYSK_ERR_INVAL before a finished merge */
int		gysk_query_cluster_states(gysk_engine *e, const uint64_t *cluster_ids, uint32_t n, gysk_cluster_row *out);
/* one row per cluster of the map in ascending cluster id; GYSK_WINDOW_ACTIVE_ONLY keeps the clusters with nsvc > 0. Count and capacity as
 * gysk_query_logical_all */
int		gysk_query_cluster_states_all(gysk_engine *e, uint32_t flags, gysk_cluster_row *out, uint32_t cap, uint32_t *n);

/* ---- services and processes ranked across every rank (GYSK_FLAG_MERGE_TOPN): madhava-wide top listeners and top processes ----
 * The multi-host rankings of web_curr_top_listeners (server/gy_mnodehandle.cc:2884-3074, the LISTEN_TOPN::is_comp_* comparators,
 * server/gy_msocket.h:745-795) and web_curr_top_aggr_procs (:5653-5677). gysk_merge_prepare ranks this rank's services by each of
 * GYSK_TOPN_QPS, _CONNS, _NET, _ISSUE and _ACTIVE, and its processes by each GYSK_TOPN_TASK_* metric, as gysk_topn_svcs(metric, -1, 64) /
 * gysk_topn_tasks(metric, 64) do (GYSK_TOPN_ACTIVE scores the nconns_active of the service's row), and keeps each list's 64 best with
 * their rows. gysk_merge_finish picks the 64 best of every rank's lists in the order score descending, then rank ascending, then the
 * rank's own order (a later slot first on equal scores): exact, since each of them is among its own rank's 64 best, and the same on
 * every rank. At world 1 the entries are those of gysk_topn_svcs / gysk_topn_tasks.
 * out: the n (1 .. 64) best, best first, entries with a zero score left out, so *nout may be below n. host_idx is the host that created
 * the slot, for MULTI_HOST_IDENT. rows (NULL: not wanted): each entry's gysk_query_svcs / gysk_query_tasks row on its owning rank at the
 * merge, byte for byte; a service row becomes LISTEN_TOPN::state_ through gysk_encode_listener_state.
 * GYSK_ERR_NOTSUP without the flag; GYSK_ERR_INVAL before a finished merge, for another metric or n.
 * Limits: each rank ranks its own last closed window, as the other merged reads do. The reference's madhava ranks only each partha's
 * 10 queued entries (MAX_LISTEN_TOPN), so it can miss a service its host ranks 11th; these calls rank every service. */
int		gysk_topn_global(gysk_engine *e, int metric, uint32_t n, gysk_topn_entry *out, gysk_svc_summary *rows, uint32_t *nout);
int		gysk_topn_global_tasks(gysk_engine *e, int metric, uint32_t n, gysk_topn_entry *out, gysk_task_summary *rows, uint32_t *nout);

int		gysk_query_flows_global(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_est *out);

/* per-kernel device timing (CUDA events on the launching stream around the ingest kernel and around the sort +
 * t-digest chain of every device batch). read() synchronises, returns the sums since the last read and resets. */
int		gysk_profile_enable(gysk_engine *e, int on);
int		gysk_profile_read(gysk_engine *e, double *ms_ingest, double *ms_tdigest, uint64_t *nbatches);

/* CUDA stream the engine launches on (cudaStream_t as void*), for callers timing with events */
void *		gysk_stream(gysk_engine *e);

#ifdef __cplusplus
}
#endif

#endif /* GYSKETCH_H */
