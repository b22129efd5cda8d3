// TEST INFRASTRUCTURE ONLY (see oracle/README.md). Never linked into the product.
//
// C-ABI wrapper around the REFERENCE's own wire and eBPF record types, compiled from where they lie under the reference
// tree: oracle/Makefile generates oracle/_ref/gy_wire_trim.h from the struct blocks of common/gy_comm_proto.h (located by
// name) and the few definitions they use; common/gy_ebpf_kernel.h and common/gy_proto_common.h (API_TRAN) are included as
// they are. Nothing from the reference is copied into the repository; oracle/_ref/ is git-ignored.
//
// Exports
//   - a layout table: sizeof / alignof of every record type, and the offset and size of every field that the library's
//     decoders, gyeeta_b200/wire.py or the shim touch (tests/test_wire_layout_host.py holds gysk_wire.h and wire.py to it);
//   - builders: records written through the reference's own types, fields set by name, trailing strings and padding by the
//     type's own set_padding_len() / get_elem_size(), whole messages by COMM_HEADER's own constructor
//     (tests/golden/make_wire_golden.py).

#include "gy_ebpf_kernel.h"		// before gy_proto_common.h: API_TRAN's comm_ takes TASK_COMM_LEN from it
#include "gy_common_inc.h"
#include "gy_proto_common.h"
#include "gy_wire_trim.h"		// generated into oracle/_ref by the Makefile

#include <cstddef>
#include <cstdint>
#include <cstring>
#include <new>
#include <type_traits>

using namespace gyeeta;
using namespace gyeeta::comm;

namespace {

// GY_IP_ADDR keeps its members protected: a derived view names them for offsetof
struct IP_ADDR_VIEW : GY_IP_ADDR
{
	static constexpr uint32_t ip128() { return offsetof(IP_ADDR_VIEW, ip128_be_); }
	static constexpr uint32_t ip32() { return offsetof(IP_ADDR_VIEW, ip32_be_); }
	static constexpr uint32_t aftype() { return offsetof(IP_ADDR_VIEW, aftype_); }
	static constexpr uint32_t ipflags() { return offsetof(IP_ADDR_VIEW, ipflags_); }
};

struct StructRow { const char *name; uint32_t size, align; };
struct FieldRow { const char *strct, *field; uint32_t off, size; };

#define S(T)		{ #T, (uint32_t)sizeof(T), (uint32_t)alignof(T) }
#define F(T, M)		{ #T, #M, (uint32_t)offsetof(T, M), (uint32_t)sizeof(((T *)nullptr)->M) }

const StructRow structs[] = {
	S(COMM_HEADER),
	S(EVENT_NOTIFY),
	S(GY_IP_ADDR),
	S(IP_PORT),
	S(TCP_CONN_NOTIFY),
	S(AGGR_TASK_STATE_NOTIFY),
	S(LISTENER_STATE_NOTIFY),
	S(HOST_STATE_NOTIFY),
	S(ACTIVE_CONN_STATS),
	S(LISTENER_DAY_STATS),
	S(AGGR_TASK_HIST_STATS),
	S(API_TRAN),
	S(tcp_ipv4_event_t),
	S(tcp_ipv6_event_t),
	S(tcp_ipv4_resp_event_t),
	S(tcp_ipv6_resp_event_t),
};

const FieldRow fields[] = {
	F(COMM_HEADER, magic_),
	F(COMM_HEADER, total_sz_),
	F(COMM_HEADER, data_type_),
	F(COMM_HEADER, padding_sz_),

	F(EVENT_NOTIFY, subtype_),
	F(EVENT_NOTIFY, nevents_),

	{ "GY_IP_ADDR", "ip128_be_", IP_ADDR_VIEW::ip128(), 16 },
	{ "GY_IP_ADDR", "ip32_be_", IP_ADDR_VIEW::ip32(), 4 },
	{ "GY_IP_ADDR", "aftype_", IP_ADDR_VIEW::aftype(), 2 },
	{ "GY_IP_ADDR", "ipflags_", IP_ADDR_VIEW::ipflags(), 2 },

	F(IP_PORT, ipaddr_),
	F(IP_PORT, port_),

	F(TCP_CONN_NOTIFY, cli_),
	F(TCP_CONN_NOTIFY, ser_),
	F(TCP_CONN_NOTIFY, nat_cli_),
	F(TCP_CONN_NOTIFY, nat_ser_),
	F(TCP_CONN_NOTIFY, tusec_start_),
	F(TCP_CONN_NOTIFY, tusec_close_),
	F(TCP_CONN_NOTIFY, cli_task_aggr_id_),
	F(TCP_CONN_NOTIFY, cli_related_listen_id_),
	F(TCP_CONN_NOTIFY, cli_madhava_id_),
	F(TCP_CONN_NOTIFY, cli_ser_machine_id_),
	F(TCP_CONN_NOTIFY, ser_related_listen_id_),
	F(TCP_CONN_NOTIFY, ser_glob_id_),
	F(TCP_CONN_NOTIFY, ser_madhava_id_),
	F(TCP_CONN_NOTIFY, bytes_sent_),
	F(TCP_CONN_NOTIFY, bytes_rcvd_),
	F(TCP_CONN_NOTIFY, cli_pid_),
	F(TCP_CONN_NOTIFY, ser_pid_),
	F(TCP_CONN_NOTIFY, ser_conn_hash_),
	F(TCP_CONN_NOTIFY, ser_sock_inode_),
	F(TCP_CONN_NOTIFY, cli_comm_),
	F(TCP_CONN_NOTIFY, ser_comm_),
	F(TCP_CONN_NOTIFY, cli_cmdline_len_),
	F(TCP_CONN_NOTIFY, is_tcp_connect_event_),
	F(TCP_CONN_NOTIFY, is_tcp_accept_event_),
	F(TCP_CONN_NOTIFY, is_loopback_conn_),
	F(TCP_CONN_NOTIFY, is_pre_existing_),
	F(TCP_CONN_NOTIFY, notified_before_),
	F(TCP_CONN_NOTIFY, padding_len_),

	F(AGGR_TASK_STATE_NOTIFY, aggr_task_id_),
	F(AGGR_TASK_STATE_NOTIFY, onecomm_),
	F(AGGR_TASK_STATE_NOTIFY, pid_arr_),
	F(AGGR_TASK_STATE_NOTIFY, tcp_kbytes_),
	F(AGGR_TASK_STATE_NOTIFY, tcp_conns_),
	F(AGGR_TASK_STATE_NOTIFY, total_cpu_pct_),
	F(AGGR_TASK_STATE_NOTIFY, rss_mb_),
	F(AGGR_TASK_STATE_NOTIFY, cpu_delay_msec_),
	F(AGGR_TASK_STATE_NOTIFY, vm_delay_msec_),
	F(AGGR_TASK_STATE_NOTIFY, blkio_delay_msec_),
	F(AGGR_TASK_STATE_NOTIFY, ntasks_total_),
	F(AGGR_TASK_STATE_NOTIFY, ntasks_issue_),
	F(AGGR_TASK_STATE_NOTIFY, curr_state_),
	F(AGGR_TASK_STATE_NOTIFY, curr_issue_),
	F(AGGR_TASK_STATE_NOTIFY, issue_bit_hist_),
	F(AGGR_TASK_STATE_NOTIFY, severe_issue_bit_hist_),
	F(AGGR_TASK_STATE_NOTIFY, issue_string_len_),
	F(AGGR_TASK_STATE_NOTIFY, padding_len_),

	F(LISTENER_STATE_NOTIFY, glob_id_),
	F(LISTENER_STATE_NOTIFY, nqrys_5s_),
	F(LISTENER_STATE_NOTIFY, total_resp_5sec_),
	F(LISTENER_STATE_NOTIFY, nconns_),
	F(LISTENER_STATE_NOTIFY, nconns_active_),
	F(LISTENER_STATE_NOTIFY, ntasks_),
	F(LISTENER_STATE_NOTIFY, p95_5s_resp_ms_),
	F(LISTENER_STATE_NOTIFY, p95_5min_resp_ms_),
	F(LISTENER_STATE_NOTIFY, curr_kbytes_inbound_),
	F(LISTENER_STATE_NOTIFY, curr_kbytes_outbound_),
	F(LISTENER_STATE_NOTIFY, ser_errors_),
	F(LISTENER_STATE_NOTIFY, cli_errors_),
	F(LISTENER_STATE_NOTIFY, tasks_delay_usec_),
	F(LISTENER_STATE_NOTIFY, tasks_cpudelay_usec_),
	F(LISTENER_STATE_NOTIFY, tasks_blkiodelay_usec_),
	F(LISTENER_STATE_NOTIFY, tasks_user_cpu_),
	F(LISTENER_STATE_NOTIFY, tasks_sys_cpu_),
	F(LISTENER_STATE_NOTIFY, tasks_rss_mb_),
	F(LISTENER_STATE_NOTIFY, ntasks_issue_),
	F(LISTENER_STATE_NOTIFY, is_http_svc_),
	F(LISTENER_STATE_NOTIFY, curr_state_),
	F(LISTENER_STATE_NOTIFY, curr_issue_),
	F(LISTENER_STATE_NOTIFY, issue_bit_hist_),
	F(LISTENER_STATE_NOTIFY, high_resp_bit_hist_),
	F(LISTENER_STATE_NOTIFY, last_issue_subsrc_),
	F(LISTENER_STATE_NOTIFY, query_flags_),
	F(LISTENER_STATE_NOTIFY, issue_string_len_),
	F(LISTENER_STATE_NOTIFY, padding_len_),

	F(HOST_STATE_NOTIFY, curr_time_usec_),
	F(HOST_STATE_NOTIFY, ntasks_issue_),
	F(HOST_STATE_NOTIFY, ntasks_severe_),
	F(HOST_STATE_NOTIFY, ntasks_),
	F(HOST_STATE_NOTIFY, nlisten_issue_),
	F(HOST_STATE_NOTIFY, nlisten_severe_),
	F(HOST_STATE_NOTIFY, nlisten_),
	F(HOST_STATE_NOTIFY, curr_state_),
	F(HOST_STATE_NOTIFY, issue_bit_hist_),
	F(HOST_STATE_NOTIFY, cpu_issue_),
	F(HOST_STATE_NOTIFY, mem_issue_),
	F(HOST_STATE_NOTIFY, severe_cpu_issue_),
	F(HOST_STATE_NOTIFY, severe_mem_issue_),
	F(HOST_STATE_NOTIFY, total_cpu_delayms_),
	F(HOST_STATE_NOTIFY, total_vm_delayms_),
	F(HOST_STATE_NOTIFY, total_io_delayms_),

	F(ACTIVE_CONN_STATS, listener_glob_id_),
	F(ACTIVE_CONN_STATS, cli_aggr_task_id_),
	F(ACTIVE_CONN_STATS, ser_comm_),
	F(ACTIVE_CONN_STATS, cli_comm_),
	F(ACTIVE_CONN_STATS, remote_machine_id_),
	F(ACTIVE_CONN_STATS, remote_madhava_id_),
	F(ACTIVE_CONN_STATS, bytes_sent_),
	F(ACTIVE_CONN_STATS, bytes_received_),
	F(ACTIVE_CONN_STATS, cli_delay_msec_),
	F(ACTIVE_CONN_STATS, ser_delay_msec_),
	F(ACTIVE_CONN_STATS, max_rtt_msec_),
	F(ACTIVE_CONN_STATS, active_conns_),

	F(LISTENER_DAY_STATS, glob_id_),
	F(LISTENER_DAY_STATS, tcount_5d_),
	F(LISTENER_DAY_STATS, tsum_5d_),
	F(LISTENER_DAY_STATS, p95_5d_respms_),
	F(LISTENER_DAY_STATS, p25_5d_respms_),
	F(LISTENER_DAY_STATS, p95_qps_),
	F(LISTENER_DAY_STATS, p25_qps_),
	F(LISTENER_DAY_STATS, p95_nactive_),
	F(LISTENER_DAY_STATS, p25_nactive_),

	F(AGGR_TASK_HIST_STATS, aggr_task_id_),
	F(AGGR_TASK_HIST_STATS, starttimeusec_),
	F(AGGR_TASK_HIST_STATS, p95_cpu_pct_),
	F(AGGR_TASK_HIST_STATS, p95_cpu_delay_ms_),
	F(AGGR_TASK_HIST_STATS, p95_blkio_delay_ms_),
	F(AGGR_TASK_HIST_STATS, nprocs_),
	F(AGGR_TASK_HIST_STATS, nthreads_),
	F(AGGR_TASK_HIST_STATS, max_cores_allowed_),
	F(AGGR_TASK_HIST_STATS, cpu_cg_pct_limit_),
	F(AGGR_TASK_HIST_STATS, max_mem_cg_pct_rss_),

	F(API_TRAN, treq_usec_),
	F(API_TRAN, tres_usec_),
	F(API_TRAN, tupd_usec_),
	F(API_TRAN, reqlen_),
	F(API_TRAN, reslen_),
	F(API_TRAN, reqnum_),
	F(API_TRAN, response_usec_),
	F(API_TRAN, reaction_usec_),
	F(API_TRAN, tconnect_usec_),
	F(API_TRAN, cliip_),
	F(API_TRAN, serip_),
	F(API_TRAN, glob_id_),
	F(API_TRAN, conn_id_),
	F(API_TRAN, comm_),
	F(API_TRAN, errorcode_),
	F(API_TRAN, app_sleep_ms_),
	F(API_TRAN, tran_type_),
	F(API_TRAN, proto_),
	F(API_TRAN, cliport_),
	F(API_TRAN, serport_),
	F(API_TRAN, request_len_),
	F(API_TRAN, lenext_),
	F(API_TRAN, padlen_),

	F(tcp_ipv4_event_t, ts_ns),
	F(tcp_ipv4_event_t, bytes_received),
	F(tcp_ipv4_event_t, bytes_acked),
	F(tcp_ipv4_event_t, pid),
	F(tcp_ipv4_event_t, tid),
	F(tcp_ipv4_event_t, comm),
	F(tcp_ipv4_event_t, saddr),
	F(tcp_ipv4_event_t, daddr),
	F(tcp_ipv4_event_t, netns),
	F(tcp_ipv4_event_t, sport),
	F(tcp_ipv4_event_t, dport),
	F(tcp_ipv4_event_t, ipver),
	F(tcp_ipv4_event_t, type),

	F(tcp_ipv6_event_t, ts_ns),
	F(tcp_ipv6_event_t, bytes_received),
	F(tcp_ipv6_event_t, bytes_acked),
	F(tcp_ipv6_event_t, pid),
	F(tcp_ipv6_event_t, tid),
	F(tcp_ipv6_event_t, comm),
	F(tcp_ipv6_event_t, saddr),
	F(tcp_ipv6_event_t, daddr),
	F(tcp_ipv6_event_t, netns),
	F(tcp_ipv6_event_t, sport),
	F(tcp_ipv6_event_t, dport),
	F(tcp_ipv6_event_t, ipver),
	F(tcp_ipv6_event_t, type),

	F(tcp_ipv4_resp_event_t, tup.saddr),
	F(tcp_ipv4_resp_event_t, tup.daddr),
	F(tcp_ipv4_resp_event_t, tup.netns),
	F(tcp_ipv4_resp_event_t, tup.sport),
	F(tcp_ipv4_resp_event_t, tup.dport),
	F(tcp_ipv4_resp_event_t, lsndtime),
	F(tcp_ipv4_resp_event_t, lrcvtime),

	F(tcp_ipv6_resp_event_t, tup.saddr),
	F(tcp_ipv6_resp_event_t, tup.daddr),
	F(tcp_ipv6_resp_event_t, tup.netns),
	F(tcp_ipv6_resp_event_t, tup.sport),
	F(tcp_ipv6_resp_event_t, tup.dport),
	F(tcp_ipv6_resp_event_t, lsndtime),
	F(tcp_ipv6_resp_event_t, lrcvtime),
};

#undef S
#undef F

// One value column is VAL_BYTES wide, little endian. A scalar field takes the column through its own type (an integer or enum
// its low bytes, a bool whether the first byte is non-zero, a float the bit pattern of its width); any other field (arrays,
// __int128, GY_MACHINE_ID, GY_IP_ADDR) takes the column's first sizeof(field) bytes.
constexpr size_t VAL_BYTES = 32;

template <typename M>
void put(M &dst, const uint8_t *src)
{
	if constexpr (std::is_same_v<M, bool>) dst = src[0] != 0;
	else if constexpr (std::is_floating_point_v<M>) std::memcpy(&dst, src, sizeof(M));
	else if constexpr ((std::is_integral_v<M> || std::is_enum_v<M>) && sizeof(M) <= 8) {
		uint64_t v; std::memcpy(&v, src, 8); dst = (M)v;
	}
	else {
		static_assert(sizeof(M) <= VAL_BYTES, "value column too narrow");
		std::memcpy((void *)&dst, src, sizeof(M));
	}
}

template <typename T> using Setter = void (*)(T &, const uint8_t *);
template <typename T> struct Named { const char *name; Setter<T> set; };

#define N(T, M)		{ #M, [](T &r, const uint8_t *v) { put(r.M, v); } }
#define B(T, M)		{ #M, [](T &r, const uint8_t *v) { r.M = v[0] != 0; } }		// bit-fields

template <typename T> struct Setters;

template <> struct Setters<TCP_CONN_NOTIFY> { static constexpr Named<TCP_CONN_NOTIFY> v[] = {
	N(TCP_CONN_NOTIFY, cli_), N(TCP_CONN_NOTIFY, ser_), N(TCP_CONN_NOTIFY, nat_cli_), N(TCP_CONN_NOTIFY, nat_ser_),
	N(TCP_CONN_NOTIFY, tusec_start_), N(TCP_CONN_NOTIFY, tusec_close_), N(TCP_CONN_NOTIFY, cli_task_aggr_id_),
	N(TCP_CONN_NOTIFY, cli_related_listen_id_), N(TCP_CONN_NOTIFY, cli_madhava_id_), N(TCP_CONN_NOTIFY, cli_ser_machine_id_),
	N(TCP_CONN_NOTIFY, ser_related_listen_id_), N(TCP_CONN_NOTIFY, ser_glob_id_), N(TCP_CONN_NOTIFY, ser_madhava_id_),
	N(TCP_CONN_NOTIFY, bytes_sent_), N(TCP_CONN_NOTIFY, bytes_rcvd_), N(TCP_CONN_NOTIFY, cli_pid_), N(TCP_CONN_NOTIFY, ser_pid_),
	N(TCP_CONN_NOTIFY, ser_conn_hash_), N(TCP_CONN_NOTIFY, ser_sock_inode_), N(TCP_CONN_NOTIFY, cli_comm_), N(TCP_CONN_NOTIFY, ser_comm_),
	N(TCP_CONN_NOTIFY, is_tcp_connect_event_), N(TCP_CONN_NOTIFY, is_tcp_accept_event_), N(TCP_CONN_NOTIFY, is_loopback_conn_),
	N(TCP_CONN_NOTIFY, is_pre_existing_), N(TCP_CONN_NOTIFY, notified_before_),
}; };

template <> struct Setters<AGGR_TASK_STATE_NOTIFY> { static constexpr Named<AGGR_TASK_STATE_NOTIFY> v[] = {
	N(AGGR_TASK_STATE_NOTIFY, aggr_task_id_), N(AGGR_TASK_STATE_NOTIFY, onecomm_), N(AGGR_TASK_STATE_NOTIFY, pid_arr_),
	N(AGGR_TASK_STATE_NOTIFY, tcp_kbytes_), N(AGGR_TASK_STATE_NOTIFY, tcp_conns_), N(AGGR_TASK_STATE_NOTIFY, total_cpu_pct_),
	N(AGGR_TASK_STATE_NOTIFY, rss_mb_), N(AGGR_TASK_STATE_NOTIFY, cpu_delay_msec_), N(AGGR_TASK_STATE_NOTIFY, vm_delay_msec_),
	N(AGGR_TASK_STATE_NOTIFY, blkio_delay_msec_), N(AGGR_TASK_STATE_NOTIFY, ntasks_total_), N(AGGR_TASK_STATE_NOTIFY, ntasks_issue_),
	N(AGGR_TASK_STATE_NOTIFY, curr_state_), N(AGGR_TASK_STATE_NOTIFY, curr_issue_), N(AGGR_TASK_STATE_NOTIFY, issue_bit_hist_),
	N(AGGR_TASK_STATE_NOTIFY, severe_issue_bit_hist_),
}; };

template <> struct Setters<LISTENER_STATE_NOTIFY> { static constexpr Named<LISTENER_STATE_NOTIFY> v[] = {
	N(LISTENER_STATE_NOTIFY, glob_id_), N(LISTENER_STATE_NOTIFY, nqrys_5s_), N(LISTENER_STATE_NOTIFY, total_resp_5sec_),
	N(LISTENER_STATE_NOTIFY, nconns_), N(LISTENER_STATE_NOTIFY, nconns_active_), N(LISTENER_STATE_NOTIFY, ntasks_),
	N(LISTENER_STATE_NOTIFY, p95_5s_resp_ms_), N(LISTENER_STATE_NOTIFY, p95_5min_resp_ms_), N(LISTENER_STATE_NOTIFY, curr_kbytes_inbound_),
	N(LISTENER_STATE_NOTIFY, curr_kbytes_outbound_), N(LISTENER_STATE_NOTIFY, ser_errors_), N(LISTENER_STATE_NOTIFY, cli_errors_),
	N(LISTENER_STATE_NOTIFY, tasks_delay_usec_), N(LISTENER_STATE_NOTIFY, tasks_cpudelay_usec_), N(LISTENER_STATE_NOTIFY, tasks_blkiodelay_usec_),
	N(LISTENER_STATE_NOTIFY, tasks_user_cpu_), N(LISTENER_STATE_NOTIFY, tasks_sys_cpu_), N(LISTENER_STATE_NOTIFY, tasks_rss_mb_),
	N(LISTENER_STATE_NOTIFY, ntasks_issue_), N(LISTENER_STATE_NOTIFY, is_http_svc_), N(LISTENER_STATE_NOTIFY, curr_state_),
	N(LISTENER_STATE_NOTIFY, curr_issue_), N(LISTENER_STATE_NOTIFY, issue_bit_hist_), N(LISTENER_STATE_NOTIFY, high_resp_bit_hist_),
	N(LISTENER_STATE_NOTIFY, last_issue_subsrc_), N(LISTENER_STATE_NOTIFY, query_flags_),
}; };

template <> struct Setters<HOST_STATE_NOTIFY> { static constexpr Named<HOST_STATE_NOTIFY> v[] = {
	N(HOST_STATE_NOTIFY, curr_time_usec_), N(HOST_STATE_NOTIFY, ntasks_issue_), N(HOST_STATE_NOTIFY, ntasks_severe_),
	N(HOST_STATE_NOTIFY, ntasks_), N(HOST_STATE_NOTIFY, nlisten_issue_), N(HOST_STATE_NOTIFY, nlisten_severe_), N(HOST_STATE_NOTIFY, nlisten_),
	N(HOST_STATE_NOTIFY, curr_state_), N(HOST_STATE_NOTIFY, issue_bit_hist_), N(HOST_STATE_NOTIFY, cpu_issue_), N(HOST_STATE_NOTIFY, mem_issue_),
	N(HOST_STATE_NOTIFY, severe_cpu_issue_), N(HOST_STATE_NOTIFY, severe_mem_issue_), N(HOST_STATE_NOTIFY, total_cpu_delayms_),
	N(HOST_STATE_NOTIFY, total_vm_delayms_), N(HOST_STATE_NOTIFY, total_io_delayms_),
}; };

template <> struct Setters<ACTIVE_CONN_STATS> { static constexpr Named<ACTIVE_CONN_STATS> v[] = {
	N(ACTIVE_CONN_STATS, listener_glob_id_), N(ACTIVE_CONN_STATS, cli_aggr_task_id_), N(ACTIVE_CONN_STATS, ser_comm_),
	N(ACTIVE_CONN_STATS, cli_comm_), N(ACTIVE_CONN_STATS, remote_machine_id_), N(ACTIVE_CONN_STATS, remote_madhava_id_),
	N(ACTIVE_CONN_STATS, bytes_sent_), N(ACTIVE_CONN_STATS, bytes_received_), N(ACTIVE_CONN_STATS, cli_delay_msec_),
	N(ACTIVE_CONN_STATS, ser_delay_msec_), N(ACTIVE_CONN_STATS, max_rtt_msec_), N(ACTIVE_CONN_STATS, active_conns_),
	B(ACTIVE_CONN_STATS, cli_listener_proc_), B(ACTIVE_CONN_STATS, is_remote_listen_), B(ACTIVE_CONN_STATS, is_remote_cli_),
}; };

template <> struct Setters<API_TRAN> { static constexpr Named<API_TRAN> v[] = {
	N(API_TRAN, treq_usec_), N(API_TRAN, tres_usec_), N(API_TRAN, tupd_usec_), N(API_TRAN, reqlen_), N(API_TRAN, reslen_),
	N(API_TRAN, reqnum_), N(API_TRAN, response_usec_), N(API_TRAN, reaction_usec_), N(API_TRAN, tconnect_usec_), N(API_TRAN, cliip_),
	N(API_TRAN, serip_), N(API_TRAN, glob_id_), N(API_TRAN, conn_id_), N(API_TRAN, comm_), N(API_TRAN, errorcode_),
	N(API_TRAN, app_sleep_ms_), N(API_TRAN, tran_type_), N(API_TRAN, proto_), N(API_TRAN, cliport_), N(API_TRAN, serport_),
	N(API_TRAN, lenext_),
}; };

template <> struct Setters<tcp_ipv4_event_t> { static constexpr Named<tcp_ipv4_event_t> v[] = {
	N(tcp_ipv4_event_t, ts_ns), N(tcp_ipv4_event_t, bytes_received), N(tcp_ipv4_event_t, bytes_acked), N(tcp_ipv4_event_t, pid),
	N(tcp_ipv4_event_t, tid), N(tcp_ipv4_event_t, comm), N(tcp_ipv4_event_t, saddr), N(tcp_ipv4_event_t, daddr), N(tcp_ipv4_event_t, netns),
	N(tcp_ipv4_event_t, sport), N(tcp_ipv4_event_t, dport), N(tcp_ipv4_event_t, ipver), N(tcp_ipv4_event_t, type),
}; };

template <> struct Setters<tcp_ipv6_event_t> { static constexpr Named<tcp_ipv6_event_t> v[] = {
	N(tcp_ipv6_event_t, ts_ns), N(tcp_ipv6_event_t, bytes_received), N(tcp_ipv6_event_t, bytes_acked), N(tcp_ipv6_event_t, pid),
	N(tcp_ipv6_event_t, tid), N(tcp_ipv6_event_t, comm), N(tcp_ipv6_event_t, saddr), N(tcp_ipv6_event_t, daddr), N(tcp_ipv6_event_t, netns),
	N(tcp_ipv6_event_t, sport), N(tcp_ipv6_event_t, dport), N(tcp_ipv6_event_t, ipver), N(tcp_ipv6_event_t, type),
}; };

template <> struct Setters<tcp_ipv4_resp_event_t> { static constexpr Named<tcp_ipv4_resp_event_t> v[] = {
	N(tcp_ipv4_resp_event_t, tup.saddr), N(tcp_ipv4_resp_event_t, tup.daddr), N(tcp_ipv4_resp_event_t, tup.netns),
	N(tcp_ipv4_resp_event_t, tup.sport), N(tcp_ipv4_resp_event_t, tup.dport), N(tcp_ipv4_resp_event_t, lsndtime),
	N(tcp_ipv4_resp_event_t, lrcvtime),
}; };

template <> struct Setters<tcp_ipv6_resp_event_t> { static constexpr Named<tcp_ipv6_resp_event_t> v[] = {
	N(tcp_ipv6_resp_event_t, tup.saddr), N(tcp_ipv6_resp_event_t, tup.daddr), N(tcp_ipv6_resp_event_t, tup.netns),
	N(tcp_ipv6_resp_event_t, tup.sport), N(tcp_ipv6_resp_event_t, tup.dport), N(tcp_ipv6_resp_event_t, lsndtime),
	N(tcp_ipv6_resp_event_t, lrcvtime),
}; };

#undef N
#undef B

// The trailing string of the variable-stride kinds: its length field set to the string's length, then the type's own padding rule
inline void set_tail(TCP_CONN_NOTIFY &r, uint32_t len)		{ r.cli_cmdline_len_ = len; r.set_padding_len(); }
inline void set_tail(AGGR_TASK_STATE_NOTIFY &r, uint32_t len)	{ r.issue_string_len_ = len; r.set_padding_len(); }
inline void set_tail(LISTENER_STATE_NOTIFY &r, uint32_t len)	{ r.issue_string_len_ = len; r.set_padding_len(); }
inline void set_tail(API_TRAN &r, uint32_t len)			{ r.request_len_ = len; r.set_padding_len(); }
template <typename T> inline void set_tail(T &, uint32_t)	{}

template <typename T> inline size_t elem_size(const T &r)	{ return r.get_elem_size(); }
inline size_t elem_size(const tcp_ipv4_event_t &)		{ return sizeof(tcp_ipv4_event_t); }
inline size_t elem_size(const tcp_ipv6_event_t &)		{ return sizeof(tcp_ipv6_event_t); }
inline size_t elem_size(const tcp_ipv4_resp_event_t &)		{ return sizeof(tcp_ipv4_resp_event_t); }
inline size_t elem_size(const tcp_ipv6_resp_event_t &)		{ return sizeof(tcp_ipv6_resp_event_t); }

// n records of T: record i takes vals[i][j] (VAL_BYTES each) into the field names[j], then tails[toff[i] .. toff[i+1]) as its
// trailing string (kinds without one ignore it). Returns the bytes written, -1 for an unknown field name, -2 when out is too small.
template <typename T>
int64_t build(uint32_t n, const char *const *names, uint32_t nnames, const uint8_t *vals, const uint8_t *tails, const uint64_t *toff,
		uint8_t *out, uint64_t cap)
{
	Setter<T> set[256];
	if (nnames > 256) return -1;
	for (uint32_t j = 0; j < nnames; ++j) {
		set[j] = nullptr;
		for (const auto &s : Setters<T>::v) if (!std::strcmp(s.name, names[j])) set[j] = s.set;
		if (!set[j]) return -1;
	}
	uint64_t pos = 0;
	for (uint32_t i = 0; i < n; ++i) {
		alignas(T) uint8_t mem[sizeof(T)];
		std::memset(mem, 0, sizeof(mem));		// padding and the fields a default constructor leaves unset read as zero
		T *r = new (mem) T;
		for (uint32_t j = 0; j < nnames; ++j) set[j](*r, vals + ((size_t)i * nnames + j) * VAL_BYTES);
		const uint32_t tl = toff ? (uint32_t)(toff[i + 1] - toff[i]) : 0;
		set_tail(*r, tl);
		const size_t es = elem_size(*r);
		if (pos + es > cap) return -2;
		std::memset(out + pos, 0, es);
		std::memcpy(out + pos, mem, sizeof(T));
		if (es > sizeof(T) && tl) std::memcpy(out + pos + sizeof(T), tails + toff[i], tl);
		pos += es;
		r->~T();
	}
	return (int64_t)pos;
}

} // namespace

extern "C" {

uint32_t gyref_wire_val_bytes(void)		{ return VAL_BYTES; }
uint32_t gyref_wire_nstructs(void)		{ return sizeof(structs) / sizeof(structs[0]); }
uint32_t gyref_wire_nfields(void)		{ return sizeof(fields) / sizeof(fields[0]); }

void gyref_wire_struct(uint32_t i, const char **name, uint32_t *size, uint32_t *align)
{
	*name = structs[i].name; *size = structs[i].size; *align = structs[i].align;
}

void gyref_wire_field(uint32_t i, const char **strct, const char **field, uint32_t *off, uint32_t *size)
{
	*strct = fields[i].strct; *field = fields[i].field; *off = fields[i].off; *size = fields[i].size;
}

// Records of the named type, see build() above
int64_t gyref_wire_build(const char *strct, uint32_t n, const char *const *names, uint32_t nnames, const uint8_t *vals,
		const uint8_t *tails, const uint64_t *toff, uint8_t *out, uint64_t cap)
{
#define K(T) if (!std::strcmp(strct, #T)) return build<T>(n, names, nnames, vals, tails, toff, out, cap);
	K(TCP_CONN_NOTIFY) K(AGGR_TASK_STATE_NOTIFY) K(LISTENER_STATE_NOTIFY) K(HOST_STATE_NOTIFY) K(ACTIVE_CONN_STATS) K(API_TRAN)
	K(tcp_ipv4_event_t) K(tcp_ipv6_event_t) K(tcp_ipv4_resp_event_t) K(tcp_ipv6_resp_event_t)
#undef K
	return -3;
}

// One partha -> madhava event message: COMM_HEADER (its own constructor sets magic, length and padding) + EVENT_NOTIFY +
// body + the header's padding. Returns the bytes written, or -2 when out is too small, -3 when the header refuses the length.
int64_t gyref_wire_msg(uint32_t subtype, uint32_t nevents, const uint8_t *body, uint64_t bodylen, uint8_t *out, uint64_t cap)
{
	COMM_HEADER hdr(COMM_EVENT_NOTIFY, (uint32_t)(sizeof(COMM_HEADER) + sizeof(EVENT_NOTIFY) + bodylen), COMM_HEADER::PM_HDR_MAGIC);
	if (hdr.magic_ == COMM_HEADER::INV_HDR_MAGIC) return -3;
	EVENT_NOTIFY ev((NOTIFY_TYPE_E)subtype, nevents);
	const uint64_t total = hdr.get_total_len();
	if (total > cap) return -2;
	std::memset(out, 0, total);
	std::memcpy(out, &hdr, sizeof(hdr));
	std::memcpy(out + sizeof(hdr), &ev, sizeof(ev));
	if (bodylen) std::memcpy(out + sizeof(hdr) + sizeof(ev), body, bodylen);
	return (int64_t)total;
}

// The reference's record caps and notify subtypes, for the golden sets' limits
uint32_t gyref_wire_const(const char *name)
{
#define C(X, V) if (!std::strcmp(name, X)) return (uint32_t)(V);
	C("TCP_CONN_NOTIFY::MAX_NUM_CONNS", TCP_CONN_NOTIFY::MAX_NUM_CONNS)
	C("AGGR_TASK_STATE_NOTIFY::MAX_NUM_TASKS", AGGR_TASK_STATE_NOTIFY::MAX_NUM_TASKS)
	C("LISTENER_STATE_NOTIFY::MAX_NUM_LISTENERS", LISTENER_STATE_NOTIFY::MAX_NUM_LISTENERS)
	C("ACTIVE_CONN_STATS::MAX_NUM_CONNS", ACTIVE_CONN_STATS::MAX_NUM_CONNS)
	C("API_TRAN::MAX_NUM_REQS", API_TRAN::MAX_NUM_REQS)
	C("NOTIFY_TCP_CONN", NOTIFY_TCP_CONN)
	C("NOTIFY_AGGR_TASK_STATE", NOTIFY_AGGR_TASK_STATE)
	C("NOTIFY_LISTENER_STATE", NOTIFY_LISTENER_STATE)
	C("NOTIFY_HOST_STATE", NOTIFY_HOST_STATE)
	C("NOTIFY_ACTIVE_CONN_STATS", NOTIFY_ACTIVE_CONN_STATS)
	C("COMM_EVENT_NOTIFY", COMM_EVENT_NOTIFY)
	C("PM_HDR_MAGIC", COMM_HEADER::PM_HDR_MAGIC)
#undef C
	return 0xFFFFFFFFu;
}

} // extern "C"
