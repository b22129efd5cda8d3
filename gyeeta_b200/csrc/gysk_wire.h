// gysk_wire.h — host-side restatement of the wire records that reach MCONN_HANDLER::handle_l2_misc
// (server/gy_mconnhdlr.cc:4700-4800) and of their L1 validators (common/gy_comm_proto.cc:840-996).
// Plain-old-data mirrors with static_asserts on size and the offsets the decoder reads; the layouts follow
// common/gy_comm_proto.h (alignas(8), host endian, variable stride = sizeof + string + padding_len_).
#pragma once

#include <cstdint>
#include <cstddef>
#include <cstring>

#include "../../include/gysketch.h"

namespace gysk { namespace wire {

static constexpr uint32_t COMM_EVENT_NOTIFY = 14;			// common/gy_comm_proto.h:144
static constexpr uint32_t PM_HDR_MAGIC = 0x05666605u;			// :346 partha -> madhava
static constexpr uint32_t MAX_COMM_DATA_SZ = 16u << 20;			// :31

struct alignas(8) COMM_HEADER						// :336-372
{
	uint32_t	magic_;
	uint32_t	total_sz_;
	uint32_t	data_type_;
	uint32_t	padding_sz_;

	uint32_t get_act_len() const noexcept { return total_sz_ - padding_sz_; }
};
static_assert(sizeof(COMM_HEADER) == 16, "COMM_HEADER");

struct alignas(8) EVENT_NOTIFY						// :486-500
{
	uint32_t	subtype_;
	uint32_t	nevents_;
};
static_assert(sizeof(EVENT_NOTIFY) == 8, "EVENT_NOTIFY");

// GY_IP_ADDR is packed, aligned(8), 24 bytes (common/gy_common_inc.h:10488-10506); IP_PORT adds a u16 port -> 32 bytes (:11162)
struct alignas(8) IP_PORT
{
	uint8_t		ip128_be_[16];
	uint32_t	ip32_be_;
	int16_t		aftype_;
	uint16_t	ipflags_;
	uint16_t	port_;
	uint8_t		pad_[6];
};
static_assert(sizeof(IP_PORT) == 32, "IP_PORT");

struct alignas(8) TCP_CONN_NOTIFY					// common/gy_comm_proto.h:1665-1742
{
	IP_PORT		cli_, ser_, nat_cli_, nat_ser_;
	uint64_t	tusec_start_;
	uint64_t	tusec_close_;
	uint64_t	cli_task_aggr_id_;
	uint64_t	cli_related_listen_id_;
	uint64_t	cli_madhava_id_;
	uint64_t	cli_ser_machine_id_[2];				// GY_MACHINE_ID (common/gy_sys_hardware.h:20)
	uint64_t	ser_related_listen_id_;
	uint64_t	ser_glob_id_;
	uint64_t	ser_madhava_id_;
	uint64_t	bytes_sent_;
	uint64_t	bytes_rcvd_;
	int32_t		cli_pid_;
	int32_t		ser_pid_;
	uint32_t	ser_conn_hash_;
	uint32_t	ser_sock_inode_;
	char		cli_comm_[16];
	char		ser_comm_[16];
	uint16_t	cli_cmdline_len_;
	bool		is_tcp_connect_event_;
	bool		is_tcp_accept_event_;
	bool		is_loopback_conn_;
	bool		is_pre_existing_;
	bool		notified_before_;
	uint8_t		padding_len_;

	static constexpr size_t MAX_NUM_CONNS = 2048;			// :1711
	size_t get_elem_size() const noexcept { return sizeof(*this) + cli_cmdline_len_ + padding_len_; }
};
static_assert(sizeof(TCP_CONN_NOTIFY) == 280 && offsetof(TCP_CONN_NOTIFY, ser_glob_id_) == 192 &&
		offsetof(TCP_CONN_NOTIFY, cli_cmdline_len_) == 272 && offsetof(TCP_CONN_NOTIFY, padding_len_) == 279, "TCP_CONN_NOTIFY");

struct alignas(8) AGGR_TASK_STATE_NOTIFY				// common/gy_comm_proto.h:2114-2169
{
	uint64_t	aggr_task_id_;
	char		onecomm_[16];
	int32_t		pid_arr_[2];
	uint32_t	tcp_kbytes_;
	uint32_t	tcp_conns_;
	float		total_cpu_pct_;
	uint32_t	rss_mb_;
	uint32_t	cpu_delay_msec_;
	uint32_t	vm_delay_msec_;
	uint32_t	blkio_delay_msec_;
	uint16_t	ntasks_total_;
	uint16_t	ntasks_issue_;
	uint8_t		curr_state_;
	uint8_t		curr_issue_;
	uint8_t		issue_bit_hist_;
	uint8_t		severe_issue_bit_hist_;
	uint8_t		issue_string_len_;
	uint8_t		padding_len_;

	static constexpr size_t MAX_NUM_TASKS = 1200;			// :2138
	size_t get_elem_size() const noexcept { return sizeof(*this) + issue_string_len_ + padding_len_; }
};
static_assert(sizeof(AGGR_TASK_STATE_NOTIFY) == 72 && offsetof(AGGR_TASK_STATE_NOTIFY, padding_len_) == 69, "AGGR_TASK_STATE_NOTIFY");

static constexpr uint8_t LISTEN_FLAG_DELETE = (1 << 7) | (1 << 6);		// LISTENER_QUERY_FLAGS, common/gy_comm_proto.h:2180
// OBJ_STATE_E, common/gy_json_field_maps.h:242-251
enum : uint8_t { STATE_IDLE = 0, STATE_GOOD = 1, STATE_OK = 2, STATE_BAD = 3, STATE_SEVERE = 4, STATE_DOWN = 5 };

struct alignas(8) LISTENER_STATE_NOTIFY					// common/gy_comm_proto.h:2183-2254
{
	uint64_t	glob_id_;
	uint32_t	nqrys_5s_, total_resp_5sec_, nconns_, nconns_active_, ntasks_;
	uint32_t	p95_5s_resp_ms_, p95_5min_resp_ms_, curr_kbytes_inbound_, curr_kbytes_outbound_, ser_errors_, cli_errors_;
	uint32_t	tasks_delay_usec_, tasks_cpudelay_usec_, tasks_blkiodelay_usec_, tasks_user_cpu_, tasks_sys_cpu_, tasks_rss_mb_;
	uint16_t	ntasks_issue_;
	bool		is_http_svc_;
	uint8_t		curr_state_, curr_issue_, issue_bit_hist_, high_resp_bit_hist_, last_issue_subsrc_, query_flags_;
	uint8_t		issue_string_len_;
	uint8_t		padding_len_;

	static constexpr size_t MAX_NUM_LISTENERS = 512;		// :2222
	size_t get_elem_size() const noexcept { return sizeof(*this) + issue_string_len_ + padding_len_; }
};
static_assert(sizeof(LISTENER_STATE_NOTIFY) == 88 && offsetof(LISTENER_STATE_NOTIFY, padding_len_) == 86, "LISTENER_STATE_NOTIFY");

// the per-process p95 records madhava fills in handle_aggr_task_hist_stats (server/gy_mconnhdlr.cc:14648-14706)
struct alignas(8) AGGR_TASK_HIST_STATS					// common/gy_comm_proto.h:2966-2977
{
	uint64_t	aggr_task_id_;
	uint64_t	starttimeusec_;
	uint32_t	p95_cpu_pct_, p95_cpu_delay_ms_, p95_blkio_delay_ms_;
	uint32_t	nprocs_, nthreads_;
	uint16_t	max_cores_allowed_;
	uint8_t		cpu_cg_pct_limit_, max_mem_cg_pct_rss_;

	static constexpr size_t MAX_NUM_TASKS = 1200;
};
static_assert(sizeof(AGGR_TASK_HIST_STATS) == 40 && offsetof(AGGR_TASK_HIST_STATS, p95_cpu_pct_) == 16 &&
		offsetof(AGGR_TASK_HIST_STATS, max_cores_allowed_) == 36, "AGGR_TASK_HIST_STATS");

// raw eBPF records, common/gy_ebpf_kernel.h:37-52,106-111 ; common/gy_ebpf_bpf_common.h:23-30
struct tcp_ipv4_event_t
{
	uint64_t	ts_ns, bytes_received, bytes_acked;
	uint32_t	pid, tid;
	char		comm[16];
	uint32_t	saddr, daddr, netns;
	uint16_t	sport, dport;
	uint8_t		ipver, type;
};
static_assert(sizeof(tcp_ipv4_event_t) == 72, "tcp_ipv4_event_t");

struct tcp_ipv4_resp_event_t
{
	uint32_t	saddr, daddr, netns;
	uint16_t	sport, dport;
	uint32_t	lsndtime, lrcvtime;
};
static_assert(sizeof(tcp_ipv4_resp_event_t) == 24, "tcp_ipv4_resp_event_t");

struct alignas(16) tcp_ipv6_event_t					// common/gy_ebpf_kernel.h:54-68 (unsigned __int128 addresses)
{
	uint64_t	ts_ns, bytes_received, bytes_acked;
	uint32_t	pid, tid;
	char		comm[16];
	uint32_t	saddr[4], daddr[4];
	uint32_t	netns;
	uint16_t	sport, dport;
	uint8_t		ipver, type;
};
static_assert(sizeof(tcp_ipv6_event_t) == 96 && offsetof(tcp_ipv6_event_t, saddr) == 48 && offsetof(tcp_ipv6_event_t, type) == 89, "tcp_ipv6_event_t");

struct alignas(16) tcp_ipv6_resp_event_t				// common/gy_ebpf_kernel.h:113-118 over ipv6_tuple_t (gy_ebpf_bpf_common.h:32-39)
{
	uint32_t	saddr[4], daddr[4];
	uint32_t	netns;
	uint16_t	sport, dport;
	uint32_t	pad_[2];						// ipv6_tuple_t is padded to its 16-byte alignment
	uint32_t	lsndtime, lrcvtime;
};
static_assert(sizeof(tcp_ipv6_resp_event_t) == 64 && offsetof(tcp_ipv6_resp_event_t, lsndtime) == 48, "tcp_ipv6_resp_event_t");

struct alignas(8) ACTIVE_CONN_STATS					// common/gy_comm_proto.h:2766-2810 (fixed stride)
{
	uint64_t	listener_glob_id_;
	uint64_t	cli_aggr_task_id_;
	char		ser_comm_[16];
	char		cli_comm_[16];
	uint64_t	remote_machine_id_[2];					// GY_MACHINE_ID
	uint64_t	remote_madhava_id_;
	uint64_t	bytes_sent_;
	uint64_t	bytes_received_;
	uint32_t	cli_delay_msec_;
	uint32_t	ser_delay_msec_;
	float		max_rtt_msec_;
	uint16_t	active_conns_;
	uint8_t		flags_;							// cli_listener_proc_ : 1, is_remote_listen_ : 1, is_remote_cli_ : 1
	uint8_t		pad_;

	static constexpr size_t MAX_NUM_CONNS = 2048;			// :2786
	size_t get_elem_size() const noexcept { return sizeof(*this); }
};
static_assert(sizeof(ACTIVE_CONN_STATS) == 104 && offsetof(ACTIVE_CONN_STATS, bytes_sent_) == 72 && offsetof(ACTIVE_CONN_STATS, active_conns_) == 100, "ACTIVE_CONN_STATS");

struct alignas(8) LISTENER_DAY_STATS					// common/gy_comm_proto.h:1620-1653 (fixed stride)
{
	uint64_t	glob_id_;
	int64_t		tcount_5d_;
	int64_t		tsum_5d_;
	uint32_t	p95_5d_respms_;
	uint32_t	p25_5d_respms_;
	uint32_t	p95_qps_;
	uint32_t	p25_qps_;
	uint32_t	p95_nactive_;
	uint32_t	p25_nactive_;

	static constexpr size_t MAX_NUM_LISTENERS = 2048;			// :1632, records per NOTIFY_LISTENER_DAY_STATS message
};
static_assert(sizeof(LISTENER_DAY_STATS) == 48 && sizeof(gysk_listener_day_stats) == 48, "LISTENER_DAY_STATS");
static_assert(offsetof(LISTENER_DAY_STATS, tcount_5d_) == offsetof(gysk_listener_day_stats, tcount_5d) &&
		offsetof(LISTENER_DAY_STATS, tsum_5d_) == offsetof(gysk_listener_day_stats, tsum_5d) &&
		offsetof(LISTENER_DAY_STATS, p95_5d_respms_) == offsetof(gysk_listener_day_stats, p95_5d_respms) &&
		offsetof(LISTENER_DAY_STATS, p25_5d_respms_) == offsetof(gysk_listener_day_stats, p25_5d_respms) &&
		offsetof(LISTENER_DAY_STATS, p95_qps_) == offsetof(gysk_listener_day_stats, p95_qps) &&
		offsetof(LISTENER_DAY_STATS, p25_qps_) == offsetof(gysk_listener_day_stats, p25_qps) &&
		offsetof(LISTENER_DAY_STATS, p95_nactive_) == offsetof(gysk_listener_day_stats, p95_nactive) &&
		offsetof(LISTENER_DAY_STATS, p25_nactive_) == offsetof(gysk_listener_day_stats, p25_nactive), "gysk_listener_day_stats = LISTENER_DAY_STATS");

struct alignas(8) HOST_STATE_NOTIFY					// common/gy_comm_proto.h:2289-2330 (one record per message)
{
	uint64_t	curr_time_usec_;
	uint32_t	ntasks_issue_;
	uint32_t	ntasks_severe_;
	uint32_t	ntasks_;
	uint32_t	nlisten_issue_;
	uint32_t	nlisten_severe_;
	uint32_t	nlisten_;
	uint8_t		curr_state_;
	uint8_t		issue_bit_hist_;
	bool		cpu_issue_;
	bool		mem_issue_;
	bool		severe_cpu_issue_;
	bool		severe_mem_issue_;
	alignas(8) uint32_t total_cpu_delayms_;
	uint32_t	total_vm_delayms_;
	uint32_t	total_io_delayms_;
};
static_assert(sizeof(HOST_STATE_NOTIFY) == 56 && offsetof(HOST_STATE_NOTIFY, nlisten_issue_) == 20 && offsetof(HOST_STATE_NOTIFY, nlisten_) == 28 &&
		offsetof(HOST_STATE_NOTIFY, curr_state_) == 32 && offsetof(HOST_STATE_NOTIFY, severe_mem_issue_) == 37 &&
		offsetof(HOST_STATE_NOTIFY, total_cpu_delayms_) == 40, "HOST_STATE_NOTIFY");

// The shape shared by TCP_CONN_NOTIFY::validate / AGGR_TASK_STATE_NOTIFY::validate / LISTENER_STATE_NOTIFY::validate
// (common/gy_comm_proto.cc:840-881, :912-953, :955-996): nevents <= MAX, every element size a multiple of 8 and
// inside the remaining length, trailing string NUL-forced in place, success iff all nevents were walked.
template <typename T>
static inline bool validate_batch(T *recs, uint32_t nevents, const uint8_t *endptr, size_t maxn, size_t strlen_of(const T &))
{
	if (nevents > maxn) return false;
	const uint8_t *p = reinterpret_cast<const uint8_t *>(recs);
	ptrdiff_t totallen = endptr - p;
	uint32_t i;

	for (i = 0; i < nevents && totallen >= (ptrdiff_t)sizeof(T); ++i) {
		T *pone = reinterpret_cast<T *>(const_cast<uint8_t *>(p));
		const ptrdiff_t elem_sz = (ptrdiff_t)pone->get_elem_size();

		if (totallen < elem_sz) return false;
		if (elem_sz & 7) return false;
		const size_t sl = strlen_of(*pone);
		if (sl) *(const_cast<uint8_t *>(p) + sizeof(T) + sl - 1) = '\0';
		totallen -= elem_sz;
		p += elem_sz;
	}
	return i == nevents;
}

}} // namespace gysk::wire
