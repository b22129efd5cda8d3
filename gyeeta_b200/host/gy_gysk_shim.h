// gy_gysk_shim.h — the host-side mirror of the reference's ingest interface for this path (C++17, header only).
//
// The handlers below keep the names, argument meaning and bool return of the reference's member functions
//     MCONN_HANDLER::partha_tcp_conn_info     server/gy_mconnhdlr.h:2091   (definition gy_mconnhdlr.cc:9052)
//     MCONN_HANDLER::partha_aggr_task_state   server/gy_mconnhdlr.h:2098   (definition gy_mconnhdlr.cc:9959)
//     MCONN_HANDLER::partha_listener_state    server/gy_mconnhdlr.h:2129   (definition gy_mconnhdlr.cc:10993)
//     MCONN_HANDLER::handle_partha_active_conns server/gy_mconnhdlr.h:2155 (definition gy_mconnhdlr.cc:7705)
//     MCONN_HANDLER::handle_aggr_task_hist_stats server/gy_mconnhdlr.h:2109 (definition gy_mconnhdlr.cc:14648; reads the engine)
// and forward the record batch to the GPU engine through the C ABI of include/gysketch.h. window_listener_day_stats and host_state
// produce from the engine what a raw-forward partha no longer sends for MCONN_HANDLER::handle_listener_day_stats (gy_mconnhdlr.cc:12805)
// and handle_host_state (gy_mconnhdlr.cc:12971). The template parameters
// stand for the reference's own types (std::shared_ptr<PARTHA_INFO>, comm::TCP_CONN_NOTIFY, POOL_ALLOC_ARRAY, PGConnPool) so
// that this header compiles both inside gy_mconnhdlr.cc (with the real types) and stand-alone in this repository's tests (with
// the POD mirrors of gyeeta_b200/csrc/gysk_wire.h). See INTEGRATION.md for the call-site patch.
#pragma once

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <memory>
#include <mutex>
#include <new>
#include <utility>
#include <vector>

#include "../../include/gysketch.h"

namespace gysk_shim {

// What the shim needs from PARTHA_INFO: the 16-byte machine id (GY_MACHINE_ID machine_id_, server/gy_mconnhdlr.h:1110) and a
// dense per-madhava host index (the engine shards by it). Specialise / overload for the real PARTHA_INFO.
template <typename ParthaInfo>
struct partha_traits
{
	static const uint8_t *machine_id(const ParthaInfo & p) noexcept { return reinterpret_cast<const uint8_t *>(&p.machine_id_); }
	static uint32_t host_index(const ParthaInfo & p) noexcept { return p.gysk_host_idx_; }
};

class GYSK_HANDLER
{
public :
	explicit GYSK_HANDLER(gysk_engine *engine) noexcept : engine_(engine) {}
	// a copy starts with host_state's rows unread
	GYSK_HANDLER(const GYSK_HANDLER & o) : engine_(o.engine_), evicted_(o.evicted_), summ_(o.summ_) {}
	GYSK_HANDLER & operator=(const GYSK_HANDLER & o) { if (this != &o) { GYSK_HANDLER t(o); *this = std::move(t); } return *this; }
	GYSK_HANDLER(GYSK_HANDLER &&) noexcept = default;
	GYSK_HANDLER & operator=(GYSK_HANDLER &&) noexcept = default;

	// bool partha_tcp_conn_info(const std::shared_ptr<PARTHA_INFO> &, comm::TCP_CONN_NOTIFY *, int nconns, uint8_t *pendptr, POOL_ALLOC_ARRAY *)
	template <typename ParthaInfo, typename TcpConnNotify, typename PoolArr>
	bool partha_tcp_conn_info(const std::shared_ptr<ParthaInfo> & partha_shr, TcpConnNotify *pone, int nconns, uint8_t *pendptr, PoolArr * /*pthrpoolarr*/) noexcept
	{
		return forward(partha_shr, GYSK_NOTIFY_TCP_CONN, pone, nconns, pendptr);
	}

	// bool partha_aggr_task_state(const std::shared_ptr<PARTHA_INFO> &, const comm::AGGR_TASK_STATE_NOTIFY *, int ntasks, uint8_t *pendptr, PGConnPool &)
	template <typename ParthaInfo, typename AggrTaskStateNotify, typename DbPool>
	bool partha_aggr_task_state(const std::shared_ptr<ParthaInfo> & partha_shr, const AggrTaskStateNotify *ptask, int ntasks, uint8_t *pendptr, DbPool & /*dbpool*/) noexcept
	{
		return forward(partha_shr, GYSK_NOTIFY_AGGR_TASK_STATE, const_cast<AggrTaskStateNotify *>(ptask), ntasks, pendptr);
	}

	// bool partha_listener_state(const std::shared_ptr<PARTHA_INFO> &, const comm::LISTENER_STATE_NOTIFY *, int nitems, uint8_t *pendptr,
	//                            POOL_ALLOC_ARRAY *, PGConnPool &, bool isdummycall = false)
	template <typename ParthaInfo, typename ListenerStateNotify, typename PoolArr, typename DbPool>
	bool partha_listener_state(const std::shared_ptr<ParthaInfo> & partha_shr, const ListenerStateNotify *plist, int nitems, uint8_t *pendptr,
			PoolArr * /*pthrpoolarr*/, DbPool & /*dbpool*/, bool isdummycall = false) noexcept
	{
		if (isdummycall) return true;
		return forward(partha_shr, GYSK_NOTIFY_LISTENER_STATE, const_cast<ListenerStateNotify *>(plist), nitems, pendptr);
	}

	// bool handle_partha_active_conns(const std::shared_ptr<PARTHA_INFO> &, const comm::ACTIVE_CONN_STATS *, int nitems, uint8_t *pendptr,
	//                                 POOL_ALLOC_ARRAY *, PGConnPool &)
	template <typename ParthaInfo, typename ActiveConnStats, typename PoolArr, typename DbPool>
	bool handle_partha_active_conns(const std::shared_ptr<ParthaInfo> & partha_shr, const ActiveConnStats *pconn, int nitems, uint8_t *pendptr,
			PoolArr * /*pthrpoolarr*/, DbPool & /*dbpool*/) noexcept
	{
		return forward(partha_shr, GYSK_NOTIFY_ACTIVE_CONN_STATS, const_cast<ActiveConnStats *>(pconn), nitems, pendptr);
	}

	// the lifted per-sample paths (partha built with -DGYSK_RAW_FORWARD ships its perf-buffer pages unreduced): the callbacks of
	// GY_EBPF::tcp_response_ipv4/ipv6_thread and tcp_conn_ipv4/ipv6_thread (partha/gy_ebpf_bpf.cc:181-199,316-323) ->
	// TCP_SOCK_HANDLER::handle_ipv4_resp_event / handle_ipv6_resp_event / handle_ipv4_conn_event / handle_ipv6_conn_event
	template <typename ParthaInfo, typename RespEvent>
	bool handle_resp_events(const std::shared_ptr<ParthaInfo> & partha_shr, const RespEvent *pevents, uint32_t n) noexcept
	{
		static_assert(sizeof(RespEvent) == 24 || sizeof(RespEvent) == 64, "tcp_ipv4_resp_event_t / tcp_ipv6_resp_event_t");
		return partha_shr && 0 == gysk_ingest_raw(engine_, partha_traits<ParthaInfo>::machine_id(*partha_shr), partha_traits<ParthaInfo>::host_index(*partha_shr),
				sizeof(RespEvent) == 24 ? GYSK_RAW_TCP_IPV4_RESP : GYSK_RAW_TCP_IPV6_RESP, pevents, n);
	}
	template <typename ParthaInfo, typename ConnEvent>
	bool handle_conn_events(const std::shared_ptr<ParthaInfo> & partha_shr, const ConnEvent *pevents, uint32_t n) noexcept
	{
		static_assert(sizeof(ConnEvent) == 72 || sizeof(ConnEvent) == 96, "tcp_ipv4_event_t / tcp_ipv6_event_t");
		return partha_shr && 0 == gysk_ingest_raw(engine_, partha_traits<ParthaInfo>::machine_id(*partha_shr), partha_traits<ParthaInfo>::host_index(*partha_shr),
				sizeof(ConnEvent) == 72 ? GYSK_RAW_TCP_IPV4_EVENT : GYSK_RAW_TCP_IPV6_EVENT, pevents, n);
	}
	// SVC_INFO_CAP::upd_stats_on_req (common/gy_proto_parser.cc:2678): a run of API_TRAN records (variable stride) of one host
	template <typename ParthaInfo>
	bool handle_api_trans(const std::shared_ptr<ParthaInfo> & partha_shr, const void *ptran, uint32_t n) noexcept
	{
		return partha_shr && 0 == gysk_ingest_raw(engine_, partha_traits<ParthaInfo>::machine_id(*partha_shr), partha_traits<ParthaInfo>::host_index(*partha_shr),
				GYSK_RAW_API_TRAN, ptran, n);
	}

	// handle_trace_requests (server/gy_mconnhdlr.cc:5883-6060) with trace rows (gysk_config.max_trace_svcs): the records go to the engine,
	// which stages each one's RESP and trace events, instead of one tracereqtbl row per request. What reaches the database is one row per
	// traced service and window: trace_window_rows after each flush_window.
	template <typename ParthaInfo>
	bool handle_trace_requests(const std::shared_ptr<ParthaInfo> & partha_shr, const void *ptran, uint32_t n) noexcept
	{
		return handle_api_trans(partha_shr, ptran, n);
	}

	// the closed window of every traced service with requests in it, ascending glob_id: on_row(row, pgtext) once per service, with the
	// window's compression-100 digest as Postgres tdigest text for the row's digest column (NULL when it has no digested sample)
	template <typename OnRow>
	bool trace_window_rows(OnRow && on_row) noexcept
	{
		uint32_t n = 0;
		if (0 != gysk_query_trace_window(engine_, -1, GYSK_WINDOW_ACTIVE_ONLY, nullptr, 0, &n)) return false;
		std::vector<gysk_trace_row> rows(n);
		if (n && 0 != gysk_query_trace_window(engine_, -1, GYSK_WINDOW_ACTIVE_ONLY, rows.data(), n, &n)) return false;
		std::vector<char> buf(8192);
		for (const gysk_trace_row & r : rows) {
			const int len = r.last.td_count ? gysk_export_trace_tdigest_pgtext(engine_, r.glob_id, 1, buf.data(), (uint32_t)buf.size()) : 0;
			on_row(r, len > 0 ? (const char *)buf.data() : (const char *)nullptr);
		}
		return true;
	}

	// the 5-s reducer tick (TCP_SOCK_HANDLER::listener_stats_update cadence, common/gy_socket_stat.cc:3898)
	bool flush_window(uint32_t tsec) noexcept
	{
		if (0 != gysk_flush(engine_, tsec)) return false;
		if (hl_) hl_->flushes.fetch_add(1);
		return true;
	}

	// The tick plus what the reference does when a partha reports a deleted listener (LISTENER_STATE_NOTIFY with
	// query_flags_ == LISTEN_FLAG_DELETE, common/gy_socket_stat.cc:4023-4033): with gysk_config.idle_evict_secs set, the ids the
	// engine evicted at this flush are handed to `on_delete(glob_id)` — the place to drop the MTCP_LISTENER of that id.
	template <typename OnDelete>
	bool flush_window(uint32_t tsec, OnDelete && on_delete) noexcept
	{
		if (!flush_window(tsec)) return false;
		try {
			uint32_t n = 0;
			evicted_.resize(evicted_.size() < 1024 ? 1024 : evicted_.size());
			if (0 != gysk_evicted_ids(engine_, evicted_.data(), (uint32_t)evicted_.size(), &n)) return false;
			if (n > evicted_.size()) {
				evicted_.resize(n);
				if (0 != gysk_evicted_ids(engine_, evicted_.data(), (uint32_t)evicted_.size(), &n)) return false;
			}
			for (uint32_t i = 0; i < n && i < evicted_.size(); ++i) on_delete(evicted_[i]);
		}
		catch (...) { return false; }
		return true;
	}

	// The same, plus what MCONN_HANDLER::cleanup_partha_unused_aggr_tasks does with an aggregated process idle for 30 minutes
	// (server/gy_mconnhdlr.cc:16492-16541, a PING_TASK_AGGR with keep_task_ = false): with gysk_config.task_idle_evict_secs set, the
	// process ids the engine evicted at this flush are handed to `on_task_delete(aggr_task_id)` — the place to drop the MAGGR_TASK of
	// that id from the partha's task_aggr_tbl_ and its row from the aggregated-task table of the database.
	template <typename OnDelete, typename OnTaskDelete>
	bool flush_window(uint32_t tsec, OnDelete && on_delete, OnTaskDelete && on_task_delete) noexcept
	{
		if (!flush_window(tsec, on_delete)) return false;
		try {
			uint32_t n = 0;
			if (0 != gysk_evicted_task_ids(engine_, evicted_.data(), (uint32_t)evicted_.size(), &n)) return false;
			if (n > evicted_.size()) {
				evicted_.resize(n);
				if (0 != gysk_evicted_task_ids(engine_, evicted_.data(), (uint32_t)evicted_.size(), &n)) return false;
			}
			for (uint32_t i = 0; i < n && i < evicted_.size(); ++i) on_task_delete(evicted_[i]);
		}
		catch (...) { return false; }
		return true;
	}

	// aggregated processes the engine has evicted so far (-1 on failure)
	int64_t task_evict_count() noexcept
	{
		uint64_t t = 0;
		return 0 == gysk_task_evict_count(engine_, &t) ? (int64_t)t : -1;
	}

	// Engine output in the reference's own record form: the LISTENER_STATE_NOTIFY batch of the given listeners (<= 512 per call,
	// common/gy_comm_proto.h:2222), ready for the unchanged partha_listener_state / MTCP_LISTENER::set_state path.
	// `out` must hold n * 88 bytes. Returns the number of records written, -1 on failure.
	int listener_state_records(const uint64_t *glob_ids, uint32_t n, void *out, uint32_t cap_bytes) noexcept
	{
		try {
			summ_.resize(n);
			uint32_t nrecs = 0, nbytes = 0;
			if (0 != gysk_query_svcs(engine_, glob_ids, n, summ_.data())) return -1;
			if (0 != gysk_encode_listener_state(summ_.data(), n, out, cap_bytes, &nrecs, &nbytes)) return -1;
			return (int)nrecs;
		}
		catch (...) { return -1; }
	}

	// The 5-s tick's read side in raw-forward mode: every listener the engine holds, as LISTENER_STATE_NOTIFY batches of at most 512
	// records (MAX_NUM_LISTENERS, common/gy_comm_proto.h:2222), host by host in ascending host index, ids ascending within a host,
	// from one gysk_query_window_hosts snapshot. Call after flush_window. on_batch(uint32_t host_idx, const void *recs, uint32_t nrecs,
	// uint32_t nbytes) is where madhava calls its unchanged partha_listener_state; handing the same buffer to
	// gysk_ingest(GYSK_NOTIFY_LISTENER_STATE) fills the engine's per-host summaries, top-N lists and cluster state. Returns false on
	// failure. Its scratch is local: safe to call while other threads use this handler.
	template <typename OnBatch>
	bool window_listener_states(OnBatch && on_batch) noexcept
	{
		try {
			std::vector<gysk_svc_summary> rows;
			std::vector<uint32_t> hosts;
			uint32_t n = 0, cap = 0;
			// count, then read; listeners created in between make the read report more rows than room: read again, larger
			for (int tries = 0; ; ++tries) {
				rows.resize(cap); hosts.resize(cap);
				if (0 != gysk_query_window_hosts(engine_, -1, 0, cap ? rows.data() : nullptr, cap ? hosts.data() : nullptr, cap, &n)) return false;
				if (n <= cap) break;
				if (tries == 3) return false;
				cap = n + n / 8 + 64;
			}
			std::vector<uint8_t> recs(MAX_BATCH * RECORD_BYTES);
			for (uint32_t a = 0; a < n; ) {
				uint32_t b = a + 1;
				while (b < n && b - a < MAX_BATCH && hosts[b] == hosts[a]) ++b;
				uint32_t nrecs = 0, nbytes = 0;
				if (0 != gysk_encode_listener_state(rows.data() + a, b - a, recs.data(), (uint32_t)recs.size(), &nrecs, &nbytes)) return false;
				on_batch(hosts[a], (const void *)recs.data(), nrecs, nbytes);
				a = b;
			}
			return true;
		}
		catch (...) { return false; }
	}

	// The 5-minute half of the listener walk in raw-forward mode (listener_stats_update sends it when tcurr > next_listen_stat_tsec_,
	// common/gy_socket_stat.cc:3916-3919, :4417-4421): every listener older than 15 minutes as LISTENER_DAY_STATS records (48 bytes) in
	// batches of at most 2048 (MAX_NUM_LISTENERS, common/gy_comm_proto.h:1632), host by host in ascending host index, ids ascending
	// within a host, from one gysk_query_day_stats snapshot. Call after flush_window, every 5 minutes. on_batch(uint32_t host_idx,
	// const void *recs, uint32_t nrecs) is where madhava calls its unchanged handle_listener_day_stats. Returns false on failure. Its
	// scratch is local: safe to call while other threads use this handler.
	template <typename OnBatch>
	bool window_listener_day_stats(OnBatch && on_batch) noexcept
	{
		try {
			std::vector<gysk_listener_day_stats> rows;
			std::vector<uint32_t> hosts;
			uint32_t n = 0, cap = 0;
			for (int tries = 0; ; ++tries) {
				rows.resize(cap); hosts.resize(cap);
				if (0 != gysk_query_day_stats(engine_, -1, cap ? rows.data() : nullptr, cap ? hosts.data() : nullptr, cap, &n)) return false;
				if (n <= cap) break;
				if (tries == 3) return false;
				cap = n + n / 8 + 64;
			}
			for (uint32_t a = 0; a < n; ) {
				uint32_t b = a + 1;
				while (b < n && b - a < MAX_DAY_BATCH && hosts[b] == hosts[a]) ++b;
				on_batch(hosts[a], (const void *)(rows.data() + a), b - a);
				a = b;
			}
			return true;
		}
		catch (...) { return false; }
	}

	// Before madhava's handle_host_state (server/gy_mconnhdlr.cc:12971-13026) when the listeners live in the engine: a raw-forward partha
	// has no listener walk, so its HOST_STATE_NOTIFY (common/gy_comm_proto.h:2289-2330) reports no listeners. This fills nlisten_,
	// nlisten_issue_ and nlisten_severe_ from gysk_query_host_listen for the partha's host, recomputes curr_state_ with
	// host_status_update's rule (gysk_classify_host, common/gy_socket_stat.cc:4455-4528) from the message's own cpu, memory and task
	// fields, and rewrites bit 0 of issue_bit_hist_ (:4540-4541). cpu_idle is not on the wire: it is taken as curr_state_ == IDLE. The
	// rule reads cpu_idle only when nothing has an issue, and then partha's own evaluation, with zero listeners, took that same branch.
	// A host without live services keeps zero counts. Returns false on failure (the message is then unchanged).
	// Every partha sends one HOST_STATE_NOTIFY per 5 s, and the counts change only at a flush: the first call after each flush_window of
	// this handler reads the rows of every host with one gysk_query_host_listen call, and every other call answers from those rows
	// without entering the engine. Safe to call from any number of threads.
	template <typename ParthaInfo, typename HostStateNotify>
	bool host_state(const std::shared_ptr<ParthaInfo> & partha_shr, HostStateNotify *p) noexcept
	{
		if (!partha_shr || !p || !hl_) return false;
		try {
			const uint32_t host = partha_traits<ParthaInfo>::host_index(*partha_shr);
			gysk_host_listen hl {host, 0, 0, 0};
			{
				std::lock_guard<std::mutex> g(hl_->m);
				const uint64_t gen = hl_->flushes.load();
				if (hl_->read_at != gen) {
					if (hl_->rows.size() < HOST_ROWS) hl_->rows.resize(HOST_ROWS);
					uint32_t n = 0;
					if (0 != gysk_query_host_listen(engine_, hl_->rows.data(), (uint32_t)hl_->rows.size(), &n)) return false;
					if (n > hl_->rows.size()) {			// more hosts than ever before: once more, with room
						hl_->rows.resize(n + n / 8 + 64);
						if (0 != gysk_query_host_listen(engine_, hl_->rows.data(), (uint32_t)hl_->rows.size(), &n)) return false;
					}
					hl_->n = n < hl_->rows.size() ? n : (uint32_t)hl_->rows.size();
					hl_->read_at = gen;
				}
				const auto end = hl_->rows.begin() + hl_->n;		// ascending host_idx
				const auto it = std::lower_bound(hl_->rows.begin(), end, host, [](const gysk_host_listen &r, uint32_t h) { return r.host_idx < h; });
				if (it != end && it->host_idx == host) hl = *it;
			}
			gysk_host_state_in in {};
			in.cpu_issue = p->cpu_issue_; in.mem_issue = p->mem_issue_;
			in.severe_cpu_issue = p->severe_cpu_issue_; in.severe_mem_issue = p->severe_mem_issue_;
			in.cpu_idle = p->curr_state_ == GYSK_STATE_IDLE;
			in.ntasks_issue = p->ntasks_issue_; in.ntasks_severe = p->ntasks_severe_;
			in.nlisten_issue = hl.nlisten_issue; in.nlisten_severe = hl.nlisten_severe;
			uint8_t state = 0;
			if (0 != gysk_classify_host(&in, &state)) return false;
			p->nlisten_ = hl.nlisten; p->nlisten_issue_ = hl.nlisten_issue; p->nlisten_severe_ = hl.nlisten_severe;
			p->curr_state_ = state;
			p->issue_bit_hist_ = (uint8_t)((p->issue_bit_hist_ & ~1u) | (state >= GYSK_STATE_BAD ? 1u : 0u));
			return true;
		}
		catch (...) { return false; }
	}

	// bool handle_aggr_task_hist_stats(const std::shared_ptr<MCONNTRACK> &, AGGR_TASK_HIST_STATS *, int nevents, POOL_ALLOC_ARRAY *, PGConnPool &)
	// (server/gy_mconnhdlr.cc:14648-14706) when the process histograms live in the engine: fills p95_cpu_pct_, p95_cpu_delay_ms_ and
	// p95_blkio_delay_ms_ of the records whose aggregated process the engine holds for this partha (the reference looks each id up in
	// the partha's own task_aggr_tbl_, :14693; here the process's host_idx must be the partha's host index), with get_percentiles({95})
	// of the three MTASK_HIST histograms, the int result stored into the uint32 fields like the reference's assignment. Other records
	// stay as they are. madhava keeps the rest of its handler (pmtask->histstats_ = *pone). Its scratch is local: L2 threads may call
	// it concurrently.
	template <typename ParthaInfo, typename AggrTaskHistStats>
	bool handle_aggr_task_hist_stats(const std::shared_ptr<ParthaInfo> & partha_shr, AggrTaskHistStats *ptask, int n) noexcept
	{
		if (!partha_shr || !ptask || n < 0) return false;
		try {
			const uint32_t host = partha_traits<ParthaInfo>::host_index(*partha_shr);
			std::vector<uint64_t> ids(n);
			std::vector<gysk_task_summary> tasks(n);
			for (int i = 0; i < n; ++i) ids[i] = ptask[i].aggr_task_id_;
			if (0 != gysk_query_tasks(engine_, ids.data(), (uint32_t)n, tasks.data())) return false;
			for (int i = 0; i < n; ++i) {
				if (!tasks[i].found || tasks[i].host_idx != host) continue;
				ptask[i].p95_cpu_pct_ = tasks[i].p95_cpu_pct;
				ptask[i].p95_cpu_delay_ms_ = tasks[i].p95_cpu_delay_ms;
				ptask[i].p95_blkio_delay_ms_ = tasks[i].p95_blkio_delay_ms;
			}
		}
		catch (...) { return false; }
		return true;
	}

	gysk_engine * engine() const noexcept { return engine_; }

private :
	template <typename ParthaInfo, typename T>
	bool forward(const std::shared_ptr<ParthaInfo> & partha_shr, uint32_t subtype, T *recs, int nevents, uint8_t *pendptr) noexcept
	{
		if (!partha_shr || !recs || nevents < 0) return false;
		// same contract as the reference handlers: true = ok, false = failure, nothing thrown, caller memory not retained
		return 0 == gysk_ingest(engine_, partha_traits<ParthaInfo>::machine_id(*partha_shr), partha_traits<ParthaInfo>::host_index(*partha_shr),
				subtype, recs, (uint32_t)nevents, pendptr);
	}

	static constexpr uint32_t MAX_BATCH = 512, RECORD_BYTES = 88;		// records per NOTIFY_LISTENER_STATE message, sizeof(LISTENER_STATE_NOTIFY)
	static constexpr uint32_t MAX_DAY_BATCH = 2048;				// records per NOTIFY_LISTENER_DAY_STATS message

	static constexpr uint32_t HOST_ROWS = 1024;				// host_state's first read: MAX_PARTHA_PER_MADHAVA (512) hosts fit

	// host_state's per-host rows, read once per flush_window (a separate object: the handler stays movable and copyable)
	struct HostListenCache
	{
		std::mutex			m;
		std::atomic<uint64_t>		flushes {1};		// flush_window calls so far + 1
		uint64_t			read_at {0};		// ... when the rows were read
		std::vector<gysk_host_listen>	rows;
		uint32_t			n {0};
	};

	gysk_engine		*engine_;
	std::unique_ptr<HostListenCache> hl_ {new (std::nothrow) HostListenCache};
	std::vector<uint64_t>	evicted_;		// scratch of flush_window(tsec, on_delete) and listener_state_records: one caller at a time
	std::vector<gysk_svc_summary> summ_;
};

// MCONN_HANDLER::send_cluster_state (server/gy_mconnhdlr.cc:16052-16110) with GYSK_FLAG_MERGE_CLUSTERS: the service half of one
// MS_CLUSTER_STATE::STATE_ONE (common/gy_comm_proto.h:3181-3216) from a gysk_query_cluster_states row, every rank's hosts included.
// StateOne is comm::MS_CLUSTER_STATE::STATE_ONE (or a POD mirror); its other fields are left as they are.
template <typename StateOne>
void cluster_state_one(const gysk_cluster_row & r, StateOne & one) noexcept
{
	one.nhosts_		= r.st.nhosts;
	one.nsvc_issue_		= r.st.nsvc_issue;
	one.nsvcissue_hosts_	= r.st.nsvcissue_hosts;
	one.nsvc_		= r.st.nsvc;
	one.total_qps_		= r.st.total_qps;
	one.svc_net_mb_		= r.st.svc_net_mb;
}

// ... and the rest of CLUSTER_STATE_ONE::update_from_state (:16032-16050) for one of this madhava's hosts of the cluster, from its
// HOST_STATE_NOTIFY (comm::HOST_STATE_NOTIFY, as host_state filled it): the task, cpu and memory counters, and nhosts_ for a host the
// engine did not count because it has no live service (nlisten_ == 0)
template <typename StateOne, typename HostStateNotify>
void cluster_add_host_state(StateOne & one, const HostStateNotify & state) noexcept
{
	one.nhosts_		+= !state.nlisten_;
	one.ntasks_issue_	+= state.ntasks_issue_;
	one.ntaskissue_hosts_	+= !!state.ntasks_issue_;
	one.ntasks_		+= state.ntasks_;
	one.ncpu_issue_		+= state.cpu_issue_;
	one.nmem_issue_		+= state.mem_issue_;
}

} // namespace gysk_shim
