// gy_gysk_shim.h — the host-side mirror of the reference's ingest interface for this path (C++17, header only).
//
// The three handlers below keep the names, argument meaning and bool return of the reference's member functions
//     MCONN_HANDLER::partha_tcp_conn_info     server/gy_mconnhdlr.h:2091   (definition gy_mconnhdlr.cc:9052)
//     MCONN_HANDLER::partha_aggr_task_state   server/gy_mconnhdlr.h:2098   (definition gy_mconnhdlr.cc:9959)
//     MCONN_HANDLER::partha_listener_state    server/gy_mconnhdlr.h:2129   (definition gy_mconnhdlr.cc:10993)
//     MCONN_HANDLER::handle_partha_active_conns server/gy_mconnhdlr.h:2155 (definition gy_mconnhdlr.cc:7705)
// and forward the record batch to the GPU engine through the C ABI of include/gysketch.h. The template parameters
// stand for the reference's own types (std::shared_ptr<PARTHA_INFO>, comm::TCP_CONN_NOTIFY, POOL_ALLOC_ARRAY, PGConnPool) so
// that this header compiles both inside gy_mconnhdlr.cc (with the real types) and stand-alone in this repository's tests (with
// the POD mirrors of gyeeta_b200/csrc/gysk_wire.h). See INTEGRATION.md for the call-site patch.
#pragma once

#include <cstdint>
#include <memory>
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

	// the 5-s reducer tick (TCP_SOCK_HANDLER::listener_stats_update cadence, common/gy_socket_stat.cc:3898)
	bool flush_window(uint32_t tsec) noexcept { return 0 == gysk_flush(engine_, tsec); }

	// The tick plus what the reference does when a partha reports a deleted listener (LISTENER_STATE_NOTIFY with
	// query_flags_ == LISTEN_FLAG_DELETE, common/gy_socket_stat.cc:4023-4033): with gysk_config.idle_evict_secs set, the ids the
	// engine evicted at this flush are handed to `on_delete(glob_id)` — the place to drop the MTCP_LISTENER of that id.
	template <typename OnDelete>
	bool flush_window(uint32_t tsec, OnDelete && on_delete) noexcept
	{
		if (0 != gysk_flush(engine_, tsec)) return false;
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

	gysk_engine		*engine_;
	std::vector<uint64_t>	evicted_;
	std::vector<gysk_svc_summary> summ_;
};

} // namespace gysk_shim
