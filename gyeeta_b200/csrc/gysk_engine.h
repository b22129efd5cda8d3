// gysk_engine.h — engine object shared by gysk_engine.cu (ingest / query) and gysk_merge.cu (multi-GPU merge).
#pragma once

#include "gysk_kernels.cuh"

#include <algorithm>
#include <atomic>
#include <memory>
#include <map>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <vector>

namespace gysk {

constexpr int NBUF = 2;
constexpr uint32_t QCHUNK = 1024;		// ids per query kernel launch
constexpr uint32_t WIN_ROWS = 8192;		// rows per pass of a window read (the page-locked stage holds WIN_ROWS service rows)
constexpr uint32_t THREAD_STAGE_EVENTS = 1u << 16;	// events per per-thread staging chunk (2 MB page-locked, two chunks per thread)
constexpr uint32_t RAW_BULK_MIN = 16384;		// raw fixed-stride batches from this size on are expanded on the device: below it the
							// per-call copy / launch / event calls under the engine mutex cost more than the
							// ~20 ns per record of expanding on the calling thread (bench.py e2e_wire)

// a calling thread's page-locked staging: filled without the engine mutex (see gysk_engine.cu). Invariant whenever m is released:
// buf[cur] has no H2D copy in flight, so a staging write into it never waits (the other chunk's copy may still be queued)
struct ThreadStage
{
	std::mutex		m;
	gysk_event		*buf[2] {};
	cudaEvent_t		copied[2] {};
	int			cur {0};
	uint32_t		fill {0}, cap {0};
	std::atomic<bool>	orphan {false};		// its thread has exited: the next new thread of this engine takes it over
};

// bounded top-N of one host's last message: BOUNDED_PRIO_QUEUE::try_emplace_locked semantics (common/gy_statistics.h:385-414:
// keep the N largest by the comparator; an element enters only when the queue has room or it beats the current minimum)
struct TopEntry { uint64_t id; uint64_t score; };
struct TopQueue
{
	static constexpr size_t N = 10;			// MAX_LISTEN_TOPN / MAX_TASK_TOPN per host, server/gy_mconnhdlr.h:961,975
	std::vector<TopEntry>	v;
	void offer(uint64_t id, uint64_t score)
	{
		if (!score) return;
		if (v.size() < N) { v.push_back({id, score}); std::push_heap(v.begin(), v.end(), [](const TopEntry &a, const TopEntry &b) { return a.score > b.score; }); return; }
		if (score <= v.front().score) return;
		std::pop_heap(v.begin(), v.end(), [](const TopEntry &a, const TopEntry &b) { return a.score > b.score; });
		v.back() = {id, score};
		std::push_heap(v.begin(), v.end(), [](const TopEntry &a, const TopEntry &b) { return a.score > b.score; });
	}
};

// the four listener rankings of partha_listener_state (server/gy_mconnhdlr.cc:11262-11304; comparators LISTEN_TOPN
// server/gy_msocket.h:720-797): by issue (state, then qps), qps, active connections, network kbytes
struct HostTopn
{
	TopQueue	q[4];			// GYSK_HOSTTOP_SVC_ISSUE, _QPS, _CONNS, _NET
	template <typename L> void offer(const L &l)
	{
		if (l.curr_state_ > 2) q[0].offer(l.glob_id_, ((uint64_t)l.curr_state_ << 32) | l.tasks_delay_usec_);	// is_comp_issue: state, then task delay (:745)
		if (l.nqrys_5s_ >= 5) q[1].offer(l.glob_id_, l.nqrys_5s_);						// :11273
		if (l.nconns_active_ >= 1) q[2].offer(l.glob_id_, l.nconns_active_);					// :11284
		q[3].offer(l.glob_id_, (uint64_t)l.curr_kbytes_inbound_ + l.curr_kbytes_outbound_);			// :11295 (offer skips 0)
	}
};
// the seven process rankings of partha_aggr_task_state (server/gy_mconnhdlr.cc:10012-10079; comparators MAGGR_TASK_STATE
// server/gy_msocket.h:454-531, MTASK_ISSUE :602): issue, net, cpu, rss, cpu delay, vm delay, blkio delay
struct HostTaskTopn
{
	TopQueue	q[7];
	template <typename T> void offer(const T &t)
	{
		// is_comp_issue (:602-606): more tasks with issues first; a severe aggregate beats a non-severe one
		if (t.curr_state_ > 2) q[0].offer(t.aggr_task_id_, ((uint64_t)((t.severe_issue_bit_hist_ & 1u) && t.ntasks_issue_) << 32) | ((uint64_t)t.ntasks_issue_ + 1));
		if (t.tcp_kbytes_ > 0) q[1].offer(t.aggr_task_id_, t.tcp_kbytes_);
		if (t.total_cpu_pct_ >= 0.1f) { uint32_t bits; memcpy(&bits, &t.total_cpu_pct_, 4); q[2].offer(t.aggr_task_id_, bits); }	// positive floats order like their bits
		if (t.rss_mb_ >= 5) q[3].offer(t.aggr_task_id_, t.rss_mb_);
		q[4].offer(t.aggr_task_id_, t.cpu_delay_msec_);
		q[5].offer(t.aggr_task_id_, t.vm_delay_msec_);
		q[6].offer(t.aggr_task_id_, t.blkio_delay_msec_);
	}
};

// one logical service's t-digest in the merge step: fixed size, so that the slabs all-gather as bytes
struct SlabEntry { TdHead head; Centroid cent[TD_CAP]; };
// GYSK_FLAG_MERGE_TRACES: one logical service's trace digest (compression TRACE_TD_DELTA keeps at most TRACE_TD_CAP centroids)
struct TraceSlab { TdHead head; Centroid cent[TRACE_TD_CAP]; };
static_assert(sizeof(TraceSlab) == 1632 && sizeof(TraceSlab) % 16 == 0, "TraceSlab: 32-byte head, 100 centroids");
// the trace digests of nl logical services in whole SlabEntrys, packed after the rank's digests and top-N candidates
inline uint32_t trace_slab_entries(uint32_t nl) { return (uint32_t)(((size_t)nl * sizeof(TraceSlab) + sizeof(SlabEntry) - 1) / sizeof(SlabEntry)); }
// GYSK_FLAG_SVC_TOP_CLIENTS: the two summaries of nl logical services (TopcSet [nl][2]: GYSK_TOPC_LAST, GYSK_TOPC_5MIN) in whole
// SlabEntrys, packed after the rest of a rank's slab
static_assert(2 * sizeof(TopcSet) == 528 && sizeof(SlabEntry) == 4128, "a logical service's two summaries are 528 bytes of a 4128-byte entry");
inline uint32_t topc_slab_entries(uint32_t nl) { return (uint32_t)(((size_t)nl * 2 * sizeof(TopcSet) + sizeof(SlabEntry) - 1) / sizeof(SlabEntry)); }
// u64 SUM words of one logical service's merged trace window: the sums of gysk_trace_window in its order, then the members holding a row
enum { LT_NREQ = 0, LT_NERR, LT_NCONNS, LT_SUM_US, LT_BYTES_IN, LT_BYTES_OUT, LT_BKT /* 8 words */, LT_TD_COUNT = LT_BKT + 8, LT_NTRACED,
	LT_WORDS };
// i64 MAX words: max_resp_us, max_bytes_in, max_bytes_out
enum { LT_MAX_US = 0, LT_MAX_IN, LT_MAX_OUT, LT_MAX_WORDS };
static_assert(LT_WORDS == 16, "15 sums and ntraced");

// LISTEN_SUMM_STATS words of one logical service: the 15 int32 fields of gysk_host_summary before its pad, nstates[0..7] first
constexpr int STATE_WORDS = 15;
static_assert(sizeof(gysk_host_summary) == (STATE_WORDS + 1) * sizeof(int32_t), "gysk_host_summary: 15 fields and a pad");

// The merged arrays of the nl logical services: the merge arena's per-logical arrays and the t-digest slabs, passed by value to the
// merge kernels. lvl .. rtt exist with GYSK_FLAG_MERGE_LEVELS only, flush with it, a count-min level or GYSK_FLAG_MERGE_TRACES, states with
// GYSK_FLAG_MERGE_STATES only (nullptr without).
struct LogicalArrays
{
	uint32_t		nl {0};
	HistCell		*last {nullptr}, *all {nullptr};	// SUM [nl][16]: last-window / all-time histograms, cells 0..14
	unsigned long long	*conn {nullptr};			// SUM [nl][4]: last cnt, last kb, all cnt, all kb
	HistCell		*lvl {nullptr};				// SUM [2][nl][16]: the live ring slots of the 300-s / 5-day levels, cells 0..14
	unsigned long long	*aux {nullptr};				// SUM [nl][4]: active conns, active kbytes, client errors, server errors
	unsigned long long	*states {nullptr};			// SUM [nl][STATE_WORDS]: the members' LISTEN_SUMM_STATS, each word mod 2^32
	long long		*hmax {nullptr};			// MAX [nl][2]: max_val_seen_ of last, all
	long long		*lvl_max {nullptr};			// MAX [nl][2]: max_val_seen_ of the 300-s / 5-day levels
	long long		*rtt {nullptr};				// MAX [nl]: the largest rtt_last bit pattern (a non-negative float's order)
	long long		*flush {nullptr};			// MAX [2]: {last_flush_tsec, -last_flush_tsec} of this engine
	uint8_t			*hll {nullptr};				// MAX [nl][1 << hll_p]
	SlabEntry		*slab {nullptr};			// [nl] this engine's folded digests
	SlabEntry		*final_slab {nullptr};			// [nl] merged over ranks
	// GYSK_FLAG_MERGE_TRACES (nullptr without): the members' last trace windows
	unsigned long long	*traces {nullptr};			// SUM [nl][LT_WORDS]
	long long		*trace_max {nullptr};			// MAX [nl][LT_MAX_WORDS]
	TraceSlab		*trace_slab {nullptr};			// [nl] this engine's folded trace digests, inside the slab (MergeState::trace_off)
	TraceSlab		*trace_final {nullptr};			// [nl] merged over ranks

	// histogram `which` (GYSK_HIST_RESP_LAST, _ALL, _5MIN or _5DAY) of logical service l: its cells 0..14 and its max_val_seen_
	struct Hist { HistCell *cells; long long *max; };
	__host__ __device__ __forceinline__ Hist hist(int which, uint32_t l) const
	{
		if (which == GYSK_HIST_RESP_LAST) return Hist {last + (size_t)l * HIST_CELLS, hmax + 2 * (size_t)l};
		if (which == GYSK_HIST_RESP_ALL) return Hist {all + (size_t)l * HIST_CELLS, hmax + 2 * (size_t)l + 1};
		const int k = which - GYSK_HIST_RESP_5MIN;
		return Hist {lvl + ((size_t)k * nl + l) * HIST_CELLS, lvl_max + 2 * (size_t)l + k};
	}
	// cell c of that histogram as a row shows it: cell 15 holds max_val_seen_
	__device__ __forceinline__ HistCell cell(int which, uint32_t l, int c) const
	{
		const Hist h = hist(which, l);
		HistCell x = h.cells[c];
		if (c == HIST_MAX_CELL) x.sum = *h.max;
		return x;
	}
	__host__ __device__ __forceinline__ unsigned long long *conn_of(uint32_t l) const { return conn + 4 * (size_t)l; }
	__host__ __device__ __forceinline__ unsigned long long *aux_of(uint32_t l) const { return aux + 4 * (size_t)l; }
	__host__ __device__ __forceinline__ unsigned long long *states_of(uint32_t l) const { return states + STATE_WORDS * (size_t)l; }
	// member listeners in STATE_BAD, STATE_SEVERE or STATE_DOWN: MS_CLUSTER_STATE's nsvc_issue (gysk_query_cluster_state)
	__host__ __device__ __forceinline__ uint32_t nsvc_issue(uint32_t l) const
	{
		const unsigned long long *w = states_of(l);
		return (uint32_t)(w[GYSK_STATE_BAD] + w[GYSK_STATE_SEVERE] + w[GYSK_STATE_DOWN]);
	}
	__host__ __device__ __forceinline__ uint8_t *hll_of(uint32_t l, uint32_t hll_p) const { return hll + ((size_t)l << hll_p); }
	__host__ __device__ __forceinline__ unsigned long long *traces_of(uint32_t l) const { return traces + LT_WORDS * (size_t)l; }
	__host__ __device__ __forceinline__ long long *trace_max_of(uint32_t l) const { return trace_max + LT_MAX_WORDS * (size_t)l; }
};

// The members of each logical service on this GPU, CSR in map order: slots[offs[l] .. offs[l + 1]) are logical l's. A member whose id
// holds no slot here is written as null_slot (resolve_members_kernel): the engine's null slot max_svcs, which every fold skips.
struct Members
{
	uint32_t		*offs {nullptr}, *slots {nullptr};
	uint32_t		null_slot {0};

	// f(slot) for each member of logical l that holds a slot, in map order. The walk only reads the map: __restrict__ lets its loads
	// take the read-only path.
	template <typename F> __device__ __forceinline__ void each(uint32_t l, F f) const
	{
		const uint32_t *__restrict__ o = offs, *__restrict__ sl = slots;
		for (uint32_t m = o[l]; m < o[l + 1]; ++m) {
			const uint32_t s = sl[m];
			if (s != null_slot) f(s);
		}
	}
};

// SUM words of one host cluster (GYSK_FLAG_MERGE_CLUSTERS): the fields of gysk_cluster_state before its pad, in its order
constexpr int CLUSTER_WORDS = 6;
static_assert(sizeof(gysk_cluster_state) == (CLUSTER_WORDS + 2) * sizeof(uint32_t), "gysk_cluster_state: 6 fields and a pad");
static_assert(sizeof(gysk_cluster_row) == 48, "gysk_cluster_row is 48 bytes");
constexpr uint32_t MAX_CLUSTER_HOST = 1u << 24;		// gysk_set_cluster_map: host_of is indexed by host_idx

// The host clusters on the device, passed by value to the cluster kernels. Each mapped host has a dense index, a cluster's hosts next to
// each other in map order. host_acc gathers this engine's per-host sums during gysk_merge_prepare and is zero between merges (the host
// pass clears what it reads).
struct Clusters
{
	uint32_t		nc {0}, nh {0};				// clusters, mapped hosts
	uint32_t		ntab {0};				// entries of host_of: 1 + the largest mapped host_idx
	uint32_t		*host_of {nullptr};			// [ntab] host_idx -> dense host index, ~0u: in no cluster
	uint32_t		*offs {nullptr};			// [nc + 1] the dense hosts of cluster c are offs[c] .. offs[c + 1] - 1
	uint4			*host_acc {nullptr};			// [nh] {nlisten, nlisten_issue, tot_qps, tot_kb_inbound}, each mod 2^32
	unsigned long long	*words {nullptr};			// SUM [nc][CLUSTER_WORDS] in the merge arena

	__host__ __device__ __forceinline__ unsigned long long *words_of(uint32_t c) const { return words + CLUSTER_WORDS * (size_t)c; }
};

// the cluster map of gysk_set_cluster_map (GYSK_FLAG_MERGE_CLUSTERS)
struct ClusterMap
{
	std::vector<uint64_t>	ids;					// dense index -> cluster id
	std::unordered_map<uint64_t, uint32_t> index;		// cluster id -> dense index
	Clusters		cl;
	unsigned long long	*d_ids {nullptr};			// [nc] ids on the device: the ids of the rows
	int32_t			*d_sorted {nullptr};			// [nc] dense indices by ascending cluster id (gysk_query_cluster_states_all)
	int32_t			*d_sel {nullptr};			// [nc] the part of d_sorted an ACTIVE_ONLY read selects
};

// GYSK_FLAG_MERGE_TOPN: the TOPN_K best services by each service metric (GYSK_TOPN_QPS .. GYSK_TOPN_ACTIVE) and processes by each task
// metric (GYSK_TOPN_TASK_CPU .. _BLKIO_DELAY), list m = the service metric or TOPN_SVC_LISTS + the task metric. One rank's candidates
// (appended to its t-digest slab, so the all-gather carries them) and the merge's winners have the same layout: the entries of every list
// [TOPN_LISTS][TOPN_K], best first, then the rows of the service lists and of the task lists, each row its owner's gysk_query_svcs /
// gysk_query_tasks row (the service rows before the host's hll_finish). Every offset is 16-byte aligned.
constexpr uint32_t TOPN_K = 64, TOPN_SVC_LISTS = 5, TOPN_LISTS = TOPN_SVC_LISTS + 3;
struct TopnLists
{
	static constexpr size_t ENT = 0, SVC_ROW = ENT + (size_t)TOPN_LISTS * TOPN_K * sizeof(gysk_topn_entry),
		TASK_ROW = SVC_ROW + (size_t)TOPN_SVC_LISTS * TOPN_K * sizeof(gysk_svc_summary),
		BYTES = TASK_ROW + (size_t)(TOPN_LISTS - TOPN_SVC_LISTS) * TOPN_K * sizeof(gysk_task_summary);
	uint8_t			*base;

	__host__ __device__ __forceinline__ gysk_topn_entry *ent(uint32_t m) const { return reinterpret_cast<gysk_topn_entry *>(base + ENT) + (size_t)m * TOPN_K; }
	__host__ __device__ __forceinline__ static size_t row_bytes(uint32_t m) { return m < TOPN_SVC_LISTS ? sizeof(gysk_svc_summary) : sizeof(gysk_task_summary); }
	// row i of list m
	__host__ __device__ __forceinline__ uint8_t *row(uint32_t m, uint32_t i) const
	{
		return m < TOPN_SVC_LISTS ? base + SVC_ROW + ((size_t)m * TOPN_K + i) * sizeof(gysk_svc_summary)
					  : base + TASK_ROW + ((size_t)(m - TOPN_SVC_LISTS) * TOPN_K + i) * sizeof(gysk_task_summary);
	}
};
static_assert(TopnLists::SVC_ROW % 16 == 0 && TopnLists::TASK_ROW % 16 == 0 && sizeof(SlabEntry) % 16 == 0, "16-byte aligned rows");
// the candidates' whole SlabEntrys after a rank's nl digests
constexpr uint32_t TOPN_SLAB_ENTRIES = (uint32_t)((TopnLists::BYTES + sizeof(SlabEntry) - 1) / sizeof(SlabEntry));

// The count-min tables an engine can hold, each [cms_depth][1 << cms_log2_width] cells of one or more u64 words (CMS_TABLES below says
// which flag each one needs, its array in the merge arena, where the engine keeps it and its words per cell). Each windowed pair is an
// open table and, right after it, the table of the window the last flush closed. A new table goes last, so that every engine without it
// keeps its merge arena.
enum CmsTable { CMS_CUR, CMS_LAST, CMS_5MIN, CMS_QRY_CUR, CMS_QRY_LAST, CMS_QRY_5MIN, CMS_RESP_CUR, CMS_RESP_LAST, CMS_RESP_5MIN, CMS_ERR_CUR,
	CMS_ERR_LAST, CMS_ERR_5MIN, NCMS };
// the flow query table of the same window as flow error table t (gysk_flow_err_est.queries)
constexpr int cms_err_queries(int t) { return t - CMS_ERR_CUR + CMS_QRY_CUR; }

// GYSK_FLAG_FLOW_TOPK (every pointer nullptr without): the candidate lists and the open / last heaviest-flow sets ([TOPK_SET_WORDS]
// each) of the connection table [0] and, with GYSK_FLAG_FLOW_QUERIES, the flow query table [1]; with GYSK_FLAG_FLOW_TOPK_SLOW the slow
// set of the response histogram table [2], b_slow its first slow bucket (gysk_set_flow_slow); with GYSK_FLAG_FLOW_ERRORS the server-error
// set of the flow error table [3] (its candidates are FlowErrors::list, topk_list). Outside DevState, so that the kernels without the
// flag keep their parameter layout; not per slot, so gysk_grow and eviction leave them.
constexpr int TOPK_SETS = 4;
struct TopkSets { FlowTopk tk; unsigned long long *open[TOPK_SETS], *last[TOPK_SETS]; uint32_t b_slow; };
// the count-min table of each set, and the half of its cells that scores (1: kbytes, the high half; 0: queries, the low half; the slow
// set's score is topk_score's; 1: ser_errors, the high half)
constexpr int TOPK_TABLE[TOPK_SETS] = {CMS_CUR, CMS_QRY_CUR, CMS_RESP_CUR, CMS_ERR_CUR}, TOPK_HALF[TOPK_SETS] = {1, 0, 0, 1};
// the score of set w (launch_topk_select): TOPK_HALF[w], or the slow score from bucket b_slow
inline int topk_score(const TopkSets &t, int w) { return w != 2 ? TOPK_HALF[w] : TOPK_SCORE_SLOW | (int)t.b_slow; }
// GYSK_FLAG_FLOW_TOPK_SLOW's default threshold: a sample above 300 ms is slow (RESP_TIME_HASH bucket 9 and up)
constexpr uint32_t TOPK_SLOW_DEFAULT_B = 9;
// nsets sets of a rank in the merge slab, in whole SlabEntrys after the rest of its content
constexpr uint32_t topk_slab_entries(uint32_t nsets)
{
	return (uint32_t)((nsets * TOPK_SET_WORDS * sizeof(unsigned long long) + sizeof(SlabEntry) - 1) / sizeof(SlabEntry));
}
constexpr uint32_t TOPK_SLAB_ENTRIES = topk_slab_entries(2);

// GYSK_FLAG_FLOW_TOPK_5MIN (every pointer nullptr without): per held level [w] (w as TopkSets; the level of CMS_RINGS[w]) the sets of
// its NSLOTS ring slots ([NSLOTS][TOPK_SET_WORDS], word 1 each slot's bound B_s) and the level set L ([TOPK_SET_WORDS], word 1 B_L);
// one candidate list of NSLOTS x K keys for the flush chain, and a word for its partial bound. Outside DevState and not per slot, as
// TopkSets.
// [2]: GYSK_FLAG_FLOW_TOPK_SLOW's slow set of the response level (with GYSK_FLAG_FLOW_QUERY_LEVEL), scored as the window's; [3]:
// GYSK_FLAG_FLOW_ERRORS's server-error set of the error level, alike.
struct Topk5min { unsigned long long *slots[TOPK_SETS], *level[TOPK_SETS]; TopkList list; unsigned long long *acc; };
// the level table of each set (the score is topk_score's)
constexpr int TOPK5_LEVEL[TOPK_SETS] = {CMS_5MIN, CMS_QRY_5MIN, CMS_RESP_5MIN, CMS_ERR_5MIN};

// the cells of one count-min table
inline size_t cms_cells(const gysk_config &cfg) { return (size_t)cfg.cms_depth << cfg.cms_log2_width; }

// per-logical-service state of the merge step (SURVEY.md §8e)
struct MergeState
{
	std::vector<uint64_t>	logical_ids;		// dense index -> logical id
	std::unordered_map<uint64_t, uint32_t> index;	// logical id -> dense index
	Members			members;
	unsigned long long	*d_member_ids {nullptr};			// id each member slot held when the map was set
	unsigned long long	*d_logical_ids {nullptr};			// [nl] logical_ids on the device: the ids of the rows and top-N entries
	int32_t			*d_sorted {nullptr};				// [nl] dense indices by ascending logical id (gysk_query_logical_all)
	int32_t			*d_sel {nullptr};				// [nl] the part of d_sorted an ACTIVE_ONLY read selects
	uint32_t		nmembers {0};
	// one arena so that each reduction kind is a single collective
	uint8_t			*arena {nullptr};
	size_t			arena_bytes {0};
	size_t			off_sum {0}, bytes_sum {0};		// u64 SUM : cms cur/last [, 5min] [, cmsq cur/last [, 5min]] [, cmsr cur/last [, 5min]], hist
									//           last/all, conn [, levels, aux] [, states] [, clusters] [, traces]
	size_t			off_maxi64 {0}, bytes_maxi64 {0};	// i64 MAX : histogram max_val_seen_ [, level maxima, rtt] [, flush tsec]
									//           [, trace max]
	size_t			off_maxu8 {0}, bytes_maxu8 {0};		// u8  MAX : HLL registers
	std::string		name_sum, name_maxi64, name_maxu8;	// the regions' gysk_buffer_desc names: their arrays, in order
	unsigned long long	*g_cms[NCMS] {};			// the engine's count-min tables summed over ranks (nullptr: not held)
	LogicalArrays		lg;
	ClusterMap		clusters;				// kept across gysk_set_logical_map
	bool			prepared {false}, finished {false};
	void			*comm {nullptr};			// ncclComm_t of gysk_nccl_comm_init
	uint32_t		comm_world {0};
	bool			comm_owned {false};
	SlabEntry		*gathered {nullptr};			// [world] slabs, target of the all-gather
	uint32_t		gathered_world {0};
	// GYSK_FLAG_MERGE_TOPN: lg.slab holds slab_entries = nl + TOPN_SLAB_ENTRIES (nl without the flag), the candidates from lg.slab + nl;
	// GYSK_FLAG_MERGE_TRACES: trace_slab_entries(nl) more from lg.slab + trace_off, the trace digests
	uint32_t		slab_entries {0};
	uint32_t		trace_off {0};
	unsigned long long	*topn_slots {nullptr};			// [TOPN_LISTS][TOPN_K] this rank's candidate slots (the rows' input)
	uint8_t			*topn_final {nullptr};			// TopnLists::BYTES: the winners of the last finished merge
	// GYSK_FLAG_FLOW_TOPK: the rank's last-window sets ride from slab entry topk_off (TOPK_SLAB_ENTRIES); the merged sets of the last
	// finished merge ([2][TOPK_SET_WORDS]); the union's candidates and sort buffers (3 x topk_cap keys, with their look-back tiles)
	uint32_t		topk_off {0};
	unsigned long long	*topk_final {nullptr};
	bool			topk_done {false};
	unsigned long long	*topk_buf {nullptr}, *topk_n {nullptr}, *topk_tiles {nullptr};
	uint64_t		topk_cap {0};
	// GYSK_FLAG_FLOW_TOPK_5MIN: the rank's level sets ride from slab entry topk5_off (TOPK_SLAB_ENTRIES); the merged sets of the last
	// finished merge with their bounds ([2][TOPK_SET_WORDS]). They share the window sets' union buffers.
	uint32_t		topk5_off {0};
	unsigned long long	*topk5_final {nullptr};
	// GYSK_FLAG_FLOW_TOPK_SLOW: the rank's last-window slow set and, with its 300-s level, L with B_L ride from slab entry topks_off
	// (topk_slab_entries(1 or 2)); the merged ones land as set [2] of topk_final and topk5_final, which then hold three sets.
	uint32_t		topks_off {0};
	// GYSK_FLAG_FLOW_ERRORS with GYSK_FLAG_FLOW_TOPK: the rank's last-window server-error set and, with its 300-s level, L with B_L ride
	// from slab entry topke_off, after the slow sets (topk_slab_entries(1 or 2)); the merged ones land as set [3] of topk_final and
	// topk5_final, which then hold four sets.
	uint32_t		topke_off {0};
	// GYSK_FLAG_SVC_TOP_CLIENTS: the rank's per-logical summaries (fold_topc_kernel) ride from slab entry topc_off, after everything else
	// (topc_slab_entries(nl)); the merged ones of the last finished merge, [nl][2] as in the slab (nullptr without)
	uint32_t		topc_off {0};
	TopcSet			*topc_final {nullptr};
	// GYSK_FLAG_CLIENT_LEVELS: MAX [nl][2][CL_REGS] in the u8 MAX region after the all-time registers, each logical service's last-window
	// and 300-s client sets (nullptr without)
	uint8_t			*cl_hll {nullptr};
	__host__ __device__ __forceinline__ uint8_t *cl_of(uint32_t l, int which) const { return cl_hll + ((size_t)l * 2 + which) * CL_REGS; }
};

} // namespace gysk

struct gysk_engine
{
	gysk_config		cfg {};
	int			dev {0};
	cudaStream_t		stream {nullptr}, copy_stream {nullptr};
	gysk::DevState		st {};
	gysk::SortTemp		tmp {};
	gysk::FlowQueries	fq {};				// GYSK_FLAG_FLOW_QUERIES (every pointer nullptr without)
	gysk::FlowRespHist	fr {};				// GYSK_FLAG_FLOW_RESP_HIST (every pointer nullptr without)
	gysk::TopkSets		topk {};			// GYSK_FLAG_FLOW_TOPK (every pointer nullptr without)
	gysk::Topk5min		topk5 {};			// GYSK_FLAG_FLOW_TOPK_5MIN (every pointer nullptr without)
	gysk::ClientLevels	cl {};				// GYSK_FLAG_CLIENT_LEVELS (every pointer nullptr without)
	gysk::FlowErrors	fe {};				// GYSK_FLAG_FLOW_ERRORS (every pointer nullptr without)
	gysk::SvcTopClients	tc {};				// GYSK_FLAG_SVC_TOP_CLIENTS (every pointer nullptr without)
	std::atomic<bool>	fed {false};			// an event was handed in or gysk_flush ran (gysk_set_flow_slow refuses after)
	std::vector<std::pair<void *, size_t>> dallocs;		// every device buffer and its bytes
	size_t			dbytes {0};			// their sum (gysk_capacity_info's device_bytes)
	std::vector<void *>	hallocs;

	// capacity growth (gysk_grow, gysk_set_auto_grow): the auto-grow ceilings (0 = never), and the slot counts as of the last flush,
	// copied behind its kernels and read at the next one ({services handed out, services on the free stack, processes handed out,
	// processes on the free stack})
	uint32_t		grow_limit_svcs {0}, grow_limit_tasks {0};
	uint32_t		ngrows {0};
	uint32_t		*h_used {nullptr};
	cudaEvent_t		ev_used {nullptr};
	bool			used_pending {false};

	// staging: per-thread page-locked chunks -> device event buffers (double-buffered) -> kernels
	uint64_t		uid {0};
	std::mutex		tstage_mtx;
	std::vector<std::unique_ptr<gysk::ThreadStage>> tstages;
	gysk_event		*d_events[gysk::NBUF] {};
	cudaEvent_t		ev_copied[gysk::NBUF] {}, ev_done[gysk::NBUF] {};
	uint32_t		stage_fill {0};			// events of d_events[stage_cur] whose copies are enqueued
	int			stage_cur {0};
	uint8_t			*d_raw[gysk::NBUF] {};		// raw records on their way to decode_raw_kernel
	size_t			raw_bytes {0};
	cudaEvent_t		ev_raw_done[gysk::NBUF] {};
	int			raw_cur {0};

	// query scratch (staged_read). The stage is only valid under mtx: every read copies its result out of it before it returns.
	unsigned long long	*d_qids {nullptr}, *h_qids {nullptr};		// a piece of a read's input: QCHUNK ids, keys or logical indices
	unsigned long long	*h_counters {nullptr};
	uint8_t			*d_wstage {nullptr}, *h_wstage {nullptr};	// every read's output: WIN_ROWS summary rows per window-read pass,
										// QCHUNK rows per by-id pass, one id's raw state, the top-N entries
	std::vector<uint64_t>	win_keys, win_ids;			// a window read's {host | slot} keys and their ids on the host
	std::vector<std::pair<uint64_t, uint64_t>> win_rows;		// ... as {id, slot}, ordered within each host

	// optional per-kernel timing
	bool			profiling {false};
	std::vector<cudaEvent_t> prof_events;		// triples: before ingest, after the drain passes, after t-digest chain
	size_t			prof_used {0};

	// rolling levels: epoch held by each ring slot (~0 = never written; roll_levels) and the time of the last flush
	uint64_t		ring_epoch[gysk::NLEVELS][gysk::NSLOTS];
	uint32_t		last_flush_tsec {0};

	// idle-service eviction: ids evicted by the last flush arrive lagged (copied behind the flush kernels, read at the next call)
	unsigned long long	*h_evict {nullptr};			// [0] = count, [1..] = ids (pinned)
	cudaEvent_t		ev_evict {nullptr};
	bool			evict_pending {false};
	std::vector<uint64_t>	evicted_ids;				// of the last completed flush
	uint64_t		tombstones {0}, evicted_total {0};
	uint64_t		h_evict_fail {0};			// CTR_INSERT_FAIL as of the last collected flush
	uint64_t		insert_fail_seen {0};			// CTR_INSERT_FAIL at the last table rebuild
	// process eviction (task_idle_evict_secs): the eviction kernel writes the count and ids of each flush straight into h_tevict (page-
	// locked and mapped, d_tevict on the device: [0] = count, [1 .. max_tasks] = ids); collected with the services' list, under ev_evict
	unsigned long long	*h_tevict {nullptr}, *d_tevict {nullptr};
	std::vector<uint64_t>	evicted_task_ids;			// of the last completed flush, ascending
	uint64_t		task_tombstones {0}, task_evicted_total {0};
	uint32_t		sort_epoch {0};				// radix passes launched so far (tags the look-back status words)

	std::mutex		host_mtx;					// the per-host control-plane state below
	std::unordered_map<uint32_t, gysk_host_summary> host_summ;	// last LISTEN_SUMM_STATS per host (control-plane sized: <= 512 hosts)
	std::unordered_map<uint32_t, gysk::HostTopn> host_topn;		// top-N listeners of each host's last NOTIFY_LISTENER_STATE
	std::unordered_map<uint32_t, gysk::HostTaskTopn> host_task_topn;	// top-N aggregated processes of each host's last NOTIFY_AGGR_TASK_STATE

	gysk::MergeState	mg;

	std::mutex		mtx;
	std::string		err;
	bool			sticky {false};
	std::atomic<uint64_t>	wire_ok {0}, wire_bad {0};
	uint64_t		kernel_launches {0}, batches {0}, merges {0};
};

namespace gysk {

// slot_last_active of the window the last flush closed (state_kernel): the active_mark of svc_evaluated / svc_issue
inline uint32_t active_mark(const gysk_engine *e) { return e->last_flush_tsec ? e->last_flush_tsec : 1u; }

// one count-min table of CmsTable: the gysk_config flags it needs (0: every engine holds it), its array in the merge arena's SUM region
// (gysk_merge_buffers), the engine's live table, and the u64 words of one cell
struct CmsTableDesc
{
	uint32_t		flag;
	const char		*name;
	unsigned long long	*&(*live)(gysk_engine *);
	uint32_t		words;
};
inline const CmsTableDesc CMS_TABLES[NCMS] = {
	{0, "cms_cur", [](gysk_engine *e) -> unsigned long long *& { return e->st.cms_cur; }, 1},
	{0, "cms_last", [](gysk_engine *e) -> unsigned long long *& { return e->st.cms_last; }, 1},
	{GYSK_FLAG_FLOW_LEVEL, "cms_5min", [](gysk_engine *e) -> unsigned long long *& { return e->st.cms_5min; }, 1},
	{GYSK_FLAG_FLOW_QUERIES, "cms_qry_cur", [](gysk_engine *e) -> unsigned long long *& { return e->fq.cur; }, 1},
	{GYSK_FLAG_FLOW_QUERIES, "cms_qry_last", [](gysk_engine *e) -> unsigned long long *& { return e->fq.last; }, 1},
	{GYSK_FLAG_FLOW_QUERY_LEVEL, "cms_qry_5min", [](gysk_engine *e) -> unsigned long long *& { return e->fq.level; }, 1},
	{GYSK_FLAG_FLOW_RESP_HIST, "cms_resp_cur", [](gysk_engine *e) -> unsigned long long *& { return e->fr.cur; }, RESP_HIST_WORDS},
	{GYSK_FLAG_FLOW_RESP_HIST, "cms_resp_last", [](gysk_engine *e) -> unsigned long long *& { return e->fr.last; }, RESP_HIST_WORDS},
	{GYSK_FLAG_FLOW_RESP_HIST | GYSK_FLAG_FLOW_QUERY_LEVEL, "cms_resp_5min", [](gysk_engine *e) -> unsigned long long *& { return e->fr.level; },
			RESP_HIST_WORDS},
	{GYSK_FLAG_FLOW_ERRORS, "cms_err_cur", [](gysk_engine *e) -> unsigned long long *& { return e->fe.cur; }, 1},
	{GYSK_FLAG_FLOW_ERRORS, "cms_err_last", [](gysk_engine *e) -> unsigned long long *& { return e->fe.last; }, 1},
	{GYSK_FLAG_FLOW_ERRORS | GYSK_FLAG_FLOW_QUERY_LEVEL, "cms_err_5min", [](gysk_engine *e) -> unsigned long long *& { return e->fe.level; }, 1},
};
inline bool cms_held(const gysk_config &cfg, int t) { return (cfg.flags & CMS_TABLES[t].flag) == CMS_TABLES[t].flag; }
// the u64 words of count-min table t
inline size_t cms_words(const gysk_config &cfg, int t) { return cms_cells(cfg) * CMS_TABLES[t].words; }

// A rolling 300-s level of a windowed pair: at each flush the open table `open` goes into a ring of NSLOTS tables by level 0's decision of
// roll_levels, and the level table `level` becomes the sum of the live slots (launch_cms_level_roll). The engine holds the ring with the
// level table.
struct CmsRingDesc
{
	int			open, level;
	unsigned long long	*&(*ring)(gysk_engine *);
};
inline const CmsRingDesc CMS_RINGS[] = {
	{CMS_CUR, CMS_5MIN, [](gysk_engine *e) -> unsigned long long *& { return e->st.cms_ring; }},
	{CMS_QRY_CUR, CMS_QRY_5MIN, [](gysk_engine *e) -> unsigned long long *& { return e->fq.ring; }},
	{CMS_RESP_CUR, CMS_RESP_5MIN, [](gysk_engine *e) -> unsigned long long *& { return e->fr.ring; }},
	{CMS_ERR_CUR, CMS_ERR_5MIN, [](gysk_engine *e) -> unsigned long long *& { return e->fe.ring; }},
};

// the candidate list of heaviest-flow set w: FlowTopk's, or for the server-error set FlowErrors'
inline TopkList &topk_list(gysk_engine *e, int w) { return w < 3 ? e->topk.tk.list[w] : e->fe.list; }

int fail(gysk_engine *e, int code, const char *what, cudaError_t ce = cudaSuccess);
int post_launch(gysk_engine *e, const char *what);
int submit_stage(gysk_engine *e);
int drain_all(gysk_engine *e);
int sync_locked(gysk_engine *e);
void merge_release(gysk_engine *e);
// the Postgres text and the quantiles of one exported digest; export_td is gysk_export_tdigest or gysk_export_logical_tdigest
using ExportTd = int (*)(gysk_engine *, uint64_t, double *, uint64_t *, uint32_t, uint32_t *, double *, double *);
int tdigest_pgtext(gysk_engine *e, uint64_t id, ExportTd export_td, char *buf, uint32_t cap);
int tdigest_quantiles(gysk_engine *e, uint64_t id, ExportTd export_td, const double *qs, uint32_t nq, double *out);
// HIST_SERIAL of 16 cells (cell HIST_MAX_CELL holds max_val_seen_ in .sum); total = the sum of the first nb counts
void hist_from_cells(const HistCell *cells, int nb, gysk_hist_serial *out, uint64_t *total, int64_t *maxv, bool t_is_int);
// a 5-minute or 5-day level as gysk_export_hist answers it: hist_from_cells, and maxv = INT64_MIN while the level is empty
void level_from_cells(const HistCell *cells, gysk_hist_serial *out, uint64_t *total, int64_t *maxv);
// the gysk_export_tdigest answer of one digest: up to min(cap, TD_CAP) centroids, min and max; GYSK_ERR_NOSPC when it has more than cap
int tdigest_out(const TdHead &head, const Centroid *cent, double *means, uint64_t *weights, uint32_t cap, uint32_t *n, double *minv, double *maxv);
// The count-min point queries of the flow query ABI calls on table t: the engine's own (the batch of the events handed in runs first) or,
// merged, the last merge's sum over the ranks. GYSK_ERR_NOTSUP when the engine does not hold t; `what` names the call.
int query_cms(gysk_engine *e, int t, bool merged, const uint64_t *keys, uint32_t n, gysk_flow_est *out, const char *what);
// GYSK_FLAG_FLOW_TOPK: the first min(n, K) flows of heaviest-flow set `which` (0: connections, 1: flow queries, 2: slow responses), best
// first, with their estimates on its table: the engine's open (last_window = 0) or last set, or merged, the last finished merge's set on
// the summed table. level (GYSK_FLAG_FLOW_TOPK_5MIN): the 300-s level set instead, on the level (merged: the summed level), last_window
// ignored. Flows with a zero score are left out; *bound (if not nullptr) = the set's word 1. Row: gysk_flow_est for sets 0 and 1,
// gysk_flow_resp_est for set 2, gysk_flow_err_est for set 3 (server errors).
template <typename Row>
int topk_read(gysk_engine *e, int which, int last_window, bool level, bool merged, uint32_t n, Row *out, uint32_t *nout,
		uint64_t *bound, const char *what);
// the same on a flow error table (CMS_ERR_*), each row's queries from the flow query table of the same window
int query_cms_err(gysk_engine *e, int t, bool merged, const uint64_t *keys, uint32_t n, gysk_flow_err_est *out, const char *what);
// the same on a flow response histogram table (CMS_RESP_*)
int query_cms_resp(gysk_engine *e, int t, bool merged, const uint64_t *keys, uint32_t n, gysk_flow_resp_est *out, const char *what);

#define CU(e, call) do { cudaError_t ce__ = (call); if (ce__ != cudaSuccess) return gysk::fail((e), GYSK_ERR_CUDA, #call, ce__); } while (0)
#define CHECK_ENGINE(e) do { if (!(e)) return GYSK_ERR_INVAL; if ((e)->sticky) return GYSK_ERR_CUDA; } while (0)

// What an ABI call does with the events of the current device buffer when it enters: leave them (Drain: only every thread's
// partial chunk is handed over), run their batch (Submit: the call sees every event handed in before it), or run it and wait for
// both streams (Sync: the call reads results on the host).
enum class Pending { Drain, Submit, Sync };

// One ABI call's hold on the engine: every thread's partial chunk goes to the device, then the engine mutex is taken, the device
// selected and the pending events handled as `mode` says. A non-zero rc is the call's error; the mutex is held only when rc is 0.
struct Entry
{
	std::unique_lock<std::mutex> lk;
	int rc;
	Entry(gysk_engine *e, Pending mode) : rc(drain_all(e))
	{
		if (rc) return;
		lk = std::unique_lock<std::mutex>(e->mtx);
		const cudaError_t ce = cudaSetDevice(e->dev);
		if (ce != cudaSuccess) rc = fail(e, GYSK_ERR_CUDA, "cudaSetDevice(e->dev)", ce);
		else if (mode == Pending::Submit) rc = submit_stage(e);
		else if (mode == Pending::Sync) rc = sync_locked(e);
	}
};
#define GYSK_ENTER(e, mode) gysk::Entry entry__((e), gysk::Pending::mode); if (entry__.rc) return entry__.rc

template <typename T>
int dalloc(gysk_engine *e, T **p, size_t n, bool zero = true)
{
	void *q = nullptr;
	cudaError_t ce = cudaMalloc(&q, n * sizeof(T));

	if (ce != cudaSuccess) {
		cudaGetLastError();		// an allocation failure is not sticky: it must not surface at the next launch check
		return fail(e, GYSK_ERR_NOMEM, "cudaMalloc", ce);
	}
	e->dallocs.emplace_back(q, n * sizeof(T));
	e->dbytes += n * sizeof(T);
	if (zero) {
		ce = cudaMemsetAsync(q, 0, n * sizeof(T), e->stream);
		if (ce != cudaSuccess) return fail(e, GYSK_ERR_CUDA, "cudaMemsetAsync", ce);
	}
	*p = static_cast<T *>(q);
	return 0;
}

// frees a buffer of dalloc (nullptr: nothing to free) and clears the pointer
template <typename T>
void dfree(gysk_engine *e, T *&p)
{
	if (!p) return;
	cudaFree(p);
	for (size_t i = 0; i < e->dallocs.size(); ++i) {
		if (e->dallocs[i].first != (void *)p) continue;
		e->dbytes -= e->dallocs[i].second;
		e->dallocs.erase(e->dallocs.begin() + i);
		break;
	}
	p = nullptr;
}

// frees a buffer of halloc and clears the pointer
template <typename T>
void hfree(gysk_engine *e, T *&p)
{
	if (!p) return;
	cudaFreeHost(p);
	e->hallocs.erase(std::remove(e->hallocs.begin(), e->hallocs.end(), (void *)p), e->hallocs.end());
	p = nullptr;
}

template <typename T>
int halloc(gysk_engine *e, T **p, size_t n, unsigned flags = cudaHostAllocDefault)
{
	void *q = nullptr;
	cudaError_t ce = cudaHostAlloc(&q, n * sizeof(T), flags);

	if (ce != cudaSuccess) {
		cudaGetLastError();
		return fail(e, GYSK_ERR_NOMEM, "cudaHostAlloc", ce);
	}
	e->hallocs.push_back(q);
	*p = static_cast<T *>(q);
	return 0;
}

// ---- the read path: one stage for every read -------------------------------------------------------------------

constexpr size_t STAGE_BYTES = (size_t)WIN_ROWS * sizeof(gysk_svc_summary);
constexpr size_t HLL_STAGE_REGS = 16;		// gysk_export_hll: the found word at the head of the stage, the registers from here on
static_assert(sizeof(gysk_task_summary) <= sizeof(gysk_svc_summary) && QCHUNK <= WIN_ROWS, "the stage holds a chunk of rows");
static_assert(sizeof(SvcRaw) <= STAGE_BYTES && sizeof(TaskRaw) <= STAGE_BYTES, "the stage holds one id's raw state");
static_assert(HLL_STAGE_REGS + (1u << 16) <= STAGE_BYTES, "the stage holds the found word and 2^16 HLL registers");
static_assert(QCHUNK * sizeof(gysk_flow_est) <= STAGE_BYTES && 64 * sizeof(gysk_topn_entry) <= STAGE_BYTES, "the stage holds the flow and top-N rows");
static_assert(sizeof(SlabEntry) <= STAGE_BYTES, "the stage holds one merged digest");
static_assert(sizeof(gysk_logical_state) == 80 && sizeof(gysk_logical_state) <= sizeof(gysk_svc_summary), "the stage holds WIN_ROWS state rows");
static_assert(sizeof(gysk_svc_clients) == 32 && sizeof(gysk_svc_clients) <= sizeof(gysk_svc_summary), "the stage holds WIN_ROWS client rows");
static_assert(sizeof(gysk_cluster_row) <= sizeof(gysk_svc_summary), "the stage holds WIN_ROWS cluster rows");
static_assert(sizeof(gysk_svc_top_clients) == 280 && QCHUNK * sizeof(gysk_svc_top_clients) <= STAGE_BYTES, "the stage holds a chunk of top-client rows");
static_assert(sizeof(gysk_logical_trace) == 168 && sizeof(gysk_logical_trace) <= sizeof(gysk_svc_summary), "the stage holds WIN_ROWS logical trace rows");
static_assert(sizeof(TraceSlab) <= STAGE_BYTES, "the stage holds one merged trace digest");

// A staged read, engine mutex held. The optional input (ids, flow keys or logical indices) travels through h_qids / d_qids in pieces
// of `piece` entries; without one (the window reads) the pieces only cut the n rows. For each piece, launch(d_in, off, m) writes m
// rows of row_bytes into d_wstage and returns its kernel launches; the rows come back into h_wstage, the stream is synchronised, and
// finish(h_wstage, off, m) copies them out.
template <typename In, typename Launch, typename Finish>
int staged_read(gysk_engine *e, const In *in, uint32_t n, uint32_t piece, size_t row_bytes, const char *what, Launch launch, Finish finish)
{
	static_assert(sizeof(In) <= sizeof(unsigned long long), "h_qids holds a piece of the input");
	for (uint32_t off = 0; off < n; off += piece) {
		const uint32_t m = std::min(piece, n - off);
		if (in) {
			memcpy(e->h_qids, in + off, (size_t)m * sizeof(In));
			CU(e, cudaMemcpyAsync(e->d_qids, e->h_qids, (size_t)m * sizeof(In), cudaMemcpyHostToDevice, e->stream));
		}
		e->kernel_launches += launch(in ? e->d_qids : nullptr, off, m);
		if (row_bytes) CU(e, cudaMemcpyAsync(e->h_wstage, e->d_wstage, m * row_bytes, cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaStreamSynchronize(e->stream));
		int rc = post_launch(e, what);
		if (rc) return rc;
		finish(e->h_wstage, off, m);
	}
	return 0;
}

// finish callbacks: the rows as they are; service rows, whose HLL estimate the host finishes (hll_finish); or nothing, when the
// read has no rows (gysk_register_ids) or its caller reads them from the stage itself (the single-id exports)
template <typename T> struct CopyRows
{
	T *out;
	void operator()(const uint8_t *rows, uint32_t off, uint32_t m) const { memcpy(out + off, rows, (size_t)m * sizeof(T)); }
};
struct SvcRows
{
	uint32_t hll_p;
	gysk_svc_summary *out;
	void operator()(const uint8_t *rows, uint32_t off, uint32_t m) const;
};
struct RowsStay { void operator()(const uint8_t *, uint32_t, uint32_t) const {} };
// client rows (GYSK_FLAG_CLIENT_LEVELS), whose two estimates the host finishes (hll_finish at GYSK_HLL_WINDOW_P)
struct ClientRows
{
	gysk_svc_clients *out;
	void operator()(const uint8_t *rows, uint32_t off, uint32_t m) const;
};

} // namespace gysk
