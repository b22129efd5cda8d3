// gysk_kernels.cuh — launch interface between the engine runtime (gysk_engine.cu) and the kernels.
#pragma once

#include "gysk_device.cuh"
#include "gysk_tdigest.cuh"
#include "../../include/gysketch.h"

#include <climits>

namespace gysk {

static constexpr int NLEVELS = 2;			// rolling levels beyond the 5-s window: 300 s, 432000 s (gy_statistics.h:1548)
static constexpr int NSLOTS = 10;			// slots per level (gy_statistics.h:1105)

// The rolling 300-s / 5-day levels: per level NSLOTS ring slots, each a plane of `stride` service rows of 16 cells
// ([NLEVELS][NSLOTS][stride][16]). stride is max_svcs: the null slot (index max_svcs) has no ring row. live, cur and fresh are set by
// the host at every flush (roll_levels in gysk_engine.cu); all are 0 until the first one. The count-min levels of GYSK_FLAG_FLOW_LEVEL
// and GYSK_FLAG_FLOW_QUERY_LEVEL follow level 0's decision (cms_level_roll_kernel).
struct LevelRing
{
	HistCell		*ring;
	uint32_t		stride;
	uint32_t		live[NLEVELS];		// the ring slots inside each level's span at the last flush
	uint32_t		cur[NLEVELS];		// the ring slot of each level the last flush wrote
	uint32_t		fresh;			// bit l: the last flush started a new epoch in level l's slot cur (its old content cleared)

	__host__ __device__ __forceinline__ HistCell *row(int l, uint32_t k, uint32_t slot) const
	{
		return ring + (((size_t)l * NSLOTS + k) * stride + slot) * HIST_CELLS;
	}
	// f(row) for each live ring slot of level l, in slot order
	template <typename F> __device__ __forceinline__ void each_live(int l, uint32_t slot, F f) const
	{
		for (int k = 0; k < NSLOTS; ++k) if ((live[l] >> k) & 1u) f(row(l, k, slot));
	}
	// cell c of level l as a service's row shows it: cells 0..14 sum the live slots, cell 15 is their max_val_seen_ (LLONG_MIN: none)
	__device__ __forceinline__ HistCell cell(int l, uint32_t slot, int c) const
	{
		HistCell a {0, c == HIST_MAX_CELL ? LLONG_MIN : 0};
		each_live(l, slot, [&](const HistCell *r) {		// one walk for all 16 lanes of a warp that reads a whole row
			const HistCell x = r[c];
			if (c == HIST_MAX_CELL) a.sum = max(a.sum, x.sum);
			else { a.count += x.count; a.sum += x.sum; }
		});
		return a;
	}
};

// Trace rows (gysk_config.max_trace_svcs): per row two windows, half `par` the open one. A window is TRACE_WORDS counters — line 0
// the ones ingest_kernel adds per event (nerr, nconns, bytes), line 1 the ones trace_keys_kernel takes from the sorted keys — a digest
// header ({total, n} used; the extremes are counter words) and TRACE_TD_CAP centroids. A trace sample's sort key carries the pseudo-slot
// base + row in its slot field, so it rides the batch's radix sort and bins_merge_kernel compresses its segment into the row's digest.
static constexpr int TRACE_WORDS = 32;
static constexpr int TRACE_TD_DELTA = 100;		// public.tdigest(response, 100) of the trace view
static constexpr int TRACE_TD_CAP = TRACE_TD_DELTA;	// the K_1 compress keeps at most delta clusters
static constexpr uint32_t TRACE_BUSY = 0xFFFFFFFFu;	// row_of entry of a slot whose row is being taken
enum {
	TW_NERR = 0, TW_NCONNS, TW_BYTES_IN, TW_MAX_IN, TW_BYTES_OUT, TW_MAX_OUT,
	TW_NREQ = 16, TW_SUM_US, TW_MAX_US, TW_BKT /* 8 words */, TW_TD_NMIN = TW_BKT + 8 /* max of ~usec of the digested samples */, TW_TD_MAX,
};
static_assert(TW_TD_MAX < TRACE_WORDS, "a window's counters fit TRACE_WORDS");
struct TraceTable
{
	uint32_t		*row_of;			// [max_svcs + 1] 1 + the trace row of a service slot, 0 = none, TRACE_BUSY
	uint32_t		*row_slot;			// [rows] service slot of a row, ~0u = free
	unsigned long long	*cnt;				// [2][rows][TRACE_WORDS]
	TdHead			*head;				// [2][rows]
	Centroid		*cent;				// [2][rows][TRACE_TD_CAP]
	uint32_t		*count;				// rows handed out so far
	int32_t			*free_n;			// freed rows on the stack
	uint32_t		*free_rows;			// [rows]
	unsigned long long	*dropped;			// events dropped for want of a row
	uint32_t		rows;				// capacity; 0 = off (every pointer nullptr)
	uint32_t		par;				// the half of every array that holds the open window
	uint32_t		base;				// pseudo-slot of row 0 in the sort keys: max_svcs + 1
	TdParams		td;				// compression TRACE_TD_DELTA
	__host__ __device__ __forceinline__ unsigned long long *words(uint32_t half, uint32_t r) const { return cnt + ((size_t)half * rows + r) * TRACE_WORDS; }
	__host__ __device__ __forceinline__ TdHead *hd(uint32_t half, uint32_t r) const { return head + (size_t)half * rows + r; }
	__host__ __device__ __forceinline__ Centroid *cents(uint32_t half, uint32_t r) const { return cent + ((size_t)half * rows + r) * TRACE_TD_CAP; }
};
// bucket of a response time in the trace view's eight response columns
__host__ __device__ __forceinline__ uint32_t trace_bucket(uint32_t us)
{
	return (us >= 300u) + (us >= 1000u) + (us >= 10000u) + (us >= 30000u) + (us >= 100000u) + (us >= 300000u) + (us >= 1000000u);
}

struct DevState
{
	// id tables
	IdTable			svc_tbl, task_tbl;
	// per-service state, indexed by slot
	HistCell		*hist_cur, *hist_last, *hist_all;	// [max_svcs][16]
	LevelRing		levels;
	unsigned long long	*conn_cur, *conn_last;			// packed {count:32, kbytes:32}
	unsigned long long	*slot_id;				// [max_svcs] slot -> glob_id (written by the inserter)
	uint32_t		*slot_host;				// [max_svcs] slot -> host_idx of the first event seen
	uint32_t		*slot_first_seen, *slot_last_active;	// [max_svcs] tsec of the first flush that saw the slot / of the last window with events
	uint32_t		*evict_list;				// [max_svcs] slots evicted by the last flush; evict_ids: their ids
	unsigned long long	*evict_ids;
	unsigned long long	*conn_all_cnt, *conn_all_kb;
	uint32_t		*bm_cur, *bm_last;			// [max_svcs][16] CONN_BITMAP transposed: per bucket a mask over (client port & 31)
	SlotBatch		*slot_batch;				// [max_svcs] exact extremes of the batch's RESP samples, hot row
	unsigned long long	*hot_rows;				// [hot_cap][HOT_ROW_WORDS] dense value bins of the hot services (nullptr: feature off)
	uint32_t		*hot_slot;				// [hot_cap] row -> slot
	uint32_t		hot_cap, hot_min, hot_max, hot_bin_max;	// rows; a service turns hot with hot_min..hot_max samples in one batch, its fullest bin <= hot_bin_max
	SlotAux			*slot_aux;				// [max_svcs] active-conn roll-up, error counters
	HistCell		*qps_hist, *act_hist;			// [max_svcs][16] TCP_LISTENER::qps_hist_ / active_conn_hist_: one sample per closed window
	SlotState		*slot_state;				// [max_svcs] listener state of the last evaluated window
	uint8_t			*hll;					// [max_svcs][1 << hll_p]
	Centroid		*td_cent;				// [max_svcs][TD_CAP]
	TdHead			*td_head;				// [max_svcs]
	// per-task state
	HistCell		*task_hist;				// [max_tasks][3][16]
	HistCell		*task_prev, *task_last;			// [max_tasks][3] {count, sum}: totals at the last flush / of the last closed window
	unsigned long long	*task_slot_id;				// [max_tasks] slot -> aggr_task_id
	uint32_t		*task_slot_host;
	// process eviction (task_idle_evict_secs; nullptr without): tsec of the last flush whose closed window held samples of the slot
	// (of the first flush that saw it until then), and the slots evicted by the last flush with their ids
	uint32_t		*task_last_active;			// [max_tasks]
	uint32_t		*task_evict_list;			// [max_tasks]
	unsigned long long	*task_evict_ids;			// [max_tasks]
	// flow sketch
	unsigned long long	*cms_cur, *cms_last;			// [depth][1 << log2w]
	unsigned long long	*cms_ring, *cms_5min;			// GYSK_FLAG_FLOW_LEVEL (nullptr without): [NSLOTS][depth][1 << log2w] level-0
									// ring slots of closed windows, and the sum of the live ones
	uint32_t		cms_depth, cms_wmask, cms_log2w, hll_p;
	uint32_t		rank, world, auto_register;
	double			td_delta;
	TdParams		td;
	unsigned long long	*counters;				// [CTR_MAX]
	TraceTable		trace;					// trace rows (trace.rows == 0: off)
};

// The service slot rules every per-host read shares (window reads, gysk_query_host_listen, the cluster fold). A slot below the table's
// count is live while it holds an id. It was evaluated at the last flush when its last window with events is the one that flush closed
// (active_mark, the rule of state_kernel). It is one of listener_stats_update's nissue (common/gy_socket_stat.cc:4242-4249) when it was
// evaluated there with issue bit 0 set.
__device__ __forceinline__ bool svc_live(const DevState &st, uint32_t slot) { return st.slot_id[slot] != 0; }
__device__ __forceinline__ bool svc_evaluated(const DevState &st, uint32_t slot, uint32_t active_mark) { return st.slot_last_active[slot] == active_mark; }
__device__ __forceinline__ bool svc_issue(const DevState &st, uint32_t slot, uint32_t active_mark)
{
	return svc_evaluated(st, slot, active_mark) && (st.slot_state[slot].issue_bits & 1u);
}

// Flow table of one batch: the TCP pass sums each flow's count-min increments {count 1 | kbytes << 32} in an entry keyed by its two
// hashes, key = h2 << 32 | h1 (0 = empty), and the TASK pass adds every entry to the flow's cells once and empties the table. u64
// addition is associative, so every cell ends as it would with one RED per record. mask + 1 entries, a power of two.
struct alignas(16) FlowEnt { unsigned long long key, inc; };
struct FlowTable { FlowEnt *ent; uint32_t mask; };
static constexpr uint32_t FLOW_PROBES = 16;		// linear probe limit; past it a record updates the count-min cells directly
static constexpr uint32_t FLOW_ENT_MAX = 1u << 21;	// 32 MB; a batch takes the smallest power of two >= 2 x its events, up to this
static constexpr uint32_t FLOW_SWEEP = 4;		// entries per thread and step of the TASK pass's sweep

// GYSK_FLAG_FLOW_QUERIES: the count-min of the response samples that reach a service histogram, cells {queries | response msec << 32}
// with the depth, width and row hashes of cms_cur / cms_last, and the batch flow table the TCP pass sums them in before the TASK pass
// applies it (as FlowTable does for the connection records). ingest_kernel queues each such sample as a connection-queue record whose
// slot is QRY_REC. Kept out of DevState so that the kernels without the flag keep their parameter layout: the drain passes take it as
// parameters of their own. Every pointer nullptr: off. ring and level: GYSK_FLAG_FLOW_QUERY_LEVEL's rolling 300-s level of the tables,
// laid out as DevState::cms_ring / cms_5min (nullptr without).
struct FlowQueries { unsigned long long *cur, *last; FlowEnt *flow; unsigned long long *ring, *level; };
static constexpr uint32_t QRY_REC = 0xFFFFFFFFu;	// slot field of a queued response sample (service slots are < 2^24)

// GYSK_FLAG_FLOW_RESP_HIST: the count-min of the same samples by RESP_TIME_HASH bucket, with the depth, width and row hashes of cms_cur.
// A cell is RESP_HIST_WORDS u64 words: bucket b counts in half b & 1 of word b >> 1 (word 7's high half stays 0), every word summed
// mod 2^64. The TCP pass sums the QRY_REC records in the batch flow table `flow` under the key resp_hist_key (the cell word and the low
// bits of the two hashes that pick the cells: flows that share it share every cell), the TASK pass applies it. Laid out and kept out of
// DevState as FlowQueries; every pointer nullptr: off. ring and level: with GYSK_FLAG_FLOW_QUERY_LEVEL too, the rolling 300-s level.
struct FlowRespHist { unsigned long long *cur, *last; FlowEnt *flow; unsigned long long *ring, *level; };
static constexpr uint32_t RESP_HIST_WORDS = 8;

static constexpr uint32_t CMS_LOG2W_MAX = 28;		// the widest count-min gysk_create accepts (1 << 28 columns)

// GYSK_FLAG_FLOW_TOPK: the candidates of one windowed table's heaviest-flow set in a batch. keys [0, *n) hold the open set (written at the
// end of the previous batch's selection, emptied by gysk_flush), then every flow key the batch brings: ingest_kernel appends each
// NOTIFY_ACTIVE_CONN_STATS record's (connection table), the TCP pass each record's that takes the direct path of flow_add, and the TASK
// pass, sweeping the batch flow table, the key its claimer stored in ekeys beside the entry. cap = K + max_batch: a record appends at most
// once, directly or by claiming an entry. Every pointer nullptr: not held.
struct TopkList { unsigned long long *keys, *n, *ekeys; unsigned long long cap; };
// a heaviest-flow set: [TOPK_SET_WORDS] u64, word 0 its size, word 1 zero (GYSK_FLAG_FLOW_TOPK_5MIN's sets: their bound), then the K
// keys best first
static constexpr uint32_t TOPK_K = GYSK_FLOW_TOPK_CAP, TOPK_SET_WORDS = TOPK_K + 2;
// the held lists: [0] the connection table's, [1] the flow query table's, [2] GYSK_FLAG_FLOW_TOPK_SLOW's (the response histogram table's,
// fed only by the TCP pass's slow samples: ekeys nullptr)
struct FlowTopk { TopkList list[3]; };
// a set's score (launch_topk_select, launch_topk_bound): 0 / 1 the low / high half of a one-word-cell table (query_flows_kernel's
// estimate); TOPK_SCORE_SLOW | b_slow the slow score of a response histogram table, the sum of its bucket counts from b_slow on
// (GYSK_FLAG_FLOW_TOPK_SLOW, resp_slow_score)
static constexpr int TOPK_SCORE_SLOW = 0x100;

// GYSK_FLAG_FLOW_ERRORS: the count-min of the QRY_REC records that carry an error bit, cells {cli_errors | ser_errors << 32} with the
// depth, width and row hashes of cms_cur, and the batch flow table the TCP pass sums them in (keyed as the query table's) before the TASK
// pass applies it. ingest_kernel's ERR instances put the event's GYSK_EVF_CLI_ERROR / GYSK_EVF_SER_ERROR bits into bits 30 / 31 of the
// record's value (a counted usec is below 1 000 001 000 < 2^30), and the drain passes' ERR instances mask them off. list: with
// GYSK_FLAG_FLOW_TOPK the server-error set's candidates, fed by the TCP pass once per record with the server-error bit (ekeys nullptr).
// Laid out and kept out of DevState and FlowTopk as FlowQueries, so that the kernels without the flag keep their parameter layout; every
// pointer nullptr: off. ring and level: with GYSK_FLAG_FLOW_QUERY_LEVEL too, the rolling 300-s level.
struct FlowErrors { unsigned long long *cur, *last; FlowEnt *flow; unsigned long long *ring, *level; TopkList list; };
static constexpr uint32_t QRY_CLI_ERR = 1u << 30, QRY_SER_ERR = 1u << 31, QRY_USEC_MASK = QRY_CLI_ERR - 1u;

// GYSK_FLAG_CLIENT_LEVELS: per service slot register sets of CL_REGS one-byte registers (precision GYSK_HLL_WINDOW_P): the open window
// and the last closed one ([max_svcs + 1][CL_REGS] each), the ring of NSLOTS 30-s slots ([NSLOTS][stride][CL_REGS], the level ring's
// layout: stride = max_svcs, no row for the null slot) and the 300-s level, the registerwise maximum of the live slots ([max_svcs + 1]
// [CL_REGS]). Outside DevState, so that the kernels without the flag keep their parameter layout. Every pointer nullptr: off.
static constexpr uint32_t CL_REGS = 1u << GYSK_HLL_WINDOW_P;
struct ClientLevels { uint8_t *open, *last, *ring, *level; uint32_t stride; };

// GYSK_FLAG_SVC_TOP_CLIENTS: per service slot summaries of TOPC_K entries (gysk_topc_entry, best first, zero past the held ones) and the
// bound delta: the open window, the last closed one and the 300-s level ([max_svcs + 1] each), and the ring of NSLOTS 30-s slots
// ([NSLOTS][stride], the client ring's layout). The batch scratch: the pair table of pmask + 1 entries keyed {flow_key, slot + 1} (hi 0:
// empty) beside their sums {kbytes, conns}, zero between batches; the counters {pairs, segments, pieces}; the piece lists of the long
// segments (TopcPiece, pieces_cap of them). Outside DevState, so that the kernels without the flag keep their parameter layout. Every
// pointer nullptr: off.
static constexpr uint32_t TOPC_K = GYSK_SVC_TOPC_K;
static constexpr uint32_t TOPC_PIECE = 1024;		// pairs per piece: a longer segment is cut into pieces, one warp each
struct TopcSet { gysk_topc_entry ent[TOPC_K]; unsigned long long delta; };
static_assert(sizeof(TopcSet) == 264, "a summary is 16 entries and its bound");
struct TopcCand { unsigned long long key, kb, conns; };
// a piece of a long segment: its sorted keys [beg, end) of service slot, then the K + 1 best of its pairs (each with the old entry of its
// client added) and the old entries it met (bit j: entry j)
struct TopcPiece { TopcCand c[TOPC_K + 1]; uint32_t n, matched, beg, end, slot, pad; };
struct SvcTopClients
{
	TopcSet			*open, *last, *ring, *level;
	uint32_t		stride;
	ulonglong2		*pkey, *pacc;
	uint32_t		pmask;
	unsigned long long	*cnt;
	TopcPiece		*pieces;
	uint32_t		pieces_cap;
};

struct SortTemp
{
	unsigned long long	*keys_a, *keys_b;	// [nkeys] RESP sort keys of the batch (also the top-N sort keys)
	uint64_t		nkeys;			// max(max_batch, max(max_svcs, max_tasks) + 1)
	unsigned long long	*tile_status;		// [max_tiles][512] look-back status words {pass epoch | state | count}: never cleared
	uint32_t		*epoch;			// HOST counter of radix passes launched (tags the status words)
	uint32_t		*os_ghist;		// [OS_GHIST_WORDS] of one sort: [OS_MAX_PASSES][RADIX_MAX] global digit histograms of its passes, then
							// from OS_GHIST_TICKETS on one tile ticket per pass
	uint32_t		*touched;		// [max_svcs] services with RESP samples in the batch
	uint4			*segs;			// [max_svcs] BatchSeg of each touched service: its keys in the sorted array, its batch row
	uint32_t		*long_slot;		// [batch rows] slot of each long segment (more than LONG_SEG keys) of the batch
	unsigned long long	*batch_rows;		// [batch rows][HOT_ROW_WORDS] dense value bins of the long segments, hot-row layout; zero
							// between batches (bins_merge_kernel zeroes what it reads)
	Centroid		*items_scratch;		// [merge warps][NBINS] a warp's list of batch items
	TdWorkBig		*big_scratch;		// [merge warps] work arrays for merged lists beyond the shared-memory work area (TD_SMEM_N entries)
	uint4			*recq;			// [recq_cap] records {slot, value, flow key}: ingest_kernel resolves the ids of connection and
							// process events and queues them, the drain passes (launch_drains) apply them. Warp w of the
							// ingest launch owns region [w * cap, (w + 1) * cap) (RecRegions): its connection records from
							// the front, its process records from the back, stored at warp-local offsets without any atomic
	uint2			*rec_cnt;		// [rec_cnt_cap] {connection, process} records of each region, written by every warp of the launch
	uint64_t		recq_cap;		// max_batch + the regions' rounding (one chunk per warp of a full ingest grid)
	uint32_t		rec_cnt_cap;		// warps of a full ingest grid
	FlowEnt			*flow;			// [flow_cap] the flow table (FlowTable): zero between batches
	uint32_t		flow_cap;		// min(FLOW_ENT_MAX, smallest power of two >= 2 x max_batch)
	uint32_t		max_tiles;
};

// the record queue regions of one ingest launch: one per warp, cap = ceil(chunks / warps) x events per chunk, the most records a
// warp can queue (chunks are dealt to the warps round-robin)
struct RecRegions { uint32_t nwarps; uint64_t cap; };

// launch shape of ingest_kernel: warps per CTA, CTAs per SM (the full grid, and __launch_bounds__), events per lane and chunk
// (DESIGN.md §7 has the measurements). It also sizes the record queue beyond max_batch; launch_ingest checks every launch against
// the buffers.
struct IngestShape { static constexpr int WARPS = 8, MIN_CTAS = 3, EPT = 2, CHUNK = 32 * EPT; };

// one service's state: what a summary warp reads (in shared memory), and what the single-id exports copy to the host
struct SvcRaw
{
	unsigned long long	id;
	int32_t			found;
	uint32_t		slot;
	HistCell		cur[HIST_CELLS], last[HIST_CELLS], all[HIST_CELLS];
	HistCell		lvl[2][HIST_CELLS];			// sums of the live slots of the rolling levels
	unsigned long long	conn_cur, conn_last, conn_all_cnt, conn_all_kb;
	uint32_t		bm_cur[HIST_CELLS], bm_last[HIST_CELLS];
	uint32_t		hll_hist[64];
	TdHead			td;
	SlotAux			aux;
	SlotState		sst;
	HistCell		qps[HIST_CELLS], act[HIST_CELLS];
	Centroid		cent[TD_CAP];
};

struct TaskRaw
{
	unsigned long long	id;
	int32_t			found;
	uint32_t		slot;
	HistCell		h[3][HIST_CELLS];
};

static constexpr int SORT_TILE = 4096;		// keys per CTA tile in the radix passes
static constexpr int RADIX_MAX_BITS = 9;
static constexpr int RADIX_MAX = 1 << RADIX_MAX_BITS;
static constexpr int OS_MAX_PASSES = 8;			// radix passes of one sort: 64 key bits in 8-bit digits
static constexpr int OS_GHIST_TICKETS = OS_MAX_PASSES * RADIX_MAX, OS_GHIST_WORDS = OS_GHIST_TICKETS + OS_MAX_PASSES;	// SortTemp::os_ghist
static constexpr int TD_MERGE_CTAS_PER_SM = 5, TD_MERGE_MAX_SMS = 192;	// bins_merge_kernel grid (<= 4 warps per CTA)
// a service segment of more than LONG_SEG sorted keys is summed into a batch row by long_sum_kernel; a shorter one is read by one warp
// of bins_merge_kernel (DESIGN.md §4). Batch rows: min(max_svcs, ceil(max_batch / LONG_SEG)).
static constexpr int LONG_SEG = 8192;

// The opt-in flow state a batch's ingest and drain passes read, every pointer nullptr where its flag is off. Each flag's bit of the
// ingest_kernel and drain_kernel instance follows from it:
// fq.cur (GYSK_FLAG_FLOW_QUERIES, QRY): the response samples are queued for the flow query table too
// fr.cur (GYSK_FLAG_FLOW_RESP_HIST, RH, only with fq.cur): the response samples also go to the flow response histograms
// tk.list[0].keys (GYSK_FLAG_FLOW_TOPK, TOPK): the flow keys of the ACTIVE records join the connection table's candidates, and the
// drain passes gather each held table's candidates
// tk.list[2].keys (GYSK_FLAG_FLOW_TOPK_SLOW, SLOW, with fr.cur and tk.list[0].keys): the TCP pass gathers the flow key of each response
// sample in bucket b_slow or above
// cl.open (GYSK_FLAG_CLIENT_LEVELS, CL): the ACTIVE records and each connection record raise the open window's client registers too
// fe.cur (GYSK_FLAG_FLOW_ERRORS, ERR, only with fq.cur): the queued response samples carry their error bits (QRY_CLI_ERR, QRY_SER_ERR),
// the error samples go to the flow error tables, and with fe.list.keys their server-error flow keys to its candidates
struct FlowPass { FlowQueries fq; FlowRespHist fr; FlowTopk tk; uint32_t b_slow; ClientLevels cl; FlowErrors fe; };

// every launcher returns the number of kernel launches it issued
// service slots [s_lo, s_hi) and process slots [t_lo, t_hi) in their just-created state (the arrays zeroed before)
int launch_init_slots(const DevState &st, uint32_t s_lo, uint32_t s_hi, uint32_t t_lo, uint32_t t_hi, cudaStream_t s);
int launch_register(const DevState &st, const unsigned long long *d_ids, uint32_t n, int is_task, cudaStream_t s);
// -1: no ingest_kernel instance for fp's flags, no sort plan for max_svcs, or the launch's record regions do not fit the buffers
// key_slots: the values the slot field of a sort key takes (max_svcs, or max_svcs + 1 + trace rows with trace rows)
int launch_ingest(const DevState &st, const SortTemp &tmp, const FlowPass &fp, const gysk_event *d_ev, uint64_t n, uint32_t key_slots,
		RecRegions &rr, cudaStream_t s);
int launch_batch_merge(const DevState &st, const SortTemp &tmp, uint64_t n_events, uint32_t key_slots, cudaStream_t s);
// the TCP and then the TASK drain pass over the records launch_ingest queued. -1: no drain_kernel instance for fp's flags
int launch_drains(const DevState &st, const SortTemp &tmp, const FlowPass &fp, const RecRegions &rr, uint64_t n_events, cudaStream_t s);
// GYSK_FLAG_FLOW_TOPK, after the batch merge (it takes tmp's sort buffers, of at least n_max keys): the *l.n candidates (n_max >= *l.n)
// sorted by key in l.keys, the distinct ones scored on table tbl (score as TOPK_SCORE_SLOW says) and the K best by (score descending,
// key ascending) written to set; then, unless reseed is false, set back into l as the next batch's first candidates. -1: no sort plan
int launch_topk_select(const SortTemp &tmp, const TopkList &l, uint64_t n_max, const unsigned long long *tbl, uint32_t depth, uint32_t log2w,
		int score, unsigned long long *set, bool reseed, cudaStream_t s);
// the merge's union into l (its count reset first): the keys of world sets, rank r's at sets + r * stride words
int launch_topk_gather(const unsigned long long *sets, uint32_t world, size_t stride, const TopkList &l, cudaStream_t s);
// GYSK_FLAG_FLOW_TOPK_5MIN: the keys of set j (at sets + j * stride words) appended to l for each bit j of mask (j < 32), l's count reset
// first when reset is true
int launch_topk_gather_mask(const unsigned long long *sets, size_t stride, uint32_t mask, const TopkList &l, bool reset, cudaStream_t s);
// GYSK_FLAG_FLOW_TOPK_5MIN: a set's bound word. thr(set) is the score on tbl (score as launch_topk_select) of its K-th key when it holds
// K, else 0; t the sum of terms[j * stride] over j < nterms with bit j % 32 of mask set. *out = sum ? thr + t : max(thr, t)
int launch_topk_bound(const unsigned long long *set, const unsigned long long *tbl, uint32_t depth, uint32_t log2w, int score,
		const unsigned long long *terms, size_t stride, uint32_t nterms, uint32_t mask, bool sum, unsigned long long *out, cudaStream_t s);
// sorts tmp.keys_a on key bits [lo, hi); *which = 1: the result is in keys_b. -1: no sort plan for the range (more than 8 passes, or
// bits outside [0, 64)), or n_max >= 2^30
int launch_radix_sort(const SortTemp &tmp, const unsigned long long *d_n, uint64_t n_max, int lo, int hi, int *which, cudaStream_t s);
// the want best services (host_filter < 0: of every host) or processes (is_task) of nslots by one metric, and with d_slots their slots;
// -1: sort failed
int launch_topn(const DevState &st, const SortTemp &tmp, uint32_t nslots, int is_task, int metric, int host_filter, uint32_t want,
		gysk_topn_entry *d_out, cudaStream_t s, unsigned long long *d_slots = nullptr);
// the second half of a top-N: the *d_n <= nkeys {score : 32 | index : 32} keys in tmp.keys_a sorted by score (stable), then the want best
// as entries {ids[index], score, hosts[index]} (hosts nullptr: host 0), the later index first on equal scores, and with d_slots each
// entry's index (0 past the keys); -1: sort failed
int launch_topn_pick(const SortTemp &tmp, const unsigned long long *d_n, uint32_t nkeys, const unsigned long long *ids, const uint32_t *hosts,
		uint32_t want, gysk_topn_entry *d_out, cudaStream_t s, unsigned long long *d_slots = nullptr);
// the closed window of every process slot; with idle_secs the process eviction too: the evicted ids go to host_ids (page-locked,
// mapped: [0] = count, [1..] = ids in eviction-list order)
int launch_task_flush(const DevState &st, uint32_t max_tasks, uint32_t tsec, uint32_t idle_secs, unsigned long long *host_ids, cudaStream_t s);
// the window roll into ring slot st.levels.cur of each level (cleared by the host when it starts a new epoch), the listener states,
// the idle-service eviction
// (GYSK_FLAG_CLIENT_LEVELS, cl.open != nullptr: an evicted slot's client sets are cleared with it)
// (GYSK_FLAG_SVC_TOP_CLIENTS, tc.open != nullptr: an evicted slot's summaries are cleared with it)
int launch_flush(const DevState &st, const ClientLevels &cl, const SvcTopClients &tc, uint32_t max_svcs, uint32_t tsec, uint32_t idle_secs,
		cudaStream_t s);
// clears table t and re-inserts the ids t.slot_id holds in slots [0, nslots)
int launch_rebuild_table(const IdTable &t, uint32_t nslots, cudaStream_t s);
// the single-id exports: the raw state of n ids (id 0 and unknown ids: found = 0); the HLL registers of the id d_ids[0]
int launch_gather_svcs(const DevState &st, const unsigned long long *d_ids, uint32_t n, SvcRaw *d_out, cudaStream_t s);
int launch_gather_tasks(const DevState &st, const unsigned long long *d_ids, uint32_t n, TaskRaw *d_out, cudaStream_t s);
int launch_gather_hll(const DevState &st, const unsigned long long *d_ids, int32_t *found, uint8_t *d_out, cudaStream_t s);
// window reads: the live slots (host filter, closed-window filter, with seen_before != ~0u only services first seen by a flush before
// that tsec) as keys {host : 32 | slot : 32}, *d_n of them; with `order` sorted by host (stable) and the ids of the sorted keys in *ids.
// *keys / *ids point into the sort buffers of tmp.
int launch_window_list(const DevState &st, const SortTemp &tmp, uint32_t nslots, int is_task, int host_filter, uint32_t active_only,
		uint32_t active_mark, uint32_t seen_before, unsigned long long *d_n, bool order, const unsigned long long **keys, const unsigned long long **ids,
		cudaStream_t s);
// LISTENER_DAY_STATS rows of n slots
int launch_day_stats(const DevState &st, const unsigned long long *d_slots, uint32_t n, gysk_listener_day_stats *d_out, cudaStream_t s);
// per-host listener counts over the n host-sorted keys of launch_window_list (*d_n on the device): the issue / severe counts of each
// host's run at acc[run head] (acc: n entries of scratch), then the rows of the runs ranked [rlo, rlo + cap) and *d_rows = runs
int launch_host_listen_count(const DevState &st, const unsigned long long *keys, const unsigned long long *d_n, uint32_t n, uint32_t active_mark,
		unsigned long long *acc, cudaStream_t s);
int launch_host_listen_rows(const unsigned long long *keys, const unsigned long long *d_n, const unsigned long long *acc, uint32_t rlo, uint32_t cap,
		gysk_host_listen *d_out, unsigned long long *d_rows, cudaStream_t s);
// service / process rows by id (d_ids) or, with d_ids == nullptr, by slot (d_slots)
int launch_svc_summaries(const DevState &st, const unsigned long long *d_ids, const unsigned long long *d_slots, uint32_t n, gysk_svc_summary *d_out,
		cudaStream_t s);
int launch_task_summaries(const DevState &st, const unsigned long long *d_ids, const unsigned long long *d_slots, uint32_t n, gysk_task_summary *d_out,
		cudaStream_t s);
// the count-min point queries of n flow keys on table tbl ([depth][1 << log2w] cells)
int launch_query_flows(const unsigned long long *tbl, uint32_t depth, uint32_t log2w, const unsigned long long *d_keys, uint32_t n, gysk_flow_est *d_out,
		cudaStream_t s);
// the same on a flow response histogram table ([depth][1 << log2w][RESP_HIST_WORDS] words): bucket counts, total and percentiles
int launch_query_flow_resp(const unsigned long long *tbl, uint32_t depth, uint32_t log2w, const unsigned long long *d_keys, uint32_t n,
		gysk_flow_resp_est *d_out, cudaStream_t s);
// a rolling count-min level at the flush, before its window pair's swap: the open table cur ([cells]) into ring slot lv.cur[0]
// (replacing it when the slot is fresh), then level = the sum of the live slots (level 0's decision of lv)
int launch_cms_level_roll(const unsigned long long *cur, unsigned long long *ring, unsigned long long *level, size_t cells, const LevelRing &lv,
		cudaStream_t s);
// GYSK_FLAG_CLIENT_LEVELS at the flush, after launch_flush and before the open / last swap: the open sets of slots [0, nslots) (the
// capacity) max-merged into ring slot lv.cur[0] (in its place when the slot is fresh) and the level = the registerwise maximum of the
// live slots (level 0's decision of lv)
int launch_client_roll(const ClientLevels &cl, uint32_t nslots, const LevelRing &lv, cudaStream_t s);
// the client rows (gysk_svc_clients) by id (d_ids) or by slot (d_slots); the estimates as hll_pending leaves them
int launch_client_rows(const DevState &st, const ClientLevels &cl, const unsigned long long *d_ids, const unsigned long long *d_slots, uint32_t n,
		gysk_svc_clients *d_out, cudaStream_t s);
// GYSK_FLAG_SVC_TOP_CLIENTS after a batch's drain passes and top-K selections (it takes tmp's sort buffers and segment array): the
// batch's exact per-(service, client) sums of the TCP regions' connection records, grouped by service and merged into each service's
// open summary. -1: no sort plan
// (rr: the regions of the batch's ingest launch)
int launch_topc_batch(const SortTemp &tmp, const SvcTopClients &tc, const RecRegions &rr, uint64_t n_events, uint32_t max_svcs, cudaStream_t s);
// GYSK_FLAG_SVC_TOP_CLIENTS at the flush, before the open / last swap: each open summary of slots [0, nslots) merged into ring slot
// lv.cur[0] (in its place when the slot is fresh), then the level = the merge of the live slots (level 0's decision of lv)
int launch_topc_roll(const SvcTopClients &tc, uint32_t nslots, const LevelRing &lv, cudaStream_t s);
// the rows of summary `which` (GYSK_TOPC_*) by id (d_ids) or by slot (d_slots)
int launch_topc_rows(const DevState &st, const SvcTopClients &tc, int which, const unsigned long long *d_ids, const unsigned long long *d_slots,
		uint32_t n, gysk_svc_top_clients *d_out, cudaStream_t s);
// the CL_REGS registers at regs + slot * CL_REGS of the id d_ids[0] (gysk_export_hll_window)
int launch_gather_hll_window(const DevState &st, const uint8_t *regs, const unsigned long long *d_ids, int32_t *found, uint8_t *d_out, cudaStream_t s);
// trace rows at gysk_flush: the half `open` (the one the flush opens) of rows [0, nrows) cleared
int launch_trace_roll(const DevState &st, uint32_t open, uint32_t nrows, cudaStream_t s);
// trace rows by id (d_ids) or by row (d_rows)
int launch_trace_rows(const DevState &st, const unsigned long long *d_ids, const unsigned long long *d_rows, uint32_t n, gysk_trace_row *d_out, cudaStream_t s);
// the rows in use of [0, nrows) that pass the host filter and (active_only) hold requests in their last window: ids at ids[i], rows at
// rows[i], *d_n of them
int launch_trace_list(const DevState &st, uint32_t nrows, int host_filter, uint32_t active_only, unsigned long long *ids, unsigned long long *rows,
		unsigned long long *d_n, cudaStream_t s);
// one id's digest of one window: TraceRaw
struct TraceRaw { int32_t found; uint32_t n; unsigned long long total; double minv, maxv; Centroid cent[TRACE_TD_CAP]; };
int launch_gather_trace(const DevState &st, const unsigned long long *d_id, int last_window, TraceRaw *d_out, cudaStream_t s);

} // namespace gysk
