// gysk_kernels.cu — hand-written sm_90a kernels of the streaming-sketch engine.
//
//   ingest_kernel        one pass over a batch of 32-byte events: id -> slot, then per event type
//                          RESP : one 64-bit sort key {slot | value bin | usec}; CONN_BITMAP bit, batch min / max when they change
//                          TCP, TASK : one 16-byte record {slot, value, flow key} in the batch's record queue
//                          ACTIVE : ACTIVE_CONN_STATS records                          server/gy_mconnhdlr.cc:7705
//   drain_kernel         the queued records, one launch per kind: TCP -> the flow's count-min increment summed in the batch flow table,
//                        HLL register max, per-service exact cell; TASK -> the flow table into the count-min cells, then
//                        MAGGR_TASK::set_local_task_state (3 histograms) server/gy_msocket.h:1009-1018
//   os_pass_kernel       stable one-sweep LSD radix pass (RESP keys of a batch on their slot; the top-N rankings)
//   segs_mark_kernel     sorted keys -> one segment per service, touched list (short segments), batch rows (long segments)
//   long_sum_kernel      keys of the long segments -> per-bin samples and exact usec sums in their batch rows
//   trace_keys_kernel    trace rows (max_trace_svcs): requests, usec sum / max, response buckets of each row from the tail of the sorted keys
//   bins_merge_kernel    per touched service: bins -> GY_HISTOGRAM::add_data for every sample (RESP_TIME_HASH, common/gy_statistics.h:
//                        596-623, :1698) and -> the merging t-digest (K_1 scale)               DESIGN.md §2
//   flush_kernel         5-s window roll                                               common/gy_socket_stat.cc:3898
//   state_kernel         listener state of the closed window (get_curr_state)          common/gy_socket_stat.cc:2020-2875
//   evict_kernel         idle listeners leave, slots recycled                          common/gy_socket_stat.cc:3968-4037
//                        idle aggregated processes too (task_idle_evict_secs)         server/gy_mconnhdlr.cc:16492-16541
//   gather_* / query_* / topn_*   read side
//   window_* / task_summary_kernel  window reads: every live id, summarised on the device (gysk_summary.cuh)
#include "gysk_kernels.cuh"
#include "gysk_state.cuh"
#include "gysk_summary.cuh"
#include "gysk_topc.cuh"

#include <cfloat>
#include <climits>
#include <cmath>
#include <algorithm>
#include <array>
#include <type_traits>
#include <cstring>
#include <utility>

namespace gysk {

// RESP sort key = {slot : 24 | bin index : 10 | usec : 30}. Bin index = td_code(usec) + RESP_TIME_HASH bucket of usec / 1000: both
// terms are monotone in usec, so the index is too and no bin straddles a histogram bucket (DESIGN.md §3). The radix passes sort on
// the slot bits only: the samples of one service end up as one contiguous SEGMENT, its bins in no particular order inside it
// (bins_merge_kernel sums them per bin itself).
static constexpr int KEY_GROUP_SHIFT = 30;				// key >> 30 = {slot, bin}
static constexpr int KEY_SLOT_SHIFT = KEY_GROUP_SHIFT + TD_CODE_BITS;
__device__ __forceinline__ uint32_t key_usec(unsigned long long k) { return (uint32_t)k & 0x3FFFFFFFu; }
__device__ __forceinline__ uint32_t key_slot(unsigned long long k) { return (uint32_t)(k >> KEY_SLOT_SHIFT); }
__device__ __forceinline__ uint32_t key_bin(unsigned long long k) { return (uint32_t)(k >> KEY_GROUP_SHIFT) & ((1u << TD_CODE_BITS) - 1u); }
// the bin index of a response time, as the key carries it
__device__ __forceinline__ uint32_t resp_bin(uint32_t usec) { return td_code(usec) + (uint32_t)bucket_resp_time((long long)(usec / 1000u)); }

static constexpr int KEY_DIGIT_MAX = 9;				// widest digit of the RESP-key passes (key_sort_plan)
static constexpr int KEY_SLOT_BITS_MAX = 24;
// passes of the longest RESP plan: ingest_kernel keeps this many digit histograms in shared memory
static constexpr int KEY_PASSES_MAX = (KEY_SLOT_BITS_MAX + KEY_DIGIT_MAX - 1) / KEY_DIGIT_MAX;
static_assert(KEY_PASSES_MAX <= OS_MAX_PASSES, "a RESP plan fits a SortPlan");
// which bits of the key each pass of the radix sort takes as its digit, lowest first: pass p sorts on bits [shift[p], shift[p] + bits[p]).
// key_sort_plan cuts the RESP keys, plain_sort_plan every other sort; ingest_kernel and os_hist_kernel fill the passes' histograms
// from the plan, os_pass_kernel gets its pass's shift and width.
struct SortPlan { int np; int shift[OS_MAX_PASSES]; int bits[OS_MAX_PASSES]; };
__device__ __forceinline__ uint32_t sort_digit(unsigned long long k, int shift, int bits) { return (uint32_t)(k >> shift) & ((1u << bits) - 1u); }

// ---------------------------------------------------------------------------------------------------
// state init / registration
// ---------------------------------------------------------------------------------------------------
// The just-created state of one service slot, written by threads t = 0 .. nt - 1 together: what a slot holds before its first id, and
// again once its id is evicted. Every per-slot array but the batch scratch (slot_batch: its hot row belongs to the slot, whoever lives
// in it) and the eviction / free lists. The null slot (index max_svcs) stays in this state for the engine's life; slot max_svcs has
// no ring row (LevelRing).
__device__ __forceinline__ void slot_reset(const DevState &st, uint32_t slot, uint32_t t, uint32_t nt)
{
	if (t == 0) {
		st.slot_id[slot] = 0; st.slot_host[slot] = 0; st.slot_first_seen[slot] = 0; st.slot_last_active[slot] = 0;
		st.conn_cur[slot] = 0; st.conn_last[slot] = 0; st.conn_all_cnt[slot] = 0; st.conn_all_kb[slot] = 0;
		st.slot_aux[slot] = SlotAux {0, 0, 0, 0, 0, 0};
		st.slot_state[slot] = SlotState {GYSK_STATE_OK, GYSK_ISSUE_NONE, 0, 0, 0};
		TdHead h; h.total = 0; h.minv = INFINITY; h.maxv = -INFINITY; h.n = 0; h.pad = 0;
		st.td_head[slot] = h;
	}
	for (uint32_t c = t; c < (uint32_t)HIST_CELLS; c += nt) {
		const size_t i = (size_t)slot * HIST_CELLS + c;
		const HistCell z {0, c == HIST_MAX_CELL ? LLONG_MIN : 0};		// max_val_seen_{numeric_limits<T>::min()} gy_statistics.h:560
		st.hist_cur[i] = z; st.hist_last[i] = z; st.hist_all[i] = z;
		st.bm_cur[i] = 0; st.bm_last[i] = 0;
		const HistCell zi {0, c == HIST_MAX_CELL ? (long long)INT_MIN : 0};	// GY_HISTOGRAM<int, ...>: numeric_limits<int>::min()
		st.qps_hist[i] = zi; st.act_hist[i] = zi;
		if (slot < st.levels.stride)
			for (int l = 0; l < NLEVELS; ++l)
				for (int k = 0; k < NSLOTS; ++k) st.levels.row(l, k, slot)[c] = HistCell {0, 0};
	}
	uint32_t *hw = reinterpret_cast<uint32_t *>(st.hll + ((size_t)slot << st.hll_p));
	for (uint32_t w = t; w < (1u << st.hll_p) / 4u; w += nt) hw[w] = 0;
	for (uint32_t w = t; w < (uint32_t)TD_CAP; w += nt) st.td_cent[(size_t)slot * TD_CAP + w] = Centroid {0.0, 0ull};
}

// The just-created state of one process slot, written by threads t = 0 .. nt - 1 together: three empty histograms, an empty last window,
// no id. What a slot holds before its first id, and again once its id is evicted. The eviction list and the free stack are not per-slot
// state.
__device__ __forceinline__ void task_slot_reset(const DevState &st, uint32_t slot, uint32_t t, uint32_t nt)
{
	for (uint32_t c = t; c < 3u * HIST_CELLS; c += nt)
		st.task_hist[(size_t)slot * 3 * HIST_CELLS + c] = HistCell {0, c % HIST_CELLS == HIST_MAX_CELL ? LLONG_MIN : 0};
	for (uint32_t h = t; h < 3u; h += nt) { st.task_prev[(size_t)slot * 3 + h] = HistCell {0, 0}; st.task_last[(size_t)slot * 3 + h] = HistCell {0, 0}; }
	if (t == 0) {
		st.task_slot_id[slot] = 0; st.task_slot_host[slot] = 0;
		if (st.task_last_active) st.task_last_active[slot] = 0;
	}
}

// An evicted service's trace row, by threads t = 0 .. nt - 1 of one CTA together: both windows zeroed, the row on the free stack, the
// slot without a row
__device__ __forceinline__ void trace_release(const TraceTable &tr, uint32_t slot, uint32_t t, uint32_t nt)
{
	const uint32_t r1 = tr.row_of[slot];
	__syncthreads();			// every thread has read the entry before thread 0 clears it
	if (r1 == 0 || r1 == TRACE_BUSY) return;
	const uint32_t r = r1 - 1u;
	for (uint32_t h = 0; h < 2u; ++h) {
		for (uint32_t w = t; w < (uint32_t)TRACE_WORDS; w += nt) tr.words(h, r)[w] = 0ull;
		for (uint32_t c = t; c < (uint32_t)TRACE_TD_CAP; c += nt) tr.cents(h, r)[c] = Centroid {0.0, 0ull};
		if (t == 0) { TdHead z; z.total = 0; z.minv = INFINITY; z.maxv = -INFINITY; z.n = 0; z.pad = 0; *tr.hd(h, r) = z; }
	}
	if (t == 0) {
		tr.row_of[slot] = 0; tr.row_slot[r] = ~0u;
		const int32_t f = atomicAdd(tr.free_n, 1);
		tr.free_rows[f] = r;
	}
}

// the slot-reset functions evict_kernel takes
struct SvcSlotReset
{
	__device__ void operator()(const DevState &st, uint32_t slot, uint32_t t, uint32_t nt) const
	{
		slot_reset(st, slot, t, nt);
		if (st.trace.rows) trace_release(st.trace, slot, t, nt);
	}
};
struct TaskSlotReset { __device__ void operator()(const DevState &st, uint32_t slot, uint32_t t, uint32_t nt) const { task_slot_reset(st, slot, t, nt); } };
// GYSK_FLAG_CLIENT_LEVELS: the service's reset and its 2 + NSLOTS + 1 client sets zeroed, so that a recycled slot starts from zero as its
// all-time registers do
struct SvcClientSlotReset
{
	ClientLevels cl;
	__device__ void operator()(const DevState &st, uint32_t slot, uint32_t t, uint32_t nt) const
	{
		constexpr uint32_t Q = CL_REGS / 16;
		for (uint32_t i = t; i < (3u + NSLOTS) * Q; i += nt) {
			const uint32_t set = i / Q, q = i % Q;
			uint8_t *base = set == 0 ? cl.open : set == 1 ? cl.last : set == 2 ? cl.level : cl.ring + (size_t)(set - 3) * cl.stride * CL_REGS;
			reinterpret_cast<uint4 *>(base + (size_t)slot * CL_REGS)[q] = make_uint4(0, 0, 0, 0);
		}
		SvcSlotReset {}(st, slot, t, nt);
	}
};
// GYSK_FLAG_SVC_TOP_CLIENTS: the reset of Inner and the slot's 3 + NSLOTS summaries zeroed
template <typename Inner>
struct SvcTopcSlotReset
{
	SvcTopClients tc;
	Inner inner;
	__device__ void operator()(const DevState &st, uint32_t slot, uint32_t t, uint32_t nt) const
	{
		constexpr uint32_t W = sizeof(TopcSet) / 8;
		for (uint32_t i = t; i < (3u + NSLOTS) * W; i += nt) {
			const uint32_t set = i / W, w = i % W;
			TopcSet *base = set == 0 ? tc.open : set == 1 ? tc.last : set == 2 ? tc.level : tc.ring + (size_t)(set - 3) * tc.stride;
			reinterpret_cast<unsigned long long *>(base + slot)[w] = 0ull;
		}
		inner(st, slot, t, nt);
	}
};

// service slots [s_lo, s_hi) and process slots [t_lo, t_hi) in their just-created state: one CTA per service slot, one thread per
// process slot (grid-stride): gysk_create over every slot, gysk_grow over the new ones
__global__ void __launch_bounds__(256) init_slots_kernel(DevState st, uint32_t s_lo, uint32_t s_hi, uint32_t t_lo, uint32_t t_hi)
{
	for (uint32_t s = s_lo + blockIdx.x; s < s_hi; s += gridDim.x) {
		slot_reset(st, s, threadIdx.x, blockDim.x);
		if (threadIdx.x == 0) st.slot_batch[s] = SlotBatch {0xFFFFFFFFu, 0u, 0u, 0u};
	}
	for (uint32_t i = t_lo + blockIdx.x * blockDim.x + threadIdx.x; i < t_hi; i += gridDim.x * blockDim.x) task_slot_reset(st, i, 0, 1);
}

__global__ void register_kernel(DevState st, const unsigned long long *ids, uint32_t n, int is_task)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;

	if (i < n && ids[i] && ids[i] != KEY_TOMBSTONE) table_lookup(is_task ? st.task_tbl : st.svc_tbl, ids[i], true);
}

// ---------------------------------------------------------------------------------------------------
// ingest
// ---------------------------------------------------------------------------------------------------
// Service popularity is Zipf-skewed: a few {count, sum} cells would take millions of same-address L2 atomics per batch and
// serialise the kernel. Two levels take that pressure off L2:
//   warp : lanes updating the same cell are grouped with match.any, reduced with a shuffle loop and represented by one leader;
//   CTA  : a two-choice shared-memory table privatises hot cells for the lifetime of the CTA (a cell is admitted when it
//          shows up ADMIT times inside one warp: twice for connection cells, once for process cells), and is flushed with one RED
//          per field and entry when the CTA retires.
// Everything stays exact integer arithmetic, so the result is independent of grouping and order.
template <int BITS_>
struct HotTableT				// structure of arrays, 20 B per entry
{
	static constexpr int BITS = BITS_;
	static constexpr int N = 1 << BITS;
	uint32_t		tag[N];			// cell id + 1, 0 = free
	uint32_t		count[N];
	unsigned long long	sum[N];
	int			vmax[N];
};
static constexpr uint32_t CELL_TASK = 1u << 30;			// cell ids: conn = slot, task = CELL_TASK | (tslot*48 + hist*16 + bucket)

// one RED per field, nothing is read back: {count, sum} (+ max_val_seen_ for histogram cells)
__device__ __forceinline__ void cell_add_global(const DevState &st, uint32_t cell, uint32_t cnt, unsigned long long sum, int vmax)
{
	if (cell & CELL_TASK) {
		HistCell *c = st.task_hist + (cell & ~CELL_TASK);
		red_add_u64(&c->count, cnt); red_add_u64((unsigned long long *)&c->sum, sum);
		// max_val_seen_ of the histogram: a fire-and-forget RED.MAX — looking first (to skip the atomic) made every process record wait
		// for an L2 round trip; the busy processes' cells
		// live in the CTA's hot table and reach this point once per CTA
		red_max_s64(&st.task_hist[(cell & ~CELL_TASK) | 15u].sum, (long long)vmax);
	}
	else red_add_u64(st.conn_cur + cell, (unsigned long long)cnt + (sum << 32));	// packed {count, kbytes}
}

// all 32 lanes call this; lanes with active == false only take part in the collectives.
// Group sums use a shuffle loop bounded by the largest group of the warp (typically 1-4): redux with per-lane masks would
// make the compiler iterate over every distinct group. No global load anywhere: the updates are fire-and-forget REDs.
// A cell that misses the table takes a free candidate entry when it shows up ADMIT times in this call (on first sight with ADMIT = 1).
template <int ADMIT = 2, typename HotTable>
__device__ __forceinline__ void cell_add(const DevState &st, HotTable &hot, bool active, uint32_t cell, int data)
{
	const int lane = threadIdx.x & 31;
	const uint32_t id = active ? cell : (0x80000000u | (uint32_t)lane);
	const uint32_t m = __match_any_sync(0xffffffffu, id);
	const uint32_t cnt = __popc(m);
	const uint32_t maxcnt = __reduce_max_sync(0xffffffffu, cnt);
	long long sum = data;
	int gmax = data;
	uint32_t rest = m & ~(1u << lane);

	for (uint32_t t = 1; t < maxcnt; ++t) {
		const int src = rest ? (__ffs(rest) - 1) : lane;
		const int other = __shfl_sync(0xffffffffu, data, src);
		if (rest) { sum += other; gmax = max(gmax, other); rest &= rest - 1; }
	}

	if (!active || (m & ((1u << lane) - 1u))) return;		// group leader = lowest lane

	// two candidate entries per cell, hashed with a per-CTA seed: which hot cells collide differs from CTA to CTA, so no cell
	// loses its privatisation everywhere at once (slot numbers, hence cell ids, depend on registration order)
	const uint32_t seed = blockIdx.x * 0x9E3779B9u;
	uint32_t h = ((cell ^ seed) * 2654435761u) >> (32 - HotTable::BITS);
	uint32_t tag = *((volatile uint32_t *)&hot.tag[h]);
	bool hit = tag == cell + 1;

	if (!hit) {
		const uint32_t h2 = ((cell ^ ~seed) * 0x85EBCA6Bu) >> (32 - HotTable::BITS);
		const uint32_t tag2 = *((volatile uint32_t *)&hot.tag[h2]);
		if (tag2 == cell + 1) { hit = true; h = h2; }
		else if (cnt >= (uint32_t)ADMIT) {
			// admission: a free candidate entry
			if (tag == 0) { tag = atomicCAS(&hot.tag[h], 0u, cell + 1); hit = tag == 0 || tag == cell + 1; }
			if (!hit && tag2 == 0) { const uint32_t t2 = atomicCAS(&hot.tag[h2], 0u, cell + 1); if (t2 == 0 || t2 == cell + 1) { hit = true; h = h2; } }
		}
	}
	if (hit) { atomicAdd(&hot.count[h], cnt); atomicAdd(&hot.sum[h], (unsigned long long)sum); atomicMax(&hot.vmax[h], gmax); }
	else cell_add_global(st, cell, cnt, (unsigned long long)sum, gmax);
}

// HLL register update in two halves, so that the caller can put other work between the load of the register word and its use
__device__ __forceinline__ uint32_t hll_peek(const uint8_t *regs, uint32_t idx)
{
	return __ldca(reinterpret_cast<const uint32_t *>(regs) + (idx >> 2));	// stale is harmless: the CAS re-validates
}

__device__ __forceinline__ void hll_raise(uint8_t *regs, uint32_t idx, uint32_t rank, uint32_t w)
{
	uint32_t *wp = reinterpret_cast<uint32_t *>(regs) + (idx >> 2);
	const uint32_t sh = (idx & 3u) * 8u;

	while (((w >> sh) & 0xFFu) < rank) {
		const uint32_t nw = (w & ~(0xFFu << sh)) | (rank << sh);
		const uint32_t old = atomicCAS(wp, w, nw);
		if (old == w) break;
		w = old;
	}
}

__device__ __forceinline__ void hll_update(uint8_t *regs, uint32_t idx, uint32_t rank)
{
	hll_raise(regs, idx, rank, hll_peek(regs, idx));
}

// The kernel is WARP-AUTONOMOUS: no block barrier anywhere in the event loop. A warp takes a chunk of 32 x EPT events and
//   (1) decodes them fully converged: 2 x 128-bit load per event, shard filter, id -> slot lookup with the first table probe
//       of all EPT events in flight together;
//   (2) a RESP sample (70 % of the stream) becomes ONE 64-bit sort key {slot : 24 | value bin : 10 | usec : 30} in the warp's key
//       queue (ballot + popc placement; the queue leaves as a coalesced run, and its digits are counted into the CTA's radix
//       histograms on the way out); beside it only what would change state: the batch extremes of the slot and the CONN_BITMAP bit,
//       each behind a load so that the atomic is issued only while the value still moves;
//   (3) TCP / TASK events join one of the warp's two private shared-memory queues (ballot + popc, no atomics: the queue
//       lengths are warp-uniform registers); a queue leaves for the warp's own region of the batch's record queue only in whole
//       multiples of 32 entries (coalesced 16-byte stores at the warp's running offset, no atomic), the < 32 left-over entries
//       move to the front. drain_kernel applies the records after this kernel: TCP = two lookup2 hashes per flow key -> the
//       flow's entry of the batch flow table (four count-min REDs per flow and batch) + HLL register + the service's exact
//       {count, kbytes} cell; TASK = the three histograms of
//       MAGGR_TASK::set_local_task_state, one record per lane and one cell_add per histogram.
// The histogram cells and the t-digest of a service are produced from its bins by bins_merge_kernel after the batch.
struct alignas(16) IngestRec { uint32_t slot; uint32_t value; unsigned long long flow_key; };		// moved as one 128-bit word
static_assert(sizeof(IngestRec) == 16, "IngestRec travels as one uint4");

// a queued record is read exactly once: evict-first, like the __stcs that wrote it, so that it does not push the drain pass's
// count-min / histogram lines out of L2
__device__ __forceinline__ IngestRec ld_rec(const IngestRec *p)
{
	const uint4 v = __ldcs(reinterpret_cast<const uint4 *>(p));
	IngestRec r; r.slot = v.x; r.value = v.y; r.flow_key = ((unsigned long long)v.w << 32) | v.z;
	return r;
}

// inc into the cells of the flow with hashes h1, h2 in count-min table cms (the geometry of st), one RED per row
__device__ __forceinline__ void cms_add(const DevState &st, unsigned long long *cms, uint32_t h1, uint32_t h2, unsigned long long inc)
{
	for (uint32_t row = 0; row < st.cms_depth; ++row)
		red_add_u64(cms + ((size_t)row << st.cms_log2w) + cms_index2(h1, h2, row, st.cms_wmask), inc);
}

// How a batch flow table entry {key, inc} reaches its cells, in the TASK pass's sweep and on the direct path of flow_add.
// CmsApply: a count-min of one u64 per cell (connections, flow queries), key = h2 << 32 | h1.
struct CmsApply
{
	const DevState &st;
	unsigned long long *cms;
	__device__ __forceinline__ void operator()(unsigned long long key, unsigned long long inc) const
	{
		cms_add(st, cms, (uint32_t)key, (uint32_t)(key >> 32), inc);
	}
};

// GYSK_FLAG_FLOW_RESP_HIST: the key of a response sample in bucket b of the flow with hashes h1, h2, one per cell word:
// ((b >> 1) + 1) << 56 | (h2 & wmask) << 28 | (h1 & wmask), its entry summing the word increments 1 << 32 * (b & 1). Row r's column
// (h1 + r * (h2 | 1)) & wmask depends only on those low bits, and each field holds every width gysk_create accepts (CMS_LOG2W_MAX), so two
// flows with the same key share every cell and their increments may be summed in one entry; the two buckets of a word share it too. The
// key is never 0.
static_assert(2 * CMS_LOG2W_MAX + 4 <= 64 && CMS_LOG2W_MAX <= 28, "resp_hist_key: two column fields of 28 bits and a word field");
__device__ __forceinline__ unsigned long long resp_hist_key(uint32_t h1, uint32_t h2, uint32_t b, uint32_t wmask)
{
	return ((unsigned long long)((b >> 1) + 1u) << 56) | ((unsigned long long)(h2 & wmask) << 28) | (h1 & wmask);
}
__device__ __forceinline__ unsigned long long resp_hist_inc(uint32_t b) { return 1ull << (32u * (b & 1u)); }

// RespHistApply: the summed increment inc of a resp_hist_key into its word of the table's cells, one RED.ADD.64 per row
struct RespHistApply
{
	const DevState &st;
	unsigned long long *tbl;
	__device__ __forceinline__ void operator()(unsigned long long key, unsigned long long inc) const
	{
		const uint32_t w = (uint32_t)(key >> 56) - 1u, h1 = (uint32_t)key & 0xFFFFFFFu, h2 = (uint32_t)(key >> 28) & 0xFFFFFFFu;
		for (uint32_t row = 0; row < st.cms_depth; ++row)
			red_add_u64(tbl + ((((size_t)row << st.cms_log2w) + cms_index2(h1, h2, row, st.cms_wmask)) * RESP_HIST_WORDS + w), inc);
	}
};

// GYSK_FLAG_FLOW_TOPK: flow key fk appended to candidate list l, one cursor atomic per group of converged lanes
__device__ __forceinline__ void topk_append(const TopkList &l, unsigned long long fk)
{
	const uint32_t am = __activemask(), lane = threadIdx.x & 31, leader = __ffs(am) - 1;
	unsigned long long base = 0;
	if (lane == leader) base = atomicAdd(l.n, (unsigned long long)__popc(am));
	base = __shfl_sync(am, base, leader) + __popc(am & ((1u << lane) - 1u));
	if (base < l.cap) l.keys[base] = fk;
}

// What flow_add and flow_sweep record of the flow keys for GYSK_FLAG_FLOW_TOPK: NoCapture nothing; TopkCapture the key of the record that
// claims an entry (beside the entry, for the sweep) and of a record on the direct path (into the candidates).
struct NoCapture
{
	__device__ __forceinline__ void claim(uint32_t, unsigned long long) const {}
	__device__ __forceinline__ void direct(unsigned long long) const {}
	__device__ __forceinline__ void swept(uint32_t) const {}
};
struct TopkCapture
{
	const TopkList &l;
	__device__ __forceinline__ void claim(uint32_t pos, unsigned long long fk) const { l.ekeys[pos] = fk; }
	__device__ __forceinline__ void direct(unsigned long long fk) const { topk_append(l, fk); }
	__device__ __forceinline__ void swept(uint32_t pos) const { topk_append(l, l.ekeys[pos]); }
};

// One connection record's count-min increment into the batch's flow table, given the key k of entry pos (the first probe): a RED into the
// flow's entry, claimed with a CAS on the key if need be. Past FLOW_PROBES entries, or for key 0, the record updates its count-min
// cells directly through apply (normal priority: nothing is left for the TASK pass to reset) and is counted in counter ctr, one RED per
// group of converged lanes, since a table too small for the batch's flows sends most records this way. Entries only go from empty to a
// key during the pass, so a record never misses its flow's entry; should a flow still hold two, the TASK pass applies both. A response
// sample of GYSK_FLAG_FLOW_QUERIES takes the same path with the query flow table, cells and counter, and with GYSK_FLAG_FLOW_RESP_HIST
// once more with the response flow table. cap records the record's flow key fk (GYSK_FLAG_FLOW_TOPK).
template <typename Apply, typename Capture = NoCapture>
__device__ __forceinline__ void flow_add(const DevState &st, const FlowTable &ft, const Apply &apply, int ctr, unsigned long long key,
		uint32_t pos, unsigned long long k, unsigned long long inc, unsigned long long pol_last, const Capture &cap = Capture {},
		unsigned long long fk = 0)
{
	if (key) {
		for (uint32_t p = 0; ; ) {
			if (k == 0) {
				k = atomicCAS(&ft.ent[pos].key, 0ull, key);
				if (k == 0) cap.claim(pos, fk);
			}
			if (k == 0 || k == key) { red_add_u64_hint(&ft.ent[pos].inc, inc, pol_last); return; }
			if (++p == FLOW_PROBES) break;
			pos = (pos + 1) & ft.mask;
			k = ld_cg_hint_u64(&ft.ent[pos].key, pol_last);
		}
	}
	const uint32_t am = __activemask();
	if ((threadIdx.x & 31) == __ffs(am) - 1) atomicAdd(st.counters + ctr, (unsigned long long)__popc(am));
	apply(key, inc);
	cap.direct(fk);
}

// m queued connection records (all 32 lanes call): two lookup2 hashes per flow key -> the flow's entry in the batch's flow table (the
// TASK pass applies it to the count-min cells, DESIGN.md §4) + the HLL register + the service's exact {count, kbytes} cell.
// L2 priorities (DESIGN.md §7): the flow table's lines are taken evict_last, the HLL register sectors evict_first, the records are read
// evict-first (ld_rec). At normal priority the 20 M HLL sectors of a 100 M-event batch, spread over hundreds of MB by the services' Zipf
// tail, pushed the 32 MB of randomly updated lines out of the 50 MB L2 and many REDs became DRAM read-modify-writes. The drain_kernel
// TASK pass sets the lines back to evict_normal. pol_hll / pol_last: l2_policy_evict_first / _last.
// QRY (GYSK_FLAG_FLOW_QUERIES): a record with slot QRY_REC is a response sample {usec, flow key}; it adds {1 | msec << 32} to its flow's
// entry of the query flow table fq (cells fq_cms past the probe limit) and touches neither the HLL nor a service cell.
// RH (GYSK_FLAG_FLOW_RESP_HIST, only with QRY): such a record also adds its word increment to the entry of its resp_hist_key in the
// response flow table fr (cells fr_cms past the probe limit).
// TOPK (GYSK_FLAG_FLOW_TOPK): the record that claims an entry of the connection or query flow table stores its flow key beside the entry,
// and a record on the direct path appends it to the table's candidates (tk).
// SLOW (GYSK_FLAG_FLOW_TOPK_SLOW, only with RH and TOPK): a response sample in bucket b >= b_slow appends its flow key to the slow set's
// candidates tk.list[2], once per record (the selection's key sort removes the repeats).
// CL (GYSK_FLAG_CLIENT_LEVELS): a connection record also raises the open window's client register (cl_open, precision GYSK_HLL_WINDOW_P),
// from the same mixed hash; its word is asked for beside the all-time one and taken with the same policy.
// ERR (GYSK_FLAG_FLOW_ERRORS, only with QRY): a response sample's value carries its error bits (QRY_CLI_ERR, QRY_SER_ERR), masked off
// before its msec and bucket are taken; a sample with either bit adds {cli | ser << 32} to its flow's entry of the error flow table
// ep.ft (cells ep.cms past the probe limit), under the query table's key, and one with the server-error bit appends its flow key to the
// server-error set's candidates ep.list when they are held.
struct ErrPass { FlowTable ft; unsigned long long *cms; TopkList list; };
template <bool QRY, bool RH, bool TOPK, bool SLOW, bool CL, bool ERR, typename HotTable>
__device__ __forceinline__ void drain_tcp_recs(const DevState &st, const FlowTable &ft, HotTable &hot, const IngestRec *q, uint32_t m,
		int lane, unsigned long long pol_hll, unsigned long long pol_last, const FlowTable &fq, unsigned long long *fq_cms, const FlowTable &fr,
		unsigned long long *fr_cms, const FlowTopk &tk, uint32_t b_slow, uint8_t *cl_open, const ErrPass &ep)
{
	for (uint32_t i = lane; i < ((m + 31u) & ~31u); i += 32) {
		const bool act = i < m;
		bool qry = false;
		uint32_t cell = 0, idx = 0, rank = 0, hw = 0, pos = 0, rpos = 0; int kb = 0;
		uint32_t widx = 0, wrank = 0, ww = 0;
		unsigned long long key = 0, inc = 0, k = 0, rkey = 0, rk = 0, rinc = 0, fk = 0;
		uint32_t eb = 0, epos = 0;
		unsigned long long ek = 0;
		if (act) {
			IngestRec r = ld_rec(q + i);
			fk = r.flow_key;
			qry = QRY && r.slot == QRY_REC;
			if (ERR && qry) { eb = r.value >> 30; r.value &= QRY_USEC_MASK; }
			FlowEnt *const tent = qry ? fq.ent : ft.ent;		// field by field: a selected reference would copy both tables to the stack
			const uint32_t tmask = qry ? fq.mask : ft.mask;
			uint32_t h1, h2;
			flow_hashes(r.flow_key, h1, h2);
			// the HLL register word and the flow table's first probe are asked for together and looked at after the cell update, which
			// hides their latency (a stale register is harmless: the CAS re-validates)
			if (!qry) {
				if (CL) {
					const unsigned long long h = hll_hash2(h1, h2);
					hll_idx_rank_h(h, st.hll_p, idx, rank);
					hll_idx_rank_h(h, GYSK_HLL_WINDOW_P, widx, wrank);
				}
				else hll_idx_rank2(h1, h2, st.hll_p, idx, rank);
				hw = ld_na_hint_u32(reinterpret_cast<const uint32_t *>(st.hll + ((size_t)r.slot << st.hll_p)) + (idx >> 2), pol_hll);
				if (CL) ww = ld_na_hint_u32(reinterpret_cast<const uint32_t *>(cl_open + (size_t)r.slot * CL_REGS) + (widx >> 2), pol_hll);
			}
			key = ((unsigned long long)h2 << 32) | h1;
			// usec -> msec as the histogram takes it (ingest_kernel)
			inc = qry ? 1ull | ((unsigned long long)(r.value / 1000u) << 32) : cms_increment(r.value);
			pos = table_hash(key) & tmask;
			if (key) k = ld_cg_hint_u64(&tent[pos].key, pol_last);
			if (RH && qry) {
				const uint32_t b = (uint32_t)bucket_resp_time((long long)(r.value / 1000u));
				rkey = resp_hist_key(h1, h2, b, st.cms_wmask);
				rinc = resp_hist_inc(b);
				rpos = table_hash(rkey) & fr.mask;
				rk = ld_cg_hint_u64(&fr.ent[rpos].key, pol_last);
				if (SLOW && b >= b_slow) topk_append(tk.list[2], fk);
			}
			if (ERR && eb) {
				epos = table_hash(key) & ep.ft.mask;
				if (key) ek = ld_cg_hint_u64(&ep.ft.ent[epos].key, pol_last);
				if (ep.list.keys && (eb & 2u)) topk_append(ep.list, fk);
			}
			cell = r.slot;
			kb = (int)(r.value >> 10);
		}
		cell_add(st, hot, act && !qry, cell, kb);
		if (act) {
			if (TOPK) {
				if (qry) flow_add(st, fq, CmsApply {st, fq_cms}, CTR_FLOWQ_DIRECT, key, pos, k, inc, pol_last, TopkCapture {tk.list[1]}, fk);
				else flow_add(st, ft, CmsApply {st, st.cms_cur}, CTR_FLOW_DIRECT, key, pos, k, inc, pol_last, TopkCapture {tk.list[0]}, fk);
			}
			else if (qry) flow_add(st, fq, CmsApply {st, fq_cms}, CTR_FLOWQ_DIRECT, key, pos, k, inc, pol_last);
			else flow_add(st, ft, CmsApply {st, st.cms_cur}, CTR_FLOW_DIRECT, key, pos, k, inc, pol_last);
			if (RH && qry) flow_add(st, fr, RespHistApply {st, fr_cms}, CTR_FLOWR_DIRECT, rkey, rpos, rk, rinc, pol_last);
			if (ERR && eb) flow_add(st, ep.ft, CmsApply {st, ep.cms}, CTR_FLOWE_DIRECT, key, epos, ek, (eb & 1u) | ((unsigned long long)(eb >> 1) << 32),
					pol_last);
		}
		if (act && !qry) hll_raise(st.hll + ((size_t)cell << st.hll_p), idx, rank, hw);
		if (CL && act && !qry) hll_raise(cl_open + (size_t)cell * CL_REGS, widx, wrank, ww);
	}
}

// one group of queued process records, one record per lane (act: the lane holds one): the three histograms of
// MAGGR_TASK::set_local_task_state, one cell_add per histogram over the whole warp, so that the records of a busy process are summed
// over the group before they reach the hot table or L2.
template <int ADMIT, typename HotTable>
__device__ __forceinline__ void drain_task_group(const DevState &st, HotTable &hot, const IngestRec &r, bool act)
{
	// GY_HISTOGRAM<int, ...>::add_data(int): the three values narrow to int (server/gy_msocket.h:1014-1016)
	const int d[3] = {(int)r.value, (int)(uint32_t)r.flow_key, (int)(uint32_t)(r.flow_key >> 32)};
	uint32_t cell[3];
#pragma unroll
	for (uint32_t h = 0; h < 3; ++h) {
		const uint32_t b = h == 0 ? (uint32_t)bucket_hash_1_3000(d[h]) : (uint32_t)bucket_duration(d[h]);
		cell[h] = CELL_TASK | (r.slot * 3u * HIST_CELLS + h * HIST_CELLS + b);
	}
#pragma unroll
	for (int h = 0; h < 3; ++h) cell_add<ADMIT>(st, hot, act, cell[h], d[h]);
}


// ---- trace rows on the ingest side ----
__device__ __forceinline__ void red_max_u64(unsigned long long *p, unsigned long long v)
{
	asm volatile("red.global.max.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// The trace row of a service slot: the one it holds, else one taken now (a freed row first, else the next fresh one), published in
// row_of; -1 when no row is left. Racing events of the same slot wait for the taker, as table_resolve_slow's readers do.
__device__ __forceinline__ int trace_row_take(const TraceTable &tr, uint32_t slot)
{
	uint32_t r1 = __ldcg(tr.row_of + slot);
	if (r1 != 0 && r1 != TRACE_BUSY) return (int)(r1 - 1u);
	if (r1 == 0 && (r1 = atomicCAS(tr.row_of + slot, 0u, TRACE_BUSY)) == 0) {
		uint32_t r = ~0u;
		const int32_t f = atomicSub(tr.free_n, 1);
		if (f > 0) r = tr.free_rows[f - 1];
		else {
			atomicAdd(tr.free_n, 1);
			const uint32_t c = atomicAdd(tr.count, 1u);
			if (c < tr.rows) r = c;
			else atomicSub(tr.count, 1u);
		}
		if (r != ~0u) tr.row_slot[r] = slot;
		st_volatile_u32(tr.row_of + slot, r == ~0u ? 0u : r + 1u);
		return r == ~0u ? -1 : (int)r;
	}
	while (r1 == TRACE_BUSY) { __nanosleep(20); r1 = ld_volatile_u32(tr.row_of + slot); }
	return r1 ? (int)(r1 - 1u) : -1;
}

// The counters ingest_kernel adds per trace event (nerr, nconns, bytes in / out and their maxima), summed over a warp's lanes of one row
// and held warp-uniform until a different row comes along or the kernel ends: one traced service brings millions of events per batch,
// and REDs on one line are applied one after the other.
struct TraceAcc
{
	int row;
	unsigned long long nerr, nconns, bin, bout;
	uint32_t min_, mout;

	__device__ __forceinline__ void clear() { row = -1; nerr = nconns = bin = bout = 0; min_ = mout = 0; }
	__device__ __forceinline__ void flush(const TraceTable &tr, int lane)
	{
		if (row >= 0 && lane == 0) {
			unsigned long long *w = tr.words(tr.par, (uint32_t)row);
			if (nerr) red_add_u64(w + TW_NERR, nerr);
			if (nconns) red_add_u64(w + TW_NCONNS, nconns);
			if (bin) red_add_u64(w + TW_BYTES_IN, bin);
			if (bout) red_add_u64(w + TW_BYTES_OUT, bout);
			if (min_) red_max_u64(w + TW_MAX_IN, min_);
			if (mout) red_max_u64(w + TW_MAX_OUT, mout);
		}
		clear();
	}
	// the lanes' events (row < 0: none), all 32 lanes
	__device__ __forceinline__ void add(const TraceTable &tr, int r_lane, uint32_t flags, unsigned long long fk, int lane)
	{
		const uint32_t lo = (uint32_t)fk, hi = (uint32_t)(fk >> 32);
		for (uint32_t todo = __ballot_sync(0xffffffffu, r_lane >= 0); todo; ) {
			const int r = __shfl_sync(0xffffffffu, r_lane, __ffs(todo) - 1);
			const bool in = r_lane == r;
			todo &= ~__ballot_sync(0xffffffffu, in);
			const uint32_t ec = __reduce_add_sync(0xffffffffu, in ? (flags & GYSK_EVF_TRACE_ERROR ? 1u : 0u) | (flags & GYSK_EVF_TRACE_NEWCONN ? 1u << 16 : 0u) : 0u);
			const unsigned long long bi = __reduce_add_sync(0xffffffffu, in ? lo & 0xFFFFu : 0u) + ((unsigned long long)__reduce_add_sync(0xffffffffu, in ? lo >> 16 : 0u) << 16);
			const unsigned long long bo = __reduce_add_sync(0xffffffffu, in ? hi & 0xFFFFu : 0u) + ((unsigned long long)__reduce_add_sync(0xffffffffu, in ? hi >> 16 : 0u) << 16);
			const uint32_t mi = __reduce_max_sync(0xffffffffu, in ? lo : 0u), mo = __reduce_max_sync(0xffffffffu, in ? hi : 0u);
			if (r != row) { flush(tr, lane); row = r; }
			nerr += ec & 0xFFFFu; nconns += ec >> 16; bin += bi; bout += bo;
			min_ = max(min_, mi); mout = max(mout, mo);
		}
	}
};

struct IngestShared
{
	static constexpr int KQ_CAP = 192, KQ_FLUSH = KQ_CAP - IngestShape::CHUNK;	// a flush leaves room for a whole chunk of RESP events
	static constexpr int RQ_CAP = 32 + IngestShape::CHUNK;		// < 32 left over + one chunk
	static constexpr int DH = 1 << KEY_DIGIT_MAX;			// digit values of a RESP-key radix pass
	struct Warp { unsigned long long kq[KQ_CAP]; IngestRec tcp[RQ_CAP], task[RQ_CAP]; };
	Warp		w[IngestShape::WARPS];
	uint32_t	dhist[KEY_PASSES_MAX][DH];			// digit histograms of this CTA's keys, one per radix pass
};

// TRACE: the engine has trace rows (a separate instance, so that an engine without them runs the kernel without the trace path).
// QRY: GYSK_FLAG_FLOW_QUERIES (a separate instance too): every response sample that reaches its service's histogram, by the key or the
// hot-row route, also joins the connection queue as a record {QRY_REC, usec, flow key} for the TCP drain pass.
// TOPK: GYSK_FLAG_FLOW_TOPK (a separate instance too): the flow key of each ACTIVE record, which updates the count-min here, joins the
// connection table's candidates tl.
// ERR: GYSK_FLAG_FLOW_ERRORS (a separate instance too, only with QRY): a queued response sample also carries its event's GYSK_EVF_CLI_ERROR
// / GYSK_EVF_SER_ERROR bits in bits 30 / 31 of its value (QRY_CLI_ERR, QRY_SER_ERR).
// ClOpen: GYSK_FLAG_CLIENT_LEVELS (a separate instance too) with one uint8_t * parameter, the open window's client registers, which each
// ACTIVE record also raises. A pack, so that the instances without the flag keep their parameter list.
__device__ __forceinline__ uint8_t *cl_open_of() { return nullptr; }
__device__ __forceinline__ uint8_t *cl_open_of(uint8_t *p) { return p; }
template <bool TRACE, bool QRY, bool TOPK, bool ERR, typename... ClOpen>
__global__ void __launch_bounds__(IngestShape::WARPS * 32, IngestShape::MIN_CTAS) ingest_kernel(DevState st, const gysk_event *__restrict__ ev, uint64_t n,
		unsigned long long *__restrict__ keys, uint32_t *__restrict__ ghist, SortPlan plan, uint4 *__restrict__ recq, uint2 *__restrict__ rec_cnt, TopkList tl,
		ClOpen... cl_open)
{
	constexpr bool CL = sizeof...(ClOpen) > 0;
	constexpr int WARPS = IngestShape::WARPS, EPT = IngestShape::EPT, CHUNK = IngestShape::CHUNK, DH = IngestShared::DH;
	extern __shared__ __align__(128) unsigned char smem_raw[];
	IngestShared &S = *reinterpret_cast<IngestShared *>(smem_raw);
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	IngestShared::Warp &W = S.w[wid];
	const uint32_t lt = (1u << lane) - 1u;
	uint32_t c_in = 0, c_foreign = 0, n_resp = 0, n_active = 0;	// per thread: < 2^32 events per launch
	uint32_t n_trace = 0, n_trace_drop = 0;				// trace events kept / dropped for want of a row
	TraceAcc tacc;
	tacc.clear();
	uint32_t nk = 0, ntcp = 0, ntask = 0;				// queue lengths (warp-uniform)
	unsigned long long t_tcp = 0, t_task = 0;			// queued in total (warp-uniform)

	for (int i = threadIdx.x; i < KEY_PASSES_MAX * DH; i += WARPS * 32) (&S.dhist[0][0])[i] = 0;
	__syncthreads();						// the only block barriers: here and before the retire step

	const uint64_t nchunks = (n + CHUNK - 1) / CHUNK;
	const uint64_t nwarps = (uint64_t)gridDim.x * WARPS;
	const uint64_t gwarp = (uint64_t)blockIdx.x * WARPS + wid;

	// ---- queue drains (all 32 lanes, m = multiple of 32 except in the final drain): handed as one coalesced run to the warp's
	//      region of the batch's record queue, which the two drain_kernel passes apply after this kernel ----
	// the region holds what the warp's chunks can bring (rcap = its number of chunks x CHUNK): connection records grow from its front,
	// process records from its back (taskq = its last entry); the offsets are the warp's totals so far, no atomic
	const uint64_t rcap = (nchunks + nwarps - 1) / nwarps * CHUNK;
	uint4 *const tcpq = recq + gwarp * rcap, *const taskq = tcpq + (rcap - 1);
	auto hand_over = [&](const IngestRec *q, uint32_t m, uint4 *gq, unsigned long long base, bool backwards) {
		for (uint32_t i = lane; i < m; i += 32) {
			const uint4 v = *reinterpret_cast<const uint4 *>(q + i);
			if (backwards) __stcs(gq - (long long)(base + i), v); else __stcs(gq + base + i, v);
		}
	};
	auto drain_tcp = [&](uint32_t m) { hand_over(W.tcp, m, tcpq, t_tcp, false); };
	auto drain_task = [&](uint32_t m) { hand_over(W.task, m, taskq, t_task, true); };
	auto keep_rest = [&](IngestRec *q, uint32_t m, uint32_t total) {		// entries [m, total) move to the front (total - m < 32)
		IngestRec r;
		const bool mv = m + lane < total;
		if (mv) r = q[m + lane];
		__syncwarp();
		if (mv) q[lane] = r;
		__syncwarp();
	};
	auto flush_keys = [&]() {
		unsigned long long base = 0;
		if (lane == 0) base = atomicAdd(st.counters + CTR_NKEYS, (unsigned long long)nk);
		base = __shfl_sync(0xffffffffu, base, 0);
		for (uint32_t q = lane; q < nk; q += 32) {
			const unsigned long long k = W.kq[q];
#pragma unroll
			for (int p = 0; p < KEY_PASSES_MAX; ++p)
				if (p < plan.np) atomicAdd(&S.dhist[p][sort_digit(k, plan.shift[p], plan.bits[p])], 1u);
			__stcs(keys + base + q, k);
		}
		nk = 0;
		__syncwarp();
	};

	for (uint64_t chunk = gwarp; chunk < nchunks; chunk += nwarps) {
		const uint64_t cbase = chunk * CHUNK;
		uint4 ra[EPT], rb[EPT];
#pragma unroll
		for (int k = 0; k < EPT; ++k) {
			const uint64_t i = cbase + (uint64_t)k * 32 + lane;
			if (i < n) {
				ra[k] = __ldcs(reinterpret_cast<const uint4 *>(ev + i));		// streamed once: evict-first, keep L2 for
				rb[k] = __ldcs(reinterpret_cast<const uint4 *>(ev + i) + 1);	// the id table / histogram / count-min lines
			}
			else { ra[k] = make_uint4(0, 0, 0, 0); rb[k] = make_uint4(0, 0, 0, 0xFFFFu); }	// type 0xFFFF: padding, not counted
		}

		// decode; put the first id-table probe of all EPT events in flight before any of them is resolved
		uint4 praw[EPT];
		uint32_t ppos[EPT];
		uint32_t kind[EPT];		// 0 none, GYSK_EV_RESP, GYSK_EV_ACCEPT (= any TCP type), GYSK_EV_TASK
#pragma unroll
		for (int k = 0; k < EPT; ++k) {
			const unsigned long long svc = ((unsigned long long)ra[k].y << 32) | ra[k].x;
			const uint32_t value = rb[k].x, host_idx = rb[k].y;
			const uint32_t type = rb[k].w & 0xFFFFu;
			const bool is_resp = type == GYSK_EV_RESP, is_task = type == GYSK_EV_TASK;
			const bool is_tcp = type >= GYSK_EV_CONNECT && type <= GYSK_EV_CLOSE_SER, is_active = type == GYSK_EV_ACTIVE;
			const bool is_trace = TRACE && type == GYSK_EV_TRACE;	// every response time: the row counts those beyond the rule too
			bool mine = type != 0xFFFFu;

			kind[k] = 0; ppos[k] = 0; praw[k] = make_uint4(0, 0, 0, 0);
			if (mine && st.world > 1 && (host_idx % st.world) != st.rank) { c_foreign++; mine = false; }
			if (mine) {
				c_in++;
				// usec -> msec as SVC_INFO_CAP::upd_stats_on_req (gy_proto_parser.cc:2678); validity rule of
				// handle_ipv4_resp_event (gy_socket_stat.cc:1519-1524): drop beyond 1 000 000 msec
				if (svc + 1ull > 1ull && (is_tcp || is_task || is_active || is_trace || (is_resp && value < 1000001000u))) {	// id not 0 / ~0 (tombstone); msec <= 1 000 000
					kind[k] = is_resp ? (uint32_t)GYSK_EV_RESP : (is_task ? (uint32_t)GYSK_EV_TASK : (is_active ? (uint32_t)GYSK_EV_ACTIVE :
							(is_trace ? (uint32_t)GYSK_EV_TRACE : (uint32_t)GYSK_EV_ACCEPT)));
					praw[k] = table_probe_first(is_task ? st.task_tbl : st.svc_tbl, svc, ppos[k]);
				}
			}
		}
		// resolve every slot, then put the second round of loads (the slot's batch record and CONN_BITMAP word) of all EPT events
		// in flight together, and fire the bin REDs — nothing below waits for them
		int slotv[EPT], trow[EPT];
		uint4 sbv[EPT];
		uint32_t mwv[EPT], bkt[EPT];
#pragma unroll
		for (int k = 0; k < EPT; ++k) {
			const bool is_resp = kind[k] == GYSK_EV_RESP, is_task = kind[k] == GYSK_EV_TASK;
			int slot = -1;
			if (kind[k]) {
				// one id lookup for all three event kinds (services and tasks live in separate tables)
				slot = table_resolve(is_task ? st.task_tbl : st.svc_tbl, ((unsigned long long)ra[k].y << 32) | ra[k].x, st.auto_register, rb[k].y, ppos[k], praw[k]);
			}
			slotv[k] = slot; sbv[k] = make_uint4(0, 0, 0, 0); mwv[k] = 0; bkt[k] = 0; trow[k] = -1;
			if (TRACE && slot >= 0 && kind[k] == GYSK_EV_TRACE) {
				trow[k] = trace_row_take(st.trace, (uint32_t)slot);
				if (trow[k] >= 0) n_trace++; else n_trace_drop++;
			}
			if (slot >= 0 && is_resp) {
				const uint32_t v = rb[k].x, ms = v / 1000u;		// usec -> msec as SVC_INFO_CAP::upd_stats_on_req (gy_proto_parser.cc:2678)
				const uint32_t b = (uint32_t)bucket_resp_time((long long)ms);
				bkt[k] = b;
				sbv[k] = ld_cg_v4(st.slot_batch + slot);
				mwv[k] = __ldcg(st.bm_cur + (size_t)slot * HIST_CELLS + b);
				n_resp++;
			}
		}
#pragma unroll
		for (int k = 0; k < EPT; ++k) {
			const bool is_resp = kind[k] == GYSK_EV_RESP, is_task = kind[k] == GYSK_EV_TASK, is_tcp = kind[k] == GYSK_EV_ACCEPT;
			const int slot = slotv[k];
			const bool ok = slot >= 0;
			// a hot service (sbv.w = 1 + its row of dense value bins, handed out by bins_merge_kernel after an earlier batch) takes its
			// sample as two REDs into the L2-resident row; everybody else's sample becomes a sort key
			const uint32_t hotrow = (ok && is_resp) ? sbv[k].w : 0u;
			// a trace sample within the RESP validity rule becomes a sort key of its row's pseudo-slot (a trace row: trow >= 0)
			const bool tr_key = TRACE && trow[k] >= 0 && rb[k].x < 1000001000u;
			const uint32_t m_resp = __ballot_sync(0xffffffffu, (ok && is_resp && !hotrow) || tr_key),
					m_tcp = __ballot_sync(0xffffffffu, ok && (is_tcp || (QRY && is_resp))), m_task = __ballot_sync(0xffffffffu, ok && is_task);
			if (ok) {
				if (is_resp) {
					const uint32_t bin = td_code(rb[k].x) + bkt[k];
					if (hotrow) {
						unsigned long long *hb = st.hot_rows + (size_t)(hotrow - 1u) * HOT_ROW_WORDS + hot_word(bin);
						const uint32_t us = rb[k].x;
						red_add_u64(hb, 1ull | ((unsigned long long)(us - (us / 1000u) * 1000u) << BIN_CNT_BITS));
						red_add_u64(hb + HOT_ROW_BINS, (unsigned long long)us);
					}
					else W.kq[nk + __popc(m_resp & lt)] = ((unsigned long long)(uint32_t)slot << KEY_SLOT_SHIFT) |
							((unsigned long long)bin << KEY_GROUP_SHIFT) | rb[k].x;
					// the rest only when it changes something: batch extremes (minv != ~0 also marks the slot as touched) and the
					// CONN_BITMAP bit — TCP_LISTENER::CONN_BITMAP::add_response (common/gy_socket_stat.h:403-410), transposed: per
					// bucket a mask over client port & 31
					const uint32_t v = rb[k].x;
					if (v < sbv[k].x) atomicMin(&st.slot_batch[slot].minv, v);
					if (v > sbv[k].y) atomicMax(&st.slot_batch[slot].maxv, v);
					const uint32_t bit = 1u << (ra[k].z & 0x1Fu);
					if (!(mwv[k] & bit)) atomicOr(st.bm_cur + (size_t)slot * HIST_CELLS + bkt[k], bit);
					const uint32_t ef = rb[k].w >> 16;			// API_TRAN error flags: rare
					if (ef & 3u) red_add_u64(&st.slot_aux[slot].err_cur, (unsigned long long)(ef & 1u) | ((unsigned long long)((ef >> 1) & 1u) << 32));
					if (QRY) {
						IngestRec r; r.slot = QRY_REC; r.value = ERR ? v | ((ef & 3u) << 30) : v; r.flow_key = ((unsigned long long)ra[k].w << 32) | ra[k].z;
						W.tcp[ntcp + __popc(m_tcp & lt)] = r;
					}
				}
				else if (TRACE && kind[k] == GYSK_EV_TRACE) {
					const uint32_t v = rb[k].x;
					// the value bins of a RESP key (td_code + RESP_TIME_HASH bucket): the batch items are those of the service digest's path
					if (tr_key) W.kq[nk + __popc(m_resp & lt)] = ((unsigned long long)(st.trace.base + (uint32_t)trow[k]) << KEY_SLOT_SHIFT) |
							((unsigned long long)resp_bin(v) << KEY_GROUP_SHIFT) | v;
					else if (trow[k] >= 0) {
						// beyond the validity rule (rare): no key, the counters the key would have brought straight into the row
						unsigned long long *w = st.trace.words(st.trace.par, (uint32_t)trow[k]);
						red_add_u64(w + TW_NREQ, 1ull);
						red_add_u64(w + TW_SUM_US, (unsigned long long)v);
						red_max_u64(w + TW_MAX_US, (unsigned long long)v);
						red_add_u64(w + TW_BKT + 7, 1ull);
					}
				}
				else if (kind[k] == GYSK_EV_ACTIVE) {
					// one pre-aggregated {listener, client process} record of the 15-s inet_diag scan (gy_socket_stat.cc:6156-6194): a few
					// per flow and minute — handled on the spot. The flow sketch takes its connections and kbytes, the service its totals.
					const unsigned long long fk = ((unsigned long long)ra[k].w << 32) | ra[k].z;
					const unsigned long long inc = (unsigned long long)(rb[k].w >> 16) | ((unsigned long long)rb[k].x << 32);
					uint32_t h1, h2, idx, rank;
					flow_hashes(fk, h1, h2);
					cms_add(st, st.cms_cur, h1, h2, inc);
					if (TOPK) topk_append(tl, fk);
					hll_idx_rank2(h1, h2, st.hll_p, idx, rank);
					hll_update(st.hll + ((size_t)slot << st.hll_p), idx, rank);
					if constexpr (CL) {		// ACTIVE records are few: the hash is mixed once more rather than kept across the all-time update
						hll_idx_rank_h(hll_hash2(h1, h2), GYSK_HLL_WINDOW_P, idx, rank);
						hll_update(cl_open_of(cl_open...) + (size_t)slot * CL_REGS, idx, rank);
					}
					red_add_u64(&st.slot_aux[slot].act_cur, inc);
					atomicMax(&st.slot_aux[slot].rtt_cur, rb[k].z);		// non-negative floats order like their bit patterns
					n_active++;
				}
				else {
					IngestRec r; r.slot = (uint32_t)slot; r.value = rb[k].x; r.flow_key = ((unsigned long long)ra[k].w << 32) | ra[k].z;
					if (is_tcp) W.tcp[ntcp + __popc(m_tcp & lt)] = r;
					else W.task[ntask + __popc(m_task & lt)] = r;
				}
			}
			nk += __popc(m_resp); ntcp += __popc(m_tcp); ntask += __popc(m_task);
			if (TRACE) tacc.add(st.trace, trow[k], rb[k].w >> 16, ((unsigned long long)ra[k].w << 32) | ra[k].z, lane);
		}
		__syncwarp();

		if (ntcp >= 32) { const uint32_t m = ntcp & ~31u; drain_tcp(m); keep_rest(W.tcp, m, ntcp); t_tcp += m; ntcp -= m; }
		if (ntask >= 32) { const uint32_t m = ntask & ~31u; drain_task(m); keep_rest(W.task, m, ntask); t_task += m; ntask -= m; }
		if (nk > (uint32_t)IngestShared::KQ_FLUSH) flush_keys();
	}
	// what is left in the queues
	if (ntcp) { drain_tcp(ntcp); t_tcp += ntcp; }
	if (ntask) { drain_task(ntask); t_task += ntask; }
	if (nk) flush_keys();
	if (TRACE) tacc.flush(st.trace, lane);
	if (lane == 0) rec_cnt[gwarp] = make_uint2((uint32_t)t_tcp, (uint32_t)t_task);	// every warp of the launch: no memset needed

	__syncthreads();
	// retire: one RED per digit this CTA saw
	for (int i = threadIdx.x; i < plan.np * DH; i += WARPS * 32) {
		const uint32_t c = (&S.dhist[0][0])[i];
		if (c) atomicAdd(ghist + (i / DH) * RADIX_MAX + (i % DH), c);		// the passes read their histogram at stride RADIX_MAX
	}

	// statsmap-style counters (gy_mconnhdlr.cc:4708-4715): warp-reduce, one atomic per warp and counter
	c_in = __reduce_add_sync(0xffffffffu, c_in);
	c_foreign = __reduce_add_sync(0xffffffffu, c_foreign);
	const unsigned long long t_resp = __reduce_add_sync(0xffffffffu, n_resp);
	if (QRY) t_tcp -= t_resp;					// each counted response sample was queued once as a QRY_REC record
	t_tcp += __reduce_add_sync(0xffffffffu, n_active);		// counted with the connection events
	const unsigned long long t_trace = __reduce_add_sync(0xffffffffu, n_trace);
	n_trace_drop = __reduce_add_sync(0xffffffffu, n_trace_drop);
	if (lane == 0) {
		if (TRACE && n_trace_drop) atomicAdd(st.trace.dropped, (unsigned long long)n_trace_drop);
		if (c_in) atomicAdd(st.counters + CTR_IN, (unsigned long long)c_in);
		if (c_foreign) atomicAdd(st.counters + CTR_FOREIGN, (unsigned long long)c_foreign);
		if (t_resp) atomicAdd(st.counters + CTR_RESP, t_resp);
		if (t_tcp) atomicAdd(st.counters + CTR_TCP, t_tcp);
		if (t_task) atomicAdd(st.counters + CTR_TASK, t_task);
		// dropped = taken in but not queued (svc_id 0, bad type or value, table full, unknown id); two's complement arithmetic
		const unsigned long long q = t_resp + t_tcp + t_task + t_trace;
		if (c_in != q) atomicAdd(st.counters + CTR_DROPPED, (unsigned long long)c_in - q);
	}
}

// ---------------------------------------------------------------------------------------------------
// drain passes: the connection and process records ingest_kernel queued, applied in two launches after it, TCP first, then TASK.
// Each pass touches only its own state (flow table + HLL + connection cells, about 33 MB at the bench's sizes, or the process
// histograms, about 19 MB), and each fits in the H100's 50 MB L2 on its own; inside ingest_kernel they competed with each other and
// with the RESP path's tables, bitmaps and hot rows for it (DESIGN.md §7). Two launches, not two phases of one kernel: CTAs would
// reach the second phase at different times and mix the two working sets again. Persistent grid; a warp takes 32 records at a time;
// hot cells are privatised per CTA (cell_add). Inside the TCP pass, L2 priorities keep the flow table resident against the HLL
// sectors (drain_tcp_recs); the TASK pass first applies the flow table to the count-min.
// ---------------------------------------------------------------------------------------------------
// Launch shape of each pass: warps per CTA and hot-table entries (2^HOT_BITS, 20 B each); CTAs per SM follow from the shared memory
// (DESIGN.md §7 has the measurements behind each choice). ADMIT: cell_add's admission threshold.
template <bool TASK> struct DrainShape;
template <> struct DrainShape<false> { static constexpr int WARPS = 8, HOT_BITS = 12, ADMIT = 2; };	// 4096 entries, 80 KB: faster than 2^11 and 2^9
// one CTA of 16 warps per SM around 8192 entries (160 KB), a cell admitted on first sight: the process cells that miss the table
// cost three L2 REDs each, and they were most of the pass's time
template <> struct DrainShape<true> { static constexpr int WARPS = 16, HOT_BITS = 13, ADMIT = 1; };

// A flow table the TCP pass filled, swept by the whole grid of the TASK pass: each entry's sum into its flow's cells through apply (the
// key holds what picks them), then the entry emptied for the next batch. The TCP pass left the table's lines evict_last, a
// priority they keep after it ends: back to normal, so that they do not hold L2 against the next batch's ingest_kernel and chain. A
// thread takes FLOW_SWEEP entries a step, one grid stride apart, their loads in flight together (the REDs' memory clobber keeps a load
// from moving past them). cap records the flow key stored beside each entry the sweep applies (GYSK_FLAG_FLOW_TOPK).
template <typename Apply, typename Capture = NoCapture>
__device__ __forceinline__ void flow_sweep(const FlowTable &t, const Apply &apply, const Capture &cap = Capture {})
{
	const uint32_t stride = gridDim.x * blockDim.x;
	for (uint32_t i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 <= t.mask; i0 += FLOW_SWEEP * stride) {
		FlowEnt f[FLOW_SWEEP];
#pragma unroll
		for (uint32_t u = 0; u < FLOW_SWEEP; ++u) if (i0 + u * stride <= t.mask) f[u] = t.ent[i0 + u * stride]; else f[u] = FlowEnt {0ull, 0ull};
#pragma unroll
		for (uint32_t u = 0; u < FLOW_SWEEP; ++u) {
			const uint32_t i = i0 + u * stride;
			if (f[u].key) {
				apply(f[u].key, f[u].inc);
				cap.swept(i);
				t.ent[i] = FlowEnt {0ull, 0ull};
			}
			if (i <= t.mask && !(i & 7u)) l2_evict_normal_line(t.ent + i);
		}
	}
}

// The records sit in the ingest launch's per-warp regions (RecRegions). Each CTA scans the regions' counts into a table of where
// each region's groups of 32 records start, and every warp takes an equal, contiguous share of all groups: the regions' sizes
// differ, the drain warps' work does not.
// QRY (GYSK_FLAG_FLOW_QUERIES): the TCP pass also sums the queued response samples in the query flow table fq, and the TASK pass applies
// that table to the query cells fq_cms after the connection flow table.
// RH (GYSK_FLAG_FLOW_RESP_HIST, only with QRY): the same once more with the response flow table fr and the response histogram cells fr_cms.
// TOPK (GYSK_FLAG_FLOW_TOPK): the TCP pass keeps the flow keys of the connection and query records (drain_tcp_recs), and the TASK pass's
// sweeps append the key beside each applied entry to that table's candidates tk.
// SLOW (GYSK_FLAG_FLOW_TOPK_SLOW, TCP pass only): the TCP pass also keeps the flow key of each response sample in bucket b_slow or above.
// CL (GYSK_FLAG_CLIENT_LEVELS, TCP pass only): the TCP pass also raises the open window's client registers cl_open.
// ERR (GYSK_FLAG_FLOW_ERRORS, only with QRY): the TCP pass also sums the error samples in the error flow table ep.ft (drain_tcp_recs), and
// the TASK pass applies that table to the error cells ep.cms after the others. A trailing parameter, so that the instances without the
// flag keep their parameter layout.
template <bool TASK, bool QRY, bool RH, bool TOPK, bool SLOW, bool CL, bool ERR>
__global__ void __launch_bounds__(DrainShape<TASK>::WARPS * 32) drain_kernel(DevState st, FlowTable ft, const uint4 *__restrict__ q, const uint2 *__restrict__ cnt,
		RecRegions rr, FlowTable fq, unsigned long long *fq_cms, FlowTable fr, unsigned long long *fr_cms, FlowTopk tk, uint32_t b_slow, uint8_t *cl_open,
		ErrPass ep)
{
	constexpr int WARPS = DrainShape<TASK>::WARPS;
	using DrainHot = HotTableT<DrainShape<TASK>::HOT_BITS>;
	if (TASK && TOPK) {
		flow_sweep(ft, CmsApply {st, st.cms_cur}, TopkCapture {tk.list[0]});
		if (QRY) flow_sweep(fq, CmsApply {st, fq_cms}, TopkCapture {tk.list[1]});
		if (RH) flow_sweep(fr, RespHistApply {st, fr_cms});
		if (ERR) flow_sweep(ep.ft, CmsApply {st, ep.cms});
	}
	else if (TASK) {
		flow_sweep(ft, CmsApply {st, st.cms_cur});
		if (QRY) flow_sweep(fq, CmsApply {st, fq_cms});
		if (RH) flow_sweep(fr, RespHistApply {st, fr_cms});
		if (ERR) flow_sweep(ep.ft, CmsApply {st, ep.cms});
	}
	const unsigned long long pol_hll = TASK ? 0 : l2_policy_evict_first(), pol_last = TASK ? 0 : l2_policy_evict_last();
	extern __shared__ __align__(16) unsigned char drain_smem[];
	DrainHot &hot = *reinterpret_cast<DrainHot *>(drain_smem);
	// [nwarps + 1] per region: first group << 5 | (records & 31); the last entry holds the number of groups << 5
	uint32_t *rstart = reinterpret_cast<uint32_t *>(drain_smem + sizeof(DrainHot));
	__shared__ uint32_t wsum[WARPS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	for (int i = threadIdx.x; i < DrainHot::N; i += WARPS * 32) { hot.tag[i] = 0; hot.count[i] = 0; hot.sum[i] = 0; hot.vmax[i] = INT_MIN; }

	// exclusive scan of the regions' group counts: thread t takes a contiguous run of regions
	const uint32_t nreg = rr.nwarps, per = (nreg + WARPS * 32 - 1) / (WARPS * 32), r0 = threadIdx.x * per;
	const uint32_t r1 = min(r0 + per, nreg);
	uint32_t s = 0;
	for (uint32_t r = r0; r < r1; ++r) {
		const uint32_t c = TASK ? cnt[r].y : cnt[r].x;
		rstart[r] = c; s += (c + 31u) >> 5;
	}
	uint32_t incl = s;
#pragma unroll
	for (int off = 1; off < 32; off <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += t; }
	if (lane == 31) wsum[wid] = incl;
	__syncthreads();
	uint32_t g0 = incl - s, ngroups = 0;
#pragma unroll
	for (int w = 0; w < WARPS; ++w) { if (w < wid) g0 += wsum[w]; ngroups += wsum[w]; }
	for (uint32_t r = r0; r < r1; ++r) { const uint32_t c = rstart[r]; rstart[r] = (g0 << 5) | (c & 31u); g0 += (c + 31u) >> 5; }
	if (threadIdx.x == 0) rstart[nreg] = ngroups << 5;
	__syncthreads();

	const uint32_t gw = blockIdx.x * WARPS + wid, nw = gridDim.x * WARPS;
	const uint32_t gbeg = (uint32_t)((unsigned long long)ngroups * gw / nw), gend = (uint32_t)((unsigned long long)ngroups * (gw + 1) / nw);
	const IngestRec *recs = reinterpret_cast<const IngestRec *>(q);
	// region of group gbeg: the last one that starts at or before it
	uint32_t r = 0;
	for (uint32_t hi = nreg; r < hi; ) { const uint32_t mid = (r + hi + 1) >> 1; if ((rstart[mid] >> 5) <= gbeg) r = mid; else hi = mid - 1; }
	// group g (< gend) -> its region r (walked forward), where it starts in the region and how many records it holds
	auto locate = [&](uint32_t g, uint32_t &off, uint32_t &m) {
		while ((rstart[r + 1] >> 5) <= g) ++r;			// empty regions start where the next one does
		const uint32_t first = rstart[r] >> 5, tail = rstart[r] & 31u;
		off = (g - first) * 32u;
		m = (g + 1 == rstart[r + 1] >> 5 && tail) ? tail : 32u;
	};
	if (TASK) {
		// one record per lane and group, read once: process records grow from the back of their region, so a group is one coalesced
		// backward read. The next group's records are in flight while the current group is applied.
		auto fetch = [&](uint32_t g, uint32_t &m) {
			uint32_t off;
			locate(g, off, m);
			IngestRec rec {0u, 0u, 0ull};
			if ((uint32_t)lane < m) rec = ld_rec(recs + (unsigned long long)r * rr.cap + (rr.cap - 1 - off - lane));
			return rec;
		};
		uint32_t m = 0;
		IngestRec next = gbeg < gend ? fetch(gbeg, m) : IngestRec {0u, 0u, 0ull};
		for (uint32_t g = gbeg; g < gend; ++g) {
			const IngestRec cur = next;
			const bool act = (uint32_t)lane < m;
			if (g + 1 < gend) next = fetch(g + 1, m);
			drain_task_group<DrainShape<TASK>::ADMIT>(st, hot, cur, act);
		}
	}
	else {
		for (uint32_t g = gbeg; g < gend; ++g) {
			uint32_t off, m;
			locate(g, off, m);
			drain_tcp_recs<QRY, RH, TOPK, SLOW, CL, ERR>(st, ft, hot, recs + (unsigned long long)r * rr.cap + off, m, lane, pol_hll, pol_last, fq, fq_cms, fr,
					fr_cms, tk, b_slow, cl_open, ep);
		}
	}

	__syncthreads();
	for (int i = threadIdx.x; i < DrainHot::N; i += WARPS * 32) {
		if (hot.tag[i] && hot.count[i]) cell_add_global(st, hot.tag[i] - 1, hot.count[i], hot.sum[i], hot.vmax[i]);
	}
}

// ---------------------------------------------------------------------------------------------------
// stable LSD radix sort of 64-bit keys on the bit range of a SortPlan, one digit of 6 to 9 bits per pass (a narrower last digit runs
// in the 6-bit kernel), tile = SORT_TILE keys per CTA of 256 threads. It sorts every batch's RESP keys by slot
// (launch_batch_merge) and, through launch_radix_sort, the window list by host, the top-N keys of services, processes and logical
// services by score, and the group-by's keys by group.
//
// one-sweep radix pass: 16 B of HBM traffic per key and pass (read once, write once)
//
//   os_hist_kernel     one read of the keys fills the GLOBAL digit histograms of every pass (a stable pass does not change how
//                      many keys carry a digit value);
//   os_pass_kernel     a CTA takes the next tile (ticket from an atomic counter, so every predecessor tile is already running),
//                      ranks its keys per digit, publishes the tile's digit counts and obtains the number of keys with the same
//                      digit in all earlier tiles by decoupled look-back over the status words of its predecessors
//                      (status word = pass epoch : 32 | state : 2 | count : 30; state 1 = this tile's count, 2 = inclusive prefix
//                      up to this tile; a word of another epoch reads as "not there yet", so the array is never cleared),
//                      reorders the tile by digit in shared memory and writes every digit's run to its final place.
// The number of keys comes from DEVICE memory: the grid is sized for the largest possible count and surplus CTAs leave at once.
// Stability: tiles are ordered by ticket = tile index, ranks inside a tile follow the input order (warp, round, lane).
// ---------------------------------------------------------------------------------------------------
static constexpr int OS_THREADS = 256;			// thread t owns digits t, t + 256 in the per-digit steps
static constexpr int OS_WARPS = OS_THREADS / 32;
static constexpr int OS_KPT = SORT_TILE / OS_THREADS;	// 16 keys per thread
static constexpr uint32_t OS_FLAG_AGG = 1u << 30, OS_FLAG_PREFIX = 2u << 30, OS_COUNT_MASK = (1u << 30) - 1u;

__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long *p)
{
	unsigned long long v;
	asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
	return v;
}
__device__ __forceinline__ void st_volatile_u64(unsigned long long *p, unsigned long long v)
{
	asm volatile("st.volatile.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// lane-privatised histogram copies (lane & (copies - 1)), skewed by one bank each: 8 copies of 257 words per pass for 8-bit
// digits, 4 copies of 513 words when a pass has 9 bits
template <int copies, int stride>
__global__ void __launch_bounds__(512) os_hist_kernel(const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ d_n, SortPlan P,
		uint32_t *__restrict__ ghist /* [np][RADIX_MAX] */)
{
	extern __shared__ __align__(16) unsigned char osh_smem[];
	uint32_t *h = reinterpret_cast<uint32_t *>(osh_smem);		// [np][copies][stride]
	const int copy = threadIdx.x & (copies - 1);
	constexpr int pstride = copies * stride;
	const uint64_t n = *d_n;

	for (int i = threadIdx.x; i < P.np * pstride; i += blockDim.x) h[i] = 0;
	__syncthreads();

	const uint64_t gstride = (uint64_t)gridDim.x * blockDim.x * 2;
	for (uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2; i < n; i += gstride) {
		unsigned long long k0, k1 = 0;
		const bool two = i + 1 < n;
		if (two) { const ulonglong2 v = __ldcs(reinterpret_cast<const ulonglong2 *>(keys + i)); k0 = v.x; k1 = v.y; }
		else k0 = keys[i];
#pragma unroll
		for (int p = 0; p < OS_MAX_PASSES; ++p) {
			if (p < P.np) {
				uint32_t *hp = h + p * pstride + copy * stride;
				atomicAdd(hp + sort_digit(k0, P.shift[p], P.bits[p]), 1u);
				if (two) atomicAdd(hp + sort_digit(k1, P.shift[p], P.bits[p]), 1u);
			}
		}
	}
	__syncthreads();
	for (int j = threadIdx.x; j < P.np * RADIX_MAX; j += blockDim.x) {
		const int p = j >> RADIX_MAX_BITS, d = j & (RADIX_MAX - 1);
		if (d >= stride - 1) continue;
		uint32_t s = 0;
		for (int c = 0; c < copies; ++c) s += h[p * pstride + c * stride + d];
		if (s) atomicAdd(&ghist[j], s);
	}
}

// exclusive scan over the 256 threads of the CTA of a packed pair {hi: < 2^32, lo: < 2^16 summed}; smem >= 8 u64.
// *total = sum over all threads (same value in every thread)
__device__ __forceinline__ unsigned long long os_block_exclusive_scan(unsigned long long v, unsigned long long *smem, unsigned long long *total)
{
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	unsigned long long incl = v;

#pragma unroll
	for (int off = 1; off < 32; off <<= 1) {
		const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, off);
		if (lane >= off) incl += t;
	}
	if (lane == 31) smem[wid] = incl;
	__syncthreads();
	unsigned long long woff = 0, tot = 0;
#pragma unroll
	for (int w = 0; w < OS_WARPS; ++w) { const unsigned long long x = smem[w]; if (w < wid) woff += x; if (total) tot += x; }
	if (total) *total = tot;
	return woff + incl - v;
}

template <int RBITS>
struct OneSweepSharedT
{
	static constexpr int RADIX = 1 << RBITS;
	unsigned long long	keys[SORT_TILE];		// tile reordered by digit
	uint32_t		whist[OS_WARPS][RADIX];		// per-warp digit counts, then exclusive prefix over the warps
	uint32_t		dstart[RADIX];			// tile-local start of each digit
	uint32_t		goff[RADIX];			// output index of tile-local position 0 of each digit's run (mod 2^32)
	unsigned long long	scan[2][OS_WARPS];
	float			fscan[OS_WARPS];
	uint32_t		tile;
};

template <int RBITS>
__global__ void __launch_bounds__(OS_THREADS, 4) os_pass_kernel(const unsigned long long *__restrict__ in, unsigned long long *__restrict__ out,
		const unsigned long long *__restrict__ d_n, int shift, int bits /* <= RBITS */, const uint32_t *__restrict__ ghist /* [RADIX] of this pass */,
		unsigned long long *__restrict__ status /* [ntiles][RADIX] */, uint32_t *__restrict__ ticket, uint32_t epoch)
{
	constexpr int RADIX = 1 << RBITS;
	constexpr int DPT = RADIX >= OS_THREADS ? RADIX / OS_THREADS : 1;	// digits per thread in the per-digit steps (threads >= RADIX idle there)
	extern __shared__ __align__(16) unsigned char os_smem[];
	OneSweepSharedT<RBITS> &S = *reinterpret_cast<OneSweepSharedT<RBITS> *>(os_smem);
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t lt_mask = (1u << lane) - 1u;
	const uint32_t n = (uint32_t)*d_n;
	const unsigned long long etag = (unsigned long long)epoch << 32;
	const int width = RBITS > 6 ? RBITS : bits;		// a digit of 7 to 9 bits has its own instantiation, narrower ones share the 6-bit one

	// persistent CTAs: the grid fills the machine once and every CTA keeps taking tile tickets until the keys are used up. The host
	// sizes nothing by the key count (it never reads it back): with most samples on the hot rows a batch may leave a fraction of
	// the tiles its event count would allow, and a CTA per POSSIBLE tile would spend more time starting and leaving than sorting.
	for (;;) {
	if (threadIdx.x == 0) S.tile = atomicAdd(ticket, 1u);
	for (int i = threadIdx.x; i < OS_WARPS * RADIX; i += OS_THREADS) (&S.whist[0][0])[i] = 0;
	__syncthreads();
	const uint32_t tile = S.tile;
	if ((uint64_t)tile * SORT_TILE >= n) return;		// no tile left
	const uint32_t wbase = tile * (uint32_t)SORT_TILE + (uint32_t)wid * (OS_KPT * 32);

	unsigned long long k[OS_KPT];
	uint32_t rk[OS_KPT / 2];			// two 16-bit ranks per word
#pragma unroll
	for (int r = 0; r < OS_KPT; ++r) {
		const uint32_t i = wbase + (uint32_t)r * 32 + lane;
		k[r] = i < n ? __ldcs(in + i) : 0ull;
	}

	// Lanes holding the same digit form a group. match.any finds the groups in one instruction, but the hardware walks the
	// distinct values of the warp one by one (the address-divergence unit stays busy on a pass whose digits are uniform); one ballot per
	// digit bit costs the same whatever the data. The CTA picks per pass: expected number of distinct digits among 32 keys,
	// from the global histogram of the pass.
	bool use_ballot;
	{
		float distinct = 0.f;
#pragma unroll
		for (int j = 0; j < DPT; ++j) {
			if (threadIdx.x + j * OS_THREADS >= RADIX) continue;
			const float pd = (float)ghist[threadIdx.x + j * OS_THREADS] / (float)n;
			float q = 1.f - pd; q *= q; q *= q; q *= q; q *= q; q *= q;		// (1 - p)^32
			distinct += 1.f - q;
		}
#pragma unroll
		for (int off = 16; off > 0; off >>= 1) distinct += __shfl_xor_sync(0xffffffffu, distinct, off);
		if (lane == 0) S.fscan[wid] = distinct;
		__syncthreads();
		float tot = 0.f;
#pragma unroll
		for (int w = 0; w < OS_WARPS; ++w) tot += S.fscan[w];
		// every thread has the same tot; taking lane 0's choice costs one shuffle and cuts the kernel's local-memory spills by a
		// third (ptxas -v)
		use_ballot = __shfl_sync(0xffffffffu, (int)(tot > 10.f), 0);
	}
	const bool partial = (tile + 1) * (uint32_t)SORT_TILE > n;

	// rank of every key among the keys of its digit inside this warp's chunk (rounds in order, lanes in order); the group
	// leader bumps the warp's digit counter and hands the previous value to its group
	uint32_t dg[OS_KPT / 2];			// two 16-bit digits per word
#pragma unroll
	for (int r = 0; r < OS_KPT; ++r) {
		const bool valid = wbase + (uint32_t)r * 32 + lane < n;
		const uint32_t d = valid ? sort_digit(k[r], shift, width) : ((uint32_t)RADIX + lane);
		if (r & 1) dg[r >> 1] |= d << 16; else dg[r >> 1] = d;
		uint32_t m;
		if (use_ballot) {
			m = 0xffffffffu;
#pragma unroll
			for (int b = 0; b < RBITS; ++b) {
				const bool bit = (d >> b) & 1u;
				const uint32_t bal = __ballot_sync(0xffffffffu, bit);
				m &= bit ? bal : ~bal;
			}
			if (partial) m &= __ballot_sync(0xffffffffu, valid);
		}
		else m = __match_any_sync(0xffffffffu, d);
		const int leader = __ffs(m) - 1;
		uint32_t old = 0;
		if (valid && lane == leader) { old = S.whist[wid][d]; S.whist[wid][d] = old + __popc(m); }
		__syncwarp();
		old = __shfl_sync(0xffffffffu, old, leader & 31);
		const uint32_t rank = old + __popc(m & lt_mask);
		if (r & 1) rk[r >> 1] |= rank << 16; else rk[r >> 1] = rank;
	}
	__syncthreads();

	// thread t owns digits t (+ 256): prefix over the warps, the tile's count of the digit -> published at once, so successors
	// can look back through it; then the scans over the digits, with a carry between the two halves of a 9-bit pass
	uint32_t dtotal[DPT];
#pragma unroll
	for (int j = 0; j < DPT; ++j) {
		const uint32_t d = threadIdx.x + j * OS_THREADS;
		uint32_t run = 0;
		dtotal[j] = 0;
		if (d >= RADIX) continue;
#pragma unroll
		for (int w = 0; w < OS_WARPS; ++w) { const uint32_t t = S.whist[w][d]; S.whist[w][d] = run; run += t; }
		dtotal[j] = run;
		st_volatile_u64(status + (size_t)tile * RADIX + d, etag | (tile == 0 ? OS_FLAG_PREFIX : OS_FLAG_AGG) | run);
	}
	unsigned long long carry = 0;
#pragma unroll
	for (int j = 0; j < DPT; ++j) {
		const uint32_t d = threadIdx.x + j * OS_THREADS;
		unsigned long long tot = 0;
		// {global count of digit d, tile count of digit d} -> exclusive scans over the digits in one go
		const bool own = d < RADIX;
		const unsigned long long sc = carry + os_block_exclusive_scan(own ? (((unsigned long long)ghist[d] << 16) | dtotal[j]) : 0ull, S.scan[j], DPT > 1 ? &tot : nullptr);
		carry += tot;
		if (!own) continue;
		const uint32_t gexcl = (uint32_t)(sc >> 16), dstart = (uint32_t)(sc & 0xFFFFu);
		// decoupled look-back: keys with digit d in the tiles before this one
		uint32_t excl = 0;
		if (tile > 0) {
			uint32_t p = tile - 1;
			for (;;) {
				const unsigned long long v = ld_volatile_u64(status + (size_t)p * RADIX + d);
				if ((v >> 32) != epoch || !((uint32_t)v >> 30)) continue;	// predecessor has its ticket, so it is running: its count will come
				excl += (uint32_t)v & OS_COUNT_MASK;
				if ((uint32_t)v & OS_FLAG_PREFIX) break;
				--p;
			}
			st_volatile_u64(status + (size_t)tile * RADIX + d, etag | OS_FLAG_PREFIX | (excl + dtotal[j]));
		}
		S.dstart[d] = dstart;
		S.goff[d] = gexcl + excl - dstart;
	}
	__syncthreads();

	// reorder the tile by digit in shared memory
#pragma unroll
	for (int r = 0; r < OS_KPT; ++r) {
		if (wbase + (uint32_t)r * 32 + lane < n) {
			const uint32_t dd = (r & 1) ? (dg[r >> 1] >> 16) : (dg[r >> 1] & 0xFFFFu);
			const uint32_t rank = (r & 1) ? (rk[r >> 1] >> 16) : (rk[r >> 1] & 0xFFFFu);
			S.keys[S.dstart[dd] + S.whist[wid][dd] + rank] = k[r];
		}
	}
	__syncthreads();

	// consecutive threads write consecutive keys: every digit's run leaves as full sectors
	const uint32_t tbase = tile * (uint32_t)SORT_TILE;
	const uint32_t nvalid = n - tbase < (uint32_t)SORT_TILE ? n - tbase : (uint32_t)SORT_TILE;
#pragma unroll 4
	for (uint32_t i = threadIdx.x; i < nvalid; i += OS_THREADS) {
		const unsigned long long key = S.keys[i];
		out[S.goff[sort_digit(key, shift, width)] + i] = key;
	}
	__syncthreads();		// the tile's shared state is free for the next ticket
	}
}

// ---------------------------------------------------------------------------------------------------
// per batch: sorted RESP keys -> one key segment per service -> histogram cells + t-digest
// ---------------------------------------------------------------------------------------------------
// (1) segs_mark_kernel   one sweep over the sorted keys: where does each service's segment start and end (the slot bits differ from
//     a neighbour's). A segment of at most LONG_SEG keys joins the list of touched services (one cursor bump per warp); a longer one
//     is handed the next batch row and joins the list of long segments.
// (2) long_sum_kernel    the keys of the long segments -> their batch rows: every 128-key chunk holding keys of a long segment adds
//     {samples | sub-msec remainders, usec sum} per bin with REDs into the row. A batch without a long segment leaves at once.
// (3) bins_merge_kernel  one warp per work item — a hot row, a long segment's batch row, or a short segment read straight from the
//     sorted keys: bins -> items {mean, weight} + GY_HISTOGRAM::add_data for every sample of the bin (count and exact msec sum per
//     bucket), then the merging t-digest step.
// Every number a bin gets is an integer sum over its samples, whichever of the three ways its service takes.
struct alignas(16) BatchSeg { uint32_t key0, row1, end, pad; };	// a touched service's keys [key0, end) in the sorted array; row1 = 1 + its
									// batch row (long segment), 0 (short)

static constexpr int SG_THREADS = 256;
static constexpr int SG_V = 8;	// keys per thread: positions wbase + t * 32 + lane; a CTA of SG_THREADS threads covers SG_THREADS * SG_V keys

__global__ void __launch_bounds__(SG_THREADS) segs_mark_kernel(const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ d_n,
		BatchSeg *__restrict__ segs /* [slot] */, uint32_t *__restrict__ touched, unsigned long long *ntouched, uint32_t *__restrict__ long_slot,
		unsigned long long *nlong)
{
	const uint64_t n = *d_n;
	const int lane = threadIdx.x & 31;
	const uint64_t wbase = ((uint64_t)blockIdx.x * SG_THREADS + threadIdx.x - lane) * SG_V;	// 32 * SG_V consecutive keys per warp
	if (wbase >= n) return;

	uint32_t s[SG_V + 2];		// slot of key wbase - 1 (lane 0 only), own keys, successor of the last (lane 31 only); ~0u: none
#pragma unroll
	for (int t = 0; t < SG_V; ++t) {
		const uint64_t i = wbase + (uint64_t)t * 32 + lane;
		s[1 + t] = i < n ? key_slot(keys[i]) : ~0u;
	}
	s[0] = (lane == 0 && wbase) ? key_slot(keys[wbase - 1]) : ~0u;
	s[SG_V + 1] = (lane == 31 && wbase + 32 * SG_V < n) ? key_slot(keys[wbase + 32 * SG_V]) : ~0u;

	uint32_t isstart = 0, isend = 0;	// bit t: own key t starts / ends a service segment
#pragma unroll
	for (int t = 0; t < SG_V; ++t) {
		const uint64_t i = wbase + (uint64_t)t * 32 + lane;
		uint32_t prev = __shfl_up_sync(0xffffffffu, s[1 + t], 1);
		const uint32_t prev0 = __shfl_sync(0xffffffffu, s[t], 31);		// key t - 1 of lane 31 (t >= 1)
		if (lane == 0) prev = t == 0 ? s[0] : prev0;
		uint32_t next = __shfl_down_sync(0xffffffffu, s[1 + t], 1);
		const uint32_t next0 = __shfl_sync(0xffffffffu, s[2 + (t < SG_V - 1 ? t : 0)], 0);	// key t + 1 of lane 0
		if (lane == 31) next = t == SG_V - 1 ? s[SG_V + 1] : next0;
		const bool valid = i < n;
		isstart |= (valid && s[1 + t] != prev ? 1u : 0u) << t;		// i == 0: prev is the sentinel
		isend |= (valid && s[1 + t] != next ? 1u : 0u) << t;		// last key: next is the sentinel
	}
	// a segment is long (more than LONG_SEG keys) when the key LONG_SEG places after its start still belongs to it: the keys are sorted
	uint32_t islong = 0;
#pragma unroll
	for (int t = 0; t < SG_V; ++t) {
		const uint64_t i = wbase + (uint64_t)t * 32 + lane;
		if (((isstart >> t) & 1u) && i + LONG_SEG < n && key_slot(keys[i + LONG_SEG]) == s[1 + t]) islong |= 1u << t;
	}

	// one cursor bump per warp for all the short segments that start in it
	const uint32_t nstart = __popc(isstart & ~islong);
	uint32_t incl = nstart;
#pragma unroll
	for (int off = 1; off < 32; off <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += v; }
	const uint32_t wtotal = __shfl_sync(0xffffffffu, incl, 31);
	unsigned long long tb = 0;
	if (wtotal && lane == 0) tb = atomicAdd(ntouched, (unsigned long long)wtotal);
	tb = __shfl_sync(0xffffffffu, tb, 0) + (incl - nstart);
	// the next batch rows for the long ones (rare: one bump per lane that has any). A batch has at most max_batch / (LONG_SEG + 1)
	// long segments: the rows never run out (engine allocation).
	uint32_t rb = 0;
	if (islong) rb = (uint32_t)atomicAdd(nlong, (unsigned long long)__popc(islong));

#pragma unroll
	for (int t = 0; t < SG_V; ++t) {
		const uint64_t i = wbase + (uint64_t)t * 32 + lane;
		const uint32_t slot = s[1 + t];
		if ((isstart >> t) & 1u) {
			uint32_t row1 = 0;
			if ((islong >> t) & 1u) { long_slot[rb] = slot; row1 = ++rb; }
			else touched[tb++] = slot;
			*reinterpret_cast<uint2 *>(&segs[slot].key0) = make_uint2((uint32_t)i, row1);
		}
		if ((isend >> t) & 1u) segs[slot].end = (uint32_t)(i + 1);
	}
}

static constexpr int LS_V = 4;			// consecutive sorted keys per lane: a warp reads one 128-key chunk

// one 128-key chunk's keys of long segments into their batch rows: keys of slot sf go to row rf - 1, of slot sl to row rl - 1 (0:
// a short segment's, skipped); a slot in between has fewer than 128 keys, all of them in this chunk — a short segment
__device__ __forceinline__ void long_sum_chunk(const unsigned long long *__restrict__ keys, uint64_t n, uint64_t base, uint32_t sf, uint32_t rf,
		uint32_t sl, uint32_t rl, unsigned long long *__restrict__ rows)
{
	const int lane = threadIdx.x & 31;
	const uint64_t i0 = base + (uint64_t)lane * LS_V;
	unsigned long long kk[LS_V];
	if (i0 + LS_V <= n) {
		const ulonglong2 a = *reinterpret_cast<const ulonglong2 *>(keys + i0), c = *reinterpret_cast<const ulonglong2 *>(keys + i0 + 2);
		kk[0] = a.x; kk[1] = a.y; kk[2] = c.x; kk[3] = c.y;
	}
	else {
#pragma unroll
		for (int t = 0; t < LS_V; ++t) kk[t] = i0 + t < n ? keys[i0 + t] : ~0ull;
	}
	// where a key's sample goes: {batch row : 22 | bin : 10}, ~0u: nowhere (no key, or a short segment's)
	auto dest = [&](unsigned long long k) -> uint32_t {
		if (k == ~0ull) return ~0u;
		const uint32_t s = key_slot(k), r1 = s == sf ? rf : (s == sl ? rl : 0u);
		return r1 ? ((r1 - 1u) << TD_CODE_BITS) | key_bin(k) : ~0u;
	};
	auto red_bin = [&](uint32_t d, unsigned long long cw, unsigned long long us) {
		unsigned long long *row = rows + (size_t)(d >> TD_CODE_BITS) * HOT_ROW_WORDS;
		const uint32_t w = hot_word(d & ((1u << TD_CODE_BITS) - 1u));
		red_add_u64(row + w, cw);
		red_add_u64(row + w + HOT_ROW_BINS, us);
	};

	// whole chunk inside one bin of a long segment (a popular bin of a big service): one RED pair for 128 samples. The keys are sorted
	// by slot only, so every key is checked against the chunk's first one
	const uint32_t dfirst = __shfl_sync(0xffffffffu, dest(kk[0]), 0);
	bool same = dfirst != ~0u;
#pragma unroll
	for (int t = 0; t < LS_V; ++t) same = same && dest(kk[t]) == dfirst;
	if (__all_sync(0xffffffffu, same)) {
		unsigned long long us = 0;
		uint32_t rem = 0;
#pragma unroll
		for (int t = 0; t < LS_V; ++t) { const uint32_t v = key_usec(kk[t]); us += v; rem += v - (v / 1000u) * 1000u; }
		const unsigned long long gsum = (unsigned long long)__reduce_add_sync(0xffffffffu, (uint32_t)us & 0xFFFFFu) +
				((unsigned long long)__reduce_add_sync(0xffffffffu, (uint32_t)(us >> 20)) << 20);	// us < 2^32: 20 + 12 bits, x 32 lanes fits
		rem = __reduce_add_sync(0xffffffffu, rem);
		if (lane == 0) red_bin(dfirst, (unsigned long long)(32 * LS_V) | ((unsigned long long)rem << BIN_CNT_BITS), gsum);
		return;
	}

	// own samples -> lane-local runs of one destination; sample t carries the totals of its run so far, only the last one is emitted
	uint32_t pd[LS_V], pc[LS_V], prem[LS_V];
	unsigned long long ps[LS_V];
	bool tail[LS_V];
#pragma unroll
	for (int t = 0; t < LS_V; ++t) {
		const uint32_t d = dest(kk[t]);
		const bool valid = d != ~0u;
		tail[t] = valid;
		const uint32_t v = key_usec(kk[t]);
		pd[t] = valid ? d : (0x80000000u | (uint32_t)lane); pc[t] = valid ? 1u : 0u; ps[t] = valid ? v : 0u; prem[t] = valid ? v - (v / 1000u) * 1000u : 0u;
		if (t > 0 && valid && pd[t] == pd[t - 1]) { pc[t] += pc[t - 1]; ps[t] += ps[t - 1]; prem[t] += prem[t - 1]; tail[t - 1] = false; }
	}
	// lanes ending a run of the same destination add up across the warp; the lowest of them issues the RED pair
#pragma unroll
	for (int t = 0; t < LS_V; ++t) {
		const bool act = tail[t];
		if (!__any_sync(0xffffffffu, act)) continue;
		const uint32_t did = act ? pd[t] : (0x80000000u | (uint32_t)lane);
		const unsigned long long v = act ? ps[t] : 0ull;
		uint32_t cnt = act ? pc[t] : 0u, rem = act ? prem[t] : 0u;
		const uint32_t m = __match_any_sync(0xffffffffu, did);
		unsigned long long gsum = v;
		const uint32_t maxcnt = __reduce_max_sync(0xffffffffu, (uint32_t)__popc(m));
		uint32_t rest = m & ~(1u << lane);
		const uint32_t cnt0 = cnt, rem0 = rem;
		for (uint32_t u = 1; u < maxcnt; ++u) {
			const int src = rest ? (__ffs(rest) - 1) : lane;
			const unsigned long long ov = __shfl_sync(0xffffffffu, v, src);
			const uint32_t oc = __shfl_sync(0xffffffffu, cnt0, src), orr = __shfl_sync(0xffffffffu, rem0, src);
			if (rest) { gsum += ov; cnt += oc; rem += orr; rest &= rest - 1; }
		}
		if (act && (m & ((1u << lane) - 1u)) == 0) red_bin(did, (unsigned long long)cnt | ((unsigned long long)rem << BIN_CNT_BITS), gsum);
	}
}

__global__ void __launch_bounds__(256) long_sum_kernel(const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ d_n,
		const BatchSeg *__restrict__ segs, const unsigned long long *__restrict__ nlong, unsigned long long *__restrict__ rows)
{
	if (*nlong == 0) return;		// no service brought more than LONG_SEG keys
	const uint64_t n = *d_n;
	const uint64_t nchunks = (n + 127) >> 7;
	const int lane = threadIdx.x & 31;
	const uint64_t gw = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
	// lane l looks at chunk c0 + l: it has work only if its first or its last key belongs to a long segment
	for (uint64_t c0 = gw * 32; c0 < nchunks; c0 += nwarps * 32) {
		const uint64_t c = c0 + lane;
		uint32_t sf = 0, sl = 0, rf = 0, rl = 0;
		if (c < nchunks) {
			const uint64_t f = c << 7, l = f + 127 < n ? f + 127 : n - 1;
			sf = key_slot(keys[f]); sl = key_slot(keys[l]);
			rf = segs[sf].row1; rl = segs[sl].row1;
		}
		for (uint32_t todo = __ballot_sync(0xffffffffu, (rf | rl) != 0); todo; todo &= todo - 1) {
			const int src = __ffs(todo) - 1;
			long_sum_chunk(keys, n, (c0 + (uint64_t)src) << 7, __shfl_sync(0xffffffffu, sf, src), __shfl_sync(0xffffffffu, rf, src),
					__shfl_sync(0xffffffffu, sl, src), __shfl_sync(0xffffffffu, rl, src), rows);
		}
	}
}

// The counters of the trace rows that their keys carry: requests, usec sum and maximum, the eight response buckets and the digest's
// extremes. Trace keys have the highest slot numbers (pseudo-slots base + row), so they form the tail of the sorted array; each warp
// takes an even share of the tail in rounds of 32 consecutive keys, sums each round per row with warp reductions and adds a row's sums to
// it when the next row comes along (one RED per counter and row, not per key). A batch without trace keys leaves after the search.
struct TraceKeyAcc
{
	int row;
	unsigned long long nreq, sum, bkt[8];
	uint32_t maxv, nmin;

	__device__ __forceinline__ void clear() { row = -1; nreq = sum = 0; maxv = nmin = 0;
#pragma unroll
		for (int b = 0; b < 8; ++b) bkt[b] = 0;
	}
	__device__ __forceinline__ void flush(const TraceTable &tr, int lane)
	{
		if (row >= 0 && lane == 0) {
			unsigned long long *w = tr.words(tr.par, (uint32_t)row);
			red_add_u64(w + TW_NREQ, nreq);
			red_add_u64(w + TW_SUM_US, sum);
			red_max_u64(w + TW_MAX_US, maxv);
#pragma unroll
			for (int b = 0; b < 8; ++b) if (bkt[b]) red_add_u64(w + TW_BKT + b, bkt[b]);
			red_max_u64(w + TW_TD_NMIN, nmin);
			red_max_u64(w + TW_TD_MAX, maxv);
		}
		clear();
	}
};

__global__ void __launch_bounds__(256) trace_keys_kernel(TraceTable tr, const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ d_n)
{
	const uint64_t n = *d_n;
	uint64_t lo = 0, hi = n;		// the first trace key
	while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if (key_slot(keys[mid]) < tr.base) lo = mid + 1; else hi = mid; }
	if (lo == n) return;
	const int lane = threadIdx.x & 31;
	const uint64_t gw = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
	const uint64_t rounds = (n - lo + 31) >> 5, per = (rounds + nwarps - 1) / nwarps;
	const uint64_t q1 = min(rounds, (gw + 1) * per);
	TraceKeyAcc a;
	a.clear();
	for (uint64_t q = gw * per; q < q1; ++q) {
		const uint64_t i = lo + (q << 5) + lane;
		int row = -1;
		uint32_t v = 0;
		if (i < n) { const unsigned long long k = keys[i]; row = (int)(key_slot(k) - tr.base); v = key_usec(k); }
		const uint32_t b = trace_bucket(v);
		for (uint32_t todo = __ballot_sync(0xffffffffu, row >= 0); todo; ) {
			const int r = __shfl_sync(0xffffffffu, row, __ffs(todo) - 1);
			const bool in = row == r;
			const uint32_t m = __ballot_sync(0xffffffffu, in);
			todo &= ~m;
			// per-bucket counts of the round (<= 32 each) packed 8 bits apiece; v < 2^30: 16-bit halves sum without overflow
			const uint32_t pk0 = __reduce_add_sync(0xffffffffu, in && b < 4u ? 1u << (8u * b) : 0u);
			const uint32_t pk1 = __reduce_add_sync(0xffffffffu, in && b >= 4u ? 1u << (8u * (b - 4u)) : 0u);
			const unsigned long long sm = __reduce_add_sync(0xffffffffu, in ? v & 0xFFFFu : 0u) +
					((unsigned long long)__reduce_add_sync(0xffffffffu, in ? v >> 16 : 0u) << 16);
			const uint32_t mx = __reduce_max_sync(0xffffffffu, in ? v : 0u), nmn = __reduce_max_sync(0xffffffffu, in ? ~v : 0u);
			if (r != a.row) { a.flush(tr, lane); a.row = r; }
			a.nreq += __popc(m); a.sum += sm; a.maxv = max(a.maxv, mx); a.nmin = max(a.nmin, nmn);
#pragma unroll
			for (int j = 0; j < 4; ++j) { a.bkt[j] += (pk0 >> (8 * j)) & 0xFFu; a.bkt[4 + j] += (pk1 >> (8 * j)) & 0xFFu; }
		}
	}
	a.flush(tr, lane);
}

static constexpr int TD_WARPS = 3;		// warps (= services in flight) per CTA
// longest merged list (old centroids + batch items) that works in shared memory, 14.6 KB per warp: 5 CTAs x 3 warps fill the SM's
// 228 KB. A list that does not fit is merged in the L2 scratch at several times the cost of one that does, so a larger area that
// fits more lists beats more services in flight (measured on the bench workload, DESIGN.md §7: 384 entries at 7 CTAs 1.48 ms,
// 440 at 6 CTAs 1.36 ms, 540 at 5 CTAs 1.25 ms; 540 is the most a CTA's 48 KB of static shared memory holds)
static constexpr int TD_SMEM_N = 540;

// One warp per touched service. Its non-empty bins become the batch's items {mean = exact usec sum / samples, weight = samples} — in
// value order, because the bin index is monotone — and every bin adds {samples, exact msec sum} to its bucket of the window
// histogram: GY_HISTOGRAM::add_data for each of its samples (common/gy_statistics.h:596-623); max_val_seen_ and the digest's ends
// come from the batch's exact extremes. The items are then merged with the old centroids (old first on equal means) and the greedy
// K_1 pass cuts the list to at most TD_CAP clusters (warp_merge_compress). Lists of up to TD_SMEM_N entries work in shared memory;
// longer ones (a first batch can fill several hundred bins) in the warp's L2-resident scratch — same code, same result.
// Work items, in this order: the hot rows, the batch rows of the long segments (both: dense bins, read in bin order and zeroed),
// then the short segments, whose keys the warp reads itself.
template <bool TRACE>
__global__ void __launch_bounds__(TD_WARPS * 32, TD_MERGE_CTAS_PER_SM) bins_merge_kernel(DevState st, const unsigned long long *__restrict__ keys,
		const uint32_t *__restrict__ touched, const unsigned long long *__restrict__ ntouched_p, const uint32_t *__restrict__ long_slot,
		const unsigned long long *__restrict__ nlong_p, unsigned long long *__restrict__ batch_rows, const BatchSeg *__restrict__ segs,
		Centroid *__restrict__ items_scratch /* [nwarps][NBINS] */, TdWorkBig *__restrict__ big_scratch /* [nwarps] */)
{
	__shared__ TdWorkT<TD_SMEM_N> work[TD_WARPS];
	// window histogram of the service's batch: 32-bit shared-memory atomics (native; a 64-bit shared atomicAdd is a CAS loop). A bucket's
	// sample count of one batch fits 32 bits (max_batch < 2^27); the msec sum is kept as {low word, carries + high words}
	__shared__ uint32_t hcnt[TD_WARPS][16], hsum_lo[TD_WARPS][16], hsum_hi[TD_WARPS][16];
	// histogram bucket of every bin, per group of 8 bins: {bucket of the group's first bin : 4 | offset of the next bucket's first bin in
	// the group, 8: none : 4}. Buckets 2..14 start at least 14 bins apart, so a group holds at most one start
	__shared__ uint8_t bk_tab[NBINS / 8];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t gw = blockIdx.x * TD_WARPS + wid, nwarps = gridDim.x * TD_WARPS;

	Centroid *items = items_scratch + (size_t)gw * NBINS;
	const uint32_t ntouched = (uint32_t)*ntouched_p, nlong = (uint32_t)*nlong_p;

	for (uint32_t g = threadIdx.x; g < (uint32_t)NBINS / 8; g += blockDim.x) {
		// thresholds of RESP_TIME_HASH in msec (gy_statistics.h:1677): bucket b >= 2 starts at (thr[b-2] + 1) msec, bucket 1 at 0;
		// bin index = td_code(usec) + bucket, so bucket b's bins start at td_code(first usec of the bucket) + b
		constexpr uint32_t thr[13] = {1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000};
		auto bucket = [&](uint32_t bin) {
			uint32_t bk = bin >= 1u;
			for (int q = 2; q < 15; ++q) bk += bin >= td_code((thr[q - 2] + 1u) * 1000u) + (uint32_t)q;
			return bk;
		};
		const uint32_t b0 = bucket(g * 8);
		uint32_t off = 8;
		for (uint32_t o = 7; o >= 1; --o) if (bucket(g * 8 + o) != b0) off = o;
		bk_tab[g] = (uint8_t)(b0 | (off << 4));
	}
	__syncthreads();

	// the batch's work list: first the hot services (rows in use; the heavy ones start first), then the long and the short segments
	// segs_mark_kernel found in the sorted keys. CTR_NHOT does not move while this kernel runs: rows handed out below count in
	// CTR_NHOT_NEXT.
	const uint32_t nhot = st.hot_rows ? (uint32_t)st.counters[CTR_NHOT] : 0u;
	const uint32_t nrow = nhot + nlong, total = nrow + ntouched;
	const uint32_t lt = (1u << lane) - 1u;
	auto slot_of = [&](uint32_t t) { return t < nhot ? st.hot_slot[t] : (t < nrow ? long_slot[t - nhot] : touched[t - nrow]); };
	uint32_t nslot = gw < total ? slot_of(gw) : 0u;
	// a trace row's segment (slot >= the pseudo-slot base): its digest at compression TRACE_TD_DELTA, no histogram, no hot row
	const uint32_t tbase = TRACE ? st.trace.base : 0xFFFFFFFFu;
	for (uint32_t t = gw; t < total; t += nwarps) {
		const uint32_t slot = nslot;
		const bool trace = TRACE && slot >= tbase;		// warp-uniform
		const bool has_next = t + nwarps < total;
		// the loads of item t + nwarps go out before item t is merged: its slot here; its batch extremes, digest header and centroid
		// lines (TD_CAP x 16 B = 32 lines, one per lane) as L2 prefetches as soon as the slot arrives, its segment as a value and
		// its first keys as L2 prefetches further down. The chain of the next item then starts from L2 instead of DRAM.
		nslot = has_next ? slot_of(t + nwarps) : 0u;
		const SlotBatch sb = trace ? SlotBatch {0xFFFFFFFFu, 0u, 0u, 0u} : st.slot_batch[slot];
		BatchSeg seg {0u, 0u, 0u, 0u};
		if (t >= nrow) seg = segs[slot];
		uint2 nseg = make_uint2(0u, 0u);
		if (TRACE && has_next && nslot >= tbase) {
			if (lane * 8 < TRACE_TD_CAP) prefetch_l2(st.trace.cents(st.trace.par, nslot - tbase) + lane * 8);
		}
		else if (has_next) {
			prefetch_l2(st.td_cent + (size_t)nslot * TD_CAP + lane * (TD_CAP / 32));
			if (lane == 0) prefetch_l2(st.slot_batch + nslot);
			else if (lane == 1) prefetch_l2(st.td_head + nslot);
		}
		if (has_next) {
			if (t + nwarps >= nrow) { const BatchSeg ns = segs[nslot]; nseg = make_uint2(ns.key0, ns.end); }
		}
		if (t < nhot && sb.minv == 0xFFFFFFFFu) continue;			// a hot service without a sample in this batch (warp-uniform)
		if (lane < 16) { hcnt[wid][lane] = 0; hsum_lo[wid][lane] = 0; hsum_hi[wid][lane] = 0; }
		__syncwarp();
		TdHead *const hp = trace ? st.trace.hd(st.trace.par, slot - tbase) : st.td_head + slot;
		const uint32_t na = hp->n;		// old centroids of the digest
		TdWorkT<TD_SMEM_N> &W = work[wid];
		// one non-empty bin {samples | remainders, usec sum} -> item j of the batch + GY_HISTOGRAM::add_data of its samples. The item
		// goes to items[j], or with `staged` straight to where warp_merge_compress_staged reads it: mean at W.src[na + j], weight
		// (a short segment's bin: <= LONG_SEG samples) at W.nxt[j]
		auto take_bin = [&](uint32_t j, unsigned long long cw, unsigned long long us, uint32_t bin, bool staged) {
			const unsigned long long cnt = cw & BIN_CNT_MASK, rem = cw >> BIN_CNT_BITS;
			const double mean = __ddiv_rn((double)us, (double)cnt);	// exact integer sum, one rounding
			if (staged) { W.src[na + j] = mean; W.nxt[j] = (uint16_t)cnt; }
			else { Centroid c; c.mean = mean; c.weight = cnt; items[j] = c; }
			if (trace) return;
			const uint32_t e = bk_tab[bin >> 3], bk = (e & 15u) + ((bin & 7u) >= (e >> 4) ? 1u : 0u);
			atomicAdd(&hcnt[wid][bk], (uint32_t)cnt);
			const unsigned long long ms = (us - rem) / 1000ull;		// sum of (usec / 1000) over the bin's samples
			const uint32_t mlo = (uint32_t)ms, mhi = (uint32_t)(ms >> 32);
			const uint32_t old = atomicAdd(&hsum_lo[wid][bk], mlo);
			const uint32_t up = mhi + (old + mlo < old ? 1u : 0u);		// carry out of the low word
			if (up) atomicAdd(&hsum_hi[wid][bk], up);
		};
		uint32_t nitems = 0, nsamples, binmax = 0;	// binmax: samples in the fullest bin (per lane, reduced when needed)
		bool staged = false;				// the batch items wait in the work area for warp_merge_compress_staged
		if (t >= nrow) {
			// a short segment, read straight from the sorted keys in blocks of 256: lane l holds keys [b0 + 8 l, b0 + 8 l + 8), four
			// 16-byte loads, and the next block's loads go out before this one is summed. The keys arrive in slot order only, so each
			// lane adds each of its samples to its bin's accumulator in the warp's work area with shared atomics of its own. (Joining
			// the lanes of one bin first with match.any, then one set of atomics per bin, made the kernel 1.9 to 2.7 times slower on the
			// bench workload, DESIGN.md §7.) Then the warp walks the bins in order, 32 per step, and packs every non-empty one
			// {usec sum, samples | remainders | bin} at its item index j (j <= its bin: the walk overwrites only bins it has read),
			// and every lane takes every 32nd item, as for a row.
			nsamples = seg.end - seg.key0;
			// a short segment's bin: samples <= LONG_SEG and remainders < 1000 x LONG_SEG fit below bit 54 of cw
			constexpr int RAW_BIN_SHIFT = 54;
			static_assert(BIN_CNT_BITS + 10 + 14 <= RAW_BIN_SHIFT && LONG_SEG <= (1 << 14), "cw of a short segment's bin below the bin bits");
			// every bin of the segment lies in [blo, bhi]: the bins of the service's batch extremes (ingest_kernel keeps them for every
			// sample it makes a key of), every bin for a trace row's segment. Accumulator of bin b: 4 words at acc[4 (b - blo)],
			// {sum of usec & 0x3FFFF < 2^31, sum of usec >> 18 < 2^25, samples, remainders < 2^23} — 32-bit shared atomics (native; a
			// 64-bit one is a CAS loop) that cannot overflow over LONG_SEG samples. It aliases the start of the work area, which is free
			// until the items are taken: the packed items fill [0, 16 nitems), below the staged means and weights (W.src, W.nxt). The
			// merge writes over all of it, so each short segment zeroes its bins' accumulators first.
			const uint32_t blo = trace ? 0u : resp_bin(sb.minv), nb = (trace ? (uint32_t)NBINS - 1u : resp_bin(sb.maxv)) - blo + 1u;
			static_assert(sizeof(TdWorkT<TD_SMEM_N>) >= NBINS * 16 && offsetof(TdWorkT<TD_SMEM_N>, nxt) >= TD_SMEM_N * 16 &&
					offsetof(TdWorkT<TD_SMEM_N>, src) >= TD_SMEM_N * 16, "the bin accumulators and packed items fit below the staged items");
			uint32_t *const acc = reinterpret_cast<uint32_t *>(W.mean);
			unsigned long long *const packed = reinterpret_cast<unsigned long long *>(W.mean);
			for (uint32_t i = lane; i < 2u * nb; i += 32) reinterpret_cast<uint2 *>(acc)[i] = make_uint2(0u, 0u);
			auto load8 = [&](uint32_t b0, unsigned long long (&k)[8]) {	// ~0ull: no key of the segment (never a key: bin <= 845)
				const uint32_t i0 = b0 + (uint32_t)lane * 8u;
				if (i0 >= seg.key0 && i0 + 8u <= seg.end) {
#pragma unroll
					for (int q = 0; q < 4; ++q) {
						const ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(keys + i0 + 2 * q);
						k[2 * q] = v.x; k[2 * q + 1] = v.y;
					}
				}
				else {
#pragma unroll
					for (int u = 0; u < 8; ++u) k[u] = i0 + u >= seg.key0 && i0 + u < seg.end ? keys[i0 + u] : ~0ull;
				}
			};
			const uint32_t a0 = seg.key0 & ~1u;		// even: every lane's keys start 16-byte aligned
			unsigned long long kk[8], nk[8];
			load8(a0, kk);
			__syncwarp();
			for (uint32_t b0 = a0; b0 < seg.end; b0 += 256) {
				if (b0 + 256u < seg.end) load8(b0 + 256u, nk);
				else {
#pragma unroll
					for (int u = 0; u < 8; ++u) nk[u] = ~0ull;
				}
#pragma unroll
				for (int u = 0; u < 8; ++u) {
					if (kk[u] != ~0ull) {
						const uint32_t v = key_usec(kk[u]);
						uint32_t *const a = acc + 4u * (key_bin(kk[u]) - blo);
						atomicAdd(a, v & 0x3FFFFu);
						atomicAdd(a + 1, v >> 18);
						atomicAdd(a + 2, 1u);
						atomicAdd(a + 3, v - (v / 1000u) * 1000u);
					}
				}
#pragma unroll
				for (int u = 0; u < 8; ++u) kk[u] = nk[u];
			}
			__syncwarp();
			for (uint32_t b0 = 0; b0 < nb; b0 += 32) {
				const uint32_t i = b0 + lane;
				uint2 us2 = make_uint2(0u, 0u), cr = make_uint2(0u, 0u);
				if (i < nb) { us2 = reinterpret_cast<const uint2 *>(acc)[2u * i]; cr = reinterpret_cast<const uint2 *>(acc)[2u * i + 1u]; }
				const bool ne = cr.x != 0u;
				const uint32_t m = __ballot_sync(0xffffffffu, ne);
				if (ne) {
					const uint32_t j = nitems + __popc(m & lt);
					packed[2u * j] = (unsigned long long)us2.x + ((unsigned long long)us2.y << 18);
					packed[2u * j + 1u] = (unsigned long long)cr.x | ((unsigned long long)cr.y << BIN_CNT_BITS) |
							((unsigned long long)(blo + i) << RAW_BIN_SHIFT);
					binmax = max(binmax, cr.x);
				}
				nitems += __popc(m);
				__syncwarp();
			}
			staged = na + nitems <= (uint32_t)TD_SMEM_N;
			for (uint32_t j = lane; j < nitems; j += 32) {
				const unsigned long long us = packed[2u * j], cw = packed[2u * j + 1u];
				take_bin(j, cw & ((1ull << RAW_BIN_SHIFT) - 1u), us, (uint32_t)(cw >> RAW_BIN_SHIFT), staged);
			}
		}
		else {
			// the service's dense row — its hot row, or the batch row of its long segment — in bin order (= value order); the row is
			// left zeroed for the next batch
			unsigned long long *row = t < nhot ? st.hot_rows + (size_t)t * HOT_ROW_WORDS : batch_rows + (size_t)(t - nhot) * HOT_ROW_WORDS;
			uint32_t mine = 0;
			for (uint32_t b0 = 0; b0 < (uint32_t)NBINS; b0 += 32) {
				const uint32_t bin = b0 + lane;
				const uint32_t i0 = hot_word(bin), i1 = i0 + (uint32_t)HOT_ROW_BINS;
				ulonglong2 v = make_ulonglong2(0ull, 0ull);
				if (bin < (uint32_t)NBINS) { v.x = __ldcg(row + i0); v.y = __ldcg(row + i1); }
				const bool ne = (v.x & BIN_CNT_MASK) != 0;
				const uint32_t m = __ballot_sync(0xffffffffu, ne);
				if (ne) {
					take_bin(nitems + __popc(m & lt), v.x, v.y, bin, false);
					row[i0] = 0ull; row[i1] = 0ull;
					mine += (uint32_t)(v.x & BIN_CNT_MASK);
					binmax = max(binmax, (uint32_t)(v.x & BIN_CNT_MASK));
				}
				nitems += __popc(m);
			}
			nsamples = __reduce_add_sync(0xffffffffu, mine);
		}
		if (has_next && t + nwarps >= nrow) {		// the next item is a short segment: its first 32 lines of keys (16 keys per line)
			const uint32_t l0 = nseg.x >> 4, l1 = (nseg.y - 1u) >> 4;
			if (l0 + lane <= l1) prefetch_l2(keys + (size_t)(l0 + lane) * 16);
		}
		binmax = __reduce_max_sync(0xffffffffu, binmax);
		__syncwarp();
		// nobody else touches this slot's window histogram while the batch is merged (same stream as the flush): plain updates
		if (trace) {}
		else if (lane < HIST_MAX_CELL) {
			if (hcnt[wid][lane]) {
				HistCell *c = st.hist_cur + (size_t)slot * HIST_CELLS + lane;
				c->count += hcnt[wid][lane]; c->sum += (long long)(((unsigned long long)hsum_hi[wid][lane] << 32) | hsum_lo[wid][lane]);
			}
		}
		else if (lane == HIST_MAX_CELL) {
			HistCell *c = st.hist_cur + (size_t)slot * HIST_CELLS + HIST_MAX_CELL;
			const long long mx = (long long)(sb.maxv / 1000u);		// max_val_seen_ of add_data (gy_statistics.h:609-611)
			if (mx > c->sum) c->sum = mx;
			// a service that brought hot_min samples in one batch gets a row of dense bins for the batches to come (rows are never
			// taken back: a row belongs to the SLOT, whoever lives in it — routing only, the numbers are the same either way).
			// Not one whose fullest bin holds more than hot_bin_max samples: atomics on one 128-byte line are applied one after the
			// other (measured: ~8 ns each), a few hundred thousand of them on one line would outlast the rest of ingest_kernel —
			// such a service sorts well instead (its keys form long runs).
			uint32_t hot = sb.hot;
			if (!hot && st.hot_rows && nsamples >= st.hot_min && nsamples <= st.hot_max && binmax <= st.hot_bin_max) {
				const unsigned long long h = atomicAdd(st.counters + CTR_NHOT_NEXT, 1ull);
				if (h < (unsigned long long)st.hot_cap) { st.hot_slot[h] = slot; hot = (uint32_t)h + 1u; }
				else atomicAdd(st.counters + CTR_NHOT_NEXT, ~0ull);
			}
			st.slot_batch[slot] = SlotBatch {0xFFFFFFFFu, 0u, 0u, hot};
		}
		__syncwarp();

		TdHead head = *hp;
		Centroid *cent = trace ? st.trace.cents(st.trace.par, slot - tbase) : st.td_cent + (size_t)slot * TD_CAP;
		const TdParams P = trace ? st.trace.td : st.td;
		uint32_t nout;
		if (staged) nout = warp_merge_compress_staged(W, cent, na, nitems, cent, P);
		else if (na + nitems <= (uint32_t)TD_SMEM_N) nout = warp_merge_compress(W, cent, na, items, nitems, cent, P);
		else nout = warp_merge_compress(big_scratch[gw], cent, na, items, nitems, cent, P);
		if (lane == 0) {
			head.n = nout;
			head.total += nsamples;
			// a trace digest's extremes are counter words of its window (trace_keys_kernel)
			if (!trace && (double)sb.minv < head.minv) head.minv = (double)sb.minv;
			if (!trace && (double)sb.maxv > head.maxv) head.maxv = (double)sb.maxv;
			*hp = head;
		}
		__syncwarp();
	}
}

// ---------------------------------------------------------------------------------------------------
// 5-second window roll: last = cur; all += cur; cur = 0  (one thread per histogram cell)
// ---------------------------------------------------------------------------------------------------
//
// Idle services (SURVEY §8f-1): the reference deletes a listener that produced no statistics for TIMEOUT_INET_DIAG_SECS
// (300 s, common/gy_socket_stat.h:997) once it is older than twice that (common/gy_socket_stat.cc:3968-3982: tclock != 0,
// tclock + 300 s < now, tstart + 600 s < now) and tells madhava with LISTEN_FLAG_DELETE (:4023-4033). Here the flush records,
// per slot, the first flush that saw it and the last window that held events, and lists the slots that meet the rule.
__global__ void flush_kernel(DevState st, uint32_t nslots, uint32_t tsec, uint32_t idle_secs)
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	const bool valid = i < (uint64_t)nslots * HIST_CELLS;		// nslots * 16: whole half-warps are valid or not
	const int cell = (int)(i & (HIST_CELLS - 1));
	HistCell c {0, 0};
	unsigned long long cc = 0;
	const uint32_t slot = (uint32_t)(i >> 4);

	if (valid) {
		c = st.hist_cur[i];
		if (cell == HIST_MAX_CELL) cc = st.conn_cur[slot];
	}
	// did the closing window hold any event of this service? (16 lanes = the 15 buckets + the max / conn cell)
	bool auxact = false;				// ACTIVE_CONN_STATS records / API_TRAN errors count as activity of the window too
	if (valid && cell == HIST_MAX_CELL) { const SlotAux a0 = st.slot_aux[slot]; auxact = (a0.act_cur | a0.err_cur) != 0; }
	const uint32_t bal = __ballot_sync(0xffffffffu, valid && (cell == HIST_MAX_CELL ? (cc != 0 || auxact) : c.count != 0));
	const bool active = ((bal >> (threadIdx.x & 16)) & 0xFFFFu) != 0;
	if (!valid) return;

	st.bm_last[i] = st.bm_cur[i]; st.bm_cur[i] = 0;		// CONN_BITMAP::clear every 5 s (gy_socket_stat.h:436)
	st.hist_last[i] = c;
	// rolling levels: the window is added to the current slot of each level (cleared by the host when its epoch changed).
	// A cleared slot's max cell reads 0, which is below any recorded response time or equal to it: harmless for max().
	HistCell &r0 = st.levels.row(0, st.levels.cur[0], slot)[cell], &r1 = st.levels.row(1, st.levels.cur[1], slot)[cell];
	if (cell == HIST_MAX_CELL) {
		if (c.sum > r0.sum) r0.sum = c.sum;
		if (c.sum > r1.sum) r1.sum = c.sum;
	}
	else {
		r0.count += c.count; r0.sum += c.sum;
		r1.count += c.count; r1.sum += c.sum;
	}
	if (cell == HIST_MAX_CELL) {
		if (c.sum > st.hist_all[i].sum) st.hist_all[i].sum = c.sum;
		st.hist_cur[i].count = 0; st.hist_cur[i].sum = LLONG_MIN;
		st.conn_last[slot] = cc;
		st.conn_all_cnt[slot] += (uint32_t)cc;
		st.conn_all_kb[slot] += cc >> 32;
		st.conn_cur[slot] = 0;
		{
			SlotAux a = st.slot_aux[slot];
			a.act_last = a.act_cur; a.act_cur = 0; a.err_last = a.err_cur; a.err_cur = 0; a.rtt_last = a.rtt_cur; a.rtt_cur = 0;
			st.slot_aux[slot] = a;
		}

		const unsigned long long id = st.slot_id[slot];
		if (id) {
			uint32_t first = st.slot_first_seen[slot], last = st.slot_last_active[slot];
			if (!first) { first = tsec ? tsec : 1u; st.slot_first_seen[slot] = first; }
			if (active) { last = tsec ? tsec : 1u; st.slot_last_active[slot] = last; }
			if (idle_secs && last && (uint64_t)last + idle_secs < tsec && (uint64_t)first + 2ull * idle_secs < tsec) {
				const unsigned long long k = atomicAdd(st.counters + CTR_NEVICT, 1ull);
				st.evict_list[k] = slot;
				st.evict_ids[k] = id;
			}
		}
	}
	else {
		st.hist_all[i].count += c.count;
		st.hist_all[i].sum += c.sum;
		st.hist_cur[i].count = 0; st.hist_cur[i].sum = 0;
	}
}

// ---------------------------------------------------------------------------------------------------
// The state decision of the 5-s reducer, one thread per service slot, right behind flush_kernel: what listener_stats_update does per
// listener around get_curr_state (common/gy_socket_stat.cc:4111-4130 samples of qps_hist_ / active_conn_hist_, :4158-4173 connection
// counts, :4222-4233 level statistics + get_curr_state, :4242-4272 issue_bit_hist_). A slot whose closing window held no event is
// "stale" (:4098-4107): the reference leaves such a listener's state alone, and so does this kernel.
// ---------------------------------------------------------------------------------------------------
struct LevelStat { int64_t p95, p99, p25; uint64_t cnt, sum; double mean; };

__device__ __forceinline__ LevelStat level_stat(const uint64_t *counts, uint64_t sum)
{
	LevelStat r;
	uint64_t c = 0;
	for (int b = 0; b < HIST_MAX_CELL; ++b) c += counts[b];
	r.p95 = resp_bucket_value(hist_pct_bucket(counts, HIST_MAX_CELL, c, 95.0f), c);
	r.p99 = resp_bucket_value(hist_pct_bucket(counts, HIST_MAX_CELL, c, 99.0f), c);
	r.p25 = resp_bucket_value(hist_pct_bucket(counts, HIST_MAX_CELL, c, 25.0f), c);
	r.cnt = c; r.sum = sum;
	r.mean = (double)(long long)sum / (double)(c ? (long long)c : 1ll);		// TIME_HISTOGRAM::get_stats, gy_statistics.h:1358
	return r;
}

// p95 / p25 of qps_hist_ and active_conn_hist_ from their bucket counts (cnt is scratch). The active-connection histogram is read over
// its 14 buckets (HASH_1_3000).
struct QpsActPct { int64_t qps_p95, qps_p25, act_p95, act_p25; };
__device__ __forceinline__ QpsActPct qps_act_pct(const HistCell *q, const HistCell *a, uint64_t *cnt)
{
	QpsActPct r;
	uint64_t tot = 0;
	for (int b = 0; b < HIST_MAX_CELL; ++b) { cnt[b] = q[b].count; tot += cnt[b]; }
	r.qps_p95 = qps_bucket_value(hist_pct_bucket(cnt, HIST_MAX_CELL, tot, 95.0f), tot);
	r.qps_p25 = qps_bucket_value(hist_pct_bucket(cnt, HIST_MAX_CELL, tot, 25.0f), tot);
	tot = 0;
	for (int b = 0; b < HIST_MAX_CELL; ++b) { cnt[b] = b < 14 ? a[b].count : 0; tot += cnt[b]; }
	r.act_p95 = act_bucket_value(hist_pct_bucket(cnt, 14, tot, 95.0f), tot);
	r.act_p25 = act_bucket_value(hist_pct_bucket(cnt, 14, tot, 25.0f), tot);
	return r;
}

__global__ void __launch_bounds__(128) state_kernel(DevState st, uint32_t nslots, uint32_t tsec)
{
	const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= nslots || !st.slot_id[slot]) return;
	if (st.slot_last_active[slot] != (tsec ? tsec : 1u)) return;			// stale window: state stays

	const size_t base = (size_t)slot * HIST_CELLS;
	uint64_t cnt[HIST_MAX_CELL];
	uint64_t sum;
	gysk_listener_state_in in;
	memset(&in, 0, sizeof(in));

	sum = 0;
	for (int b = 0; b < HIST_MAX_CELL; ++b) { const HistCell c = st.hist_last[base + b]; cnt[b] = c.count; sum += (uint64_t)c.sum; }
	const LevelStat s5 = level_stat(cnt, sum);
	LevelStat lv[NLEVELS];
	for (int l = 0; l < NLEVELS; ++l) {
		for (int b = 0; b < HIST_MAX_CELL; ++b) cnt[b] = 0;
		sum = 0;
		// LevelRing::cell's sums, a ring row at a time: each thread reads its rows front to back
		st.levels.each_live(l, slot, [&](const HistCell *ring) {
			for (int b = 0; b < HIST_MAX_CELL; ++b) { const HistCell c = ring[b]; cnt[b] += c.count; sum += (uint64_t)c.sum; }
		});
		lv[l] = level_stat(cnt, sum);
	}
	sum = 0;
	for (int b = 0; b < HIST_MAX_CELL; ++b) { const HistCell c = st.hist_all[base + b]; cnt[b] = c.count; sum += (uint64_t)c.sum; }
	const LevelStat sa = level_stat(cnt, sum);

	in.r5p95 = s5.p95; in.r5p99 = s5.p99; in.nqrys_5s = s5.cnt; in.total_resp_msec = s5.sum; in.mean5 = s5.mean;
	in.r300p95 = lv[0].p95; in.r300p99 = lv[0].p99; in.mean300 = lv[0].mean;
	in.r5dp95 = lv[1].p95; in.r5dp99 = lv[1].p99; in.r5dp25 = lv[1].p25; in.tcount_5d = lv[1].cnt; in.mean5d = lv[1].mean;
	in.rallp95 = sa.p95; in.rallp99 = sa.p99; in.meanall = sa.mean;

	SlotState ss = st.slot_state[slot];
	const SlotAux aux = st.slot_aux[slot];
	in.last_qps_count = (int32_t)(s5.cnt / 5);
	if ((uint32_t)aux.act_last) ss.nconn_active = (uint32_t)aux.act_last;		// an ACTIVE_CONN_STATS report arrived in this window

	// GY_HISTOGRAM<int, ...>::add_data of the two per-window samples, then their p95 / p25
	{
		HistCell *q = st.qps_hist + base, *a = st.act_hist + base;
		const int qv = in.last_qps_count, av = (int)ss.nconn_active;
		const int qb = bucket_semi_log_lo(qv), ab = bucket_hash_1_3000(av);
		q[qb].count += 1; q[qb].sum += qv; if ((long long)qv > q[HIST_MAX_CELL].sum) q[HIST_MAX_CELL].sum = qv;
		a[ab].count += 1; a[ab].sum += av; if ((long long)av > a[HIST_MAX_CELL].sum) a[HIST_MAX_CELL].sum = av;
		const QpsActPct p = qps_act_pct(q, a, cnt);
		in.qps_p95 = p.qps_p95; in.qps_p25 = p.qps_p25; in.act_p95 = p.act_p95; in.act_p25 = p.act_p25;
	}

	in.nconn = (int32_t)ss.nconn_active;
	in.curr_active_conn = in.nconn;
	for (int b = 0; b < HIST_MAX_CELL; ++b) {
		const int c = __popc(st.bm_last[base + b]);					// CONN_BITMAP::get_conn_breakup
		in.nactive_conn_arr[b] = (uint8_t)c;
		if (in.curr_active_conn < c) in.curr_active_conn = c;
	}
	in.ser_errors = (uint32_t)(aux.err_last >> 32);
	const uint32_t first = st.slot_first_seen[slot];
	const uint32_t age = tsec > first ? tsec - first : 0u;
	in.secs_5d = age + 1u < 432000u ? age + 1u : 432000u;

	classify_listener(in, ss.high_bits, ss.state, ss.issue);
	apply_issue_history(age, in.ser_errors, ss.state, ss.issue, ss.issue_bits);
	st.slot_state[slot] = ss;
}

// The LISTENER_DAY_STATS record of a listener (get_curr_state, common/gy_socket_stat.cc:2101-2117), one warp per listed slot: lanes
// 0..15 gather one cell each of the 5-day level's live ring slots and of qps_hist_ / active_conn_hist_, lane 0 takes the percentiles
// with state_kernel's helpers. The int64 values go into the uint32 fields by plain conversion, as the reference's assignments do.
static constexpr int DAY_WARPS = 4;
__global__ void __launch_bounds__(DAY_WARPS * 32) day_stats_kernel(DevState st, const unsigned long long *__restrict__ slots, uint32_t n,
		gysk_listener_day_stats *__restrict__ out)
{
	__shared__ HistCell lvl[DAY_WARPS][HIST_CELLS], qa[DAY_WARPS][2][HIST_CELLS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t q = blockIdx.x * DAY_WARPS + wid;

	if (q >= n) return;
	const uint32_t slot = (uint32_t)slots[q];
	if (lane < HIST_CELLS) {
		if (lane < HIST_MAX_CELL) lvl[wid][lane] = st.levels.cell(1, slot, lane);		// level_stat reads cells 0..14 only
		qa[wid][0][lane] = st.qps_hist[(size_t)slot * HIST_CELLS + lane];
		qa[wid][1][lane] = st.act_hist[(size_t)slot * HIST_CELLS + lane];
	}
	__syncwarp();
	if (lane) return;
	uint64_t cnt[HIST_MAX_CELL], sum = 0;
	for (int b = 0; b < HIST_MAX_CELL; ++b) { cnt[b] = lvl[wid][b].count; sum += (uint64_t)lvl[wid][b].sum; }
	const LevelStat d = level_stat(cnt, sum);
	const QpsActPct p = qps_act_pct(qa[wid][0], qa[wid][1], cnt);
	gysk_listener_day_stats r;
	r.glob_id = st.slot_id[slot];
	r.tcount_5d = (int64_t)d.cnt; r.tsum_5d = (int64_t)d.sum;
	r.p95_5d_respms = (uint32_t)d.p95; r.p25_5d_respms = (uint32_t)d.p25;
	r.p95_qps = (uint32_t)p.qps_p95; r.p25_qps = (uint32_t)p.qps_p25;
	r.p95_nactive = (uint32_t)p.act_p95; r.p25_nactive = (uint32_t)p.act_p25;
	out[q] = r;
}

// one CTA per evicted slot (grid-stride) of the list {slots, ids} of *nev entries: the id's entry of table t becomes a tombstone, the
// slot returns to its just-created state (reset) and its number goes on t's free stack for the next unknown id. Services and processes
// alike; host_ids (optional, page-locked and mapped) receives the count and the ids.
template <typename Reset>
__global__ void __launch_bounds__(256) evict_kernel(DevState st, IdTable t, const uint32_t *__restrict__ slots, const unsigned long long *__restrict__ ids,
		const unsigned long long *nev_p, unsigned long long *total, unsigned long long *host_ids, Reset reset)
{
	const uint32_t nev = (uint32_t)*nev_p;

	if (host_ids && blockIdx.x == 0 && threadIdx.x == 0) host_ids[0] = nev;
	for (uint32_t q = blockIdx.x; q < nev; q += gridDim.x) {
		const uint32_t slot = slots[q];
		const unsigned long long id = ids[q];

		if (threadIdx.x == 0) {
			uint32_t pos = table_hash(id) & t.mask;
			for (uint32_t probe = 0; probe <= t.mask; ++probe, pos = (pos + 1) & t.mask) {
				TblEntry *e = &t.ent[pos];
				if (e->key == id) { e->key = KEY_TOMBSTONE; e->slot1 = 0; break; }
				if (e->key == 0) break;
			}
			const int32_t f = atomicAdd(t.free_n, 1);
			t.free_slots[f] = slot;
			if (total) atomicAdd(total, 1ull);
			if (host_ids) host_ids[1 + q] = id;
		}
		reset(st, slot, threadIdx.x, blockDim.x);
	}
}

// tombstones (and the dead entries of lost insert races) only go away by rebuilding: clear the table, re-insert the ids of the live
// slots (slot numbers stay). Services at gysk_flush; both tables at gysk_grow, into their new capacity.
__global__ void rebuild_table_kernel(IdTable t, uint32_t nslots)
{
	const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= nslots) return;
	const unsigned long long id = t.slot_id[slot];
	if (!id) return;
	uint32_t pos = table_hash(id) & t.mask;
	for (;;) {
		const unsigned long long k = atomicCAS(&t.ent[pos].key, 0ull, id);
		if (k == 0) { t.ent[pos].slot1 = slot + 1; return; }
		pos = (pos + 1) & t.mask;
	}
}

// ---------------------------------------------------------------------------------------------------
// read side: one warp per queried id
// ---------------------------------------------------------------------------------------------------

// row q of a warp's read: by id (ids != nullptr: lane 0 looks it up, id 0 and unknown ids give slot -1) or by slot (the window reads:
// the id from the table's slot -> id array)
struct Resolved { int slot; unsigned long long id; };
__device__ __forceinline__ Resolved resolve_warp(const IdTable &t, const unsigned long long *__restrict__ ids, const unsigned long long *__restrict__ slots,
		uint32_t q, int lane)
{
	Resolved r;
	if (ids) {
		r.id = ids[q];
		r.slot = -1;
		if (lane == 0 && r.id) r.slot = table_lookup(t, r.id, false);
		r.slot = __shfl_sync(0xffffffffu, r.slot, 0);
	}
	else { r.slot = (int)(uint32_t)slots[q]; r.id = t.slot_id[r.slot]; }
	return r;
}

// the warp's copy of one slot's state (all but id / found / slot and the HLL register histogram)
__device__ __forceinline__ void gather_slot(const DevState &st, int slot, SvcRaw &o, int lane)
{
	if (lane < HIST_CELLS) {
		o.cur[lane] = st.hist_cur[(size_t)slot * HIST_CELLS + lane];
		o.last[lane] = st.hist_last[(size_t)slot * HIST_CELLS + lane];
		o.all[lane] = st.hist_all[(size_t)slot * HIST_CELLS + lane];
		o.bm_cur[lane] = st.bm_cur[(size_t)slot * HIST_CELLS + lane]; o.bm_last[lane] = st.bm_last[(size_t)slot * HIST_CELLS + lane];
		for (int l = 0; l < NLEVELS; ++l) o.lvl[l][lane] = st.levels.cell(l, slot, lane);
	}
	if (lane == 0) {
		o.conn_cur = st.conn_cur[slot]; o.conn_last = st.conn_last[slot];
		o.conn_all_cnt = st.conn_all_cnt[slot]; o.conn_all_kb = st.conn_all_kb[slot];
		o.td = st.td_head[slot];
		o.aux = st.slot_aux[slot];
		o.sst = st.slot_state[slot];
	}
	if (lane < HIST_CELLS) { o.qps[lane] = st.qps_hist[(size_t)slot * HIST_CELLS + lane]; o.act[lane] = st.act_hist[(size_t)slot * HIST_CELLS + lane]; }
	for (int i = lane; i < TD_CAP; i += 32) o.cent[i] = st.td_cent[(size_t)slot * TD_CAP + i];
}

// the single-id exports (gysk_export_hist / _conn_bitmap / _tdigest): the raw state of the id
__global__ void __launch_bounds__(128) gather_svcs_kernel(DevState st, const unsigned long long *__restrict__ ids, uint32_t n, SvcRaw *__restrict__ out)
{
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t q = blockIdx.x * 4 + wid;

	if (q >= n) return;
	SvcRaw &o = out[q];
	const Resolved r = resolve_warp(st.svc_tbl, ids, nullptr, q, lane);
	if (lane == 0) { o.id = r.id; o.found = r.slot >= 0; o.slot = (uint32_t)r.slot; }
	if (r.slot < 0) return;
	gather_slot(st, r.slot, o, lane);
}

// ---- window reads (gysk_query_window / gysk_query_task_window) ----

// live slots below nslots (host filter, closed-window filter) -> keys {host : 32 | slot : 32} in any order, *d_n of them. A service is
// active when its last window with events is the one the last flush closed (active_mark, the rule of state_kernel); a process when
// one of its histograms took samples in that window. seen_before != ~0u keeps only services whose slot a flush before that tsec saw
// (the day-stats read).
__global__ void window_select_kernel(DevState st, uint32_t nslots, int is_task, int host_filter, uint32_t active_only, uint32_t active_mark,
		uint32_t seen_before, unsigned long long *__restrict__ keys, unsigned long long *d_n)
{
	const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
	bool take = false;
	uint32_t host = 0;
	if (slot < nslots) {
		host = is_task ? st.task_slot_host[slot] : st.slot_host[slot];
		take = (is_task ? st.task_slot_id[slot] != 0 : svc_live(st, slot)) && (host_filter < 0 || host == (uint32_t)host_filter);
		if (take && active_only) {
			if (is_task) {
				const HistCell *l = st.task_last + (size_t)slot * 3;
				take = (l[0].count | l[1].count | l[2].count) != 0;
			}
			else take = svc_evaluated(st, slot, active_mark);
		}
		if (take && seen_before != ~0u) {
			const uint32_t first = st.slot_first_seen[slot];
			take = first && first < seen_before;
		}
	}
	const unsigned mask = __ballot_sync(0xffffffffu, take);
	if (!mask) return;
	const int lane = threadIdx.x & 31;
	unsigned long long base = 0;
	if (lane == __ffs(mask) - 1) base = atomicAdd(d_n, (unsigned long long)__popc(mask));
	base = __shfl_sync(0xffffffffu, base, __ffs(mask) - 1);
	if (take) keys[base + __popc(mask & ((1u << lane) - 1u))] = ((unsigned long long)host << 32) | slot;
}

// ids of the slots of the (sorted) keys
__global__ void window_ids_kernel(DevState st, int is_task, const unsigned long long *__restrict__ keys, const unsigned long long *d_n,
		unsigned long long *__restrict__ ids)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= *d_n) return;
	const uint32_t slot = (uint32_t)keys[i];
	ids[i] = is_task ? st.task_slot_id[slot] : st.slot_id[slot];
}

// ---- per-host listener counts (gysk_query_host_listen) over the host-sorted keys of the window list ----

// first position in [lo, hi) whose key's host is > h (above = true) or >= h
__device__ __forceinline__ uint32_t host_bound(const unsigned long long *keys, uint32_t lo, uint32_t hi, uint32_t h, bool above)
{
	while (lo < hi) {
		const uint32_t mid = lo + ((hi - lo) >> 1);
		const uint32_t hm = (uint32_t)(keys[mid] >> 32);
		if (hm < h || (above && hm == h)) lo = mid + 1; else hi = mid;
	}
	return lo;
}

// Every listed service adds {issue : 32 | severe : 32} to acc[head of its host's run] (acc zeroed): issue = evaluated at the last flush
// (slot_last_active == active_mark) with issue bit 0 set there, severe = issue and state >= SEVERE (listener_stats_update's nissue /
// nsevere, common/gy_socket_stat.cc:4242-4252). Lanes of one run add once per warp.
__global__ void host_listen_count_kernel(DevState st, const unsigned long long *__restrict__ keys, const unsigned long long *d_n, uint32_t active_mark,
		unsigned long long *__restrict__ acc)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, n = (uint32_t)*d_n;
	const unsigned live = __ballot_sync(0xffffffffu, i < n);
	if (i >= n) return;
	const unsigned long long key = keys[i];
	const uint32_t slot = (uint32_t)key, head = host_bound(keys, 0, i, (uint32_t)(key >> 32), false);
	const bool issue = svc_issue(st, slot, active_mark), severe = issue && st.slot_state[slot].state >= GYSK_STATE_SEVERE;
	const unsigned run = __match_any_sync(live, head);
	const unsigned bi = __ballot_sync(run, issue), bs = __ballot_sync(run, severe);
	if ((threadIdx.x & 31) == __ffs(run) - 1 && bi)
		atomicAdd(acc + head, ((unsigned long long)__popc(bi) << 32) | (unsigned long long)__popc(bs));
}

// One CTA walks the keys in order and writes the row of every host run whose rank lies in [rlo, rlo + cap): {host, run length, issue,
// severe}; *d_rows = number of runs. tile_rank ranks the run heads of each 1024-key tile.
__global__ void __launch_bounds__(1024) host_listen_rows_kernel(const unsigned long long *__restrict__ keys, const unsigned long long *d_n,
		const unsigned long long *__restrict__ acc, uint32_t rlo, uint32_t cap, gysk_host_listen *__restrict__ out, unsigned long long *d_rows)
{
	__shared__ uint32_t wcnt[32];
	const uint32_t n = (uint32_t)*d_n;
	uint32_t running = 0;

	for (uint32_t t = 0; t < n; t += 1024) {
		const uint32_t i = t + threadIdx.x;
		const uint32_t h = i < n ? (uint32_t)(keys[i] >> 32) : 0;
		const bool head = i < n && (i == 0 || (uint32_t)(keys[i - 1] >> 32) != h);
		tile_rank(head, wcnt, running, [&](uint32_t r) {
			if (r < rlo || r - rlo >= cap) return;
			const unsigned long long a = acc[i];
			out[r - rlo] = gysk_host_listen {h, host_bound(keys, i + 1, n, h, true) - i, (uint32_t)(a >> 32), (uint32_t)a};
		});
	}
	if (threadIdx.x == 0) *d_rows = running;
}

// one warp per service: by id (ids != nullptr: looked up, id 0 and unknown ids give found = 0) or by slot (the window read). The
// slot's state goes into shared memory, then summarize_warp makes the row.
static constexpr int SUMM_WARPS = 4;
__global__ void __launch_bounds__(SUMM_WARPS * 32) svc_summary_kernel(DevState st, const unsigned long long *__restrict__ ids,
		const unsigned long long *__restrict__ slots, uint32_t n, gysk_svc_summary *__restrict__ out)
{
	__shared__ SvcRaw raw[SUMM_WARPS];
	__shared__ unsigned long long summ[SUMM_WARPS][sizeof(gysk_svc_summary) / 8];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t q = blockIdx.x * SUMM_WARPS + wid;

	if (q >= n) return;
	SvcRaw &r = raw[wid];
	const Resolved s = resolve_warp(st.svc_tbl, ids, slots, q, lane);
	if (lane == 0) { r.id = s.id; r.found = s.slot >= 0; r.slot = (uint32_t)s.slot; }
	if (s.slot >= 0) {
		gather_slot(st, s.slot, r, lane);
		hll_hist_warp(st.hll + ((size_t)s.slot << st.hll_p), st.hll_p, r.hll_hist, lane);
	}
	summarize_warp(r, s.id, st.hll_p, summ[wid], out + q, lane);
}

// one warp per process: by id (ids != nullptr: looked up, unknown ids give found = 0) or by slot (the window read)
__global__ void __launch_bounds__(128) task_summary_kernel(DevState st, const unsigned long long *__restrict__ ids,
		const unsigned long long *__restrict__ slots, uint32_t n, gysk_task_summary *__restrict__ out)
{
	__shared__ HistCell h[4][3 * HIST_CELLS + 3];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t q = blockIdx.x * 4 + wid;

	if (q >= n) return;
	const Resolved s = resolve_warp(st.task_tbl, ids, slots, q, lane);
	if (s.slot < 0) {
		if (lane == 0) { gysk_task_summary z; memset(&z, 0, sizeof(z)); z.aggr_task_id = s.id; out[q] = z; }
		return;
	}
	for (int i = lane; i < 3 * HIST_CELLS; i += 32) h[wid][i] = st.task_hist[(size_t)s.slot * 3 * HIST_CELLS + i];
	if (lane < 3) h[wid][3 * HIST_CELLS + lane] = st.task_last[(size_t)s.slot * 3 + lane];
	__syncwarp();
	if (lane == 0) summarize_task(h[wid], h[wid] + 3 * HIST_CELLS, s.id, st.task_slot_host[s.slot], out[q]);
}

// the single-id export gysk_export_task_hist: one warp per id, the id's three histograms
__global__ void __launch_bounds__(128) gather_tasks_kernel(DevState st, const unsigned long long *__restrict__ ids, uint32_t n, TaskRaw *__restrict__ out)
{
	const int lane = threadIdx.x & 31;
	const uint32_t q = blockIdx.x * 4 + (threadIdx.x >> 5);

	if (q >= n) return;
	const Resolved r = resolve_warp(st.task_tbl, ids, nullptr, q, lane);
	if (lane == 0) { out[q].id = r.id; out[q].found = r.slot >= 0; out[q].slot = (uint32_t)r.slot; }
	if (r.slot < 0) return;
	for (int i = lane; i < 3 * HIST_CELLS; i += 32) (&out[q].h[0][0])[i] = st.task_hist[(size_t)r.slot * 3 * HIST_CELLS + i];
}

// gysk_export_hll: the registers of one id (ids[0]); every warp resolves the id itself. With a Set parameter, set (gysk_export_hll_window,
// GYSK_FLAG_CLIENT_LEVELS): the CL_REGS registers of the id's slot in that client set instead of its all-time ones. A pack, so that the
// all-time instance keeps its parameter list.
__device__ __forceinline__ const uint8_t *hll_regs_of(const DevState &st, int slot) { return st.hll + ((size_t)slot << st.hll_p); }
__device__ __forceinline__ const uint8_t *hll_regs_of(const DevState &, int slot, const uint8_t *set) { return set + (size_t)slot * CL_REGS; }
template <typename... Set>
__global__ void gather_hll_kernel(DevState st, const unsigned long long *__restrict__ ids, int32_t *found, uint8_t *__restrict__ out, Set... set)
{
	const int slot = resolve_warp(st.svc_tbl, ids, nullptr, 0, threadIdx.x & 31).slot;
	if (threadIdx.x == 0) *found = slot >= 0;
	if (slot < 0) return;
	const uint8_t *regs = hll_regs_of(st, slot, set...);
	const uint32_t nregs = sizeof...(Set) ? CL_REGS : 1u << st.hll_p;
	for (uint32_t i = threadIdx.x; i < nregs; i += blockDim.x) out[i] = regs[i];
}

// the point estimate of a flow key on a count-min of one u64 per cell: the minimum over rows of each half
__device__ __forceinline__ void cms_point(const unsigned long long *__restrict__ tbl, uint32_t depth, uint32_t log2w, unsigned long long key,
		uint32_t &lo, uint32_t &hi)
{
	lo = 0xFFFFFFFFu; hi = 0xFFFFFFFFu;
	for (uint32_t r = 0; r < depth; ++r) {
		const unsigned long long c = tbl[((size_t)r << log2w) + cms_index(key, r, (1u << log2w) - 1)];
		lo = min(lo, (uint32_t)c);
		hi = min(hi, (uint32_t)(c >> 32));
	}
}

__global__ void query_flows_kernel(const unsigned long long *__restrict__ tbl, uint32_t depth, uint32_t log2w, const unsigned long long *__restrict__ keys,
		uint32_t n, gysk_flow_est *__restrict__ out)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const unsigned long long key = keys[i];
	uint32_t cnt, kb;
	cms_point(tbl, depth, log2w, key, cnt, kb);
	out[i].flow_key = key; out[i].count = cnt; out[i].kbytes = kb;
}

// GYSK_FLAG_FLOW_RESP_HIST: the point estimate of a flow key on a response histogram table, per bucket b the minimum over rows of its
// count (mn[15], word 7's high half, ends 0). The one definition of a flow's bucket counts: the point query, and the slow score of
// GYSK_FLAG_FLOW_TOPK_SLOW (resp_slow_score) read it.
__device__ __forceinline__ void resp_point(const unsigned long long *__restrict__ tbl, uint32_t depth, uint32_t log2w, unsigned long long key,
		uint32_t (&mn)[16])
{
#pragma unroll
	for (int b = 0; b < 16; ++b) mn[b] = 0xFFFFFFFFu;
	for (uint32_t r = 0; r < depth; ++r) {
		const ulonglong2 *c = reinterpret_cast<const ulonglong2 *>(tbl + (((size_t)r << log2w) + cms_index(key, r, (1u << log2w) - 1)) * RESP_HIST_WORDS);
#pragma unroll
		for (int w = 0; w < (int)RESP_HIST_WORDS / 2; ++w) {
			const ulonglong2 v = c[w];
			mn[4 * w] = min(mn[4 * w], (uint32_t)v.x); mn[4 * w + 1] = min(mn[4 * w + 1], (uint32_t)(v.x >> 32));
			mn[4 * w + 2] = min(mn[4 * w + 2], (uint32_t)v.y); mn[4 * w + 3] = min(mn[4 * w + 3], (uint32_t)(v.y >> 32));
		}
	}
}

// GYSK_FLAG_FLOW_TOPK_SLOW: a flow's slow score S, the sum of its bucket counts from b_slow (2..14) on, saturated at 2^32 - 1 so that it
// fits a rank key's 32 score bits and stays monotone in every count
__device__ __forceinline__ uint32_t resp_slow_score(const unsigned long long *__restrict__ tbl, uint32_t depth, uint32_t log2w, unsigned long long key,
		uint32_t b_slow)
{
	uint32_t mn[16];
	resp_point(tbl, depth, log2w, key, mn);
	unsigned long long s = 0;
#pragma unroll
	for (uint32_t b = 0; b < 15; ++b) if (b >= b_slow) s += mn[b];
	return (uint32_t)min(s, 0xFFFFFFFFull);
}

// GYSK_FLAG_FLOW_RESP_HIST: per key and bucket the minimum over rows of the 8-word cells, then the response percentiles of those counts by
// the rule of the service summaries' p95_5s_resp_ms (hist_percentile of RESP_TIME_HASH: GY_HISTOGRAM::get_percentiles), the full sum as the
// total
__global__ void query_flow_resp_kernel(const unsigned long long *__restrict__ tbl, uint32_t depth, uint32_t log2w, const unsigned long long *__restrict__ keys,
		uint32_t n, gysk_flow_resp_est *__restrict__ out)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const unsigned long long key = keys[i];
	uint32_t mn[16];
	resp_point(tbl, depth, log2w, key, mn);
	uint64_t counts[15], total = 0;
#pragma unroll
	for (int b = 0; b < 15; ++b) { counts[b] = mn[b]; total += mn[b]; out[i].counts[b] = mn[b]; }
	out[i].flow_key = key;
	out[i].total = (uint32_t)total;
	out[i].p25_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 25.0f);
	out[i].p95_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 95.0f);
	out[i].p99_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 99.0f);
}

// A rolling count-min level (GYSK_FLAG_FLOW_LEVEL, GYSK_FLAG_FLOW_QUERY_LEVEL) at a flush, one grid-stride pass over the cells in
// 16-byte pairs. Ring slot k takes the closing window cur, added to what the slot holds or, when the flush started a new epoch there,
// in its place (which stands in for clearing the slot). The level becomes the sum of the live slots, slot k's new content included. So the pass reads cur and the live
// slots and writes slot k and the level, every cell mod 2^64 as RED.ADD.64 builds cur. The ring and the level are streamed
// (evict-first) so that the pass does not push out of L2 the count-min lines the ingest path keeps resident.
__global__ void __launch_bounds__(256) cms_level_roll_kernel(const ulonglong2 *__restrict__ cur, ulonglong2 *__restrict__ ring,
		ulonglong2 *__restrict__ level, uint64_t npair, uint32_t k, uint32_t live, uint32_t fresh)
{
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npair; i += (uint64_t)gridDim.x * blockDim.x) {
		ulonglong2 r = cur[i];
		if (!fresh) {
			const ulonglong2 o = __ldcs(ring + k * npair + i);
			r.x += o.x; r.y += o.y;
		}
		__stcs(ring + k * npair + i, r);
		ulonglong2 a = make_ulonglong2(0, 0);
#pragma unroll
		for (uint32_t j = 0; j < NSLOTS; ++j) {
			if (!((live >> j) & 1u)) continue;
			const ulonglong2 x = j == k ? r : __ldcs(ring + j * npair + i);
			a.x += x.x; a.y += x.y;
		}
		__stcs(level + i, a);
	}
}

__device__ __forceinline__ uint4 vmax4(uint4 a, uint4 b) { return make_uint4(__vmaxu4(a.x, b.x), __vmaxu4(a.y, b.y), __vmaxu4(a.z, b.z), __vmaxu4(a.w, b.w)); }

// GYSK_FLAG_CLIENT_LEVELS at a flush: one grid-stride pass over the registers of service slots [0, nslots) in 16-byte pieces. Ring slot
// k takes the closing window's open set, max-merged into what it holds or, when the flush started a new epoch there, in its place
// (which stands in for clearing the slot); the level becomes the registerwise maximum of the live slots, slot k's new content included:
// the rule of cms_level_roll_kernel with max for +. nslots is the engine's capacity, which every client array holds; cl.stride is only
// the ring planes' pitch (a growth that stopped half way may have raised it alone). The ring and the level are streamed (evict-first).
__global__ void __launch_bounds__(256) client_roll_kernel(ClientLevels cl, uint32_t nslots, uint32_t k, uint32_t live, uint32_t fresh)
{
	constexpr uint32_t Q = CL_REGS / 16;
	const uint64_t npiece = (uint64_t)nslots * Q, plane = (uint64_t)cl.stride * Q;
	const uint4 *open = reinterpret_cast<const uint4 *>(cl.open);
	uint4 *ring = reinterpret_cast<uint4 *>(cl.ring), *level = reinterpret_cast<uint4 *>(cl.level);
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npiece; i += (uint64_t)gridDim.x * blockDim.x) {
		uint4 r = open[i];
		if (!fresh) r = vmax4(r, __ldcs(ring + k * plane + i));
		__stcs(ring + k * plane + i, r);
		uint4 a = make_uint4(0, 0, 0, 0);
#pragma unroll
		for (uint32_t j = 0; j < NSLOTS; ++j) {
			if (!((live >> j) & 1u)) continue;
			a = vmax4(a, j == k ? r : __ldcs(ring + j * plane + i));
		}
		__stcs(level + i, a);
	}
}

// gysk_query_svc_clients / gysk_query_clients_window: one warp per service, by id (ids != nullptr: looked up, id 0 and unknown ids give
// found = 0) or by slot (the window read): the register histograms of the last and the level sets, each estimate as hll_pending leaves it
// (the host finishes it with hll_finish at GYSK_HLL_WINDOW_P)
static constexpr int CL_WARPS = 4;
__global__ void __launch_bounds__(CL_WARPS * 32) client_rows_kernel(DevState st, ClientLevels cl, const unsigned long long *__restrict__ ids,
		const unsigned long long *__restrict__ slots, uint32_t n, gysk_svc_clients *__restrict__ out)
{
	__shared__ uint32_t hist[CL_WARPS][2][64];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t q = blockIdx.x * CL_WARPS + wid;

	if (q >= n) return;
	const Resolved s = resolve_warp(st.svc_tbl, ids, slots, q, lane);
	gysk_svc_clients o;
	memset(&o, 0, sizeof(o));
	o.glob_id = s.id;
	if (s.slot >= 0) {
		hll_hist_warp(cl.last + (size_t)s.slot * CL_REGS, GYSK_HLL_WINDOW_P, hist[wid][0], lane);
		hll_hist_warp(cl.level + (size_t)s.slot * CL_REGS, GYSK_HLL_WINDOW_P, hist[wid][1], lane);
		o.found = 1;
		o.last_5s = hll_pending(hist[wid][0], GYSK_HLL_WINDOW_P);
		o.last_5min = hll_pending(hist[wid][1], GYSK_HLL_WINDOW_P);
	}
	if (lane == 0) out[q] = o;
}

// ---------------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------------
static inline uint32_t div_up(uint64_t a, uint64_t b) { return (uint32_t)((a + b - 1) / b); }

// cudaFuncSetAttribute is per DEVICE: one process may own an engine on every GPU of the box (INTEGRATION.md §2)
static constexpr int MAX_DEVICES = 64;
static int current_device() { int dev = 0; cudaGetDevice(&dev); return dev < 0 || dev >= MAX_DEVICES ? 0 : dev; }
static int sm_count(int dev) { int nsm = 132; cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev); return nsm; }

int launch_init_slots(const DevState &st, uint32_t s_lo, uint32_t s_hi, uint32_t t_lo, uint32_t t_hi, cudaStream_t s)
{
	const uint32_t ns = s_hi - s_lo, nt = t_hi - t_lo;
	if (!ns && !nt) return 0;
	const uint32_t grid = std::min<uint32_t>(std::max(ns, div_up(nt, 256)), (uint32_t)sm_count(current_device()) * 16u);
	init_slots_kernel<<<grid, 256, 0, s>>>(st, s_lo, s_hi, t_lo, t_hi);
	return 1;
}

int launch_register(const DevState &st, const unsigned long long *d_ids, uint32_t n, int is_task, cudaStream_t s)
{
	if (!n) return 0;
	register_kernel<<<div_up(n, 256), 256, 0, s>>>(st, d_ids, n, is_task);
	return 1;
}

// the radix passes of the RESP keys sort on the slot only = key bits [40, 40 + slot bits), where key_slots covers the services and
// the trace pseudo-slots: the slot bits cut into the fewest digits of at most KEY_DIGIT_MAX bits, widths as even as possible
// (17 bits -> 9 8). A 9-bit pass costs more per key than an 8-bit one (two look-back rows per thread, nine ballots per key), but a
// pass's cost follows the bits it ranks, and a pass fewer saves one read and one write of every key.
static int key_sort_plan(uint32_t key_slots, SortPlan &P)
{
	int slot_bits = 1;
	while (slot_bits < KEY_SLOT_BITS_MAX && (1ull << slot_bits) < key_slots) slot_bits++;
	const int T = slot_bits;
	P.np = (T + KEY_DIGIT_MAX - 1) / KEY_DIGIT_MAX;
	if (P.np > KEY_PASSES_MAX) return -1;
	int at = KEY_SLOT_SHIFT;
	for (int p = 0; p < P.np; ++p) { P.bits[p] = T / P.np + (p < T % P.np ? 1 : 0); P.shift[p] = at; at += P.bits[p]; }
	return 0;
}

// every other sort: key bits [lo, hi) in 8-bit digits from lo upwards, the last one short; the first ones are 9 bits wide where
// that saves a whole pass (18 bits -> 9 9). A range outside the key's 64 bits has no plan: [0, 72) would fit in 8 passes of 9 bits,
// and a shift of 64 or more is undefined.
static int plain_sort_plan(int lo, int hi, SortPlan &P)
{
	if (lo < 0 || hi > 64 || lo > hi) return -1;
	const int T = hi - lo, p8 = (T + 7) / 8, p9 = (T + 8) / 9;
	int wide = p9 < p8 ? T - 8 * p9 : 0;	// number of 9-bit passes
	int at = lo;
	for (P.np = 0; at < hi; at += P.bits[P.np++]) {
		if (P.np == OS_MAX_PASSES) return -1;
		P.shift[P.np] = at;
		P.bits[P.np] = std::min(wide-- > 0 ? 9 : 8, hi - at);
	}
	return 0;
}

// ingest_kernel and drain_kernel each keep their instances in one table indexed by the instance's feature bits, filled from an index
// sequence. Each kernel's flag rules are stated once (ingest_reached, drain_reached): only the instances they reach are compiled, the
// other entries launch nothing, and the launcher refuses a flag set outside the rules.

// ingest_kernel's feature bits: TRACE (the engine has trace rows), then the FlowPass flags. ERR comes only with QRY: 24 instances.
enum IngestBit { ING_TRACE = 1, ING_QRY = 2, ING_TOPK = 4, ING_ERR = 8, ING_CL = 16, ING_INSTANCES = 32 };
static constexpr bool ingest_reached(int f) { return !(f & ING_ERR) || (f & ING_QRY); }

// An instance's shared-memory attribute is set at its first launch on a device, so that an engine without a flag never loads that
// flag's instances: setting the attribute loads the kernel, which can wait for the work already on the device.
template <int F>
static void launch_ingest_pass(const DevState &st, const SortTemp &tmp, const FlowPass &fp, const gysk_event *d_ev, uint64_t n, const SortPlan &plan,
		uint32_t grid, int dev, cudaStream_t s)
{
	if constexpr (ingest_reached(F)) {
		constexpr bool TRACE = F & ING_TRACE, QRY = F & ING_QRY, TOPK = F & ING_TOPK, ERR = F & ING_ERR, CL = F & ING_CL;
		static bool attr_set[MAX_DEVICES] = {};
		const auto launch = [&](auto kernel, auto... cl_open) {
			if (!attr_set[dev]) {
				cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(IngestShared));
				attr_set[dev] = true;
			}
			kernel<<<grid, IngestShape::WARPS * 32, sizeof(IngestShared), s>>>(st, d_ev, n, tmp.keys_a, tmp.os_ghist, plan, tmp.recq, tmp.rec_cnt,
					fp.tk.list[0], cl_open...);
		};
		if constexpr (CL) launch(ingest_kernel<TRACE, QRY, TOPK, ERR, uint8_t *>, fp.cl.open);
		else launch(ingest_kernel<TRACE, QRY, TOPK, ERR>);
	}
}
template <int... F>
static constexpr auto ingest_passes(std::integer_sequence<int, F...>) { return std::array {launch_ingest_pass<F>...}; }

int launch_ingest(const DevState &st, const SortTemp &tmp, const FlowPass &fp, const gysk_event *d_ev, uint64_t n, uint32_t key_slots,
		RecRegions &rr, cudaStream_t s)
{
	if (!n) return 0;
	const int f = (st.trace.rows ? ING_TRACE : 0) | (fp.fq.cur ? ING_QRY : 0) | (fp.tk.list[0].keys ? ING_TOPK : 0) | (fp.fe.cur ? ING_ERR : 0) |
			(fp.cl.open ? ING_CL : 0);
	if (!ingest_reached(f)) return -1;
	const int dev = current_device();
	SortPlan plan {};
	if (key_sort_plan(key_slots, plan) < 0) return -1;
	// the hot rows handed out by the batches so far are in use from this batch on
	if (st.hot_rows) cudaMemcpyAsync(st.counters + CTR_NHOT, st.counters + CTR_NHOT_NEXT, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s);
	// key cursor, digit histograms and tile tickets of this batch's sort
	cudaMemsetAsync(st.counters + CTR_NKEYS, 0, sizeof(unsigned long long), s);
	cudaMemsetAsync(tmp.os_ghist, 0, OS_GHIST_WORDS * sizeof(uint32_t), s);
	constexpr int WARPS = IngestShape::WARPS, CHUNK = IngestShape::CHUNK;
	const uint64_t want = (n + (uint64_t)CHUNK * WARPS - 1) / ((uint64_t)CHUNK * WARPS);
	const uint64_t full = (uint64_t)sm_count(dev) * IngestShape::MIN_CTAS;
	const uint32_t grid = (uint32_t)(want < full ? want : full);
	// the kernel computes the same regions from its grid
	const uint64_t nchunks = (n + CHUNK - 1) / CHUNK;
	rr.nwarps = grid * WARPS;
	rr.cap = (nchunks + rr.nwarps - 1) / rr.nwarps * CHUNK;
	if (rr.nwarps > tmp.rec_cnt_cap || (uint64_t)rr.nwarps * rr.cap > tmp.recq_cap) return -1;
	// a counted response sample takes a connection-queue entry, as one connection event does: the regions hold one record per event
	static constexpr auto passes = ingest_passes(std::make_integer_sequence<int, ING_INSTANCES> {});
	passes[f](st, tmp, fp, d_ev, n, plan, grid, dev, s);
	return 1;
}

// drain_kernel's feature bits: TASK (the pass), then the FlowPass flags. RH and ERR come only with QRY, SLOW only with RH and TOPK, and
// the TASK pass has neither SLOW nor CL: 24 TCP and 10 TASK instances.
enum DrainBit { DR_TASK = 1, DR_QRY = 2, DR_RH = 4, DR_TOPK = 8, DR_SLOW = 16, DR_CL = 32, DR_ERR = 64, DR_INSTANCES = 128 };
static constexpr bool drain_reached(int f)
{
	if ((f & (DR_RH | DR_ERR)) && !(f & DR_QRY)) return false;
	if ((f & DR_SLOW) && (f & (DR_RH | DR_TOPK)) != (DR_RH | DR_TOPK)) return false;
	return !((f & DR_TASK) && (f & (DR_SLOW | DR_CL)));
}

// one drain pass: as many CTAs as the SMs hold at once (at most one per 32 x WARPS events of the batch); shared memory = the hot
// table + the region start table, whose largest size sets the occupancy. mask: the batch flow tables' entries - 1. A flag's parameters
// go to the instances with its bit and zero to the others: b_slow (GYSK_FLAG_FLOW_TOPK_SLOW's first slow bucket) to the SLOW ones.
template <int F>
static void launch_drain_pass(const DevState &st, const SortTemp &tmp, const FlowPass &fp, const RecRegions &rr, uint64_t n_events, uint32_t mask,
		int dev, cudaStream_t s)
{
	if constexpr (drain_reached(F)) {
		constexpr bool TASK = F & DR_TASK, QRY = F & DR_QRY, RH = F & DR_RH, TOPK = F & DR_TOPK, SLOW = F & DR_SLOW, CL = F & DR_CL, ERR = F & DR_ERR;
		constexpr int WARPS = DrainShape<TASK>::WARPS;
		constexpr size_t HOT_BYTES = sizeof(HotTableT<DrainShape<TASK>::HOT_BITS>);
		static int per_sm[MAX_DEVICES] = {};
		if (!per_sm[dev]) {
			const size_t smem_max = HOT_BYTES + ((size_t)tmp.rec_cnt_cap + 1) * sizeof(uint32_t);
			cudaFuncSetAttribute(drain_kernel<TASK, QRY, RH, TOPK, SLOW, CL, ERR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
			int b = 0;
			cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, drain_kernel<TASK, QRY, RH, TOPK, SLOW, CL, ERR>, WARPS * 32, smem_max);
			per_sm[dev] = b > 0 ? b : 1;
		}
		const uint64_t want = (n_events + WARPS * 32 - 1) / (WARPS * 32);
		const uint64_t full = (uint64_t)sm_count(dev) * per_sm[dev];
		const size_t smem = HOT_BYTES + ((size_t)rr.nwarps + 1) * sizeof(uint32_t);
		const FlowTable none {nullptr, 0u};
		drain_kernel<TASK, QRY, RH, TOPK, SLOW, CL, ERR><<<(uint32_t)(want < full ? want : full), WARPS * 32, smem, s>>>(st, FlowTable {tmp.flow, mask},
				tmp.recq, tmp.rec_cnt, rr, QRY ? FlowTable {fp.fq.flow, mask} : none, QRY ? fp.fq.cur : nullptr, RH ? FlowTable {fp.fr.flow, mask} : none,
				RH ? fp.fr.cur : nullptr, fp.tk, SLOW ? fp.b_slow : 0u, CL ? fp.cl.open : nullptr,
				ERR ? ErrPass {FlowTable {fp.fe.flow, mask}, fp.fe.cur, fp.fe.list} : ErrPass {});
	}
}
template <int... F>
static constexpr auto drain_passes(std::integer_sequence<int, F...>) { return std::array {launch_drain_pass<F>...}; }

// the batch's queued connection records -> flow table, HLL, exact cells; then the flow table -> count-min and its process records ->
// process histograms. The TASK pass always runs: it leaves the flow table empty. The table takes the smallest power of two >= 2 x the
// batch's events (the flows are fewer than the connection records), up to what tmp holds, so that a small batch sweeps a small table.
// With GYSK_FLAG_FLOW_QUERIES (fq.cur) the queued response samples go the same way through a query flow table of the same size, and
// with GYSK_FLAG_FLOW_RESP_HIST (fr.cur) through a response flow table of that size too. With GYSK_FLAG_FLOW_ERRORS (fe.cur) the error
// samples go through an error flow table of that size as well: a batch whose samples all carry an error bit needs every entry the query
// table needs (DESIGN.md section 7).
int launch_drains(const DevState &st, const SortTemp &tmp, const FlowPass &fp, const RecRegions &rr, uint64_t n_events, cudaStream_t s)
{
	if (!n_events) return 0;
	const int tcp = (fp.fq.cur ? DR_QRY : 0) | (fp.fr.cur ? DR_RH : 0) | (fp.tk.list[0].keys ? DR_TOPK : 0) | (fp.tk.list[2].keys ? DR_SLOW : 0) |
			(fp.cl.open ? DR_CL : 0) | (fp.fe.cur ? DR_ERR : 0);
	if (!drain_reached(tcp)) return -1;
	const int dev = current_device();
	uint32_t n = 16;
	while (n < tmp.flow_cap && n < 2 * n_events) n <<= 1;
	cudaMemsetAsync(st.counters + CTR_FLOW_DIRECT, 0, sizeof(unsigned long long), s);
	if (fp.fq.cur) cudaMemsetAsync(st.counters + CTR_FLOWQ_DIRECT, 0, sizeof(unsigned long long), s);
	if (fp.fe.cur) cudaMemsetAsync(st.counters + CTR_FLOWE_DIRECT, 0, sizeof(unsigned long long), s);
	if (fp.fr.cur) cudaMemsetAsync(st.counters + CTR_FLOWR_DIRECT, 0, sizeof(unsigned long long), s);
	static constexpr auto passes = drain_passes(std::make_integer_sequence<int, DR_INSTANCES> {});
	passes[tcp](st, tmp, fp, rr, n_events, n - 1u, dev, s);
	passes[DR_TASK | (tcp & ~(DR_SLOW | DR_CL))](st, tmp, fp, rr, n_events, n - 1u, dev, s);
	return 2;
}

static void os_set_attrs(int dev)
{
	static bool attr_set[MAX_DEVICES] = {};
	if (attr_set[dev]) return;
	cudaFuncSetAttribute(os_pass_kernel<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(OneSweepSharedT<6>));
	cudaFuncSetAttribute(os_pass_kernel<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(OneSweepSharedT<7>));
	cudaFuncSetAttribute(os_pass_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(OneSweepSharedT<8>));
	cudaFuncSetAttribute(os_pass_kernel<9>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(OneSweepSharedT<9>));
	cudaFuncSetAttribute(os_hist_kernel<8, 257>, cudaFuncAttributeMaxDynamicSharedMemorySize, OS_MAX_PASSES * 8 * 257 * (int)sizeof(uint32_t));
	cudaFuncSetAttribute(os_hist_kernel<4, 513>, cudaFuncAttributeMaxDynamicSharedMemorySize, OS_MAX_PASSES * 4 * 513 * (int)sizeof(uint32_t));
	attr_set[dev] = true;
}

static uint32_t next_epoch(const SortTemp &tmp, uint32_t max_tiles, cudaStream_t s)
{
	uint32_t e = ++*tmp.epoch;
	if (e == 0) {		// 2^32 passes later: stale words could pass for current ones, start over
		cudaMemsetAsync(tmp.tile_status, 0, (size_t)max_tiles * RADIX_MAX * sizeof(unsigned long long), s);
		e = ++*tmp.epoch;
	}
	return e;
}

// the passes of a plan over the *d_n keys in tmp.keys_a, ping-pong with keys_b; tmp.os_ghist holds the passes' histograms and zeroed
// tickets. Each pass runs the kernel instantiation of its digit's width: a 7-bit digit has half the per-digit work (per-warp
// counters to clear and prefix, status words to publish and look back through, ballots per key) of an 8-bit one. The grid is
// persistent (os_pass_kernel): at most as many CTAs as the SMs hold at once, whatever the number of possible tiles.
// Returns the launches; *which = the buffer that holds the sorted keys
static int launch_sort_passes(const SortPlan &P, const SortTemp &tmp, const unsigned long long *d_n, uint32_t ntiles, int *which, cudaStream_t s)
{
	unsigned long long *bufs[2] = { tmp.keys_a, tmp.keys_b };
	const uint32_t grid = std::min<uint32_t>(ntiles, (uint32_t)sm_count(current_device()) * 4u);		// __launch_bounds__(OS_THREADS, 4)
	int w = 0;

	for (int p = 0; p < P.np; ++p, w ^= 1) {
		const uint32_t epoch = next_epoch(tmp, tmp.max_tiles, s);
		auto pass = [&](auto kernel, size_t smem) {
			kernel<<<grid, OS_THREADS, smem, s>>>(bufs[w], bufs[w ^ 1], d_n, P.shift[p], P.bits[p], tmp.os_ghist + p * RADIX_MAX, tmp.tile_status,
					tmp.os_ghist + OS_GHIST_TICKETS + p, epoch);
		};
		if (P.bits[p] > 8) pass(os_pass_kernel<9>, sizeof(OneSweepSharedT<9>));
		else if (P.bits[p] == 8) pass(os_pass_kernel<8>, sizeof(OneSweepSharedT<8>));
		else if (P.bits[p] == 7) pass(os_pass_kernel<7>, sizeof(OneSweepSharedT<7>));
		else pass(os_pass_kernel<6>, sizeof(OneSweepSharedT<6>));
	}
	*which = w;
	return P.np;
}

// stable LSD radix sort of the *d_n keys in keys_a on their bits [lo, hi): n_max >= *d_n sizes the grids
int launch_radix_sort(const SortTemp &tmp, const unsigned long long *d_n, uint64_t n_max, int lo, int hi, int *which, cudaStream_t s)
{
	SortPlan P;

	*which = 0;
	if (!n_max) return 0;
	if (plain_sort_plan(lo, hi, P) || n_max >= (1ull << 30)) return -1;	// status words carry 30-bit counts
	bool any9 = false;
	for (int p = 0; p < P.np; ++p) any9 |= P.bits[p] > 8;
	const int copies = any9 ? 4 : 8, stride = (any9 ? 512 : 256) + 1;
	const int dev = current_device();
	os_set_attrs(dev);

	cudaMemsetAsync(tmp.os_ghist, 0, OS_GHIST_WORDS * sizeof(uint32_t), s);
	const uint32_t hgrid = std::min<uint32_t>(div_up(n_max, 512 * 2 * 4), (uint32_t)sm_count(dev) * 3);
	if (any9) os_hist_kernel<4, 513><<<hgrid, 512, (size_t)P.np * copies * stride * sizeof(uint32_t), s>>>(tmp.keys_a, d_n, P, tmp.os_ghist);
	else os_hist_kernel<8, 257><<<hgrid, 512, (size_t)P.np * copies * stride * sizeof(uint32_t), s>>>(tmp.keys_a, d_n, P, tmp.os_ghist);
	return 1 + launch_sort_passes(P, tmp, d_n, div_up(n_max, SORT_TILE), which, s);
}

// after the ingest kernel of a batch: sort its RESP keys by slot, find every service's key segment, reduce the long ones into
// batch rows and fold every touched service's bins into its window histogram and its digest. Nothing here needs a number from the
// device on the host: the key count lives in st.counters[CTR_NKEYS], the digit histograms in tmp.os_ghist (both written by
// ingest_kernel); grids are sized by n_events, the largest possible key count, and surplus CTAs leave at once.
int launch_batch_merge(const DevState &st, const SortTemp &tmp, uint64_t n_events, uint32_t key_slots, cudaStream_t s)
{
	if (!n_events) return 0;
	unsigned long long *d_nkeys = st.counters + CTR_NKEYS, *d_ntouched = st.counters + CTR_NTOUCHED;
	const int dev = current_device();
	const int nsm = sm_count(dev);
	os_set_attrs(dev);

	SortPlan plan {};
	if (key_sort_plan(key_slots, plan) < 0) return -1;
	int which = 0;
	const int launches = launch_sort_passes(plan, tmp, d_nkeys, div_up(n_events, SORT_TILE), &which, s);
	const unsigned long long *src = which ? tmp.keys_b : tmp.keys_a;

	static_assert(CTR_NLONG == CTR_NTOUCHED + 1, "one memset clears both segment counters");
	unsigned long long *d_nlong = st.counters + CTR_NLONG;
	BatchSeg *segs = reinterpret_cast<BatchSeg *>(tmp.segs);
	cudaMemsetAsync(d_ntouched, 0, 2 * sizeof(unsigned long long), s);
	segs_mark_kernel<<<div_up(n_events, SG_THREADS * SG_V), SG_THREADS, 0, s>>>(src, d_nkeys, segs, tmp.touched, d_ntouched, tmp.long_slot, d_nlong);
	long_sum_kernel<<<nsm * 8, 256, 0, s>>>(src, d_nkeys, segs, d_nlong, tmp.batch_rows);
	if (st.trace.rows) trace_keys_kernel<<<nsm * 4, 256, 0, s>>>(st.trace, src, d_nkeys);
	const int merge_ctas = std::min(nsm, TD_MERGE_MAX_SMS) * TD_MERGE_CTAS_PER_SM;
	if (st.trace.rows)
		bins_merge_kernel<true><<<merge_ctas, TD_WARPS * 32, 0, s>>>(st, src, tmp.touched, d_ntouched, tmp.long_slot, d_nlong, tmp.batch_rows, segs,
				tmp.items_scratch, tmp.big_scratch);
	else
		bins_merge_kernel<false><<<merge_ctas, TD_WARPS * 32, 0, s>>>(st, src, tmp.touched, d_ntouched, tmp.long_slot, d_nlong, tmp.batch_rows, segs,
				tmp.items_scratch, tmp.big_scratch);
	return launches + 3 + (st.trace.rows ? 1 : 0);
}

// ---------------------------------------------------------------------------------------------------
// top-N services of the last closed window (BOUNDED_PRIO_QUEUE uses of partha_listener_state, gy_mconnhdlr.cc:11262-11304:
// top listeners by qps / active conns / network): score every service, radix-sort (score, slot) keys, read the tail
// ---------------------------------------------------------------------------------------------------
__global__ void topn_score_kernel(DevState st, uint32_t nslots, int metric, int host_filter, unsigned long long *__restrict__ keys,
		unsigned long long *d_n)
{
	const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot == 0) *d_n = nslots;
	if (slot >= nslots) return;
	unsigned long long score = 0;

	if (host_filter < 0 || st.slot_host[slot] == (uint32_t)host_filter) {
		if (metric == GYSK_TOPN_QPS) {
			for (int b = 0; b < HIST_MAX_CELL; ++b) score += st.hist_last[(size_t)slot * HIST_CELLS + b].count;
		}
		else if (metric == GYSK_TOPN_CONNS) score = (uint32_t)st.conn_last[slot];
		else if (metric == GYSK_TOPN_ISSUE) {
			// ptopissue of partha_listener_state (gy_mconnhdlr.cc:11262-11271): listeners with curr_state_ > STATE_OK, worse state first
			// (LISTEN_TOPN::is_comp_issue, gy_msocket.h:745; its tie-break, tasks_delay_usec_, is not on this path)
			const SlotState ss = st.slot_state[slot];
			score = ss.state > GYSK_STATE_OK && ss.state <= GYSK_STATE_DOWN ? ss.state : 0;
		}
		else if (metric == GYSK_TOPN_ACTIVE) score = (uint32_t)st.slot_aux[slot].act_last;	// nconns_active (is_comp_active_conn; gysk_topn_global only)
		else score = st.conn_last[slot] >> 32;
	}
	if (score > 0xFFFFFFFFull) score = 0xFFFFFFFFull;
	keys[slot] = (score << 32) | slot;
}

// top-N aggregated processes of the last closed window by cpu / cpu delay / blkio delay: the atask_top_cpu_ / _cpu_delay_ /
// _io_delay_ queues of partha_aggr_task_state (server/gy_mconnhdlr.cc:10020-10065; entries with a zero metric never enter)
__global__ void topn_task_score_kernel(DevState st, uint32_t ntasks, int metric, unsigned long long *__restrict__ keys, unsigned long long *d_n)
{
	const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot == 0) *d_n = ntasks;
	if (slot >= ntasks) return;
	unsigned long long score = st.task_slot_id[slot] ? (unsigned long long)st.task_last[(size_t)slot * 3 + metric].sum : 0ull;
	if ((long long)score < 0) score = 0;
	if (score > 0xFFFFFFFFull) score = 0xFFFFFFFFull;
	keys[slot] = (score << 32) | slot;
}

// the want best of the sorted keys, with the id and host of their slots (services' or processes'; logical services: host 0); with
// slots != nullptr also the slot (index) of each entry, 0 past the end of the keys
__global__ void topn_pick_kernel(const unsigned long long *__restrict__ slot_id, const uint32_t *__restrict__ slot_host,
		const unsigned long long *__restrict__ sorted, uint32_t nslots, uint32_t want, gysk_topn_entry *__restrict__ out,
		unsigned long long *__restrict__ slots)
{
	const uint32_t i = threadIdx.x;
	if (i >= want) return;
	gysk_topn_entry o; o.glob_id = 0; o.score = 0; o.host_idx = 0; o.pad = 0;
	uint32_t slot = 0;
	if (i < nslots) {
		const unsigned long long k = sorted[nslots - 1 - i];		// descending
		slot = (uint32_t)k;
		o.glob_id = slot_id[slot]; o.score = k >> 32; o.host_idx = slot_host ? slot_host[slot] : 0u;
	}
	out[i] = o;
	if (slots) slots[i] = slot;
}

int launch_topn_pick(const SortTemp &tmp, const unsigned long long *d_n, uint32_t nkeys, const unsigned long long *ids, const uint32_t *hosts,
		uint32_t want, gysk_topn_entry *d_out, cudaStream_t s, unsigned long long *d_slots)
{
	int which = 0;
	const int sorted = launch_radix_sort(tmp, d_n, nkeys, 32, 64, &which, s);
	if (sorted < 0) return sorted;
	topn_pick_kernel<<<1, 64, 0, s>>>(ids, hosts, which ? tmp.keys_b : tmp.keys_a, nkeys, want, d_out, d_slots);
	return sorted + 1;
}

int launch_topn(const DevState &st, const SortTemp &tmp, uint32_t nslots, int is_task, int metric, int host_filter, uint32_t want,
		gysk_topn_entry *d_out, cudaStream_t s, unsigned long long *d_slots)
{
	if (!nslots) return 0;
	unsigned long long *d_n = st.counters + CTR_NKEYS;
	if (is_task) topn_task_score_kernel<<<div_up(nslots, 256), 256, 0, s>>>(st, nslots, metric, tmp.keys_a, d_n);
	else topn_score_kernel<<<div_up(nslots, 256), 256, 0, s>>>(st, nslots, metric, host_filter, tmp.keys_a, d_n);
	const int picked = launch_topn_pick(tmp, d_n, nslots, is_task ? st.task_slot_id : st.slot_id, is_task ? st.task_slot_host : st.slot_host,
			want, d_out, s, d_slots);
	return picked < 0 ? picked : 1 + picked;
}

// ---------------------------------------------------------------------------------------------------
// GYSK_FLAG_FLOW_TOPK: the heaviest-flow set of one table after a batch (or the merge's union): the candidates sorted by key, each
// distinct one scored, the rank keys sorted by score, the K best read from the end
// ---------------------------------------------------------------------------------------------------
// The rank key of candidate i of the *d_n sorted keys: a distinct key (not equal to its predecessor) is {score : 32 | 1 : 1 | i : 31},
// a repeat only i, below every distinct key. It goes to position n - 1 - i, so the stable sort by bits [31, 64) leaves a larger key
// before a smaller one of equal score, and the read from the end takes the smaller key first.
__global__ void __launch_bounds__(256) topk_score_kernel(const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ d_n,
		const unsigned long long *__restrict__ tbl, uint32_t depth, uint32_t log2w, int half, unsigned long long *__restrict__ rank)
{
	const uint64_t n = *d_n;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const unsigned long long k = keys[i];
		unsigned long long r = i;
		if (i == 0 || keys[i - 1] != k) {
			uint32_t lo, hi;
			cms_point(tbl, depth, log2w, k, lo, hi);
			r |= ((unsigned long long)(half ? hi : lo) << 32) | (1ull << 31);
		}
		rank[n - 1 - i] = r;
	}
}

// GYSK_FLAG_FLOW_TOPK_SLOW: the same rank keys scored by the slow score on a response histogram table (a sibling, so that
// topk_score_kernel keeps its code)
__global__ void __launch_bounds__(256) topk_slow_score_kernel(const unsigned long long *__restrict__ keys, const unsigned long long *__restrict__ d_n,
		const unsigned long long *__restrict__ tbl, uint32_t depth, uint32_t log2w, uint32_t b_slow, unsigned long long *__restrict__ rank)
{
	const uint64_t n = *d_n;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const unsigned long long k = keys[i];
		unsigned long long r = i;
		if (i == 0 || keys[i - 1] != k) r |= ((unsigned long long)resp_slow_score(tbl, depth, log2w, k, b_slow) << 32) | (1ull << 31);
		rank[n - 1 - i] = r;
	}
}

// the K best of the sorted rank keys into set (word 0 its size, then the keys, 0 past the size): the distinct keys are a suffix
__global__ void __launch_bounds__(256) topk_pick_kernel(const unsigned long long *__restrict__ rank, const unsigned long long *__restrict__ d_n,
		const unsigned long long *__restrict__ keys, unsigned long long *__restrict__ set)
{
	const uint64_t n = *d_n;
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= TOPK_K) return;
	auto valid = [&](uint64_t q) { return q < n && ((rank[n - 1 - q] >> 31) & 1ull); };
	const bool v = valid(j);
	set[2 + j] = v ? keys[rank[n - 1 - j] & 0x7FFFFFFFull] : 0ull;
	if (v && (j + 1 == TOPK_K || !valid(j + 1))) set[0] = j + 1;
	if (j == 0) { if (!v) set[0] = 0; set[1] = 0; }
}

int launch_topk_select(const SortTemp &tmp, const TopkList &l, uint64_t n_max, const unsigned long long *tbl, uint32_t depth, uint32_t log2w,
		int score, unsigned long long *set, bool reseed, cudaStream_t s)
{
	// three buffers of at least n_max keys: the candidates, and tmp's two; the key sort ping-pongs between the first two, the rank sort
	// between the two the sorted keys leave free
	unsigned long long *buf[3] = {l.keys, tmp.keys_a, tmp.keys_b};
	SortTemp t = tmp;
	t.keys_a = buf[0]; t.keys_b = buf[1];
	int which = 0;
	const int n1 = launch_radix_sort(t, l.n, n_max, 0, 64, &which, s);
	if (n1 < 0) return -1;
	const unsigned long long *sorted = buf[which];
	t.keys_a = buf[which ^ 1]; t.keys_b = buf[2];
	const uint32_t grid = std::min<uint32_t>(div_up(n_max, 256), (uint32_t)sm_count(current_device()) * 8u);
	if (score & TOPK_SCORE_SLOW) topk_slow_score_kernel<<<grid ? grid : 1, 256, 0, s>>>(sorted, l.n, tbl, depth, log2w, score & 0xFF, t.keys_a);
	else topk_score_kernel<<<grid ? grid : 1, 256, 0, s>>>(sorted, l.n, tbl, depth, log2w, score, t.keys_a);
	const unsigned long long *ranked[2] = {t.keys_a, t.keys_b};
	const int n2 = launch_radix_sort(t, l.n, n_max, 31, 64, &which, s);
	if (n2 < 0) return -1;
	topk_pick_kernel<<<div_up(TOPK_K, 256), 256, 0, s>>>(ranked[which], l.n, sorted, set);
	if (reseed) {		// the set opens the next batch's candidates
		cudaMemcpyAsync(l.keys, set + 2, (size_t)TOPK_K * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s);
		cudaMemcpyAsync(l.n, set, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s);
	}
	return n1 + n2 + 2;
}

// one CTA per rank: the size-word-counted keys of its set appended to l
__global__ void __launch_bounds__(256) topk_gather_kernel(const unsigned long long *__restrict__ sets, size_t stride, TopkList l)
{
	const unsigned long long *set = sets + blockIdx.x * stride;
	const uint32_t m = (uint32_t)min(set[0], (unsigned long long)TOPK_K);
	__shared__ unsigned long long base;
	if (threadIdx.x == 0) base = atomicAdd(l.n, (unsigned long long)m);
	__syncthreads();
	for (uint32_t j = threadIdx.x; j < m; j += blockDim.x) l.keys[base + j] = set[2 + j];
}

int launch_topk_gather(const unsigned long long *sets, uint32_t world, size_t stride, const TopkList &l, cudaStream_t s)
{
	cudaMemsetAsync(l.n, 0, sizeof(unsigned long long), s);
	topk_gather_kernel<<<world, 256, 0, s>>>(sets, stride, l);
	return 1;
}

// GYSK_FLAG_FLOW_TOPK_5MIN: one CTA per bit of mask, the set of a set bit appended to l as topk_gather_kernel does (a sibling, so that
// the merge's gather keeps its code)
__global__ void __launch_bounds__(256) topk_gather_mask_kernel(const unsigned long long *__restrict__ sets, size_t stride, uint32_t mask, TopkList l)
{
	if (!((mask >> blockIdx.x) & 1u)) return;
	const unsigned long long *set = sets + blockIdx.x * stride;
	const uint32_t m = (uint32_t)min(set[0], (unsigned long long)TOPK_K);
	__shared__ unsigned long long base;
	if (threadIdx.x == 0) base = atomicAdd(l.n, (unsigned long long)m);
	__syncthreads();
	for (uint32_t j = threadIdx.x; j < m; j += blockDim.x) l.keys[base + j] = set[2 + j];
}

int launch_topk_gather_mask(const unsigned long long *sets, size_t stride, uint32_t mask, const TopkList &l, bool reset, cudaStream_t s)
{
	if (reset) cudaMemsetAsync(l.n, 0, sizeof(unsigned long long), s);
	if (!mask) return 0;
	topk_gather_mask_kernel<<<32 - __builtin_clz(mask), 256, 0, s>>>(sets, stride, mask, l);
	return 1;
}

// GYSK_FLAG_FLOW_TOPK_5MIN: the bound word of launch_topk_bound, one thread (a set's K-th key and at most world terms)
__global__ void topk_bound_kernel(const unsigned long long *__restrict__ set, const unsigned long long *__restrict__ tbl, uint32_t depth,
		uint32_t log2w, int half, const unsigned long long *terms, size_t stride, uint32_t nterms, uint32_t mask, int sum,
		unsigned long long *out)
{
	unsigned long long thr = 0, t = 0;
	if (set[0] >= TOPK_K) {
		uint32_t lo, hi;
		cms_point(tbl, depth, log2w, set[2 + TOPK_K - 1], lo, hi);
		thr = half ? hi : lo;
	}
	for (uint32_t j = 0; j < nterms; ++j) if ((mask >> (j & 31u)) & 1u) t += terms[j * stride];
	*out = sum ? thr + t : max(thr, t);
}

// GYSK_FLAG_FLOW_TOPK_SLOW: the same with thr(set) the slow score on a response histogram table (a sibling, so that topk_bound_kernel
// keeps its code)
__global__ void topk_slow_bound_kernel(const unsigned long long *__restrict__ set, const unsigned long long *__restrict__ tbl, uint32_t depth,
		uint32_t log2w, uint32_t b_slow, const unsigned long long *terms, size_t stride, uint32_t nterms, uint32_t mask, int sum,
		unsigned long long *out)
{
	unsigned long long t = 0;
	const unsigned long long thr = set[0] >= TOPK_K ? resp_slow_score(tbl, depth, log2w, set[2 + TOPK_K - 1], b_slow) : 0;
	for (uint32_t j = 0; j < nterms; ++j) if ((mask >> (j & 31u)) & 1u) t += terms[j * stride];
	*out = sum ? thr + t : max(thr, t);
}

int launch_topk_bound(const unsigned long long *set, const unsigned long long *tbl, uint32_t depth, uint32_t log2w, int score,
		const unsigned long long *terms, size_t stride, uint32_t nterms, uint32_t mask, bool sum, unsigned long long *out, cudaStream_t s)
{
	if (score & TOPK_SCORE_SLOW) topk_slow_bound_kernel<<<1, 1, 0, s>>>(set, tbl, depth, log2w, score & 0xFF, terms, stride, nterms, mask, sum ? 1 : 0, out);
	else topk_bound_kernel<<<1, 1, 0, s>>>(set, tbl, depth, log2w, score, terms, stride, nterms, mask, sum ? 1 : 0, out);
	return 1;
}

// per-task window of the three MTASK_HIST histograms: totals now minus totals at the previous flush (nothing on the ingest path).
// With idle_secs, the process eviction (MCONN_HANDLER::cleanup_partha_unused_aggr_tasks, server/gy_mconnhdlr.cc:16492-16541: a MAGGR_TASK
// whose last_tusec_ is older than 30 min goes): the thread of a live slot's first histogram stamps the slot with tsec when the window
// it closes holds samples (every sample adds to all three histograms) or the slot has no stamp yet, and lists it when its stamp
// + idle_secs < tsec.
__global__ void task_flush_kernel(DevState st, uint32_t max_tasks, uint32_t tsec, uint32_t idle_secs)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;		// (task, histogram)
	if (i >= max_tasks * 3u) return;
	const HistCell *h = st.task_hist + (size_t)i * HIST_CELLS;
	HistCell tot {0, 0};
	for (int b = 0; b < HIST_MAX_CELL; ++b) { tot.count += h[b].count; tot.sum += h[b].sum; }
	const HistCell prev = st.task_prev[i];
	const HistCell last {tot.count - prev.count, tot.sum - prev.sum};
	st.task_last[i] = last;
	st.task_prev[i] = tot;

	const uint32_t slot = i / 3u;
	if (!idle_secs || i % 3u || !st.task_slot_id[slot]) return;
	uint32_t t = st.task_last_active[slot];
	if (last.count || !t) { t = tsec ? tsec : 1u; st.task_last_active[slot] = t; }
	if ((uint64_t)t + idle_secs < tsec) {
		const unsigned long long k = atomicAdd(st.counters + CTR_TASK_NEVICT, 1ull);
		st.task_evict_list[k] = slot;
		st.task_evict_ids[k] = st.task_slot_id[slot];
	}
}

int launch_task_flush(const DevState &st, uint32_t max_tasks, uint32_t tsec, uint32_t idle_secs, unsigned long long *host_ids, cudaStream_t s)
{
	if (idle_secs) cudaMemsetAsync(st.counters + CTR_TASK_NEVICT, 0, sizeof(unsigned long long), s);
	task_flush_kernel<<<div_up((uint64_t)max_tasks * 3, 256), 256, 0, s>>>(st, max_tasks, tsec, idle_secs);
	if (!idle_secs) return 1;
	evict_kernel<<<296, 256, 0, s>>>(st, st.task_tbl, st.task_evict_list, st.task_evict_ids, st.counters + CTR_TASK_NEVICT, nullptr, host_ids,
			TaskSlotReset {});
	return 2;
}

int launch_flush(const DevState &st, const ClientLevels &cl, const SvcTopClients &tc, uint32_t nslots, uint32_t tsec, uint32_t idle_secs,
		cudaStream_t s)
{
	if (!nslots) return 0;
	cudaMemsetAsync(st.counters + CTR_NEVICT, 0, sizeof(unsigned long long), s);
	flush_kernel<<<div_up((uint64_t)nslots * HIST_CELLS, 256), 256, 0, s>>>(st, nslots, tsec, idle_secs);
	state_kernel<<<div_up(nslots, 128), 128, 0, s>>>(st, nslots, tsec);
	if (!idle_secs) return 2;
	if (tc.open && cl.open) evict_kernel<<<296, 256, 0, s>>>(st, st.svc_tbl, st.evict_list, st.evict_ids, st.counters + CTR_NEVICT,
			st.counters + CTR_EVICTED_TOTAL, nullptr, SvcTopcSlotReset<SvcClientSlotReset> {tc, SvcClientSlotReset {cl}});
	else if (tc.open) evict_kernel<<<296, 256, 0, s>>>(st, st.svc_tbl, st.evict_list, st.evict_ids, st.counters + CTR_NEVICT,
			st.counters + CTR_EVICTED_TOTAL, nullptr, SvcTopcSlotReset<SvcSlotReset> {tc, SvcSlotReset {}});
	else if (cl.open) evict_kernel<<<296, 256, 0, s>>>(st, st.svc_tbl, st.evict_list, st.evict_ids, st.counters + CTR_NEVICT, st.counters + CTR_EVICTED_TOTAL,
			nullptr, SvcClientSlotReset {cl});
	else evict_kernel<<<296, 256, 0, s>>>(st, st.svc_tbl, st.evict_list, st.evict_ids, st.counters + CTR_NEVICT, st.counters + CTR_EVICTED_TOTAL, nullptr,
			SvcSlotReset {});		// grid-stride over the (device-side) eviction list
	return 3;
}

int launch_rebuild_table(const IdTable &t, uint32_t nslots, cudaStream_t s)
{
	cudaMemsetAsync(t.ent, 0, ((size_t)t.mask + 1) * sizeof(TblEntry), s);
	rebuild_table_kernel<<<div_up(nslots, 256), 256, 0, s>>>(t, nslots);
	return 1;
}

int launch_gather_svcs(const DevState &st, const unsigned long long *d_ids, uint32_t n, SvcRaw *d_out, cudaStream_t s)
{
	if (!n) return 0;
	gather_svcs_kernel<<<div_up(n, 4), 128, 0, s>>>(st, d_ids, n, d_out);
	return 1;
}

int launch_gather_tasks(const DevState &st, const unsigned long long *d_ids, uint32_t n, TaskRaw *d_out, cudaStream_t s)
{
	if (!n) return 0;
	gather_tasks_kernel<<<div_up(n, 4), 128, 0, s>>>(st, d_ids, n, d_out);
	return 1;
}

int launch_gather_hll(const DevState &st, const unsigned long long *d_ids, int32_t *found, uint8_t *d_out, cudaStream_t s)
{
	gather_hll_kernel<<<1, 256, 0, s>>>(st, d_ids, found, d_out);
	return 1;
}

int launch_gather_hll_window(const DevState &st, const uint8_t *regs, const unsigned long long *d_ids, int32_t *found, uint8_t *d_out, cudaStream_t s)
{
	gather_hll_kernel<<<1, 256, 0, s>>>(st, d_ids, found, d_out, regs);
	return 1;
}

int launch_client_rows(const DevState &st, const ClientLevels &cl, const unsigned long long *d_ids, const unsigned long long *d_slots, uint32_t n,
		gysk_svc_clients *d_out, cudaStream_t s)
{
	if (!n) return 0;
	client_rows_kernel<<<div_up(n, CL_WARPS), CL_WARPS * 32, 0, s>>>(st, cl, d_ids, d_slots, n, d_out);
	return 1;
}

int launch_client_roll(const ClientLevels &cl, uint32_t nslots, const LevelRing &lv, cudaStream_t s)
{
	if (!nslots) return 0;
	const uint64_t npiece = (uint64_t)nslots * (CL_REGS / 16);
	client_roll_kernel<<<(uint32_t)std::min<uint64_t>(div_up(npiece, 256), (uint64_t)sm_count(current_device()) * 8), 256, 0, s>>>(cl, nslots,
			lv.cur[0], lv.live[0], lv.fresh & 1u);
	return 1;
}

int launch_query_flows(const unsigned long long *tbl, uint32_t depth, uint32_t log2w, const unsigned long long *d_keys, uint32_t n, gysk_flow_est *d_out,
		cudaStream_t s)
{
	if (!n) return 0;
	query_flows_kernel<<<div_up(n, 256), 256, 0, s>>>(tbl, depth, log2w, d_keys, n, d_out);
	return 1;
}

int launch_query_flow_resp(const unsigned long long *tbl, uint32_t depth, uint32_t log2w, const unsigned long long *d_keys, uint32_t n,
		gysk_flow_resp_est *d_out, cudaStream_t s)
{
	if (!n) return 0;
	query_flow_resp_kernel<<<div_up(n, 128), 128, 0, s>>>(tbl, depth, log2w, d_keys, n, d_out);
	return 1;
}

int launch_cms_level_roll(const unsigned long long *cur, unsigned long long *ring, unsigned long long *level, size_t cells, const LevelRing &lv,
		cudaStream_t s)
{
	const uint64_t npair = cells / 2;		// log2w >= 4: whole pairs
	const uint32_t grid = std::min<uint32_t>(div_up(npair, 256), (uint32_t)sm_count(current_device()) * 8u);
	cms_level_roll_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const ulonglong2 *>(cur), reinterpret_cast<ulonglong2 *>(ring),
			reinterpret_cast<ulonglong2 *>(level), npair, lv.cur[0], lv.live[0], lv.fresh & 1u);
	return 1;
}

int launch_window_list(const DevState &st, const SortTemp &tmp, uint32_t nslots, int is_task, int host_filter, uint32_t active_only,
		uint32_t active_mark, uint32_t seen_before, unsigned long long *d_n, bool order, const unsigned long long **keys, const unsigned long long **ids,
		cudaStream_t s)
{
	cudaMemsetAsync(d_n, 0, sizeof(unsigned long long), s);
	*keys = tmp.keys_a; *ids = tmp.keys_b;
	if (!nslots) return 0;
	window_select_kernel<<<div_up(nslots, 256), 256, 0, s>>>(st, nslots, is_task, host_filter, active_only, active_mark, seen_before, tmp.keys_a, d_n);
	if (!order) return 1;
	int which = 0;
	const int sorted = launch_radix_sort(tmp, d_n, nslots, 32, 64, &which, s);
	if (sorted < 0) return sorted;
	*keys = which ? tmp.keys_b : tmp.keys_a; *ids = which ? tmp.keys_a : tmp.keys_b;
	window_ids_kernel<<<div_up(nslots, 256), 256, 0, s>>>(st, is_task, *keys, d_n, const_cast<unsigned long long *>(*ids));
	return 2 + sorted;
}

int launch_svc_summaries(const DevState &st, const unsigned long long *d_ids, const unsigned long long *d_slots, uint32_t n, gysk_svc_summary *d_out,
		cudaStream_t s)
{
	if (!n) return 0;
	svc_summary_kernel<<<div_up(n, SUMM_WARPS), SUMM_WARPS * 32, 0, s>>>(st, d_ids, d_slots, n, d_out);
	return 1;
}

int launch_task_summaries(const DevState &st, const unsigned long long *d_ids, const unsigned long long *d_slots, uint32_t n, gysk_task_summary *d_out,
		cudaStream_t s)
{
	if (!n) return 0;
	task_summary_kernel<<<div_up(n, 4), 128, 0, s>>>(st, d_ids, d_slots, n, d_out);
	return 1;
}

int launch_day_stats(const DevState &st, const unsigned long long *d_slots, uint32_t n, gysk_listener_day_stats *d_out, cudaStream_t s)
{
	if (!n) return 0;
	day_stats_kernel<<<div_up(n, DAY_WARPS), DAY_WARPS * 32, 0, s>>>(st, d_slots, n, d_out);
	return 1;
}

int launch_host_listen_count(const DevState &st, const unsigned long long *keys, const unsigned long long *d_n, uint32_t n, uint32_t active_mark,
		unsigned long long *acc, cudaStream_t s)
{
	if (!n) return 0;
	cudaMemsetAsync(acc, 0, (size_t)n * sizeof(unsigned long long), s);
	host_listen_count_kernel<<<div_up(n, 256), 256, 0, s>>>(st, keys, d_n, active_mark, acc);
	return 1;
}

int launch_host_listen_rows(const unsigned long long *keys, const unsigned long long *d_n, const unsigned long long *acc, uint32_t rlo, uint32_t cap,
		gysk_host_listen *d_out, unsigned long long *d_rows, cudaStream_t s)
{
	host_listen_rows_kernel<<<1, 1024, 0, s>>>(keys, d_n, acc, rlo, cap, d_out, d_rows);
	return 1;
}

// ---------------------------------------------------------------------------------------------------
// trace rows: window roll, reads
// ---------------------------------------------------------------------------------------------------
// gysk_flush: the half that becomes the open window, cleared in every row handed out (its centroids are dead behind n = 0)
__global__ void trace_roll_kernel(TraceTable tr, uint32_t open, uint32_t nrows)
{
	const uint64_t nw = (uint64_t)nrows * TRACE_WORDS;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nw; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t r = (uint32_t)(i / TRACE_WORDS), w = (uint32_t)(i % TRACE_WORDS);
		tr.words(open, r)[w] = 0ull;
		if (w == 0) { TdHead z; z.total = 0; z.minv = INFINITY; z.maxv = -INFINITY; z.n = 0; z.pad = 0; *tr.hd(open, r) = z; }
	}
}

// one window of a row as gysk_trace_window
__device__ __forceinline__ void trace_window_out(const TraceTable &tr, uint32_t half, uint32_t r, gysk_trace_window &o)
{
	const unsigned long long *w = tr.words(half, r);
	o.nreq = w[TW_NREQ]; o.nerr = w[TW_NERR]; o.nconns = w[TW_NCONNS];
	o.sum_resp_us = w[TW_SUM_US]; o.max_resp_us = w[TW_MAX_US];
	o.bytes_in = w[TW_BYTES_IN]; o.bytes_out = w[TW_BYTES_OUT]; o.max_bytes_in = w[TW_MAX_IN]; o.max_bytes_out = w[TW_MAX_OUT];
	for (int b = 0; b < 8; ++b) o.resp_buckets[b] = w[TW_BKT + b];
	const TdHead h = *tr.hd(half, r);
	o.td_count = h.total;
	o.p99_resp_us = h.n ? td_quantile_seq(TdCentroids {tr.cents(half, r)}, h.n, (double)(0xFFFFFFFFu - (uint32_t)w[TW_TD_NMIN]), (double)w[TW_TD_MAX], 0.99)
			: (double)NAN;
}

// one thread per row: by id (ids: the service table's lookup, then the slot's row) or by row (rows)
__global__ void trace_rows_kernel(DevState st, const unsigned long long *__restrict__ ids, const unsigned long long *__restrict__ rows, uint32_t n,
		gysk_trace_row *__restrict__ out)
{
	const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= n) return;
	gysk_trace_row o;
	memset(&o, 0, sizeof(o));
	int r = -1, slot = -1;
	if (ids) {
		const unsigned long long id = ids[q];
		o.glob_id = id;
		slot = id + 1ull > 1ull ? table_lookup(st.svc_tbl, id, false) : -1;
		if (slot >= 0) { const uint32_t r1 = st.trace.row_of[slot]; if (r1 != 0 && r1 != TRACE_BUSY) r = (int)(r1 - 1u); }
	}
	else {
		r = (int)rows[q];
		slot = (int)st.trace.row_slot[r];
		o.glob_id = st.slot_id[slot];
	}
	if (r >= 0) {
		o.found = 1;
		o.host_idx = st.slot_host[slot];
		trace_window_out(st.trace, st.trace.par, (uint32_t)r, o.cur);
		trace_window_out(st.trace, st.trace.par ^ 1u, (uint32_t)r, o.last);
	}
	out[q] = o;
}

__global__ void trace_list_kernel(DevState st, uint32_t nrows, int host_filter, uint32_t active_only, unsigned long long *__restrict__ ids,
		unsigned long long *__restrict__ rows, unsigned long long *d_n)
{
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	bool keep = false;
	uint32_t slot = 0;
	if (r < nrows) {
		slot = st.trace.row_slot[r];
		keep = slot != ~0u && (host_filter < 0 || st.slot_host[slot] == (uint32_t)host_filter) &&
				(!active_only || st.trace.words(st.trace.par ^ 1u, r)[TW_NREQ] != 0);
	}
	const uint32_t m = __ballot_sync(0xffffffffu, keep);
	unsigned long long base = 0;
	if ((threadIdx.x & 31) == 0 && m) base = atomicAdd(d_n, (unsigned long long)__popc(m));
	base = __shfl_sync(0xffffffffu, base, 0);
	if (keep) {
		const unsigned long long i = base + __popc(m & ((1u << (threadIdx.x & 31)) - 1u));
		ids[i] = st.slot_id[slot]; rows[i] = r;
	}
}

// one id's digest of one window, by one warp
__global__ void gather_trace_kernel(DevState st, const unsigned long long *__restrict__ d_id, int last_window, TraceRaw *__restrict__ out)
{
	const int lane = threadIdx.x & 31;
	const unsigned long long id = *d_id;
	int r = -1;
	if (id + 1ull > 1ull) {
		const int slot = table_lookup(st.svc_tbl, id, false);
		if (slot >= 0) { const uint32_t r1 = st.trace.row_of[slot]; if (r1 != 0 && r1 != TRACE_BUSY) r = (int)(r1 - 1u); }
	}
	if (r < 0) { if (lane == 0) out->found = 0; return; }
	const uint32_t half = st.trace.par ^ (last_window ? 1u : 0u);
	const TdHead h = *st.trace.hd(half, (uint32_t)r);
	const Centroid *c = st.trace.cents(half, (uint32_t)r);
	for (uint32_t i = lane; i < h.n; i += 32) out->cent[i] = c[i];
	if (lane == 0) {
		const unsigned long long *w = st.trace.words(half, (uint32_t)r);
		out->found = 1; out->n = h.n; out->total = h.total;
		out->minv = h.n ? (double)(0xFFFFFFFFu - (uint32_t)w[TW_TD_NMIN]) : INFINITY;
		out->maxv = h.n ? (double)w[TW_TD_MAX] : -INFINITY;
	}
}

int launch_trace_roll(const DevState &st, uint32_t open, uint32_t nrows, cudaStream_t s)
{
	if (!nrows) return 0;
	const uint32_t grid = std::min<uint32_t>(div_up((uint64_t)nrows * TRACE_WORDS, 256), (uint32_t)sm_count(current_device()) * 8u);
	trace_roll_kernel<<<grid, 256, 0, s>>>(st.trace, open, nrows);
	return 1;
}

int launch_trace_rows(const DevState &st, const unsigned long long *d_ids, const unsigned long long *d_rows, uint32_t n, gysk_trace_row *d_out, cudaStream_t s)
{
	if (!n) return 0;
	trace_rows_kernel<<<div_up(n, 128), 128, 0, s>>>(st, d_ids, d_rows, n, d_out);
	return 1;
}

int launch_trace_list(const DevState &st, uint32_t nrows, int host_filter, uint32_t active_only, unsigned long long *ids, unsigned long long *rows,
		unsigned long long *d_n, cudaStream_t s)
{
	cudaMemsetAsync(d_n, 0, sizeof(unsigned long long), s);
	if (!nrows) return 0;
	trace_list_kernel<<<div_up(nrows, 256), 256, 0, s>>>(st, nrows, host_filter, active_only, ids, rows, d_n);
	return 1;
}

int launch_gather_trace(const DevState &st, const unsigned long long *d_id, int last_window, TraceRaw *d_out, cudaStream_t s)
{
	gather_trace_kernel<<<1, 32, 0, s>>>(st, d_id, last_window, d_out);
	return 1;
}

// ---------------------------------------------------------------------------------------------------
// GYSK_FLAG_SVC_TOP_CLIENTS: each service's heaviest clients by kbytes, weighted Misra-Gries in its mergeable form (DESIGN.md §2).
// A batch: topc_pairs_kernel sums the connection records per (service, client) in the pair table, the claimed entries are sorted by
// service, and each service's segment is merged into its open summary, a long segment in pieces of TOPC_PIECE pairs, one warp each,
// whose K + 1 best the service's warp merges (the union's K + 1 best lie among them). A flush: topc_roll_kernel.
// ---------------------------------------------------------------------------------------------------
static constexpr int TOPC_WARPS = 4;

__device__ __forceinline__ uint32_t topc_hash(uint32_t slot, unsigned long long fk)
{
	return table_hash(fk ^ ((unsigned long long)(slot + 1u) * 0xC2B2AE3D27D4EB4Full));
}

// one warp per record region (grid-stride): each connection record (every TCP record but the QRY_REC response samples, the records of
// the service's exact cell) adds {kbytes, 1} to the entry of its (service, client) pair. The record that claims an entry with the 128-bit
// CAS appends the sort key {slot : 32 | entry}. The table holds at least 2 x max_batch entries, so a probe always ends.
__global__ void __launch_bounds__(256) topc_pairs_kernel(const uint4 *__restrict__ q, const uint2 *__restrict__ cnt, RecRegions rr, SvcTopClients tc,
		unsigned long long *__restrict__ keys)
{
	const int lane = threadIdx.x & 31;
	const IngestRec *recs = reinterpret_cast<const IngestRec *>(q);
	for (uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rr.nwarps; r += (gridDim.x * blockDim.x) >> 5) {
		const uint32_t m = cnt[r].x;
		for (uint32_t i = lane; i < m; i += 32) {
			const IngestRec rec = ld_rec(recs + (unsigned long long)r * rr.cap + i);
			if (rec.slot == QRY_REC) continue;
			const ulonglong2 want = make_ulonglong2(rec.flow_key, (unsigned long long)rec.slot + 1ull);
			uint32_t pos = topc_hash(rec.slot, rec.flow_key) & tc.pmask;
			for (;;) {
				ulonglong2 k = __ldcg(tc.pkey + pos);
				if (!k.y) {
					k = atomicCAS(tc.pkey + pos, make_ulonglong2(0ull, 0ull), want);
					if (!k.y) {
						keys[atomicAdd(tc.cnt, 1ull)] = ((unsigned long long)rec.slot << 32) | pos;
						break;
					}
				}
				if (k.x == want.x && k.y == want.y) break;
				pos = (pos + 1u) & tc.pmask;
			}
			atomicAdd(&tc.pacc[pos].x, (unsigned long long)(rec.value >> 10));
			atomicAdd(&tc.pacc[pos].y, 1ull);
		}
	}
}

// one thread per sorted key: the first key of each service's run appends its segment {begin, end, slot, first piece}; a segment of more
// than TOPC_PIECE pairs takes ceil(len / TOPC_PIECE) pieces
__global__ void __launch_bounds__(256) topc_segs_kernel(const unsigned long long *__restrict__ keys, SvcTopClients tc, uint4 *__restrict__ segs)
{
	const uint32_t n = (uint32_t)tc.cnt[0], i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t slot = (uint32_t)(keys[i] >> 32);
	if (i && (uint32_t)(keys[i - 1] >> 32) == slot) return;
	uint32_t lo = i + 1, hi = n;
	while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((uint32_t)(keys[mid] >> 32) == slot) lo = mid + 1; else hi = mid; }
	uint32_t base = 0;
	if (lo - i > TOPC_PIECE) {
		const uint32_t np = (lo - i + TOPC_PIECE - 1) / TOPC_PIECE;
		base = (uint32_t)atomicAdd(tc.cnt + 2, (unsigned long long)np);
		for (uint32_t j = 0; j < np; ++j) {
			TopcPiece &p = tc.pieces[base + j];
			p.beg = i + j * TOPC_PIECE; p.end = min(lo, i + (j + 1) * TOPC_PIECE); p.slot = slot;
		}
	}
	segs[atomicAdd(tc.cnt + 1, 1ull)] = make_uint4(i, lo, slot, base);
}

// the pairs of sorted keys [beg, end), one service's, each with the old entry of the same client added (old[0, nold) in shared memory;
// bit j of the returned mask for each old entry met), offered to the warp's list; each pair's entry emptied for the next batch
__device__ __forceinline__ uint32_t topc_take_pairs(const SvcTopClients &tc, const unsigned long long *__restrict__ keys, uint32_t beg, uint32_t end,
		const TopcCand *old, uint32_t nold, TopcCand *l, uint32_t &n, int lane)
{
	uint32_t matched = 0;
	for (uint32_t i0 = beg; i0 < end; i0 += 32) {
		const uint32_t i = i0 + (uint32_t)lane;
		TopcCand c {0ull, 0ull, 0ull};
		if (i < end) {
			const uint32_t pos = (uint32_t)keys[i];
			const ulonglong2 k = tc.pkey[pos], a = tc.pacc[pos];
			tc.pkey[pos] = make_ulonglong2(0ull, 0ull); tc.pacc[pos] = make_ulonglong2(0ull, 0ull);
			c = TopcCand {k.x, a.x, a.y};
			for (uint32_t j = 0; j < nold; ++j) {
				if (old[j].key != c.key) continue;
				c.kb += old[j].kb; c.conns += old[j].conns; matched |= 1u << j;
			}
		}
		topc_offer(l, n, c, c.kb != 0, lane);
	}
	return __reduce_or_sync(0xffffffffu, matched);
}

// one warp per piece of a long segment (grid-stride): its K + 1 best, and the old entries it met
__global__ void __launch_bounds__(TOPC_WARPS * 32) topc_piece_kernel(const unsigned long long *__restrict__ keys, SvcTopClients tc)
{
	__shared__ TopcCand list[TOPC_WARPS][TOPC_K + 1], old[TOPC_WARPS][TOPC_K];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t np = (uint32_t)tc.cnt[2];
	for (uint32_t p = blockIdx.x * TOPC_WARPS + wid; p < np; p += gridDim.x * TOPC_WARPS) {
		TopcPiece &pc = tc.pieces[p];
		const uint32_t nold = topc_gather(tc.open + pc.slot, old[wid], 0, lane);
		uint32_t n = 0;
		const uint32_t matched = topc_take_pairs(tc, keys, pc.beg, pc.end, old[wid], nold, list[wid], n, lane);
		if ((uint32_t)lane < n) pc.c[lane] = list[wid][lane];
		if (lane == 0) { pc.n = n; pc.matched = matched; }
		__syncwarp();
	}
}

// one warp per segment (grid-stride): the service's open summary merged with its batch sums, from the pairs themselves (a short segment)
// or from its pieces' lists, then the old entries no pair met
__global__ void __launch_bounds__(TOPC_WARPS * 32) topc_merge_kernel(const unsigned long long *__restrict__ keys, const uint4 *__restrict__ segs,
		SvcTopClients tc)
{
	__shared__ TopcCand list[TOPC_WARPS][TOPC_K + 1], old[TOPC_WARPS][TOPC_K];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t ns = (uint32_t)tc.cnt[1];
	for (uint32_t q = blockIdx.x * TOPC_WARPS + wid; q < ns; q += gridDim.x * TOPC_WARPS) {
		const uint4 sg = segs[q];
		TopcSet *set = tc.open + sg.z;
		const unsigned long long delta = set->delta;
		const uint32_t nold = topc_gather(set, old[wid], 0, lane);
		uint32_t n = 0, matched = 0;
		if (sg.y - sg.x <= TOPC_PIECE) matched = topc_take_pairs(tc, keys, sg.x, sg.y, old[wid], nold, list[wid], n, lane);
		else {
			const TopcPiece *pc = tc.pieces + sg.w, *pe = pc + (sg.y - sg.x + TOPC_PIECE - 1) / TOPC_PIECE;
			for (; pc < pe; ++pc) {
				const uint32_t pn = pc->n;
				matched |= pc->matched;
				TopcCand c {0ull, 0ull, 0ull};
				if ((uint32_t)lane < pn) c = pc->c[lane];
				topc_offer(list[wid], n, c, (uint32_t)lane < pn, lane);
			}
		}
		const bool left = (uint32_t)lane < nold && !((matched >> lane) & 1u);
		topc_offer(list[wid], n, left ? old[wid][lane] : TopcCand {0ull, 0ull, 0ull}, left, lane);
		topc_store(list[wid], n, delta, set, lane);
	}
}

// GYSK_FLAG_SVC_TOP_CLIENTS at a flush, one warp per service slot of [0, nslots) (grid-stride): ring slot k becomes the merge of the open
// summary and what it holds (the open summary alone when the flush started a new epoch there), then the level the merge of the live
// slots, slot k's new content included: the rule of client_roll_kernel with the summaries' merge for max
__global__ void __launch_bounds__(TOPC_WARPS * 32) topc_roll_kernel(SvcTopClients tc, uint32_t nslots, uint32_t k, uint32_t live, uint32_t fresh)
{
	__shared__ TopcCand buf[TOPC_WARPS][NSLOTS * TOPC_K], list[TOPC_WARPS][TOPC_K + 1];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	for (uint32_t slot = blockIdx.x * TOPC_WARPS + wid; slot < nslots; slot += gridDim.x * TOPC_WARPS) {
		const TopcSet *op = tc.open + slot;
		TopcSet *rk = tc.ring + (size_t)k * tc.stride + slot;
		unsigned long long delta = op->delta;
		uint32_t m = topc_gather(op, buf[wid], 0, lane);
		if (!fresh) { delta += rk->delta; m = topc_gather(rk, buf[wid], m, lane); }
		uint32_t n = 0;
		topc_offer_groups(buf[wid], m, list[wid], n, lane);
		topc_store(list[wid], n, delta, rk, lane);
		delta = 0; m = 0;
		for (uint32_t j = 0; j < NSLOTS; ++j) {
			if (!((live >> j) & 1u)) continue;
			const TopcSet *sj = tc.ring + (size_t)j * tc.stride + slot;
			delta += sj->delta;
			m = topc_gather(sj, buf[wid], m, lane);
		}
		n = 0;
		topc_offer_groups(buf[wid], m, list[wid], n, lane);
		topc_store(list[wid], n, delta, tc.level + slot, lane);
	}
}

// gysk_query_svc_top_clients / gysk_query_top_clients_window: one warp per row of summary array `sets`, by id (ids != nullptr: looked up,
// id 0 and unknown ids give found = 0 and a zero row) or by slot (the window read)
__global__ void __launch_bounds__(TOPC_WARPS * 32) topc_rows_kernel(DevState st, const TopcSet *__restrict__ sets, const unsigned long long *__restrict__ ids,
		const unsigned long long *__restrict__ slots, uint32_t n, gysk_svc_top_clients *__restrict__ out)
{
	const int lane = threadIdx.x & 31;
	const uint32_t q = blockIdx.x * TOPC_WARPS + (threadIdx.x >> 5);
	if (q >= n) return;
	const Resolved s = resolve_warp(st.svc_tbl, ids, slots, q, lane);
	gysk_topc_entry e {0ull, 0u, 0u};
	if (s.slot >= 0 && (uint32_t)lane < TOPC_K) e = sets[s.slot].ent[lane];
	if ((uint32_t)lane < TOPC_K) out[q].entries[lane] = e;
	const uint32_t held = (uint32_t)__popc(__ballot_sync(0xffffffffu, e.kbytes != 0));
	if (lane == 0) {
		out[q].glob_id = s.id; out[q].found = s.slot >= 0; out[q].n = held;
		out[q].delta = s.slot >= 0 ? sets[s.slot].delta : 0ull;
	}
}

int launch_topc_batch(const SortTemp &tmp, const SvcTopClients &tc, const RecRegions &rr, uint64_t n_events, uint32_t max_svcs, cudaStream_t s)
{
	if (!n_events) return 0;
	const int nsm = sm_count(current_device());
	cudaMemsetAsync(tc.cnt, 0, 3 * sizeof(unsigned long long), s);
	topc_pairs_kernel<<<nsm * 8, 256, 0, s>>>(tmp.recq, tmp.rec_cnt, rr, tc, tmp.keys_a);
	int slot_bits = 1;
	while ((1ull << slot_bits) < max_svcs) ++slot_bits;
	int which = 0;
	const int sorted = launch_radix_sort(tmp, tc.cnt, n_events, 32, 32 + slot_bits, &which, s);
	if (sorted < 0) return -1;
	const unsigned long long *keys = which ? tmp.keys_b : tmp.keys_a;
	topc_segs_kernel<<<div_up(n_events, 256), 256, 0, s>>>(keys, tc, tmp.segs);
	topc_piece_kernel<<<nsm * 8, TOPC_WARPS * 32, 0, s>>>(keys, tc);
	topc_merge_kernel<<<nsm * 16, TOPC_WARPS * 32, 0, s>>>(keys, tmp.segs, tc);
	return 5 + sorted;
}

int launch_topc_roll(const SvcTopClients &tc, uint32_t nslots, const LevelRing &lv, cudaStream_t s)
{
	if (!nslots) return 0;
	topc_roll_kernel<<<std::min<uint32_t>(div_up(nslots, TOPC_WARPS), (uint32_t)sm_count(current_device()) * 16u), TOPC_WARPS * 32, 0, s>>>(tc, nslots,
			lv.cur[0], lv.live[0], lv.fresh & 1u);
	return 1;
}

int launch_topc_rows(const DevState &st, const SvcTopClients &tc, int which, const unsigned long long *d_ids, const unsigned long long *d_slots,
		uint32_t n, gysk_svc_top_clients *d_out, cudaStream_t s)
{
	if (!n) return 0;
	const TopcSet *sets = which == GYSK_TOPC_OPEN ? tc.open : which == GYSK_TOPC_LAST ? tc.last : tc.level;
	topc_rows_kernel<<<div_up(n, TOPC_WARPS), TOPC_WARPS * 32, 0, s>>>(st, sets, d_ids, d_slots, n, d_out);
	return 1;
}

} // namespace gysk
