// gysk_device.cuh — device-side building blocks shared by the kernels of libgysketch.so (sm_90a only).
//
// Everything here is a from-scratch CUDA formulation of behaviour defined by the reference (citations are
// relative to the reference tree) or by the sketch definitions stated in DESIGN.md.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace gysk {

// ---------------------------------------------------------------------------------------------------
// HBM layout
// ---------------------------------------------------------------------------------------------------
// One histogram = 16 cells of {count u64, sum i64} = 256 B (two 128-B lines). Cells 0..14 are the buckets,
// byte-identical to HIST_SERIAL (common/gy_statistics.h:458); cell 15 holds {unused, max_val_seen_}.
struct HistCell { unsigned long long count; long long sum; };
static constexpr int HIST_CELLS = 16;
static constexpr int HIST_MAX_CELL = 15;

// service-id table entry: open addressing, 16 B so one 128-bit load fetches key and slot together
struct alignas(16) TblEntry { unsigned long long key; uint32_t slot1; uint32_t pad; };	// slot1 = slot + 1, 0 = not yet published
static constexpr uint32_t SLOT_INVALID = 0xFFFFFFFFu;

struct Centroid { double mean; unsigned long long weight; };
static constexpr int TD_CAP = 256;		// delta = 200 yields 200 ... 1.3 x 200 centroids (DESIGN.md §2)

// One log-linear value bin of one service for the batch being ingested (DESIGN.md §3):
//   cw += 1 | (usec % 1000) << 27        {samples : 27 | sum of the sub-millisecond remainders : 37}  — a batch holds < 2^27 events
//   us += usec
// so that the bin's exact msec sum (GY_HISTOGRAM::add_data adds usec / 1000 per sample) is (us - remainders) / 1000 and its mean
// us / samples. Bin index = td_code(usec) + RESP_TIME_HASH bucket of its msec value: both terms are monotone in usec, so the
// index is too and no bin straddles a histogram bucket. Two ways lead to the same numbers: the samples of most services travel as
// sort keys, sorted by slot and summed per bin of each service's segment (bins_merge_kernel, gysk_kernels.cu); a HOT service — one that brought at least
// hot_min samples in an earlier batch — owns a dense row of such bins (DevState::hot_rows, L2-resident; layout below) and
// every one of its samples is two 64-bit REDs into it, no key, no sort. The batch's merge kernel reads a row in order and zeroes it.
struct alignas(16) Bin { unsigned long long cw; unsigned long long us; };
static constexpr int NBINS = 848;				// 832 codes + 15 buckets, padded to a multiple of 16
static constexpr int BIN_CNT_BITS = 27;
static constexpr unsigned long long BIN_CNT_MASK = (1ull << BIN_CNT_BITS) - 1;
// A hot service's row: HOT_ROW_BINS words {samples | remainders} followed by HOT_ROW_BINS words of usec sums (the two REDs of a
// sample go to different lines), bin b at word hot_word(b) — the 32 x 32 transpose of the index, so that neighbouring bins, which
// fill up together around the mode of a service's response times, lie two 128-byte lines apart: same-line atomics are serialised
// in L2 and the fullest line of the busiest service is what the ingest kernel ends up waiting for.
static constexpr int HOT_ROW_BINS = 1024, HOT_ROW_WORDS = 2 * HOT_ROW_BINS;
static_assert(NBINS <= HOT_ROW_BINS, "a row holds every bin");
__host__ __device__ __forceinline__ uint32_t hot_word(uint32_t bin) { return ((bin & 31u) << 5) | (bin >> 5); }

// per-service counters beside the histograms: ACTIVE_CONN_STATS roll-up {active conns : 32 | kbytes : 32}, max rtt (float bits),
// API_TRAN error counters {client errors : 32 | server errors : 32}; cur = window being filled, last = last closed window
struct alignas(8) SlotAux { unsigned long long act_cur, act_last, err_cur, err_last; uint32_t rtt_cur, rtt_last; };

// per-service scratch of the batch being ingested: exact extremes of its RESP samples and "has bins to merge"
// hot = 1 + the service's row of DevState::hot_rows, 0 = its samples travel as sort keys (set by bins_merge_kernel, read by the next batch)
struct alignas(16) SlotBatch { uint32_t minv, maxv, touched, hot; };
// listener state of the last evaluated window (gysk_state.cuh): curr_state_, curr_issue_, issue_bit_hist_, high_resp_bit_hist_ and the
// active connection count last reported by an ACTIVE_CONN_STATS record (kept between the 15-s reports)
struct alignas(8) SlotState { uint8_t state, issue, issue_bits, high_bits; uint32_t nconn_active; };

// per-service t-digest header
struct TdHead { unsigned long long total; double minv, maxv; uint32_t n; uint32_t pad; };

struct IdTable
{
	TblEntry	*ent;
	uint32_t	mask;		// capacity - 1
	uint32_t	max_slots;
	uint32_t	*count;		// slots handed out so far
	unsigned long long *slot_id;	// optional: slot -> id
	uint32_t	*slot_host;	// optional: slot -> host index of the inserting event
	int32_t		*free_n;	// optional: number of recycled slots on the stack (pushed by the eviction kernel at a flush,
	uint32_t	*free_slots;	//           popped here; the two never run concurrently: same stream)
	unsigned long long *insert_fail;	// optional: entries left dead by a lost race for the last slot
};
static constexpr unsigned long long KEY_TOMBSTONE = ~0ull;	// table entry of an evicted id: never matches, never ends a probe chain

// device counters (index into Engine::d_counters). CTR_NKEYS is the sort-key cursor, which ingest_kernel bumps once per warp and
// key flush (about 160 K returning atomics per 100 M-event batch); the connection / process records need no cursor (SortTemp::recq).
enum { CTR_IN = 0, CTR_DROPPED, CTR_RESP, CTR_TCP, CTR_TASK, CTR_FOREIGN, CTR_NKEYS, CTR_INSERT_FAIL, CTR_NTOUCHED /* short key segments */,
	CTR_NLONG /* long key segments (batch rows) */, CTR_NEVICT, CTR_EVICTED_TOTAL,
	CTR_NHOT /* hot rows in use by the batch in flight */, CTR_NHOT_NEXT /* rows handed out so far */, CTR_NWINDOW /* rows of the last window read (or logical read / logical top-N) */,
	CTR_NHOSTS /* host rows of the last gysk_query_host_listen */, CTR_TASK_NEVICT /* processes evicted by the last flush */,
	CTR_FLOW_DIRECT /* connection records of the last batch whose count-min update bypassed the flow table */,
	CTR_FLOWQ_DIRECT /* response samples of the last batch whose flow query update bypassed its flow table (GYSK_FLAG_FLOW_QUERIES) */,
	CTR_FLOWR_DIRECT /* ... whose flow response histogram update bypassed its flow table (GYSK_FLAG_FLOW_RESP_HIST) */,
	CTR_FLOWE_DIRECT /* error samples of the last batch whose flow error update bypassed its flow table (GYSK_FLAG_FLOW_ERRORS) */, CTR_MAX };

// ---------------------------------------------------------------------------------------------------
// jhash: Bob Jenkins lookup2 in the form the reference uses (common/jhash.h:22-35,121-134); seed 0xceedfead
// (get_uint64_hash, common/gy_common_inc.h:1120)
// ---------------------------------------------------------------------------------------------------
static constexpr uint32_t JHASH_GOLDEN = 0x9e3779b9u;
static constexpr uint32_t GY_SEED = 0xceedfeadu;
static constexpr uint32_t FLOW_SEED_A = GY_SEED;
static constexpr uint32_t FLOW_SEED_B = GY_SEED ^ 0x5bd1e995u;

__host__ __device__ __forceinline__ uint32_t jhash_2words(uint32_t a, uint32_t b, uint32_t initval)
{
	uint32_t c = initval;

	a += JHASH_GOLDEN; b += JHASH_GOLDEN;
	a -= b; a -= c; a ^= (c >> 13);
	b -= c; b -= a; b ^= (a << 8);
	c -= a; c -= b; c ^= (b >> 13);
	a -= b; a -= c; a ^= (c >> 12);
	b -= c; b -= a; b ^= (a << 16);
	c -= a; c -= b; c ^= (b >> 5);
	a -= b; a -= c; a ^= (c >> 3);
	b -= c; b -= a; b ^= (a << 10);
	c -= a; c -= b; c ^= (b >> 15);
	return c;
}

__host__ __device__ __forceinline__ uint32_t uint64_hash(unsigned long long key)
{
	return jhash_2words((uint32_t)(key & 0xFFFFFFFFu), (uint32_t)(key >> 32), GY_SEED);
}

// Internal index of the id tables. Which entry an id lands in is not observable in any output (slot numbers follow insertion
// order, not the hash), so the table does not pay the reference's 36-instruction lookup2 per event: Fibonacci hashing, one
// 64-bit multiply. The ids themselves are CityHash outputs in the reference (common/gy_socket_stat.cc:1824).
__host__ __device__ __forceinline__ uint32_t table_hash(unsigned long long key)
{
	return (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 32);
}

// Two lookup2 words per flow key serve every sketch row (Kirsch-Mitzenmacher double hashing): count-min row r indexes
// (h1 + r * (h2 | 1)) & wmask, HyperLogLog takes the 64-bit word h2:h1. Definition shared with oracle/gysk_oracle.c.
__host__ __device__ __forceinline__ void flow_hashes(unsigned long long key, uint32_t &h1, uint32_t &h2)
{
	const uint32_t lo = (uint32_t)key, hi = (uint32_t)(key >> 32);
	h1 = jhash_2words(lo, hi, FLOW_SEED_A);
	h2 = jhash_2words(lo, hi, FLOW_SEED_B);
}

__host__ __device__ __forceinline__ uint32_t cms_index2(uint32_t h1, uint32_t h2, uint32_t row, uint32_t wmask)
{
	return (h1 + row * (h2 | 1u)) & wmask;
}

__host__ __device__ __forceinline__ uint32_t cms_index(unsigned long long key, uint32_t row, uint32_t wmask)
{
	uint32_t h1, h2;
	flow_hashes(key, h1, h2);
	return cms_index2(h1, h2, row, wmask);
}

__host__ __device__ __forceinline__ unsigned long long cms_increment(uint32_t bytes)
{
	return 1ull | ((unsigned long long)(bytes >> 10) << 32);
}

// murmur3's 64-bit finalizer. The HyperLogLog takes its register index from the top p bits of the word and its rank from the
// rest, so every output bit must depend on every key bit. Two one-round lookup2 words do not do that: on keys built as
// (client ip << 32) | port, h2's top bits reached only 3 341 of 4 096 registers at p = 12 for 20 000 keys (64 ports per ip),
// and the estimate came out 65 % low. The count-min indexes low bits of h1 + r * (h2 | 1) and keeps the unmixed words.
__host__ __device__ __forceinline__ unsigned long long fmix64(unsigned long long h)
{
	h ^= h >> 33; h *= 0xff51afd7ed558ccdull;
	h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull;
	h ^= h >> 33;
	return h;
}

// the register index and rank of the mixed hash h at precision p; one h serves several precisions (GYSK_FLAG_CLIENT_LEVELS)
__device__ __forceinline__ void hll_idx_rank_h(unsigned long long h, uint32_t p, uint32_t &idx, uint32_t &rank)
{
	const unsigned long long w = h << p;

	idx = (uint32_t)(h >> (64 - p));
	rank = w ? (uint32_t)__clzll((long long)w) + 1u : (64u - p + 1u);
}
__device__ __forceinline__ unsigned long long hll_hash2(uint32_t h1, uint32_t h2) { return fmix64(((unsigned long long)h2 << 32) | h1); }
__device__ __forceinline__ void hll_idx_rank2(uint32_t h1, uint32_t h2, uint32_t p, uint32_t &idx, uint32_t &rank)
{
	const unsigned long long h = fmix64(((unsigned long long)h2 << 32) | h1);
	const unsigned long long w = h << p;

	idx = (uint32_t)(h >> (64 - p));
	rank = w ? (uint32_t)__clzll((long long)w) + 1u : (64u - p + 1u);
}

// Log-linear value code of a response time: 32 bins per octave, exact below 32, monotone, < 1024 for usec < 2^30. The RESP
// keys are sorted by (slot, code) only (DESIGN.md §3): 10 value bits instead of 30.
static constexpr int TD_CODE_BITS = 10;
__host__ __device__ __forceinline__ uint32_t td_code(uint32_t v)
{
#ifdef __CUDA_ARCH__
	if (v < 32u) return v;
	const uint32_t sh = (31u - (uint32_t)__clz((int)v)) - 5u;
#else
	if (v < 32u) return v;
	const uint32_t sh = (31u - (uint32_t)__builtin_clz(v)) - 5u;
#endif
	return ((sh + 1u) << 5) | ((v >> sh) & 31u);
}
// smallest / largest value carrying a code
__host__ __device__ __forceinline__ uint32_t td_code_lo(uint32_t c) { return c < 32u ? c : ((32u | (c & 31u)) << ((c >> 5) - 1u)); }
__host__ __device__ __forceinline__ uint32_t td_code_hi(uint32_t c) { return c < 32u ? c : (((32u | (c & 31u)) + 1u) << ((c >> 5) - 1u)) - 1u; }

// ---------------------------------------------------------------------------------------------------
// bucket hashes (common/gy_statistics.h:1674-2063): bucket = 0 below min, nthr+1 at/after max_value,
// otherwise 1 + #thresholds strictly below the value (the reference's linear scan, mid-slot shortcut included,
// returns exactly that). Classes whose operator() takes `int` narrow the value first (:1748,:1801,:1854,:2032).
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ int bucket_resp_time(long long ms)			// RESP_TIME_HASH :1677, operator()(int64_t)
{
	constexpr int thr[13] = {1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000};
	if (ms < 0) return 0;
	if (ms >= 15001) return 14;
	int b = 1;
#pragma unroll
	for (int i = 0; i < 13; ++i) b += (ms > thr[i]);
	return b;
}

__device__ __forceinline__ int bucket_hash_1_3000(int data)			// HASH_1_3000 :2016, operator()(int)
{
	constexpr int thr[12] = {1, 5, 10, 25, 50, 75, 100, 150, 300, 500, 1000, 3000};
	if (data < 0) return 0;
	if (data >= 3001) return 13;
	int b = 1;
#pragma unroll
	for (int i = 0; i < 12; ++i) b += (data > thr[i]);
	return b;
}

__device__ __forceinline__ int bucket_duration(int data)				// DURATION_HASH :1838, operator()(int)
{
	constexpr int thr[13] = {1, 10, 25, 50, 125, 400, 1000, 3000, 6000, 10000, 25000, 40000, 65000};
	if (data < 0) return 0;
	if (data >= 65001) return 14;
	int b = 1;
#pragma unroll
	for (int i = 0; i < 13; ++i) b += (data > thr[i]);
	return b;
}

// Ordered compaction in one 1024-thread CTA that walks its input in tiles of 1024 entries, every thread calling once per tile: a
// block-wide ballot scan ranks the kept entries, and each thread whose entry is kept calls f(its rank among all entries kept so far).
// wcnt is the CTA's __shared__ uint32_t[32]; running = the entries the earlier tiles kept, advanced by this tile's.
template <typename F> __device__ __forceinline__ void tile_rank(bool keep, uint32_t *wcnt, uint32_t &running, F f)
{
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const unsigned b = __ballot_sync(0xffffffffu, keep);
	if (lane == 0) wcnt[wid] = __popc(b);
	__syncthreads();
	uint32_t before = 0, total = 0;
	for (int w = 0; w < 32; ++w) { const uint32_t c = wcnt[w]; before += w < wid ? c : 0; total += c; }
	if (keep) f(running + before + __popc(b & ((1u << lane) - 1u)));
	running += total;
	__syncthreads();
}

// ---------------------------------------------------------------------------------------------------
// memory helpers
// ---------------------------------------------------------------------------------------------------
// fire-and-forget 64-bit add: compiles to RED.E.ADD.64 (no return value travels back from L2)
__device__ __forceinline__ void red_add_u64(unsigned long long *p, unsigned long long v)
{
	asm volatile("red.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ void red_max_s64(long long *p, long long v)
{
	asm volatile("red.global.max.s64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// bring the 128-byte line holding p into L2 (no register waits for it)
__device__ __forceinline__ void prefetch_l2(const void *p)
{
	asm volatile("prefetch.global.L2 [%0];" :: "l"(p));
}

// L2 eviction priorities. A policy (createpolicy, a 64-bit register) travels with each access through .L2::cache_hint: ptxas for
// sm_90a accepts a priority written directly on ld only for 256-bit loads, so the policy operand is the form open to 32- and
// 64-bit accesses. atom.cas takes no hint at all.
__device__ __forceinline__ unsigned long long l2_policy_evict_first()
{
	unsigned long long pol;
	asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
	return pol;
}

__device__ __forceinline__ unsigned long long l2_policy_evict_last()
{
	unsigned long long pol;
	asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
	return pol;
}

__device__ __forceinline__ void red_add_u64_hint(unsigned long long *p, unsigned long long v, unsigned long long pol)
{
	asm volatile("red.global.add.L2::cache_hint.u64 [%0], %1, %2;" :: "l"(p), "l"(v), "l"(pol) : "memory");
}

// 32-bit load that does not allocate in L1 and allocates in L2 with the policy's priority
__device__ __forceinline__ uint32_t ld_na_hint_u32(const uint32_t *p, unsigned long long pol)
{
	uint32_t v;
	asm volatile("ld.global.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
	return v;
}

// 64-bit load from L2 (not cached in L1) that allocates with the policy's priority
__device__ __forceinline__ unsigned long long ld_cg_hint_u64(const unsigned long long *p, unsigned long long pol)
{
	unsigned long long v;
	asm volatile("ld.global.cg.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
	return v;
}

// a line's L2 priority back to normal (a line brought in with evict_last keeps that priority after the kernel ends)
__device__ __forceinline__ void l2_evict_normal_line(const void *p)
{
	asm volatile("applypriority.global.L2::evict_normal [%0], 128;" :: "l"(p) : "memory");
}

__device__ __forceinline__ uint4 ld_cg_v4(const void *p)
{
	uint4 v;
	asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
	return v;
}

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t *p)
{
	uint32_t v;
	asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
	return v;
}

__device__ __forceinline__ void st_volatile_u32(uint32_t *p, uint32_t v)
{
	asm volatile("st.volatile.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// id -> dense slot. Fast path = ONE 16-byte L2 load (key and published slot together), no fence: the slot number is
// self-validating (0 = not yet published) and nothing else is published through it — per-slot state is zero-initialised at
// engine creation, never by the inserter. With `insert`, an unknown id claims an empty entry with a CAS on the key, takes the
// next slot number and publishes it; racing readers of the same key spin on a volatile load. Returns -1 when absent / full.
// Replaces RCU_HASH_TABLE::lookup_single_elem_locked(glob_id, get_uint64_hash(glob_id)) (gy_mconnhdlr.cc:11183).
// The lookup is split so that a thread can put the first-probe loads of several ids in flight before resolving any of them
// (the 16-byte entry load is the latency that matters; hash collisions and inserts are the rare continuation).
__device__ __forceinline__ uint4 table_probe_first(const IdTable &t, unsigned long long key, uint32_t &pos)
{
	pos = table_hash(key) & t.mask;
	return ld_cg_v4(&t.ent[pos]);
}

__device__ __forceinline__ int table_resolve_slow(const IdTable &t, unsigned long long key, bool insert, uint32_t host_idx, uint32_t pos, uint4 raw)
{
	for (uint32_t probe = 0; probe <= t.mask; ++probe) {
		TblEntry *e = &t.ent[pos];
		unsigned long long k = ((unsigned long long)raw.y << 32) | raw.x;
		uint32_t s1 = raw.z;

		if (k == 0) {
			if (!insert) return -1;
			// no slot left (nothing on the free stack, every fresh one handed out): give up BEFORE claiming the entry, so a
			// full engine does not fill its table with dead keys (unknown ids keep arriving: one per netns/ip/port on the raw path).
			// The entry was empty when probed, but another event of this same id may have claimed it since and taken the last
			// slot — the one that filled the table: look again before dropping the event (every successful claim precedes the
			// slot-count add that made the table full, so its key is visible by now)
			if ((!t.free_n || *((volatile int32_t *)t.free_n) <= 0) && *((volatile uint32_t *)t.count) >= t.max_slots) {
				__threadfence();
				k = *((volatile unsigned long long *)&e->key);
				if (k == 0) return -1;
			}
			else if ((k = atomicCAS(&e->key, 0ull, key)) == 0) {
				// a slot recycled by an eviction first, else the next fresh one
				uint32_t s = SLOT_INVALID;
				if (t.free_n) {
					const int32_t f = atomicSub(t.free_n, 1);
					if (f > 0) s = t.free_slots[f - 1];
					else atomicAdd(t.free_n, 1);
				}
				if (s == SLOT_INVALID) {
					s = atomicAdd(t.count, 1u);
					if (s >= t.max_slots) {
						// lost the race for the last slots after the check above: the entry stays dead until the next table
						// rebuild, which gysk_flush triggers from this counter
						atomicSub(t.count, 1u);
						st_volatile_u32(&e->slot1, SLOT_INVALID);
						if (t.insert_fail) atomicAdd(t.insert_fail, 1ull);
						return -1;
					}
				}
				if (t.slot_id) { t.slot_id[s] = key; t.slot_host[s] = host_idx; }
				st_volatile_u32(&e->slot1, s + 1);
				return (int)s;
			}
			s1 = 0;
		}
		if (k == key) {
			while (s1 == 0) { __nanosleep(20); s1 = ld_volatile_u32(&e->slot1); }
			return s1 == SLOT_INVALID ? -1 : (int)(s1 - 1);
		}
		pos = (pos + 1) & t.mask;
		raw = ld_cg_v4(&t.ent[pos]);
	}
	return -1;
}

// the common case — the first probe holds the key with its slot published — costs three compares; collisions, unknown ids and
// inserts take the branch to the full probe loop
__device__ __forceinline__ int table_resolve(const IdTable &t, unsigned long long key, bool insert, uint32_t host_idx, uint32_t pos, uint4 raw)
{
	if (raw.x == (uint32_t)key && raw.y == (uint32_t)(key >> 32) && raw.z - 1u < SLOT_INVALID - 1u) return (int)(raw.z - 1u);
	return table_resolve_slow(t, key, insert, host_idx, pos, raw);
}

__device__ __forceinline__ int table_lookup(const IdTable &t, unsigned long long key, bool insert, uint32_t host_idx = 0)
{
	uint32_t pos;
	const uint4 raw = table_probe_first(t, key, pos);
	return table_resolve(t, key, insert, host_idx, pos, raw);
}

} // namespace gysk
