// gysk_merge.cu — the multi-GPU merge step (SURVEY.md §8e).
//
// Ingest is sharded by host (host_idx % world), so every per-service sketch lives wholly on one GPU and the ingest path
// has no exchange. What needs one exchange per query window are the answers for LOGICAL services spanning hosts (the
// reference's cross-host key is the svc-mesh cluster id, common/gy_comm_proto.h:2479-2506) and the global flow sketch:
//
//   gysk_set_logical_map   glob_id -> logical id (same list on every rank => same dense logical index everywhere)
//   gysk_merge_prepare     fold this GPU's member services into per-logical arrays laid out in ONE arena:
//                            [u64 SUM region : global CMS cur/last | histogram last/all | conn cells]
//                            [i64 MAX region : max_val_seen_ last/all]   [u8 MAX region : HLL registers]
//                          and a fixed t-digest slab (not element-wise mergeable); GYSK_FLAG_MERGE_LEVELS appends the rolling
//                          levels and aux sums to the SUM region, their maxima, the rtt and the flush tsec pair to the i64 MAX one;
//                          GYSK_FLAG_MERGE_STATES appends the members' LISTEN_SUMM_STATS words to the SUM region,
//                          GYSK_FLAG_MERGE_CLUSTERS the host clusters' MS_CLUSTER_STATE words after them (gysk_set_cluster_map);
//                          GYSK_FLAG_MERGE_TOPN appends this rank's 64 best services / processes per metric, with their rows, to the slab;
//                          GYSK_FLAG_FLOW_LEVEL puts the count-min level after cms cur/last and, as GYSK_FLAG_MERGE_LEVELS does,
//                          the flush tsec pair in the i64 MAX region (once when both are set); GYSK_FLAG_FLOW_QUERIES puts the
//                          flow query tables cur/last after the count-min tables, GYSK_FLAG_FLOW_QUERY_LEVEL their level after
//                          them with the flush tsec pair as GYSK_FLAG_FLOW_LEVEL; GYSK_FLAG_FLOW_RESP_HIST the flow response
//                          histograms cur/last [, 5min] after those; GYSK_FLAG_SVC_TOP_CLIENTS appends each logical service's
//                          heaviest-client summaries (its members' folded in map order) to the slab
//   (caller)             all-reduce each region once, all-gather the slab        — NCCL via torch.distributed
//   gysk_merge_finish      rank-ascending merge + compress of the gathered digests [, the global pick of the gathered top-N candidates]
//                          [, the rank-ascending fold of the gathered top-client summaries]
//   gysk_query_logical     same summary fields as gysk_query_svcs, for logical ids
//   gysk_export_logical_hist / gysk_merge_flush_range   one merged histogram / the ranks' flush tsec range
//   gysk_query_logical_states[_all]   the member listeners' state counts per logical service (GYSK_FLAG_MERGE_STATES)
//   gysk_query_cluster_states[_all]   the service half of MS_CLUSTER_STATE per host cluster (GYSK_FLAG_MERGE_CLUSTERS)
//   gysk_topn_global[_tasks]          the best services / processes of every rank, with their rows (GYSK_FLAG_MERGE_TOPN)
//
// It is the additive roll-up of MS_CLUSTER_STATE::STATE_ONE::add_stats (common/gy_comm_proto.h:3199-3214) /
// SHCONN_HANDLER::aggregate_cluster_state (server/gy_shconnhdlr.cc:4583) and of GY_HISTOGRAM::update_from_serialized
// (common/gy_statistics.h:625-650): integer sums are order independent => bit-exact at any GPU count.
#include "gysk_engine.h"
#include "gysk_summary.cuh"
#include "gysk_topc.cuh"

#include <climits>
#include <dlfcn.h>
#include <nccl.h>		// types only: the library is dlopen()ed, libgysketch.so carries no link-time dependency on it

using namespace gysk;

namespace gysk {

// The map keeps every {glob_id, logical} pair it was given; which of them live on this GPU, and in which slot, is looked up at
// every merge: a service that registers after gysk_set_logical_map takes part from its first window on, one that was evicted (or whose
// slot now belongs to another id) drops out. An id without a slot maps to the engine's null slot (index max_svcs: always in its
// just-created state, the identity of every fold), which Members::each skips.
__global__ void resolve_members_kernel(DevState st, const unsigned long long *__restrict__ member_ids, uint32_t n, Members mb)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const int slot = member_ids[i] ? table_lookup(st.svc_tbl, member_ids[i], false) : -1;
	mb.slots[i] = slot >= 0 ? (uint32_t)slot : mb.null_slot;
}

// one thread per (logical, cell)
__global__ void fold_hist_kernel(DevState st, Members mb, LogicalArrays lg)
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (uint64_t)lg.nl * HIST_CELLS) return;
	const uint32_t l = (uint32_t)(i >> 4);
	const int cell = (int)(i & 15);
	const LogicalArrays::Hist hl = lg.hist(GYSK_HIST_RESP_LAST, l), ha = lg.hist(GYSK_HIST_RESP_ALL, l);

	if (cell < HIST_MAX_CELL) {
		HistCell a {0, 0}, c {0, 0};
		mb.each(l, [&](uint32_t s) {
			const HistCell x = st.hist_last[(size_t)s * HIST_CELLS + cell], y = st.hist_all[(size_t)s * HIST_CELLS + cell];
			a.count += x.count; a.sum += x.sum; c.count += y.count; c.sum += y.sum;
		});
		hl.cells[cell] = a; ha.cells[cell] = c;
	}
	else {
		long long ml = LLONG_MIN, ma = LLONG_MIN;
		unsigned long long lc = 0, lk = 0, ac = 0, ak = 0;
		mb.each(l, [&](uint32_t s) {
			ml = max(ml, st.hist_last[(size_t)s * HIST_CELLS + HIST_MAX_CELL].sum);
			ma = max(ma, st.hist_all[(size_t)s * HIST_CELLS + HIST_MAX_CELL].sum);
			const unsigned long long cl = st.conn_last[s];
			lc += (uint32_t)cl; lk += cl >> 32; ac += st.conn_all_cnt[s]; ak += st.conn_all_kb[s];
		});
		hl.cells[cell] = HistCell {0, 0}; ha.cells[cell] = HistCell {0, 0};
		*hl.max = ml; *ha.max = ma;
		unsigned long long *cn = lg.conn_of(l);
		cn[0] = lc; cn[1] = lk; cn[2] = ac; cn[3] = ak;
	}
}

// GYSK_FLAG_MERGE_LEVELS, one thread per (logical, cell): cells 0..14 sum the members' level cells (st.levels.cell, what a member's
// own gysk_query_svcs row holds in lvl[]); the cell-15 thread takes the level maxima, the aux words of the last closed window and the
// largest rtt. Thread 0 also writes this engine's {last flush tsec, -last flush tsec}, whose i64 max over the ranks gives their
// latest and earliest flush. It streams the ring: 8 CTAs per SM (32 registers) keep enough loads in flight.
__global__ void __launch_bounds__(256, 8) fold_levels_kernel(DevState st, Members mb, long long flush_tsec, LogicalArrays lg)
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i == 0) { lg.flush[0] = flush_tsec; lg.flush[1] = -flush_tsec; }
	if (i >= (uint64_t)lg.nl * HIST_CELLS) return;
	const uint32_t l = (uint32_t)(i >> 4);
	const int cell = (int)(i & 15);

	if (cell < HIST_MAX_CELL) {
		HistCell a[NLEVELS] {};
		mb.each(l, [&](uint32_t s) {
#pragma unroll
			for (int lv = 0; lv < NLEVELS; ++lv) {
				const HistCell x = st.levels.cell(lv, s, cell);
				a[lv].count += x.count; a[lv].sum += x.sum;
			}
		});
		for (int lv = 0; lv < NLEVELS; ++lv) lg.hist(GYSK_HIST_RESP_5MIN + lv, l).cells[cell] = a[lv];
	}
	else {
		long long mx[NLEVELS] = {LLONG_MIN, LLONG_MIN};
		unsigned long long ac = 0, ak = 0, ce = 0, se = 0;
		uint32_t rtt = 0;
		mb.each(l, [&](uint32_t s) {
			for (int lv = 0; lv < NLEVELS; ++lv) mx[lv] = max(mx[lv], st.levels.cell(lv, s, HIST_MAX_CELL).sum);
			const SlotAux x = st.slot_aux[s];
			ac += (uint32_t)x.act_last; ak += x.act_last >> 32; ce += (uint32_t)x.err_last; se += x.err_last >> 32;
			rtt = max(rtt, x.rtt_last);
		});
		for (int lv = 0; lv < NLEVELS; ++lv) {
			const LogicalArrays::Hist h = lg.hist(GYSK_HIST_RESP_5MIN + lv, l);
			h.cells[cell] = HistCell {0, 0}; *h.max = mx[lv];
		}
		unsigned long long *a = lg.aux_of(l);
		a[0] = ac; a[1] = ak; a[2] = ce; a[3] = se;
		lg.rtt[l] = rtt;
	}
}

// GYSK_FLAG_MERGE_STATES, one thread per logical service: each member adds LISTEN_SUMM_STATS::update (server/gy_msocket.h:853-864) of
// the LISTENER_STATE_NOTIFY record gysk_encode_listener_state writes from its gysk_query_svcs row. Every value is the row's own, from
// the arrays summarize_fields reads: curr_state (slot_state), nqrys_5s (the last window's cells through cells_total, truncated to 32
// bits), nconns_active and ser_errors (slot_aux), kbytes_5s (conn_last). The u64 words keep the int32 sums modulo 2^32.
__global__ void fold_states_kernel(DevState st, Members mb, LogicalArrays lg)
{
	const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l >= lg.nl) return;
	unsigned long long nst[8] = {}, qps = 0, act = 0, kb_in = 0, ser = 0, nlisten = 0, nactive = 0;

	mb.each(l, [&](uint32_t s) {
		const uint8_t state = st.slot_state[s].state;
		if (state > GYSK_STATE_DOWN) return;			// never reaches summstats.update (gy_mconnhdlr.cc:11183-11251)
		uint64_t counts[15];
		const uint32_t nqrys_5s = (uint32_t)cells_total(st.hist_last + (size_t)s * HIST_CELLS, 15, counts);
		const SlotAux x = st.slot_aux[s];
#pragma unroll
		for (int k = 0; k < 8; ++k) nst[k] += state == k;
		qps += nqrys_5s / 5;
		act += (uint32_t)x.act_last;
		kb_in += (uint32_t)(st.conn_last[s] >> 32);
		ser += (uint32_t)(x.err_last >> 32);
		nlisten++;
		nactive += nqrys_5s != 0;
	});
	unsigned long long *w = lg.states_of(l);
#pragma unroll
	for (int k = 0; k < 8; ++k) w[k] = nst[k];
	w[8] = qps; w[9] = act; w[10] = kb_in; w[11] = 0; w[12] = ser; w[13] = nlisten; w[14] = nactive;	// tot_kb_outbound: the encoder's 0
}

// GYSK_FLAG_MERGE_CLUSTERS, pass 1, one thread per service slot: each live slot of a mapped host adds {1, issue, nqrys_5s / 5, kbytes_5s}
// to its host's words. The first two are the host's gysk_query_host_listen counts (svc_live, svc_issue); the last two are
// LISTEN_SUMM_STATS::update of the record gysk_encode_listener_state writes from the slot's window row, as fold_states_kernel takes them:
// nqrys_5s through cells_total truncated to 32 bits, curr_kbytes_inbound_ the last window's kbytes (curr_kbytes_outbound_ is the
// encoder's 0). Sums mod 2^32 do not depend on the order of the atomics.
__global__ void fold_cluster_hosts_kernel(DevState st, uint32_t max_svcs, uint32_t active_mark, Clusters cl)
{
	const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= min(*st.svc_tbl.count, max_svcs) || !svc_live(st, slot)) return;
	const uint32_t host = st.slot_host[slot], h = host < cl.ntab ? cl.host_of[host] : ~0u;
	if (h == ~0u) return;
	uint4 *a = cl.host_acc + h;
	atomicAdd(&a->x, 1u);
	if (svc_issue(st, slot, active_mark)) atomicAdd(&a->y, 1u);
	if (st.slot_state[slot].state > GYSK_STATE_DOWN) return;		// never reaches summstats.update (gy_mconnhdlr.cc:11183-11251)
	uint64_t counts[15];
	const uint32_t nqrys_5s = (uint32_t)cells_total(st.hist_last + (size_t)slot * HIST_CELLS, 15, counts);
	atomicAdd(&a->z, nqrys_5s / 5);
	atomicAdd(&a->w, (uint32_t)(st.conn_last[slot] >> 32));
}

// GYSK_FLAG_MERGE_CLUSTERS, pass 2, one thread per cluster: each of its hosts with a live service on this engine adds the service half of
// CLUSTER_STATE_ONE::update_from_state (server/gy_mconnhdlr.cc:16032-16050), svc_net_mb = (tot_kb_inbound + tot_kb_outbound) / 1024 in
// int32 per host (:16045). Each host's words are cleared for the next merge once read.
__global__ void fold_clusters_kernel(Clusters cl)
{
	const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= cl.nc) return;
	uint32_t nhosts = 0, issue = 0, issue_hosts = 0, nsvc = 0, qps = 0, mb = 0;
	for (uint32_t h = cl.offs[c]; h < cl.offs[c + 1]; ++h) {
		const uint4 a = cl.host_acc[h];
		if (!a.x) continue;
		cl.host_acc[h] = make_uint4(0, 0, 0, 0);
		nhosts++; issue += a.y; issue_hosts += a.y != 0; nsvc += a.x; qps += a.z;
		mb += (uint32_t)((int32_t)a.w / 1024);
	}
	unsigned long long *w = cl.words_of(c);
	w[0] = nhosts; w[1] = issue; w[2] = issue_hosts; w[3] = nsvc; w[4] = qps; w[5] = mb;
}

// one thread per (logical, 4 registers): per-byte max over the member services
__global__ void fold_hll_kernel(DevState st, Members mb, LogicalArrays lg)
{
	const uint32_t words = 1u << (st.hll_p - 2);
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (uint64_t)lg.nl * words) return;
	const uint32_t l = (uint32_t)(i / words), w = (uint32_t)(i % words);
	uint32_t acc = 0;

	mb.each(l, [&](uint32_t s) { acc = __vmaxu4(acc, reinterpret_cast<const uint32_t *>(st.hll + ((size_t)s << st.hll_p))[w]); });
	reinterpret_cast<uint32_t *>(lg.hll_of(l, st.hll_p))[w] = acc;
}

// GYSK_FLAG_CLIENT_LEVELS, one thread per (logical, set, 4 registers): per-byte max over the member services' last-window (set 0) and
// 300-s (set 1) client registers, the HLL of the union of their clients
__global__ void fold_clients_kernel(ClientLevels cl, Members mb, uint32_t nl, uint8_t *__restrict__ out)
{
	constexpr uint32_t words = CL_REGS / 4;
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (uint64_t)nl * 2 * words) return;
	const uint32_t l = (uint32_t)(i / (2 * words)), set = (uint32_t)(i / words) & 1u, w = (uint32_t)(i % words);
	const uint8_t *src = set ? cl.level : cl.last;
	uint32_t acc = 0;

	mb.each(l, [&](uint32_t s) { acc = __vmaxu4(acc, reinterpret_cast<const uint32_t *>(src + (size_t)s * CL_REGS)[w]); });
	reinterpret_cast<uint32_t *>(out)[i] = acc;
}

// GYSK_FLAG_MERGE_TRACES, one thread per (logical, word): words 0 .. LT_TD_COUNT sum the members' last closed trace windows (the half
// par ^ 1 of the row a member slot holds; a slot without a row, or whose row is being taken, adds nothing), the LT_NTRACED thread counts
// those rows and takes the three maxima.
__global__ void fold_traces_kernel(DevState st, Members mb, LogicalArrays lg)
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (uint64_t)lg.nl * LT_WORDS) return;
	const uint32_t l = (uint32_t)(i / LT_WORDS);
	const int k = (int)(i % LT_WORDS);
	const TraceTable &tr = st.trace;
	const uint32_t half = tr.par ^ 1u;
	// the row word of LT_NREQ .. LT_BYTES_OUT, 8 bits apiece; the buckets follow in both layouts
	constexpr unsigned long long SRC = (unsigned long long)TW_NREQ | (unsigned long long)TW_NERR << 8 | (unsigned long long)TW_NCONNS << 16 |
		(unsigned long long)TW_SUM_US << 24 | (unsigned long long)TW_BYTES_IN << 32 | (unsigned long long)TW_BYTES_OUT << 40;
	const int src = k < LT_BKT ? (int)((SRC >> (8 * k)) & 0xFF) : TW_BKT + (k - LT_BKT);
	unsigned long long acc = 0;
	long long mx[LT_MAX_WORDS] = {0, 0, 0};

	mb.each(l, [&](uint32_t s) {
		const uint32_t r1 = tr.row_of[s];
		if (r1 == 0 || r1 == TRACE_BUSY) return;
		const uint32_t r = r1 - 1u;
		if (k == LT_TD_COUNT) acc += tr.hd(half, r)->total;
		else if (k == LT_NTRACED) {
			const unsigned long long *w = tr.words(half, r);
			acc++;
			mx[LT_MAX_US] = max(mx[LT_MAX_US], (long long)w[TW_MAX_US]);
			mx[LT_MAX_IN] = max(mx[LT_MAX_IN], (long long)w[TW_MAX_IN]);
			mx[LT_MAX_OUT] = max(mx[LT_MAX_OUT], (long long)w[TW_MAX_OUT]);
		}
		else acc += tr.words(half, r)[src];
	});
	lg.traces_of(l)[k] = acc;
	if (k == LT_NTRACED) {
		long long *m = lg.trace_max_of(l);
		m[LT_MAX_US] = mx[LT_MAX_US]; m[LT_MAX_IN] = mx[LT_MAX_IN]; m[LT_MAX_OUT] = mx[LT_MAX_OUT];
	}
}

static constexpr int MG_WARPS = 2;		// 2 x 17.8 KB of scratch: static shared memory

// One warp folds the digests digest(b) .. digest(e - 1) into {out_head, out_cent[CAP]}, one after the other: each non-empty one is
// merged into the accumulator and compressed (warp_merge_compress), its total, min and max added. digest(i) gives {n, total, min, max,
// centroids}, n = 0 for an entry to skip.
struct DigestRef { uint32_t n; unsigned long long total; double minv, maxv; const Centroid *cent; };
__device__ __forceinline__ DigestRef digest_ref(const TdHead &h, const Centroid *c) { return DigestRef {h.n, h.total, h.minv, h.maxv, c}; }
__device__ __forceinline__ DigestRef no_digest() { return DigestRef {0, 0, 0.0, 0.0, nullptr}; }
// the last closed window's digest of the trace row a service slot holds; a trace digest's extremes are counter words of its window
__device__ __forceinline__ DigestRef trace_digest(const TraceTable &tr, uint32_t slot)
{
	const uint32_t r1 = tr.row_of[slot];
	if (r1 == 0 || r1 == TRACE_BUSY) return no_digest();
	const uint32_t r = r1 - 1u, half = tr.par ^ 1u;
	const TdHead h = *tr.hd(half, r);
	const unsigned long long *w = tr.words(half, r);
	return DigestRef {h.n, h.total, (double)(0xFFFFFFFFu - (uint32_t)w[TW_TD_NMIN]), (double)w[TW_TD_MAX], tr.cents(half, r)};
}

template <int CAP, typename Digest>
__device__ __forceinline__ void fold_digests(TdScratch &S, const TdParams &P, uint32_t b, uint32_t e, Digest digest, TdHead &out_head,
		Centroid *out_cent, int lane)
{
	uint32_t nacc = 0;
	unsigned long long total = 0;
	double mn = INFINITY, mx = -INFINITY;

	for (uint32_t i = b; i < e; ++i) {
		const DigestRef d = digest(i);
		if (!d.n) continue;
		nacc = warp_merge_compress(S, S.newc, nacc, d.cent, d.n, S.newc, P);
		total += d.total; mn = fmin(mn, d.minv); mx = fmax(mx, d.maxv);
	}
	for (uint32_t c = lane; c < (uint32_t)CAP; c += 32) out_cent[c] = c < nacc ? S.newc[c] : Centroid {0.0, 0};
	if (lane == 0) { TdHead h; h.total = total; h.minv = mn; h.maxv = mx; h.n = nacc; h.pad = 0; out_head = h; }
	__syncwarp();
}

// one warp per logical service: its members' digests in map order; with GYSK_FLAG_MERGE_TRACES (lg.trace_slab) then their last trace
// windows' digests, in map order at the trace rows' compression
__global__ void __launch_bounds__(MG_WARPS * 32) fold_td_kernel(DevState st, Members mb, LogicalArrays lg)
{
	__shared__ TdScratch scratch[MG_WARPS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;

	for (uint32_t l = blockIdx.x * MG_WARPS + wid; l < lg.nl; l += gridDim.x * MG_WARPS) {
		fold_digests<TD_CAP>(scratch[wid], st.td, mb.offs[l], mb.offs[l + 1], [&](uint32_t m) {
			const uint32_t s = mb.slots[m];
			return s == mb.null_slot ? no_digest() : digest_ref(st.td_head[s], st.td_cent + (size_t)s * TD_CAP);
		}, lg.slab[l].head, lg.slab[l].cent, lane);
		if (lg.trace_slab)
			fold_digests<TRACE_TD_CAP>(scratch[wid], st.trace.td, mb.offs[l], mb.offs[l + 1], [&](uint32_t m) {
				const uint32_t s = mb.slots[m];
				return s == mb.null_slot ? no_digest() : trace_digest(st.trace, s);
			}, lg.trace_slab[l].head, lg.trace_slab[l].cent, lane);
	}
}

// one warp per logical service over the all-gathered slabs [world][stride] (each rank's nl digests first, its trace digests from entry
// trace_off), in rank-ascending order => deterministic result
__global__ void __launch_bounds__(MG_WARPS * 32) finish_td_kernel(const SlabEntry *__restrict__ gathered, uint32_t world, uint32_t stride, LogicalArrays lg,
		TdParams P, uint32_t trace_off, TdParams PT)
{
	__shared__ TdScratch scratch[MG_WARPS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;

	for (uint32_t l = blockIdx.x * MG_WARPS + wid; l < lg.nl; l += gridDim.x * MG_WARPS) {
		fold_digests<TD_CAP>(scratch[wid], P, 0, world, [&](uint32_t r) {
			const SlabEntry &g = gathered[(size_t)r * stride + l];
			return digest_ref(g.head, g.cent);
		}, lg.final_slab[l].head, lg.final_slab[l].cent, lane);
		if (lg.trace_final)
			fold_digests<TRACE_TD_CAP>(scratch[wid], PT, 0, world, [&](uint32_t r) {
				const TraceSlab &g = reinterpret_cast<const TraceSlab *>(gathered + (size_t)r * stride + trace_off)[l];
				return digest_ref(g.head, g.cent);
			}, lg.trace_final[l].head, lg.trace_final[l].cent, lane);
	}
}

// GYSK_FLAG_SVC_TOP_CLIENTS: each logical service's two summaries (GYSK_TOPC_LAST, GYSK_TOPC_5MIN: [l][0], [l][1]) as sequential
// folds acc = merge(acc, s) from the empty summary (DESIGN.md §2): its members in map order on each rank (fold_topc_kernel), then the
// ranks' results in ascending rank order (finish_topc_kernel). Every step merges at most 2K entries, so one warp does it; the result
// does not depend on the launch shape.
static constexpr int TC_WARPS = 4;
struct TopcScratch { TopcCand buf[2 * TOPC_K], list[TOPC_K + 1]; TopcSet acc; };

// acc = the empty summary
__device__ __forceinline__ void topc_clear(TopcSet *acc, int lane)
{
	if ((uint32_t)lane < TOPC_K) acc->ent[lane] = gysk_topc_entry {0ull, 0u, 0u};
	if (lane == 0) acc->delta = 0ull;
	__syncwarp();
}

// acc = merge(acc, s): the groups of both by flow key, c = the (K + 1)-th kbytes, the groups above c less c, delta = both deltas + c
__device__ __forceinline__ void topc_fold(TopcScratch &S, const TopcSet *s, int lane)
{
	const unsigned long long delta = S.acc.delta + s->delta;
	const uint32_t m = topc_gather(s, S.buf, topc_gather(&S.acc, S.buf, 0, lane), lane);
	uint32_t n = 0;
	topc_offer_groups(S.buf, m, S.list, n, lane);
	topc_store(S.list, n, delta, &S.acc, lane);
}

__device__ __forceinline__ void topc_put(const TopcSet &acc, TopcSet *out, int lane)
{
	if ((uint32_t)lane < TOPC_K) out->ent[lane] = acc.ent[lane];
	if (lane == 0) out->delta = acc.delta;
	__syncwarp();
}

// one warp per logical service (grid-stride): its members' last-window and 300-s summaries folded in map order into out[l][0 / 1]; a
// member without a slot here is skipped (the identity)
__global__ void __launch_bounds__(TC_WARPS * 32) fold_topc_kernel(SvcTopClients tc, Members mb, uint32_t nl, TopcSet *__restrict__ out)
{
	__shared__ TopcScratch scratch[TC_WARPS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	TopcScratch &S = scratch[wid];

	for (uint32_t l = blockIdx.x * TC_WARPS + wid; l < nl; l += gridDim.x * TC_WARPS) {
		for (int set = 0; set < 2; ++set) {
			const TopcSet *src = set ? tc.level : tc.last;
			topc_clear(&S.acc, lane);
			mb.each(l, [&](uint32_t s) { topc_fold(S, src + s, lane); });
			topc_put(S.acc, out + (size_t)l * 2 + set, lane);
		}
	}
}

// one warp per logical service (grid-stride): the ranks' summaries of the all-gathered slabs [world][stride] (rank r's from entry topc_off)
// folded in ascending rank order into out[l][0 / 1]
__global__ void __launch_bounds__(TC_WARPS * 32) finish_topc_kernel(const SlabEntry *__restrict__ gathered, uint32_t world, uint32_t stride,
		uint32_t topc_off, uint32_t nl, TopcSet *__restrict__ out)
{
	__shared__ TopcScratch scratch[TC_WARPS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	TopcScratch &S = scratch[wid];

	for (uint32_t l = blockIdx.x * TC_WARPS + wid; l < nl; l += gridDim.x * TC_WARPS) {
		for (int set = 0; set < 2; ++set) {
			topc_clear(&S.acc, lane);
			for (uint32_t r = 0; r < world; ++r)
				topc_fold(S, reinterpret_cast<const TopcSet *>(gathered + (size_t)r * stride + topc_off) + (size_t)l * 2 + set, lane);
			topc_put(S.acc, out + (size_t)l * 2 + set, lane);
		}
	}
}

// GYSK_FLAG_MERGE_TOPN, one CTA per list m, one thread per candidate of the gathered slabs (rank r's lists at gathered + r * stride + nl,
// each best first). Candidates with a non-zero score are ordered by score descending, then rank ascending, then local order, so the place
// of rank r's entry i is i plus, in every other rank's list, the entries with a greater score or an equal one on a lower rank (a binary
// search: the lists are sorted). Every global winner is among its own rank's TOPN_K best, so places 0 .. TOPN_K - 1 are exact; they take the
// candidate's entry and row, the places no candidate reaches stay zero.
__global__ void __launch_bounds__(256) topn_global_kernel(const SlabEntry *__restrict__ gathered, uint32_t world, uint32_t stride, uint32_t nl,
		TopnLists out)
{
	const uint32_t m = blockIdx.x;
	const size_t row_words = TopnLists::row_bytes(m) / 8;
	auto cands = [&](uint32_t r) { return TopnLists {reinterpret_cast<uint8_t *>(const_cast<SlabEntry *>(gathered + (size_t)r * stride + nl))}; };

	for (uint32_t i = threadIdx.x; i < TOPN_K; i += blockDim.x) out.ent(m)[i] = gysk_topn_entry {0, 0, 0, 0};
	__syncthreads();
	for (uint32_t c = threadIdx.x; c < world * TOPN_K; c += blockDim.x) {
		const uint32_t r = c / TOPN_K, i = c % TOPN_K;
		const gysk_topn_entry x = cands(r).ent(m)[i];
		if (!x.score) continue;
		uint32_t place = i;
		for (uint32_t q = 0; q < world && place < TOPN_K; ++q) {
			if (q == r) continue;
			const gysk_topn_entry *l = cands(q).ent(m);
			uint32_t lo = 0, hi = TOPN_K;
			while (lo < hi) {
				const uint32_t mid = (lo + hi) >> 1;
				const unsigned long long s = l[mid].score;
				if (s > x.score || (s == x.score && q < r)) lo = mid + 1;
				else hi = mid;
			}
			place += lo;
		}
		if (place >= TOPN_K) continue;
		out.ent(m)[place] = x;
		const unsigned long long *src = reinterpret_cast<const unsigned long long *>(cands(r).row(m, i));
		unsigned long long *dst = reinterpret_cast<unsigned long long *>(out.row(m, place));
		for (size_t k = 0; k < row_words; ++k) dst[k] = src[k];
	}
}

// read side: one warp per logical service, its merged arrays into a shared-memory SvcRaw, then the row of summarize_warp (the
// summary of gysk_query_svcs). The merge folds neither the current window, the connection bitmaps nor the per-slot state / qps /
// active-connection words: they are zero; so are the rolling levels and the aux words unless the engine merges them (lg.lvl).
// glob_id is the logical id (lids[l]), 0 for an index of -1.
static constexpr int LG_WARPS = 4;
__global__ void __launch_bounds__(LG_WARPS * 32) logical_summary_kernel(const int32_t *__restrict__ lidx, uint32_t n, uint32_t hll_p, LogicalArrays lg,
		const unsigned long long *__restrict__ lids, gysk_svc_summary *__restrict__ out)
{
	__shared__ SvcRaw raw[LG_WARPS];
	__shared__ unsigned long long summ[LG_WARPS][sizeof(gysk_svc_summary) / 8];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t q = blockIdx.x * LG_WARPS + wid;

	if (q >= n) return;
	SvcRaw &r = raw[wid];
	const int32_t l = lidx[q];
	if (lane == 0) { r.id = 0; r.found = l >= 0; r.slot = (uint32_t)l; }
	if (l >= 0) {
		if (lane < HIST_CELLS) {
			r.last[lane] = lg.cell(GYSK_HIST_RESP_LAST, l, lane); r.all[lane] = lg.cell(GYSK_HIST_RESP_ALL, l, lane);
			r.cur[lane] = HistCell {0, 0};
			for (int k = 0; k < NLEVELS; ++k) r.lvl[k][lane] = lg.lvl ? lg.cell(GYSK_HIST_RESP_5MIN + k, l, lane) : HistCell {0, 0};
			r.bm_cur[lane] = 0; r.bm_last[lane] = 0;
			r.qps[lane] = HistCell {0, 0}; r.act[lane] = HistCell {0, 0};
		}
		if (lane == 0) {
			const unsigned long long *cn = lg.conn_of(l);
			r.conn_cur = 0;
			r.conn_last = (cn[0] & 0xFFFFFFFFull) | (cn[1] << 32);
			r.conn_all_cnt = cn[2]; r.conn_all_kb = cn[3];
			r.td = lg.final_slab[l].head;
			r.aux = SlotAux {0, 0, 0, 0, 0, 0};
			if (lg.lvl) {
				const unsigned long long *a = lg.aux_of(l);
				r.aux.act_last = (a[0] & 0xFFFFFFFFull) | (a[1] << 32);
				r.aux.err_last = (a[2] & 0xFFFFFFFFull) | (a[3] << 32);
				r.aux.rtt_last = (uint32_t)lg.rtt[l];
			}
			r.sst = SlotState {0, 0, 0, 0, 0};
		}
		for (int i = lane; i < TD_CAP; i += 32) r.cent[i] = lg.final_slab[l].cent[i];
		hll_hist_warp(lg.hll_of(l, hll_p), hll_p, r.hll_hist, lane);
	}
	summarize_warp(r, l >= 0 ? lids[l] : 0ull, hll_p, summ[wid], out + q, lane);
}

// GYSK_FLAG_CLIENT_LEVELS read side, one warp per row: the merged client sets (regs: [nl][2][CL_REGS]) of dense index lidx[q] as
// client_rows_kernel reads a service's, logical id lids[l]; an index of -1 gives an all-zero row
__global__ void __launch_bounds__(LG_WARPS * 32) logical_clients_kernel(const int32_t *__restrict__ lidx, uint32_t n, const uint8_t *__restrict__ regs,
		const unsigned long long *__restrict__ lids, gysk_svc_clients *__restrict__ out)
{
	__shared__ uint32_t hist[LG_WARPS][2][64];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const uint32_t q = blockIdx.x * LG_WARPS + wid;

	if (q >= n) return;
	const int32_t l = lidx[q];
	gysk_svc_clients o;
	memset(&o, 0, sizeof(o));
	if (l >= 0) {
		for (int set = 0; set < 2; ++set) hll_hist_warp(regs + ((size_t)l * 2 + set) * CL_REGS, GYSK_HLL_WINDOW_P, hist[wid][set], lane);
		o.glob_id = lids[l]; o.found = 1;
		o.last_5s = hll_pending(hist[wid][0], GYSK_HLL_WINDOW_P);
		o.last_5min = hll_pending(hist[wid][1], GYSK_HLL_WINDOW_P);
	}
	if (lane == 0) out[q] = o;
}

// a logical service whose merged last window holds response samples or connection events (GYSK_WINDOW_ACTIVE_ONLY)
__device__ __forceinline__ bool logical_active(const LogicalArrays &lg, uint32_t l)
{
	const HistCell *c = lg.hist(GYSK_HIST_RESP_LAST, l).cells;
	unsigned long long any = lg.conn_of(l)[0];
#pragma unroll
	for (int b = 0; b < HIST_MAX_CELL; ++b) any |= c[b].count;
	return any != 0;
}

// the GYSK_WINDOW_ACTIVE_ONLY rule of each all-rows read: a logical service as logical_active, a cluster with a live service on some rank
struct LogicalActive { LogicalArrays lg; __device__ __forceinline__ bool operator()(uint32_t l) const { return logical_active(lg, l); } };
struct ClusterActive { Clusters cl; __device__ __forceinline__ bool operator()(uint32_t c) const { return (uint32_t)cl.words_of(c)[3] != 0; } };
// ... and a logical service whose merged trace window holds requests
struct TraceActive { LogicalArrays lg; __device__ __forceinline__ bool operator()(uint32_t l) const { return lg.traces_of(l)[LT_NREQ] != 0; } };

// One CTA walks the n dense indices of `sorted` (ascending id) and keeps the active ones, in order: tile_rank places the kept entries
// of each 1024-entry tile. *d_n = entries kept.
template <typename Active>
__global__ void __launch_bounds__(1024) logical_select_kernel(const int32_t *__restrict__ sorted, uint32_t n, Active active, int32_t *__restrict__ sel,
		unsigned long long *d_n)
{
	__shared__ uint32_t wcnt[32];
	uint32_t running = 0;

	for (uint32_t t = 0; t < n; t += 1024) {
		const uint32_t i = t + threadIdx.x;
		const int32_t l = i < n ? sorted[i] : 0;
		const bool keep = i < n && active((uint32_t)l);
		tile_rank(keep, wcnt, running, [&](uint32_t r) { sel[r] = l; });
	}
	if (threadIdx.x == 0) *d_n = running;
}

// top-N keys {score : 32 | dense index : 32} of the logical services, scored as topn_score_kernel scores a service from the merged arrays
__global__ void logical_topn_score_kernel(LogicalArrays lg, int metric, unsigned long long *__restrict__ keys, unsigned long long *d_n)
{
	const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l == 0) *d_n = lg.nl;
	if (l >= lg.nl) return;
	unsigned long long score = 0;

	if (metric == GYSK_TOPN_QPS) {
		const HistCell *c = lg.hist(GYSK_HIST_RESP_LAST, l).cells;
		for (int b = 0; b < HIST_MAX_CELL; ++b) score += c[b].count;
		if (score > 0xFFFFFFFFull) score = 0xFFFFFFFFull;
	}
	else if (metric == GYSK_TOPN_CONNS) score = (uint32_t)lg.conn_of(l)[0];
	else if (metric == GYSK_TOPN_NET) score = (uint32_t)lg.conn_of(l)[1];
	else if (metric == GYSK_TOPN_ISSUE) score = lg.nsvc_issue(l);
	else score = (uint32_t)lg.aux_of(l)[0];		// GYSK_TOPN_ACTIVE
	keys[l] = (score << 32) | l;
}

// GYSK_FLAG_MERGE_STATES read side, one thread per row: the merged words of dense index lidx[q] as LISTEN_SUMM_STATS<int> (each word
// truncated to 32 bits: the int32 wrap-around sum), logical id lids[l]; an index of -1 gives an all-zero row
__global__ void logical_state_kernel(const int32_t *__restrict__ lidx, uint32_t n, LogicalArrays lg, const unsigned long long *__restrict__ lids,
		gysk_logical_state *__restrict__ out)
{
	const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= n) return;
	const int32_t l = lidx[q];
	gysk_logical_state o;
	memset(&o, 0, sizeof(o));
	if (l >= 0) {
		const unsigned long long *w = lg.states_of((uint32_t)l);
		int32_t f[STATE_WORDS + 1];
#pragma unroll
		for (int k = 0; k < STATE_WORDS; ++k) f[k] = (int32_t)(uint32_t)w[k];
		f[STATE_WORDS] = 0;
		memcpy(&o.summ, f, sizeof(f));
		o.logical_id = lids[l]; o.found = 1; o.nsvc_issue = lg.nsvc_issue((uint32_t)l);
	}
	out[q] = o;
}

// GYSK_FLAG_MERGE_CLUSTERS read side, one thread per row: the merged words of dense index cidx[q], each truncated to 32 bits (the uint32
// wrap-around sum), cluster id cids[c]; an index of -1 gives an all-zero row
__global__ void cluster_row_kernel(const int32_t *__restrict__ cidx, uint32_t n, Clusters cl, const unsigned long long *__restrict__ cids,
		gysk_cluster_row *__restrict__ out)
{
	const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= n) return;
	const int32_t c = cidx[q];
	gysk_cluster_row o;
	memset(&o, 0, sizeof(o));
	if (c >= 0) {
		const unsigned long long *w = cl.words_of((uint32_t)c);
		o.cluster_id = cids[c]; o.found = 1;
		o.st.nhosts = (uint32_t)w[0]; o.st.nsvc_issue = (uint32_t)w[1]; o.st.nsvcissue_hosts = (uint32_t)w[2];
		o.st.nsvc = (uint32_t)w[3]; o.st.total_qps = (uint32_t)w[4]; o.st.svc_net_mb = (uint32_t)w[5];
	}
	out[q] = o;
}

// GYSK_FLAG_MERGE_TRACES read side, one thread per row: the merged trace window of dense index lidx[q], logical id lids[l], p99 from the
// merged digest (NaN while it is empty, as trace_window_out); an index of -1 gives an all-zero row
__global__ void logical_trace_kernel(const int32_t *__restrict__ lidx, uint32_t n, LogicalArrays lg, const unsigned long long *__restrict__ lids,
		gysk_logical_trace *__restrict__ out)
{
	const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= n) return;
	const int32_t l = lidx[q];
	gysk_logical_trace o;
	memset(&o, 0, sizeof(o));
	if (l >= 0) {
		const unsigned long long *w = lg.traces_of((uint32_t)l);
		const long long *m = lg.trace_max_of((uint32_t)l);
		const TraceSlab &d = lg.trace_final[l];
		gysk_trace_window &t = o.last;
		o.logical_id = lids[l]; o.found = 1; o.ntraced = (uint32_t)w[LT_NTRACED];
		t.nreq = w[LT_NREQ]; t.nerr = w[LT_NERR]; t.nconns = w[LT_NCONNS]; t.sum_resp_us = w[LT_SUM_US];
		t.max_resp_us = (unsigned long long)m[LT_MAX_US];
		t.bytes_in = w[LT_BYTES_IN]; t.bytes_out = w[LT_BYTES_OUT];
		t.max_bytes_in = (unsigned long long)m[LT_MAX_IN]; t.max_bytes_out = (unsigned long long)m[LT_MAX_OUT];
		for (int b = 0; b < 8; ++b) t.resp_buckets[b] = w[LT_BKT + b];
		t.td_count = w[LT_TD_COUNT];
		const TdHead h = d.head;
		t.p99_resp_us = h.n ? td_quantile_seq(TdCentroids {d.cent}, h.n, h.minv, h.maxv, 0.99) : (double)NAN;
	}
	out[q] = o;
}

// GYSK_FLAG_SVC_TOP_CLIENTS read side, one warp per row: summary `set` (0: GYSK_TOPC_LAST, 1: GYSK_TOPC_5MIN) of dense index lidx[q] as
// topc_rows_kernel reads a service's, logical id lids[l]; an index of -1 gives found = 0 and a zero row
__global__ void __launch_bounds__(LG_WARPS * 32) logical_topc_kernel(const int32_t *__restrict__ lidx, uint32_t n, const TopcSet *__restrict__ sets,
		int set, const unsigned long long *__restrict__ lids, gysk_svc_top_clients *__restrict__ out)
{
	const int lane = threadIdx.x & 31;
	const uint32_t q = blockIdx.x * LG_WARPS + (threadIdx.x >> 5);
	if (q >= n) return;
	const int32_t l = lidx[q];
	const TopcSet *s = l >= 0 ? sets + (size_t)l * 2 + set : nullptr;
	gysk_topc_entry e {0ull, 0u, 0u};
	if (s && (uint32_t)lane < TOPC_K) e = s->ent[lane];
	if ((uint32_t)lane < TOPC_K) out[q].entries[lane] = e;
	const uint32_t held = (uint32_t)__popc(__ballot_sync(0xffffffffu, e.kbytes != 0));
	if (lane == 0) {
		out[q].glob_id = s ? lids[l] : 0ull; out[q].found = s != nullptr; out[q].n = held;
		out[q].delta = s ? s->delta : 0ull;
	}
}

} // namespace gysk

namespace {

inline uint32_t div_up(uint64_t a, uint64_t b) { return (uint32_t)((a + b - 1) / b); }
inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// dense index of a logical (or cluster) id, -1 for an id the map does not have
int32_t dense_index(const std::unordered_map<uint64_t, uint32_t> &index, uint64_t id)
{
	const auto it = index.find(id);
	return it == index.end() ? -1 : (int32_t)it->second;
}
int32_t logical_index(const MergeState &mg, uint64_t id) { return dense_index(mg.index, id); }

// The dense index space of a row type: the logical services (service and state rows) or the host clusters (cluster rows). sorted holds
// the n indices by ascending id, sel the ACTIVE_ONLY part of them; select launches the selection (*d_n = indices kept).
struct RowSpace
{
	const std::unordered_map<uint64_t, uint32_t> *index;
	uint32_t n;
	const int32_t *sorted;
	int32_t *sel;
};
template <typename Row> RowSpace row_space(MergeState &mg, const Row *) { return RowSpace {&mg.index, mg.lg.nl, mg.d_sorted, mg.d_sel}; }
RowSpace row_space(MergeState &mg, const gysk_cluster_row *)
{
	const ClusterMap &cm = mg.clusters;
	return RowSpace {&cm.index, cm.cl.nc, cm.d_sorted, cm.d_sel};
}
template <typename Row> void launch_select(gysk_engine *e, const Row *, unsigned long long *d_n)
{
	logical_select_kernel<<<1, 1024, 0, e->stream>>>(e->mg.d_sorted, e->mg.lg.nl, LogicalActive {e->mg.lg}, e->mg.d_sel, d_n);
}
void launch_select(gysk_engine *e, const gysk_cluster_row *, unsigned long long *d_n)
{
	const ClusterMap &cm = e->mg.clusters;
	logical_select_kernel<<<1, 1024, 0, e->stream>>>(cm.d_sorted, cm.cl.nc, ClusterActive {cm.cl}, cm.d_sel, d_n);
}
void launch_select(gysk_engine *e, const gysk_logical_trace *, unsigned long long *d_n)
{
	logical_select_kernel<<<1, 1024, 0, e->stream>>>(e->mg.d_sorted, e->mg.lg.nl, TraceActive {e->mg.lg}, e->mg.d_sel, d_n);
}

// Per row type of the logical and cluster reads: the launch that makes the rows of the dense indices lidx[0 .. m) in the device stage
// (an index of -1 gives the not-found row), the finish that copies them out, the field a by-id read stamps with the queried id, and the
// engine flag the rows need.
int launch_logical(gysk_engine *e, const int32_t *lidx, uint32_t m, gysk_svc_summary *, int = 0)
{
	logical_summary_kernel<<<div_up(m, LG_WARPS), LG_WARPS * 32, 0, e->stream>>>(lidx, m, e->cfg.hll_p, e->mg.lg, e->mg.d_logical_ids,
			reinterpret_cast<gysk_svc_summary *>(e->d_wstage));
	return 1;
}
int launch_logical(gysk_engine *e, const int32_t *lidx, uint32_t m, gysk_logical_state *, int = 0)
{
	logical_state_kernel<<<div_up(m, 256), 256, 0, e->stream>>>(lidx, m, e->mg.lg, e->mg.d_logical_ids, reinterpret_cast<gysk_logical_state *>(e->d_wstage));
	return 1;
}
int launch_logical(gysk_engine *e, const int32_t *lidx, uint32_t m, gysk_cluster_row *, int = 0)
{
	cluster_row_kernel<<<div_up(m, 256), 256, 0, e->stream>>>(lidx, m, e->mg.clusters.cl, e->mg.clusters.d_ids, reinterpret_cast<gysk_cluster_row *>(e->d_wstage));
	return 1;
}
int launch_logical(gysk_engine *e, const int32_t *lidx, uint32_t m, gysk_svc_clients *, int = 0)
{
	logical_clients_kernel<<<div_up(m, LG_WARPS), LG_WARPS * 32, 0, e->stream>>>(lidx, m, e->mg.cl_hll, e->mg.d_logical_ids,
			reinterpret_cast<gysk_svc_clients *>(e->d_wstage));
	return 1;
}
int launch_logical(gysk_engine *e, const int32_t *lidx, uint32_t m, gysk_logical_trace *, int = 0)
{
	logical_trace_kernel<<<div_up(m, 128), 128, 0, e->stream>>>(lidx, m, e->mg.lg, e->mg.d_logical_ids, reinterpret_cast<gysk_logical_trace *>(e->d_wstage));
	return 1;
}
// (which: the summary of the top-client rows)
int launch_logical(gysk_engine *e, const int32_t *lidx, uint32_t m, gysk_svc_top_clients *, int which)
{
	logical_topc_kernel<<<div_up(m, LG_WARPS), LG_WARPS * 32, 0, e->stream>>>(lidx, m, e->mg.topc_final, which == GYSK_TOPC_5MIN, e->mg.d_logical_ids,
			reinterpret_cast<gysk_svc_top_clients *>(e->d_wstage));
	return 1;
}
SvcRows logical_finish(const gysk_engine *e, gysk_svc_summary *out) { return SvcRows {e->cfg.hll_p, out}; }
CopyRows<gysk_logical_state> logical_finish(const gysk_engine *, gysk_logical_state *out) { return CopyRows<gysk_logical_state> {out}; }
CopyRows<gysk_cluster_row> logical_finish(const gysk_engine *, gysk_cluster_row *out) { return CopyRows<gysk_cluster_row> {out}; }
CopyRows<gysk_logical_trace> logical_finish(const gysk_engine *, gysk_logical_trace *out) { return CopyRows<gysk_logical_trace> {out}; }
ClientRows logical_finish(const gysk_engine *, gysk_svc_clients *out) { return ClientRows {out}; }
CopyRows<gysk_svc_top_clients> logical_finish(const gysk_engine *, gysk_svc_top_clients *out) { return CopyRows<gysk_svc_top_clients> {out}; }
uint64_t &row_id(gysk_svc_summary &r) { return r.glob_id; }
uint64_t &row_id(gysk_logical_state &r) { return r.logical_id; }
uint64_t &row_id(gysk_cluster_row &r) { return r.cluster_id; }
uint64_t &row_id(gysk_logical_trace &r) { return r.logical_id; }
uint64_t &row_id(gysk_svc_clients &r) { return r.glob_id; }
uint64_t &row_id(gysk_svc_top_clients &r) { return r.glob_id; }
template <typename Row> constexpr uint32_t logical_flag()
{
	return std::is_same<Row, gysk_logical_state>::value ? GYSK_FLAG_MERGE_STATES : std::is_same<Row, gysk_cluster_row>::value ? GYSK_FLAG_MERGE_CLUSTERS :
		std::is_same<Row, gysk_logical_trace>::value ? GYSK_FLAG_MERGE_TRACES : std::is_same<Row, gysk_svc_clients>::value ? GYSK_FLAG_CLIENT_LEVELS :
		std::is_same<Row, gysk_svc_top_clients>::value ? GYSK_FLAG_SVC_TOP_CLIENTS : 0;
}

// gysk_query_logical / gysk_query_logical_states / gysk_query_cluster_states: the rows of n ids, in QCHUNK pieces, each row carrying its
// queried id (which: the summary of the top-client rows)
template <typename Row>
int logical_query_rows(gysk_engine *e, const uint64_t *ids, uint32_t n, Row *out, const char *what, int which = 0)
{
	CHECK_ENGINE(e);
	if ((!ids || !out) && n) return GYSK_ERR_INVAL;
	if ((e->cfg.flags & logical_flag<Row>()) != logical_flag<Row>()) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, (std::string("gysk_") + what + ": no finished merge").c_str());

	const RowSpace sp = row_space(mg, out);
	std::vector<int32_t> lidx(n);
	for (uint32_t i = 0; i < n; ++i) lidx[i] = dense_index(*sp.index, ids[i]);
	const auto rows = logical_finish(e, out);
	return staged_read(e, lidx.data(), n, QCHUNK, sizeof(Row), what, [&](const unsigned long long *d_l, uint32_t, uint32_t m) {
		return launch_logical(e, reinterpret_cast<const int32_t *>(d_l), m, out, which);
	}, [&](const uint8_t *h_rows, uint32_t off, uint32_t m) {
		rows(h_rows, off, m);
		for (uint32_t i = 0; i < m; ++i) row_id(out[off + i]) = ids[off + i];
	});
}

// gysk_query_logical_all / gysk_query_logical_states_all / gysk_query_cluster_states_all: every row of the index space in ascending id
// (the uploaded permutation, compacted on the device by logical_select_kernel under ACTIVE_ONLY), in pieces of up to WIN_ROWS rows the
// stage holds; *n = rows that match (which: the summary of the top-client rows)
template <typename Row>
int logical_all_rows(gysk_engine *e, uint32_t flags, Row *out, uint32_t cap, uint32_t *n, const char *what, int which = 0)
{
	CHECK_ENGINE(e);
	if (!n || (!out && cap) || (flags & ~GYSK_WINDOW_ACTIVE_ONLY)) return GYSK_ERR_INVAL;
	if ((e->cfg.flags & logical_flag<Row>()) != logical_flag<Row>()) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, (std::string("gysk_") + what + ": no finished merge").c_str());

	const RowSpace sp = row_space(mg, out);
	uint32_t total = sp.n;
	const int32_t *sel = sp.sorted;
	if ((flags & GYSK_WINDOW_ACTIVE_ONLY) && total) {
		unsigned long long *d_n = e->st.counters + CTR_NWINDOW, cnt = 0;
		launch_select(e, out, d_n);
		e->kernel_launches++;
		CU(e, cudaMemcpyAsync(&cnt, d_n, sizeof(cnt), cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaStreamSynchronize(e->stream));
		if (int rc = post_launch(e, (std::string(what) + " select").c_str())) return rc;
		total = (uint32_t)cnt;
		sel = sp.sel;
	}
	int rc = staged_read<uint64_t>(e, nullptr, std::min(cap, total), (uint32_t)std::min<size_t>(WIN_ROWS, STAGE_BYTES / sizeof(Row)), sizeof(Row), what,
			[&](const unsigned long long *, uint32_t off, uint32_t m) { return launch_logical(e, sel + off, m, out, which); }, logical_finish(e, out));
	if (rc) return rc;
	*n = total;
	return GYSK_OK;
}

// gysk_topn_global / gysk_topn_global_tasks: the first n winners of one list and their rows, the entries with a zero score left out
SvcRows topn_finish(const gysk_engine *e, gysk_svc_summary *rows) { return SvcRows {e->cfg.hll_p, rows}; }
CopyRows<gysk_task_summary> topn_finish(const gysk_engine *, gysk_task_summary *rows) { return CopyRows<gysk_task_summary> {rows}; }
template <typename Row>
int topn_global_rows(gysk_engine *e, int metric, uint32_t n, gysk_topn_entry *out, Row *rows, uint32_t *nout, const char *what)
{
	constexpr bool task = std::is_same<Row, gysk_task_summary>::value;
	CHECK_ENGINE(e);
	if (!out || !nout || n == 0 || n > TOPN_K || metric < 0 || (uint32_t)metric >= (task ? TOPN_LISTS - TOPN_SVC_LISTS : TOPN_SVC_LISTS))
		return GYSK_ERR_INVAL;
	if (!(e->cfg.flags & GYSK_FLAG_MERGE_TOPN)) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, (std::string("gysk_") + what + ": no finished merge").c_str());
	const uint32_t m = task ? TOPN_SVC_LISTS + (uint32_t)metric : (uint32_t)metric;
	const TopnLists w {mg.topn_final};
	constexpr size_t row_off = TOPN_K * sizeof(gysk_topn_entry);
	static_assert(row_off + TOPN_K * sizeof(gysk_svc_summary) <= STAGE_BYTES, "the stage holds one list's entries and rows");
	CU(e, cudaMemcpyAsync(e->h_wstage, w.ent(m), n * sizeof(gysk_topn_entry), cudaMemcpyDeviceToHost, e->stream));
	if (rows) CU(e, cudaMemcpyAsync(e->h_wstage + row_off, w.row(m, 0), n * sizeof(Row), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	if (int rc = post_launch(e, what)) return rc;
	const gysk_topn_entry *h = reinterpret_cast<const gysk_topn_entry *>(e->h_wstage);
	const auto finish = topn_finish(e, rows);
	uint32_t k = 0;
	for (uint32_t i = 0; i < n; ++i) {
		if (!h[i].glob_id || !h[i].score) continue;
		if (rows) finish(e->h_wstage + row_off + i * sizeof(Row), k, 1);
		out[k++] = h[i];
	}
	*nout = k;
	return GYSK_OK;
}

} // namespace

// ---- NCCL inside the library (SURVEY.md §8e): the whole merge step of one query window as ONE call -------------------
//
// A C++ madhava has no torch.distributed: it calls gysk_merge_global(engine, comm) per engine (one thread per GPU, or inside its
// own ncclGroupStart/End when one thread drives all eight). libnccl.so.2 is resolved at first use with dlopen — a process that
// already carries NCCL (torch) shares that copy — so single-GPU deployments and the CPU-side ABI tests need no NCCL at all.
namespace {

struct NcclApi
{
	void *h {nullptr};
	ncclResult_t (*GetUniqueId)(ncclUniqueId *) {nullptr};
	ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) {nullptr};
	ncclResult_t (*CommDestroy)(ncclComm_t) {nullptr};
	ncclResult_t (*CommCount)(const ncclComm_t, int *) {nullptr};
	ncclResult_t (*CommUserRank)(const ncclComm_t, int *) {nullptr};
	ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) {nullptr};
	ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) {nullptr};
	ncclResult_t (*GroupStart)() {nullptr};
	ncclResult_t (*GroupEnd)() {nullptr};
	const char *(*GetErrorString)(ncclResult_t) {nullptr};
	std::string err;
};

NcclApi *nccl_api()
{
	static NcclApi api;
	static std::once_flag once;
	std::call_once(once, [] {
		for (const char *name : {"libnccl.so.2", "libnccl.so"}) { api.h = dlopen(name, RTLD_NOW | RTLD_GLOBAL); if (api.h) break; }
		if (!api.h) { api.err = std::string("dlopen(libnccl.so.2): ") + (dlerror() ? dlerror() : "not found"); return; }
		auto sym = [&](const char *n) { void *p = dlsym(api.h, n); if (!p && api.err.empty()) api.err = std::string("libnccl lacks ") + n; return p; };
		api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
		api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
		api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
		api.CommCount = (decltype(api.CommCount))sym("ncclCommCount");
		api.CommUserRank = (decltype(api.CommUserRank))sym("ncclCommUserRank");
		api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
		api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
		api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
		api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
		api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
	});
	return api.err.empty() ? &api : nullptr;
}

int nccl_fail(gysk_engine *e, const char *what, ncclResult_t r)
{
	NcclApi *a = nccl_api();
	char buf[256];
	snprintf(buf, sizeof(buf), "%s: %s", what, a && a->GetErrorString ? a->GetErrorString(r) : "nccl error");
	return fail(e, GYSK_ERR_CUDA, buf);		// sticky, like a CUDA error
}

} // namespace

namespace gysk {
void merge_release(gysk_engine *e)
{
	if (e->mg.comm && e->mg.comm_owned) { NcclApi *a = nccl_api(); if (a) a->CommDestroy((ncclComm_t)e->mg.comm); }
	e->mg.comm = nullptr;
}
} // namespace gysk


namespace {

// A map's keys as dense indices in order of first appearance (identical on every rank when the same list is passed): ids[dense] = key,
// index[key] = dense. offs / pos: the list positions of each dense index in list order, CSR. sorted: the dense indices by ascending key.
struct DenseMap { std::vector<uint32_t> offs, pos; std::vector<int32_t> sorted; };
DenseMap dense_map(const uint64_t *keys, uint32_t n, std::vector<uint64_t> &ids, std::unordered_map<uint64_t, uint32_t> &index)
{
	index.clear(); ids.clear();
	std::vector<uint32_t> dense(n);
	for (uint32_t i = 0; i < n; ++i) {
		auto it = index.find(keys[i]);
		if (it == index.end()) {
			it = index.emplace(keys[i], (uint32_t)ids.size()).first;
			ids.push_back(keys[i]);
		}
		dense[i] = it->second;
	}
	const uint32_t nd = (uint32_t)ids.size();
	DenseMap m {std::vector<uint32_t>(nd + 1, 0), std::vector<uint32_t>(n), std::vector<int32_t>(nd)};
	for (uint32_t i = 0; i < n; ++i) m.offs[dense[i] + 1]++;
	for (uint32_t d = 0; d < nd; ++d) m.offs[d + 1] += m.offs[d];
	std::vector<uint32_t> cur(m.offs.begin(), m.offs.end() - 1);
	for (uint32_t i = 0; i < n; ++i) m.pos[cur[dense[i]]++] = i;
	for (uint32_t d = 0; d < nd; ++d) m.sorted[d] = (int32_t)d;
	std::sort(m.sorted.begin(), m.sorted.end(), [&](int32_t a, int32_t b) { return ids[a] < ids[b]; });
	return m;
}

// (Re)allocates the arena for the logical and cluster maps the engine holds; the last merge's results go with the old one.
int lay_out_arena(gysk_engine *e)
{
	MergeState &mg = e->mg;
	LogicalArrays &lg = mg.lg;
	const uint32_t nl = lg.nl;
	dfree(e, mg.arena);
	mg.prepared = mg.finished = false;

	// The arena region by region, each array 256-byte aligned: layout(nullptr) sizes it, layout(arena) places the arrays. Each array's
	// name joins its region's gysk_merge_buffers name. GYSK_FLAG_MERGE_LEVELS appends its arrays to the ends of the SUM and i64 MAX
	// regions, GYSK_FLAG_MERGE_STATES its words to the end of the SUM region after them, GYSK_FLAG_MERGE_CLUSTERS its words after those.
	// GYSK_FLAG_FLOW_LEVEL puts the count-min level after the two window tables, and needs the flush tsec pair as the levels do:
	// still three regions, three collectives. GYSK_FLAG_FLOW_QUERIES puts the two flow query tables after the count-min ones, and
	// GYSK_FLAG_FLOW_QUERY_LEVEL their level after them, with the flush tsec pair. GYSK_FLAG_FLOW_RESP_HIST puts the flow response
	// histograms (and with GYSK_FLAG_FLOW_QUERY_LEVEL their level) after all of them: 8 words a cell, summed like every other word.
	// GYSK_FLAG_FLOW_ERRORS puts the flow error tables (and with GYSK_FLAG_FLOW_QUERY_LEVEL their level) after those.
	// GYSK_FLAG_MERGE_TRACES puts its words at the end of the SUM region, its maxima at the end of the i64 MAX one, and needs the flush
	// tsec pair too. Only the flags and the maps size the arena (never max_trace_svcs).
	const bool levels = e->cfg.flags & GYSK_FLAG_MERGE_LEVELS, states = e->cfg.flags & GYSK_FLAG_MERGE_STATES, clusters = e->cfg.flags & GYSK_FLAG_MERGE_CLUSTERS;
	const bool flow_level = e->cfg.flags & (GYSK_FLAG_FLOW_LEVEL | GYSK_FLAG_FLOW_QUERY_LEVEL), traces = e->cfg.flags & GYSK_FLAG_MERGE_TRACES;
	const size_t b_hist = (size_t)nl * HIST_CELLS * sizeof(HistCell);
	auto layout = [&](uint8_t *base) {
		size_t off = 0;
		std::string names;
		auto take = [&](auto *&p, size_t bytes, const char *name) {
			if (base) p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(base + off);
			off += align256(bytes);
			names += (names.empty() ? "" : "|") + std::string(name);
		};
		mg.off_sum = off;
		for (int t = 0; t < NCMS; ++t) if (cms_held(e->cfg, t)) take(mg.g_cms[t], cms_words(e->cfg, t) * 8, CMS_TABLES[t].name);
		take(lg.last, b_hist, "hist_last"); take(lg.all, b_hist, "hist_all"); take(lg.conn, (size_t)nl * 4 * 8, "conn");
		if (levels) { take(lg.lvl, NLEVELS * b_hist, "levels"); take(lg.aux, (size_t)nl * 4 * 8, "aux"); }
		if (states) take(lg.states, (size_t)nl * STATE_WORDS * 8, "states");
		if (clusters) take(mg.clusters.cl.words, (size_t)mg.clusters.cl.nc * CLUSTER_WORDS * 8, "clusters");
		if (traces) take(lg.traces, (size_t)nl * LT_WORDS * 8, "traces");
		mg.bytes_sum = off - mg.off_sum;
		mg.name_sum = "sum_u64: " + names;
		names.clear();
		mg.off_maxi64 = off;
		take(lg.hmax, (size_t)nl * 2 * 8, "hist max_val_seen");
		if (levels) { take(lg.lvl_max, (size_t)nl * NLEVELS * 8, "level max_val_seen"); take(lg.rtt, (size_t)nl * 8, "rtt"); }
		if (levels || flow_level || traces) take(lg.flush, 2 * 8, "flush tsec");
		if (traces) take(lg.trace_max, (size_t)nl * LT_MAX_WORDS * 8, "trace max");
		mg.bytes_maxi64 = off - mg.off_maxi64;
		mg.name_maxi64 = "max_i64: " + names;
		names.clear();
		mg.off_maxu8 = off;
		take(lg.hll, (size_t)nl << e->cfg.hll_p, "hll registers");
		if (e->cfg.flags & GYSK_FLAG_CLIENT_LEVELS) take(mg.cl_hll, (size_t)nl * 2 * CL_REGS, "client registers");
		mg.bytes_maxu8 = off - mg.off_maxu8;
		mg.name_maxu8 = "max_u8: " + names;
		return off;
	};
	mg.arena_bytes = layout(nullptr);
	int rc = dalloc(e, &mg.arena, mg.arena_bytes);
	if (rc) return rc;
	layout(mg.arena);
	return 0;
}

// gysk_set_logical_map, engine held
int set_logical_map(gysk_engine *e, const uint64_t *glob_ids, const uint64_t *logical_ids, uint32_t n)
{
	MergeState &mg = e->mg;

	// dense logical index in order of first appearance; CSR logical -> every {glob_id} mapped to it, in map order (the slots are looked
	// up at merge time, resolve_members_kernel); dense indices by ascending logical id: the row order of gysk_query_logical_all
	const DenseMap dm = dense_map(logical_ids, n, mg.logical_ids, mg.index);
	const uint32_t nl = (uint32_t)mg.logical_ids.size();
	std::vector<uint64_t> member_ids(n);
	for (uint32_t k = 0; k < n; ++k) member_ids[k] = glob_ids[dm.pos[k]];

	// (re)allocate the arena
	dfree(e, mg.members.offs); dfree(e, mg.members.slots); dfree(e, mg.d_member_ids); dfree(e, mg.arena); dfree(e, mg.lg.slab); dfree(e, mg.lg.final_slab);
	dfree(e, mg.d_logical_ids); dfree(e, mg.d_sorted); dfree(e, mg.d_sel); dfree(e, mg.topn_slots); dfree(e, mg.topn_final); dfree(e, mg.lg.trace_final);
	dfree(e, mg.topk_final); dfree(e, mg.topk_buf); dfree(e, mg.topk_n); dfree(e, mg.topk_tiles); dfree(e, mg.topk5_final); dfree(e, mg.topc_final);
	{
		std::vector<uint64_t> ids_keep(std::move(mg.logical_ids));
		std::unordered_map<uint64_t, uint32_t> idx_keep(std::move(mg.index));
		ClusterMap clusters_keep(std::move(mg.clusters));
		void *comm_keep = mg.comm;
		const uint32_t world_keep = mg.comm_world;
		const bool owned_keep = mg.comm_owned;
		mg = MergeState {};
		mg.logical_ids = std::move(ids_keep); mg.index = std::move(idx_keep); mg.clusters = std::move(clusters_keep);
		mg.comm = comm_keep; mg.comm_world = world_keep; mg.comm_owned = owned_keep;		// gysk_nccl_comm_init's communicator stays
	}
	LogicalArrays &lg = mg.lg;
	lg.nl = nl;
	int rc = lay_out_arena(e);
	if (rc) return rc;
	// GYSK_FLAG_MERGE_TOPN: the candidates after the digests, in whole SlabEntrys, so the slab stays one all-gather; GYSK_FLAG_MERGE_TRACES:
	// the trace digests after them, packed as TraceSlabs in whole SlabEntrys
	const bool topn = e->cfg.flags & GYSK_FLAG_MERGE_TOPN, traces = e->cfg.flags & GYSK_FLAG_MERGE_TRACES;
	// GYSK_FLAG_FLOW_TOPK: the rank's last-window heaviest-flow sets after everything else; GYSK_FLAG_FLOW_TOPK_5MIN: its level sets
	// and their bounds after those; GYSK_FLAG_FLOW_TOPK_SLOW: its last-window slow set, and with the slow level set L (and B_L) after
	// those; GYSK_FLAG_FLOW_ERRORS: its last-window server-error set, and with its level L (and B_L), after the slow sets. The merged slow
	// sets are set [2] of topk_final / topk5_final, the merged server-error sets set [3]. GYSK_FLAG_SVC_TOP_CLIENTS: each logical service's
	// two summaries after everything else.
	const bool topk = e->cfg.flags & GYSK_FLAG_FLOW_TOPK, topk5 = e->cfg.flags & GYSK_FLAG_FLOW_TOPK_5MIN, topc = e->cfg.flags & GYSK_FLAG_SVC_TOP_CLIENTS;
	const uint32_t nslow = e->topk.open[2] ? (e->topk5.level[2] ? 2 : 1) : 0, nerr = e->topk.open[3] ? (e->topk5.level[3] ? 2 : 1) : 0;
	mg.trace_off = nl + (topn ? TOPN_SLAB_ENTRIES : 0);
	mg.topk_off = mg.trace_off + (traces ? trace_slab_entries(nl) : 0);
	mg.topk5_off = mg.topk_off + (topk ? TOPK_SLAB_ENTRIES : 0);
	mg.topks_off = mg.topk5_off + (topk5 ? TOPK_SLAB_ENTRIES : 0);
	mg.topke_off = mg.topks_off + (nslow ? topk_slab_entries(nslow) : 0);
	mg.topc_off = mg.topke_off + (nerr ? topk_slab_entries(nerr) : 0);
	mg.slab_entries = mg.topc_off + (topc ? topc_slab_entries(nl) : 0);
	if ((rc = dalloc(e, &lg.slab, mg.slab_entries ? mg.slab_entries : 1))) return rc;
	if (topk) {
		if ((rc = dalloc(e, &mg.topk_final, (nerr ? 4 : nslow ? 3 : 2) * (size_t)TOPK_SET_WORDS))) return rc;
		if ((rc = dalloc(e, &mg.topk_n, 1))) return rc;
	}
	if (topk5 && (rc = dalloc(e, &mg.topk5_final, (nerr == 2 ? 4 : nslow == 2 ? 3 : 2) * (size_t)TOPK_SET_WORDS))) return rc;
	if (topn) {
		if ((rc = dalloc(e, &mg.topn_slots, (size_t)TOPN_LISTS * TOPN_K))) return rc;
		if ((rc = dalloc(e, &mg.topn_final, TopnLists::BYTES))) return rc;
	}
	if (traces) {
		lg.trace_slab = reinterpret_cast<TraceSlab *>(lg.slab + mg.trace_off);
		if ((rc = dalloc(e, &lg.trace_final, nl ? nl : 1))) return rc;
	}
	if ((rc = dalloc(e, &lg.final_slab, nl ? nl : 1))) return rc;
	if (topc && (rc = dalloc(e, &mg.topc_final, nl ? 2 * (size_t)nl : 1))) return rc;
	if ((rc = dalloc(e, &mg.members.offs, (size_t)nl + 1))) return rc;
	if ((rc = dalloc(e, &mg.members.slots, (size_t)n + 1))) return rc;
	mg.members.null_slot = e->cfg.max_svcs;
	if ((rc = dalloc(e, &mg.d_member_ids, member_ids.size() + 1))) return rc;
	if ((rc = dalloc(e, &mg.d_logical_ids, nl ? nl : 1))) return rc;
	if ((rc = dalloc(e, &mg.d_sorted, nl ? nl : 1))) return rc;
	if ((rc = dalloc(e, &mg.d_sel, nl ? nl : 1))) return rc;
	if (nl) {
		CU(e, cudaMemcpyAsync(mg.d_logical_ids, mg.logical_ids.data(), (size_t)nl * sizeof(uint64_t), cudaMemcpyHostToDevice, e->stream));
		CU(e, cudaMemcpyAsync(mg.d_sorted, dm.sorted.data(), (size_t)nl * sizeof(int32_t), cudaMemcpyHostToDevice, e->stream));
	}
	// the member slots are written by resolve_members_kernel at every merge, before any fold reads them
	mg.nmembers = n;
	if (n) CU(e, cudaMemcpyAsync(mg.d_member_ids, member_ids.data(), (size_t)n * sizeof(uint64_t), cudaMemcpyHostToDevice, e->stream));
	CU(e, cudaMemcpyAsync(mg.members.offs, dm.offs.data(), ((size_t)nl + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	return post_launch(e, "set_logical_map");
}

} // namespace

extern "C" {

int gysk_set_logical_map(gysk_engine *e, const uint64_t *glob_ids, const uint64_t *logical_ids, uint32_t n)
{
	CHECK_ENGINE(e);
	if ((!glob_ids || !logical_ids) && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Sync);
	return set_logical_map(e, glob_ids, logical_ids, n);
}

int gysk_set_cluster_map(gysk_engine *e, const uint32_t *host_idxs, const uint64_t *cluster_ids, uint32_t n)
{
	CHECK_ENGINE(e);
	if ((!host_idxs || !cluster_ids) && n) return GYSK_ERR_INVAL;
	if (!(e->cfg.flags & GYSK_FLAG_MERGE_CLUSTERS)) return GYSK_ERR_NOTSUP;
	uint32_t ntab = 0;
	for (uint32_t i = 0; i < n; ++i) {
		if (host_idxs[i] >= MAX_CLUSTER_HOST) return GYSK_ERR_INVAL;
		ntab = std::max(ntab, host_idxs[i] + 1);
	}
	// host -> dense host index: the hosts of each cluster next to each other, in map order
	std::vector<uint32_t> host_of(ntab, ~0u);
	std::vector<uint64_t> ids;
	std::unordered_map<uint64_t, uint32_t> index;
	const DenseMap dm = dense_map(cluster_ids, n, ids, index);
	for (uint32_t k = 0; k < n; ++k) {
		uint32_t &h = host_of[host_idxs[dm.pos[k]]];
		if (h != ~0u) return GYSK_ERR_INVAL;			// a host listed twice
		h = k;
	}
	GYSK_ENTER(e, Sync);
	MergeState &mg = e->mg;
	ClusterMap &cm = mg.clusters;
	dfree(e, cm.cl.host_of); dfree(e, cm.cl.offs); dfree(e, cm.cl.host_acc); dfree(e, cm.d_ids); dfree(e, cm.d_sorted); dfree(e, cm.d_sel);
	cm = ClusterMap {};
	cm.ids = std::move(ids); cm.index = std::move(index);
	Clusters &cl = cm.cl;
	cl.nc = (uint32_t)cm.ids.size(); cl.nh = n; cl.ntab = ntab;
	int rc = 0;
	if ((rc = dalloc(e, &cl.host_of, ntab ? ntab : 1, false))) return rc;
	if ((rc = dalloc(e, &cl.offs, (size_t)cl.nc + 1, false))) return rc;
	if ((rc = dalloc(e, &cl.host_acc, n ? n : 1))) return rc;			// zeroed: the host pass keeps it so between merges
	if ((rc = dalloc(e, &cm.d_ids, cl.nc ? cl.nc : 1, false))) return rc;
	if ((rc = dalloc(e, &cm.d_sorted, cl.nc ? cl.nc : 1, false))) return rc;
	if ((rc = dalloc(e, &cm.d_sel, cl.nc ? cl.nc : 1, false))) return rc;
	if (ntab) CU(e, cudaMemcpyAsync(cl.host_of, host_of.data(), (size_t)ntab * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
	CU(e, cudaMemcpyAsync(cl.offs, dm.offs.data(), ((size_t)cl.nc + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
	if (cl.nc) {
		CU(e, cudaMemcpyAsync(cm.d_ids, cm.ids.data(), (size_t)cl.nc * sizeof(uint64_t), cudaMemcpyHostToDevice, e->stream));
		CU(e, cudaMemcpyAsync(cm.d_sorted, dm.sorted.data(), (size_t)cl.nc * sizeof(int32_t), cudaMemcpyHostToDevice, e->stream));
	}
	// the arena, or with no logical map yet an empty one (which lays out the arena): a merge of clusters alone needs nothing more
	rc = mg.lg.slab ? lay_out_arena(e) : set_logical_map(e, nullptr, nullptr, 0);
	if (rc) return rc;
	CU(e, cudaStreamSynchronize(e->stream));
	return post_launch(e, "set_cluster_map");
}

int gysk_merge_prepare(gysk_engine *e)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Submit);
	MergeState &mg = e->mg;
	// GYSK_FLAG_MERGE_TOPN and GYSK_FLAG_FLOW_TOPK need no map: without one, an empty logical map (as gysk_set_cluster_map sets up)
	if (!mg.arena && (e->cfg.flags & (GYSK_FLAG_MERGE_TOPN | GYSK_FLAG_FLOW_TOPK))) {
		if (int rc = set_logical_map(e, nullptr, nullptr, 0)) return rc;
	}
	if (!mg.arena) return fail(e, GYSK_ERR_INVAL, "gysk_merge_prepare: call gysk_set_logical_map first");

	const uint32_t nl = mg.lg.nl;

	for (int t = 0; t < NCMS; ++t)
		if (mg.g_cms[t]) CU(e, cudaMemcpyAsync(mg.g_cms[t], CMS_TABLES[t].live(e), cms_words(e->cfg, t) * 8, cudaMemcpyDeviceToDevice, e->stream));
	if (nl) {
		if (mg.nmembers) {
			resolve_members_kernel<<<div_up(mg.nmembers, 256), 256, 0, e->stream>>>(e->st, mg.d_member_ids, mg.nmembers, mg.members);
			e->kernel_launches++;
		}
		fold_hist_kernel<<<div_up((uint64_t)nl * HIST_CELLS, 256), 256, 0, e->stream>>>(e->st, mg.members, mg.lg);
		fold_hll_kernel<<<div_up((uint64_t)nl << (e->cfg.hll_p - 2), 256), 256, 0, e->stream>>>(e->st, mg.members, mg.lg);
		if (mg.cl_hll) {		// GYSK_FLAG_CLIENT_LEVELS
			fold_clients_kernel<<<div_up((uint64_t)nl * 2 * (CL_REGS / 4), 256), 256, 0, e->stream>>>(e->cl, mg.members, nl, mg.cl_hll);
			e->kernel_launches++;
		}
		fold_td_kernel<<<std::min<uint32_t>(div_up(nl, MG_WARPS), 132 * 8), MG_WARPS * 32, 0, e->stream>>>(e->st, mg.members, mg.lg);
		e->kernel_launches += 3;
		if (mg.lg.states) {		// GYSK_FLAG_MERGE_STATES
			fold_states_kernel<<<div_up(nl, 256), 256, 0, e->stream>>>(e->st, mg.members, mg.lg);
			e->kernel_launches++;
		}
		if (mg.lg.traces) {		// GYSK_FLAG_MERGE_TRACES: the counter words (the digests are in fold_td_kernel's pass)
			fold_traces_kernel<<<div_up((uint64_t)nl * LT_WORDS, 256), 256, 0, e->stream>>>(e->st, mg.members, mg.lg);
			e->kernel_launches++;
		}
		if (mg.topc_final) {		// GYSK_FLAG_SVC_TOP_CLIENTS
			fold_topc_kernel<<<std::min<uint32_t>(div_up(nl, TC_WARPS), 132 * 8), TC_WARPS * 32, 0, e->stream>>>(e->tc, mg.members, nl,
					reinterpret_cast<TopcSet *>(mg.lg.slab + mg.topc_off));
			e->kernel_launches++;
		}
	}
	if (mg.lg.flush) {		// GYSK_FLAG_MERGE_LEVELS, a count-min level or GYSK_FLAG_MERGE_TRACES: also with no logical service, for the flush tsec pair
		LogicalArrays lg = mg.lg;
		if (!lg.lvl) lg.nl = 0;		// without GYSK_FLAG_MERGE_LEVELS: the pair only
		fold_levels_kernel<<<std::max<uint32_t>(div_up((uint64_t)lg.nl * HIST_CELLS, 256), 1), 256, 0, e->stream>>>(e->st, mg.members,
				(long long)e->last_flush_tsec, lg);
		e->kernel_launches++;
	}
	if (const uint32_t nc = mg.clusters.cl.nc) {		// GYSK_FLAG_MERGE_CLUSTERS with a cluster map
		fold_cluster_hosts_kernel<<<div_up(e->cfg.max_svcs, 256), 256, 0, e->stream>>>(e->st, e->cfg.max_svcs, active_mark(e), mg.clusters.cl);
		fold_clusters_kernel<<<div_up(nc, 256), 256, 0, e->stream>>>(mg.clusters.cl);
		e->kernel_launches += 2;
	}
	if (mg.topn_final) {		// GYSK_FLAG_MERGE_TOPN
		// each list: the score kernel, radix sort and pick of gysk_topn_svcs / gysk_topn_tasks over every slot (max_svcs / max_tasks: the
		// slots past the table's count score 0, and the count stays on the device), its entries into the slab, its slots beside them; then
		// the rows of all the slots through the summary path of gysk_query_svcs / gysk_query_tasks. max_svcs, max_tasks >= 1: every pick
		// writes all TOPN_K entries and slots
		const TopnLists cand {reinterpret_cast<uint8_t *>(mg.lg.slab + nl)};
		for (uint32_t m = 0; m < TOPN_LISTS; ++m) {
			const bool task = m >= TOPN_SVC_LISTS;
			const int k = launch_topn(e->st, e->tmp, task ? e->cfg.max_tasks : e->cfg.max_svcs, task, task ? (int)(m - TOPN_SVC_LISTS) : (int)m, -1,
					TOPN_K, cand.ent(m), e->stream, mg.topn_slots + (size_t)m * TOPN_K);
			if (k < 0) return fail(e, GYSK_ERR_INVAL, "gysk_merge_prepare: top-N sort failed");
			e->kernel_launches += k;
		}
		e->kernel_launches += launch_svc_summaries(e->st, nullptr, mg.topn_slots, TOPN_SVC_LISTS * TOPN_K,
				reinterpret_cast<gysk_svc_summary *>(cand.row(0, 0)), e->stream);
		e->kernel_launches += launch_task_summaries(e->st, nullptr, mg.topn_slots + (size_t)TOPN_SVC_LISTS * TOPN_K, (TOPN_LISTS - TOPN_SVC_LISTS) * TOPN_K,
				reinterpret_cast<gysk_task_summary *>(cand.row(TOPN_SVC_LISTS, 0)), e->stream);
	}
	if (mg.topk_final) {		// GYSK_FLAG_FLOW_TOPK: the last-window sets (a set the engine does not hold: empty)
		unsigned long long *dst = reinterpret_cast<unsigned long long *>(mg.lg.slab + mg.topk_off);
		for (int w = 0; w < 2; ++w) {
			unsigned long long *d = dst + (size_t)w * TOPK_SET_WORDS;
			if (e->topk.last[w]) CU(e, cudaMemcpyAsync(d, e->topk.last[w], sizeof(unsigned long long) * TOPK_SET_WORDS, cudaMemcpyDeviceToDevice, e->stream));
			else CU(e, cudaMemsetAsync(d, 0, sizeof(unsigned long long) * TOPK_SET_WORDS, e->stream));
		}
	}
	if (mg.topk5_final) {		// GYSK_FLAG_FLOW_TOPK_5MIN: the level sets with their bounds (a level the engine does not hold: empty)
		unsigned long long *dst = reinterpret_cast<unsigned long long *>(mg.lg.slab + mg.topk5_off);
		for (int w = 0; w < 2; ++w) {
			unsigned long long *d = dst + (size_t)w * TOPK_SET_WORDS;
			if (e->topk5.level[w]) CU(e, cudaMemcpyAsync(d, e->topk5.level[w], sizeof(unsigned long long) * TOPK_SET_WORDS, cudaMemcpyDeviceToDevice, e->stream));
			else CU(e, cudaMemsetAsync(d, 0, sizeof(unsigned long long) * TOPK_SET_WORDS, e->stream));
		}
	}
	if (e->topk.open[2]) {		// GYSK_FLAG_FLOW_TOPK_SLOW: the last-window slow set, then with the slow level its L and B_L
		unsigned long long *dst = reinterpret_cast<unsigned long long *>(mg.lg.slab + mg.topks_off);
		CU(e, cudaMemcpyAsync(dst, e->topk.last[2], sizeof(unsigned long long) * TOPK_SET_WORDS, cudaMemcpyDeviceToDevice, e->stream));
		if (e->topk5.level[2])
			CU(e, cudaMemcpyAsync(dst + TOPK_SET_WORDS, e->topk5.level[2], sizeof(unsigned long long) * TOPK_SET_WORDS, cudaMemcpyDeviceToDevice, e->stream));
	}
	if (e->topk.open[3]) {		// GYSK_FLAG_FLOW_ERRORS: the last-window server-error set, then with the error level its L and B_L
		unsigned long long *dst = reinterpret_cast<unsigned long long *>(mg.lg.slab + mg.topke_off);
		CU(e, cudaMemcpyAsync(dst, e->topk.last[3], sizeof(unsigned long long) * TOPK_SET_WORDS, cudaMemcpyDeviceToDevice, e->stream));
		if (e->topk5.level[3])
			CU(e, cudaMemcpyAsync(dst + TOPK_SET_WORDS, e->topk5.level[3], sizeof(unsigned long long) * TOPK_SET_WORDS, cudaMemcpyDeviceToDevice, e->stream));
	}
	// no host sync: the caller enqueues the collectives on gysk_stream(e) (stream order) or calls gysk_sync() first
	mg.prepared = true; mg.finished = false;
	return post_launch(e, "merge_prepare");
}

int gysk_merge_buffers(gysk_engine *e, gysk_buffer_desc *out, uint32_t cap, uint32_t *n)
{
	CHECK_ENGINE(e);
	if (!out || !n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.arena) return fail(e, GYSK_ERR_INVAL, "gysk_merge_buffers: call gysk_set_logical_map first");
	if (cap < 3) return GYSK_ERR_NOSPC;
	out[0] = gysk_buffer_desc {mg.name_sum.c_str(), mg.arena + mg.off_sum, mg.bytes_sum, GYSK_RED_SUM_U64, 0};
	out[1] = gysk_buffer_desc {mg.name_maxi64.c_str(), mg.arena + mg.off_maxi64, mg.bytes_maxi64, GYSK_RED_MAX_I64, 0};
	out[2] = gysk_buffer_desc {mg.name_maxu8.c_str(), mg.arena + mg.off_maxu8, mg.bytes_maxu8, GYSK_RED_MAX_U8, 0};
	*n = 3;
	return GYSK_OK;
}

int gysk_merge_tdigest_slab(gysk_engine *e, void **dptr, uint64_t *nbytes)
{
	CHECK_ENGINE(e);
	if (!dptr || !nbytes) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	if (!e->mg.lg.slab) return fail(e, GYSK_ERR_INVAL, "gysk_merge_tdigest_slab: call gysk_set_logical_map first");
	*dptr = e->mg.lg.slab; *nbytes = (uint64_t)e->mg.slab_entries * sizeof(SlabEntry);
	return GYSK_OK;
}

int gysk_merge_finish(gysk_engine *e, const void *d_gathered, uint32_t world)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.prepared) return fail(e, GYSK_ERR_INVAL, "gysk_merge_finish: call gysk_merge_prepare first");
	if (!world) world = 1;
	const SlabEntry *src = d_gathered ? static_cast<const SlabEntry *>(d_gathered) : mg.lg.slab;
	if (!d_gathered) world = 1;
	if (mg.lg.nl) {
		finish_td_kernel<<<std::min<uint32_t>(div_up(mg.lg.nl, MG_WARPS), 132 * 8), MG_WARPS * 32, 0, e->stream>>>(src, world, mg.slab_entries, mg.lg,
				e->st.td, mg.trace_off, e->st.trace.td);
		e->kernel_launches++;
	}
	if (mg.topc_final && mg.lg.nl) {		// GYSK_FLAG_SVC_TOP_CLIENTS
		finish_topc_kernel<<<std::min<uint32_t>(div_up(mg.lg.nl, TC_WARPS), 132 * 8), TC_WARPS * 32, 0, e->stream>>>(src, world, mg.slab_entries,
				mg.topc_off, mg.lg.nl, mg.topc_final);
		e->kernel_launches++;
	}
	if (mg.topn_final) {		// GYSK_FLAG_MERGE_TOPN
		topn_global_kernel<<<TOPN_LISTS, 256, 0, e->stream>>>(src, world, mg.slab_entries, mg.lg.nl, TopnLists {mg.topn_final});
		e->kernel_launches++;
	}
	if (mg.topk_final) {		// GYSK_FLAG_FLOW_TOPK: per held set the union of every rank's, scored on the summed last-window table
		const uint64_t need = (uint64_t)world * TOPK_K;
		if (need > mg.topk_cap) {
			dfree(e, mg.topk_buf); dfree(e, mg.topk_tiles);
			mg.topk_cap = 0;
			if (int rc = dalloc(e, &mg.topk_buf, 3 * (size_t)need, false)) return rc;
			if (int rc = dalloc(e, &mg.topk_tiles, (size_t)RADIX_MAX * ((need + SORT_TILE - 1) / SORT_TILE))) return rc;
			mg.topk_cap = need;
		}
		// the union's own candidates and sort buffers: the engine's stay with its open sets
		SortTemp t = e->tmp;
		t.keys_a = mg.topk_buf + mg.topk_cap; t.keys_b = mg.topk_buf + 2 * mg.topk_cap;
		t.tile_status = mg.topk_tiles; t.max_tiles = (uint32_t)((mg.topk_cap + SORT_TILE - 1) / SORT_TILE);
		const TopkList l {mg.topk_buf, mg.topk_n, nullptr, mg.topk_cap};
		const size_t stride = (size_t)mg.slab_entries * sizeof(SlabEntry) / sizeof(unsigned long long);
		// the rank's window set w in the slab (the slow and server-error sets each in their own region)
		auto slab_set = [&](int w, bool level) {
			const uint32_t off = w < 2 ? (level ? mg.topk5_off : mg.topk_off) : w == 2 ? mg.topks_off : mg.topke_off;
			const unsigned long long *base = reinterpret_cast<const unsigned long long *>(src + off);
			return base + (size_t)(w < 2 ? w : level ? 1 : 0) * TOPK_SET_WORDS;
		};
		for (int w = 0; w < TOPK_SETS; ++w) {
			unsigned long long *set = mg.topk_final + (size_t)w * TOPK_SET_WORDS;
			if (!e->topk.last[w]) continue;
			e->kernel_launches += launch_topk_gather(slab_set(w, false), world, stride, l, e->stream);
			const int k = launch_topk_select(t, l, need, mg.g_cms[TOPK_TABLE[w] + 1], e->cfg.cms_depth, e->cfg.cms_log2_width, topk_score(e->topk, w), set,
					false, e->stream);
			if (k < 0) return fail(e, GYSK_ERR_INVAL, "gysk_merge_finish: heaviest-flow sort failed");
			e->kernel_launches += k;
		}
		// GYSK_FLAG_FLOW_TOPK_5MIN: per held level the union of every rank's level set, the K best on the summed level, with
		// B_G = max(thr(G), sum over ranks of B_L)
		for (int w = 0; w < TOPK_SETS && mg.topk5_final; ++w) {
			unsigned long long *set = mg.topk5_final + (size_t)w * TOPK_SET_WORDS;
			if (!e->topk5.level[w]) continue;
			const unsigned long long *sets = slab_set(w, true);
			const unsigned long long *tbl = mg.g_cms[TOPK5_LEVEL[w]];
			const int score = topk_score(e->topk, w);
			e->kernel_launches += launch_topk_gather(sets, world, stride, l, e->stream);
			const int k = launch_topk_select(t, l, need, tbl, e->cfg.cms_depth, e->cfg.cms_log2_width, score, set, false, e->stream);
			if (k < 0) return fail(e, GYSK_ERR_INVAL, "gysk_merge_finish: 300-s heaviest-flow sort failed");
			e->kernel_launches += k + launch_topk_bound(set, tbl, e->cfg.cms_depth, e->cfg.cms_log2_width, score, sets + 1, stride, world, ~0u,
					false, set + 1, e->stream);
		}
		mg.topk_done = true;
	}
	mg.finished = true;			// stream-ordered; the query calls synchronise
	return post_launch(e, "merge_finish");
}

int gysk_query_logical(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_svc_summary *out)
{
	return logical_query_rows(e, logical_ids, n, out, "query_logical");
}

// every logical service's row in ascending logical id, each byte-equal to its gysk_query_logical row
int gysk_query_logical_all(gysk_engine *e, uint32_t flags, gysk_svc_summary *out, uint32_t cap, uint32_t *n)
{
	return logical_all_rows(e, flags, out, cap, n, "query_logical_all");
}

// GYSK_FLAG_MERGE_STATES: the members' LISTEN_SUMM_STATS of logical ids, rows made on the device (logical_state_kernel)
int gysk_query_logical_states(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_logical_state *out)
{
	return logical_query_rows(e, logical_ids, n, out, "query_logical_states");
}

// GYSK_FLAG_MERGE_STATES: every logical service's state row, the rows of gysk_query_logical_all
int gysk_query_logical_states_all(gysk_engine *e, uint32_t flags, gysk_logical_state *out, uint32_t cap, uint32_t *n)
{
	return logical_all_rows(e, flags, out, cap, n, "query_logical_states_all");
}

// GYSK_FLAG_MERGE_CLUSTERS: the merged service half of MS_CLUSTER_STATE of cluster ids, rows made on the device (cluster_row_kernel)
int gysk_query_cluster_states(gysk_engine *e, const uint64_t *cluster_ids, uint32_t n, gysk_cluster_row *out)
{
	return logical_query_rows(e, cluster_ids, n, out, "query_cluster_states");
}

// GYSK_FLAG_MERGE_CLUSTERS: every cluster's row in ascending cluster id
int gysk_query_cluster_states_all(gysk_engine *e, uint32_t flags, gysk_cluster_row *out, uint32_t cap, uint32_t *n)
{
	return logical_all_rows(e, flags, out, cap, n, "query_cluster_states_all");
}

// GYSK_FLAG_MERGE_TRACES: the members' last trace windows merged, rows made on the device (logical_trace_kernel)
int gysk_query_logical_traces(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_logical_trace *out)
{
	return logical_query_rows(e, logical_ids, n, out, "query_logical_traces");
}

// GYSK_FLAG_MERGE_TRACES: every logical service's trace row, in the order of gysk_query_logical_all
int gysk_query_logical_traces_all(gysk_engine *e, uint32_t flags, gysk_logical_trace *out, uint32_t cap, uint32_t *n)
{
	return logical_all_rows(e, flags, out, cap, n, "query_logical_traces_all");
}

// GYSK_FLAG_MERGE_TRACES: the merged trace digest of one logical service, with the contract of gysk_export_logical_tdigest
int gysk_export_logical_trace_tdigest(gysk_engine *e, uint64_t logical_id, double *means, uint64_t *weights, uint32_t cap, uint32_t *n,
		double *minv, double *maxv)
{
	CHECK_ENGINE(e);
	if (!means || !weights || !n) return GYSK_ERR_INVAL;
	if (!(e->cfg.flags & GYSK_FLAG_MERGE_TRACES)) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, "gysk_export_logical_trace_tdigest: no finished merge");
	const int32_t l = logical_index(mg, logical_id);
	if (l < 0) return GYSK_ERR_NOENT;
	CU(e, cudaMemcpyAsync(e->h_wstage, mg.lg.trace_final + l, sizeof(TraceSlab), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	const TraceSlab &s = *reinterpret_cast<const TraceSlab *>(e->h_wstage);
	return tdigest_out(s.head, s.cent, means, weights, cap, n, minv, maxv);
}

int gysk_export_logical_trace_tdigest_pgtext(gysk_engine *e, uint64_t logical_id, char *buf, uint32_t cap)
{
	double means[TRACE_TD_CAP], mn, mx;
	uint64_t weights[TRACE_TD_CAP];
	uint32_t n = 0;
	int rc = gysk_export_logical_trace_tdigest(e, logical_id, means, weights, TRACE_TD_CAP, &n, &mn, &mx);
	if (rc) return rc;
	return gysk_tdigest_to_pgtext(means, weights, n, TRACE_TD_DELTA, buf, cap);		// at compression 100 already: no recompress
}

int gysk_export_logical_hist(gysk_engine *e, uint64_t logical_id, int which, gysk_hist_serial out[GYSK_HIST_MAX_BUCKETS], uint64_t *total,
		int64_t *maxv)
{
	CHECK_ENGINE(e);
	if (!out || !total || !maxv) return GYSK_ERR_INVAL;
	const bool level = which == GYSK_HIST_RESP_5MIN || which == GYSK_HIST_RESP_5DAY;
	if (!level && which != GYSK_HIST_RESP_LAST && which != GYSK_HIST_RESP_ALL) return GYSK_ERR_INVAL;
	if (level && !(e->cfg.flags & GYSK_FLAG_MERGE_LEVELS)) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, "gysk_export_logical_hist: no finished merge");
	const int32_t l = logical_index(mg, logical_id);
	if (l < 0) return GYSK_ERR_NOENT;
	const LogicalArrays::Hist src = mg.lg.hist(which, (uint32_t)l);
	// the 15 cells, then max_val_seen_ into cell 15 (stream order: behind the merge that wrote them)
	HistCell *h = reinterpret_cast<HistCell *>(e->h_wstage);
	CU(e, cudaMemcpyAsync(h, src.cells, HIST_CELLS * sizeof(HistCell), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaMemcpyAsync(&h[HIST_MAX_CELL].sum, src.max, sizeof(long long), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	if (level) level_from_cells(h, out, total, maxv);
	else hist_from_cells(h, 15, out, total, maxv, false);
	return GYSK_OK;
}

// score every logical service, sort the keys, pick the n best: the top-N path of gysk_topn_svcs over the merged arrays
int gysk_topn_logical(gysk_engine *e, int metric, uint32_t n, gysk_topn_entry *out, uint32_t *nout)
{
	CHECK_ENGINE(e);
	if (!out || !nout || n == 0 || n > 64 || metric < GYSK_TOPN_QPS || metric > GYSK_TOPN_ACTIVE) return GYSK_ERR_INVAL;
	if (metric == GYSK_TOPN_ISSUE && !(e->cfg.flags & GYSK_FLAG_MERGE_STATES)) return GYSK_ERR_INVAL;
	if (metric == GYSK_TOPN_ACTIVE && !(e->cfg.flags & GYSK_FLAG_MERGE_LEVELS)) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, "gysk_topn_logical: no finished merge");
	const uint32_t nl = mg.lg.nl;
	*nout = 0;
	if (!nl) return GYSK_OK;
	if (nl > e->tmp.nkeys) return fail(e, GYSK_ERR_NOSPC, "gysk_topn_logical: more logical services than the sort buffers hold");
	unsigned long long *d_n = e->st.counters + CTR_NWINDOW;
	gysk_topn_entry *d_out = reinterpret_cast<gysk_topn_entry *>(e->d_wstage);
	logical_topn_score_kernel<<<div_up(nl, 256), 256, 0, e->stream>>>(mg.lg, metric, e->tmp.keys_a, d_n);
	const int picked = launch_topn_pick(e->tmp, d_n, nl, mg.d_logical_ids, nullptr, n, d_out, e->stream);
	if (picked < 0) return fail(e, GYSK_ERR_INVAL, "gysk_topn_logical: sort failed");
	e->kernel_launches += 1 + picked;
	CU(e, cudaMemcpyAsync(e->h_wstage, d_out, sizeof(gysk_topn_entry) * n, cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	if (int rc = post_launch(e, "gysk_topn_logical")) return rc;
	const gysk_topn_entry *h = reinterpret_cast<const gysk_topn_entry *>(e->h_wstage);
	uint32_t k = 0;
	for (uint32_t i = 0; i < std::min(n, nl); ++i) if (h[i].score) out[k++] = h[i];
	*nout = k;
	return GYSK_OK;
}

// the merged digest of one logical service, with the contract of gysk_export_tdigest
int gysk_export_logical_tdigest(gysk_engine *e, uint64_t logical_id, double *means, uint64_t *weights, uint32_t cap, uint32_t *n, double *minv,
		double *maxv)
{
	CHECK_ENGINE(e);
	if (!means || !weights || !n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, "gysk_export_logical_tdigest: no finished merge");
	const int32_t l = logical_index(mg, logical_id);
	if (l < 0) return GYSK_ERR_NOENT;
	CU(e, cudaMemcpyAsync(e->h_wstage, mg.lg.final_slab + l, sizeof(SlabEntry), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	const SlabEntry &s = *reinterpret_cast<const SlabEntry *>(e->h_wstage);
	return tdigest_out(s.head, s.cent, means, weights, cap, n, minv, maxv);
}

int gysk_export_logical_tdigest_pgtext(gysk_engine *e, uint64_t logical_id, char *buf, uint32_t cap)
{
	return tdigest_pgtext(e, logical_id, gysk_export_logical_tdigest, buf, cap);
}

int gysk_query_logical_quantiles(gysk_engine *e, uint64_t logical_id, const double *qs, uint32_t nq, double *out)
{
	return tdigest_quantiles(e, logical_id, gysk_export_logical_tdigest, qs, nq, out);
}

// the merged HLL registers of one logical service, with the contract of gysk_export_hll
int gysk_export_logical_hll(gysk_engine *e, uint64_t logical_id, uint8_t *regs)
{
	CHECK_ENGINE(e);
	if (!regs) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, "gysk_export_logical_hll: no finished merge");
	const int32_t l = logical_index(mg, logical_id);
	if (l < 0) return GYSK_ERR_NOENT;
	const size_t nb = (size_t)1 << e->cfg.hll_p;
	CU(e, cudaMemcpyAsync(e->h_wstage, mg.lg.hll_of((uint32_t)l, e->cfg.hll_p), nb, cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	memcpy(regs, e->h_wstage, nb);
	return GYSK_OK;
}

// GYSK_FLAG_CLIENT_LEVELS: the merged client rows of n logical ids, and one logical service's merged client registers with the contract
// of gysk_export_logical_hll
int gysk_query_logical_clients(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_svc_clients *out)
{
	return logical_query_rows(e, logical_ids, n, out, "query_logical_clients");
}

// GYSK_FLAG_SVC_TOP_CLIENTS: summary `which` (GYSK_TOPC_LAST or GYSK_TOPC_5MIN) of n logical ids from the last finished merge, and of every
// logical service in the order of gysk_query_logical_all
int gysk_query_logical_top_clients(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, int which, gysk_svc_top_clients *out)
{
	CHECK_ENGINE(e);
	if (!(e->cfg.flags & GYSK_FLAG_SVC_TOP_CLIENTS)) return GYSK_ERR_NOTSUP;
	if (which != GYSK_TOPC_LAST && which != GYSK_TOPC_5MIN) return GYSK_ERR_INVAL;
	return logical_query_rows(e, logical_ids, n, out, "query_logical_top_clients", which);
}

int gysk_query_logical_top_clients_all(gysk_engine *e, uint32_t flags, int which, gysk_svc_top_clients *out, uint32_t cap, uint32_t *n)
{
	CHECK_ENGINE(e);
	if (!(e->cfg.flags & GYSK_FLAG_SVC_TOP_CLIENTS)) return GYSK_ERR_NOTSUP;
	if (which != GYSK_TOPC_LAST && which != GYSK_TOPC_5MIN) return GYSK_ERR_INVAL;
	return logical_all_rows(e, flags, out, cap, n, "query_logical_top_clients_all", which);
}

int gysk_export_logical_hll_window(gysk_engine *e, uint64_t logical_id, int which, uint8_t *regs)
{
	CHECK_ENGINE(e);
	if (!regs || (which != GYSK_CLIENTS_LAST && which != GYSK_CLIENTS_5MIN)) return GYSK_ERR_INVAL;
	if (!(e->cfg.flags & GYSK_FLAG_CLIENT_LEVELS)) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, "gysk_export_logical_hll_window: no finished merge");
	const int32_t l = logical_index(mg, logical_id);
	if (l < 0) return GYSK_ERR_NOENT;
	CU(e, cudaMemcpyAsync(e->h_wstage, mg.cl_of((uint32_t)l, which), CL_REGS, cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	memcpy(regs, e->h_wstage, CL_REGS);
	return GYSK_OK;
}

int gysk_merge_flush_range(gysk_engine *e, uint32_t *min_tsec, uint32_t *max_tsec)
{
	CHECK_ENGINE(e);
	if (!min_tsec || !max_tsec) return GYSK_ERR_INVAL;
	if (!(e->cfg.flags & (GYSK_FLAG_MERGE_LEVELS | GYSK_FLAG_FLOW_LEVEL | GYSK_FLAG_FLOW_QUERY_LEVEL | GYSK_FLAG_MERGE_TRACES))) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, "gysk_merge_flush_range: no finished merge");
	long long *h = reinterpret_cast<long long *>(e->h_wstage);
	CU(e, cudaMemcpyAsync(h, mg.lg.flush, 2 * sizeof(long long), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	*max_tsec = (uint32_t)h[0]; *min_tsec = (uint32_t)-h[1];
	return GYSK_OK;
}

// global count-min point query on the merged table
int gysk_query_flows_global(gysk_engine *e, const uint64_t *keys, uint32_t n, int last_window, gysk_flow_est *out)
{
	return query_cms(e, last_window ? CMS_LAST : CMS_CUR, true, keys, n, out, "query_flows_global");
}

// GYSK_FLAG_FLOW_LEVEL: the point query on the count-min level summed over the ranks
int gysk_query_flows_global_5min(gysk_engine *e, const uint64_t *keys, uint32_t n, gysk_flow_est *out)
{
	return query_cms(e, CMS_5MIN, true, keys, n, out, "query_flows_global_5min");
}

// GYSK_FLAG_FLOW_QUERIES: the point query on the flow query tables summed over the ranks
int gysk_query_flow_queries_global(gysk_engine *e, const uint64_t *keys, uint32_t n, int last_window, gysk_flow_qry_est *out)
{
	return query_cms(e, last_window ? CMS_QRY_LAST : CMS_QRY_CUR, true, keys, n, reinterpret_cast<gysk_flow_est *>(out), "query_flow_queries_global");
}

// GYSK_FLAG_FLOW_QUERY_LEVEL: the point query on the flow query level summed over the ranks
int gysk_query_flow_queries_global_5min(gysk_engine *e, const uint64_t *keys, uint32_t n, gysk_flow_qry_est *out)
{
	return query_cms(e, CMS_QRY_5MIN, true, keys, n, reinterpret_cast<gysk_flow_est *>(out), "query_flow_queries_global_5min");
}

// GYSK_FLAG_FLOW_RESP_HIST: the point query on the flow response histograms (and their level) summed over the ranks
int gysk_query_flow_resp_global(gysk_engine *e, const uint64_t *keys, uint32_t n, int last_window, gysk_flow_resp_est *out)
{
	return query_cms_resp(e, last_window ? CMS_RESP_LAST : CMS_RESP_CUR, true, keys, n, out, "query_flow_resp_global");
}

int gysk_query_flow_resp_global_5min(gysk_engine *e, const uint64_t *keys, uint32_t n, gysk_flow_resp_est *out)
{
	return query_cms_resp(e, CMS_RESP_5MIN, true, keys, n, out, "query_flow_resp_global_5min");
}

// GYSK_FLAG_FLOW_ERRORS: the point query on the flow error tables (and their level) summed over the ranks, with the summed queries
int gysk_query_flow_errors_global(gysk_engine *e, const uint64_t *keys, uint32_t n, int last_window, gysk_flow_err_est *out)
{
	return query_cms_err(e, last_window ? CMS_ERR_LAST : CMS_ERR_CUR, true, keys, n, out, "query_flow_errors_global");
}

int gysk_query_flow_errors_global_5min(gysk_engine *e, const uint64_t *keys, uint32_t n, gysk_flow_err_est *out)
{
	return query_cms_err(e, CMS_ERR_5MIN, true, keys, n, out, "query_flow_errors_global_5min");
}

#define NC(e, call) do { ncclResult_t r__ = (call); if (r__ != ncclSuccess) return nccl_fail((e), #call, r__); } while (0)

int gysk_nccl_unique_id(uint8_t out[GYSK_NCCL_UNIQUE_ID_BYTES])
{
	NcclApi *a = nccl_api();
	if (!out) return GYSK_ERR_INVAL;
	if (!a) return GYSK_ERR_NOTSUP;
	static_assert(sizeof(ncclUniqueId) == GYSK_NCCL_UNIQUE_ID_BYTES, "ncclUniqueId is 128 bytes");
	ncclUniqueId id;
	if (a->GetUniqueId(&id) != ncclSuccess) return GYSK_ERR_CUDA;
	memcpy(out, &id, sizeof(id));
	return GYSK_OK;
}

int gysk_nccl_comm_init(gysk_engine *e, const uint8_t uid[GYSK_NCCL_UNIQUE_ID_BYTES], uint32_t nranks, uint32_t rank)
{
	CHECK_ENGINE(e);
	if (!uid || !nranks || rank >= nranks) return GYSK_ERR_INVAL;
	NcclApi *a = nccl_api();
	if (!a) return fail(e, GYSK_ERR_NOTSUP, "libnccl.so.2 could not be loaded");
	GYSK_ENTER(e, Drain);
	if (e->mg.comm) { a->CommDestroy((ncclComm_t)e->mg.comm); e->mg.comm = nullptr; }
	ncclUniqueId id;
	memcpy(&id, uid, sizeof(id));
	ncclComm_t c = nullptr;
	NC(e, a->CommInitRank(&c, (int)nranks, id, (int)rank));
	e->mg.comm = c; e->mg.comm_world = nranks; e->mg.comm_owned = true;
	return GYSK_OK;
}

// prepare (fold) -> one grouped NCCL launch: all-reduce per reduction kind + all-gather of the t-digest slabs -> finish.
// comm == NULL uses the communicator of gysk_nccl_comm_init. Everything is enqueued on the engine's stream; nothing blocks.
int gysk_merge_global(gysk_engine *e, void *comm)
{
	CHECK_ENGINE(e);
	NcclApi *a = nccl_api();
	if (!a) return fail(e, GYSK_ERR_NOTSUP, "libnccl.so.2 could not be loaded");
	ncclComm_t c = comm ? (ncclComm_t)comm : (ncclComm_t)e->mg.comm;
	if (!c) return fail(e, GYSK_ERR_INVAL, "gysk_merge_global: no communicator (pass one or call gysk_nccl_comm_init)");
	int rc = gysk_merge_prepare(e);
	if (rc) return rc;
	int world = 0;
	{
		GYSK_ENTER(e, Drain);
		MergeState &mg = e->mg;
		NC(e, a->CommCount(c, &world));
		if (world < 1) return fail(e, GYSK_ERR_INVAL, "gysk_merge_global: empty communicator");
		if (mg.gathered_world != (uint32_t)world) {
			dfree(e, mg.gathered);
			if ((rc = dalloc(e, &mg.gathered, (size_t)(mg.slab_entries ? mg.slab_entries : 1) * world, false))) return rc;
			mg.gathered_world = (uint32_t)world;
		}
		const size_t slab = (size_t)mg.slab_entries * sizeof(SlabEntry);
		NC(e, a->GroupStart());
		NC(e, a->AllReduce(mg.arena + mg.off_sum, mg.arena + mg.off_sum, mg.bytes_sum / 8, ncclUint64, ncclSum, c, e->stream));
		NC(e, a->AllReduce(mg.arena + mg.off_maxi64, mg.arena + mg.off_maxi64, mg.bytes_maxi64 / 8, ncclInt64, ncclMax, c, e->stream));
		NC(e, a->AllReduce(mg.arena + mg.off_maxu8, mg.arena + mg.off_maxu8, mg.bytes_maxu8, ncclUint8, ncclMax, c, e->stream));
		if (slab) NC(e, a->AllGather(mg.lg.slab, mg.gathered, slab, ncclUint8, c, e->stream));
		NC(e, a->GroupEnd());
		e->merges++;
	}
	return gysk_merge_finish(e, e->mg.slab_entries ? e->mg.gathered : nullptr, (uint32_t)world);
}

// GYSK_FLAG_MERGE_TOPN: the winners of the last finished merge (topn_global_kernel)
// GYSK_FLAG_FLOW_TOPK: the heaviest flows of the last finished merge
int gysk_topk_flows_global(gysk_engine *e, uint32_t n, gysk_flow_est *out, uint32_t *nout)
{
	return topk_read(e, 0, 1, false, true, n, out, nout, nullptr, "topk_flows_global");
}

int gysk_topk_flow_queries_global(gysk_engine *e, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout)
{
	return topk_read(e, 1, 1, false, true, n, reinterpret_cast<gysk_flow_est *>(out), nout, nullptr, "topk_flow_queries_global");
}

// GYSK_FLAG_FLOW_TOPK_5MIN: the heaviest flows of the summed 300-s levels of the last finished merge, with B_G
int gysk_topk_flows_global_5min(gysk_engine *e, uint32_t n, gysk_flow_est *out, uint32_t *nout, uint64_t *bound)
{
	return topk_read(e, 0, 0, true, true, n, out, nout, bound, "topk_flows_global_5min");
}

int gysk_topk_flow_queries_global_5min(gysk_engine *e, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout, uint64_t *bound)
{
	return topk_read(e, 1, 0, true, true, n, reinterpret_cast<gysk_flow_est *>(out), nout, bound, "topk_flow_queries_global_5min");
}

// GYSK_FLAG_FLOW_TOPK_SLOW: the flows with the most slow responses over every rank, from the last finished merge
int gysk_topk_flow_slow_global(gysk_engine *e, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout)
{
	return topk_read(e, 2, 1, false, true, n, out, nout, nullptr, "topk_flow_slow_global");
}

int gysk_topk_flow_slow_global_5min(gysk_engine *e, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout, uint64_t *bound)
{
	return topk_read(e, 2, 0, true, true, n, out, nout, bound, "topk_flow_slow_global_5min");
}

// GYSK_FLAG_FLOW_ERRORS: the flows with the most server errors over every rank, from the last finished merge
int gysk_topk_flow_errors_global(gysk_engine *e, uint32_t n, gysk_flow_err_est *out, uint32_t *nout)
{
	return topk_read(e, 3, 1, false, true, n, out, nout, nullptr, "topk_flow_errors_global");
}

int gysk_topk_flow_errors_global_5min(gysk_engine *e, uint32_t n, gysk_flow_err_est *out, uint32_t *nout, uint64_t *bound)
{
	return topk_read(e, 3, 0, true, true, n, out, nout, bound, "topk_flow_errors_global_5min");
}

int gysk_topn_global(gysk_engine *e, int metric, uint32_t n, gysk_topn_entry *out, gysk_svc_summary *rows, uint32_t *nout)
{
	return topn_global_rows(e, metric, n, out, rows, nout, "topn_global");
}

int gysk_topn_global_tasks(gysk_engine *e, int metric, uint32_t n, gysk_topn_entry *out, gysk_task_summary *rows, uint32_t *nout)
{
	return topn_global_rows(e, metric, n, out, rows, nout, "topn_global_tasks");
}

} // extern "C"
