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
//                          levels and aux sums to the SUM region, their maxima, the rtt and the flush tsec pair to the i64 MAX one
//   (caller)               all-reduce each region once, all-gather the slab        — NCCL via torch.distributed
//   gysk_merge_finish      rank-ascending merge + compress of the gathered digests
//   gysk_query_logical     same summary fields as gysk_query_svcs, for logical ids
//   gysk_export_logical_hist / gysk_merge_flush_range   one merged histogram / the ranks' flush tsec range
//
// It is the additive roll-up of MS_CLUSTER_STATE::STATE_ONE::add_stats (common/gy_comm_proto.h:3199-3214) /
// SHCONN_HANDLER::aggregate_cluster_state (server/gy_shconnhdlr.cc:4583) and of GY_HISTOGRAM::update_from_serialized
// (common/gy_statistics.h:625-650): integer sums are order independent => bit-exact at any GPU count.
#include "gysk_engine.h"
#include "gysk_summary.cuh"

#include <climits>
#include <dlfcn.h>
#include <nccl.h>		// types only: the library is dlopen()ed, libgysketch.so carries no link-time dependency on it

using namespace gysk;

namespace gysk {

struct SlabEntry { TdHead head; Centroid cent[TD_CAP]; };

// The map keeps every {glob_id, logical} pair it was given; which of them live on this GPU, and in which slot, is looked up at
// every merge: a service that registers after gysk_set_logical_map takes part from its first window on, one that was evicted (or whose
// slot now belongs to another id) drops out. An id without a slot maps to the engine's null slot (index max_svcs: always in its
// just-created state, the identity of every fold), which the fold kernels skip.
__global__ void resolve_members_kernel(DevState st, const unsigned long long *__restrict__ member_ids, uint32_t n, uint32_t *__restrict__ members,
		uint32_t null_slot)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const int slot = member_ids[i] ? table_lookup(st.svc_tbl, member_ids[i], false) : -1;
	members[i] = slot >= 0 ? (uint32_t)slot : null_slot;
}

// one thread per (logical, cell)
__global__ void fold_hist_kernel(DevState st, const uint32_t *__restrict__ offs, const uint32_t *__restrict__ members, uint32_t nl, uint32_t null_slot,
		HistCell *__restrict__ l_last, HistCell *__restrict__ l_all, unsigned long long *__restrict__ l_conn, long long *__restrict__ l_hmax)
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (uint64_t)nl * HIST_CELLS) return;
	const uint32_t l = (uint32_t)(i >> 4);
	const int cell = (int)(i & 15);
	const uint32_t b = offs[l], e = offs[l + 1];

	if (cell < HIST_MAX_CELL) {
		HistCell a {0, 0}, c {0, 0};
		for (uint32_t m = b; m < e; ++m) {
			if (members[m] == null_slot) continue;
			const HistCell x = st.hist_last[(size_t)members[m] * HIST_CELLS + cell], y = st.hist_all[(size_t)members[m] * HIST_CELLS + cell];
			a.count += x.count; a.sum += x.sum; c.count += y.count; c.sum += y.sum;
		}
		l_last[i] = a; l_all[i] = c;
	}
	else {
		long long ml = LLONG_MIN, ma = LLONG_MIN;
		unsigned long long lc = 0, lk = 0, ac = 0, ak = 0;
		for (uint32_t m = b; m < e; ++m) {
			const uint32_t s = members[m];
			if (s == null_slot) continue;
			ml = max(ml, st.hist_last[(size_t)s * HIST_CELLS + HIST_MAX_CELL].sum);
			ma = max(ma, st.hist_all[(size_t)s * HIST_CELLS + HIST_MAX_CELL].sum);
			const unsigned long long cl = st.conn_last[s];
			lc += (uint32_t)cl; lk += cl >> 32; ac += st.conn_all_cnt[s]; ak += st.conn_all_kb[s];
		}
		l_last[i] = HistCell {0, 0}; l_all[i] = HistCell {0, 0};
		l_hmax[2 * l] = ml; l_hmax[2 * l + 1] = ma;
		l_conn[4 * l] = lc; l_conn[4 * l + 1] = lk; l_conn[4 * l + 2] = ac; l_conn[4 * l + 3] = ak;
	}
}

// GYSK_FLAG_MERGE_LEVELS, one thread per (logical, cell): cells 0..14 sum the live ring slots of both rolling levels over the members
// (live0 / live1: the masks gather_slot applies, so a member adds exactly the lvl[] of its own gysk_query_svcs row); the cell-15
// thread takes the level maxima, the aux words of the last closed window and the largest rtt. Thread 0 also writes this engine's
// {last flush tsec, -last flush tsec}, whose i64 max over the ranks gives their latest and earliest flush.
__global__ void fold_levels_kernel(DevState st, const uint32_t *__restrict__ offs, const uint32_t *__restrict__ members, uint32_t nl, uint32_t null_slot,
		uint32_t live0, uint32_t live1, long long flush_tsec, HistCell *__restrict__ l_lvl, unsigned long long *__restrict__ l_aux,
		long long *__restrict__ l_lvl_max, long long *__restrict__ l_rtt, long long *__restrict__ l_flush)
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i == 0) { l_flush[0] = flush_tsec; l_flush[1] = -flush_tsec; }
	if (i >= (uint64_t)nl * HIST_CELLS) return;
	const uint32_t l = (uint32_t)(i >> 4);
	const int cell = (int)(i & 15);
	const uint32_t b = offs[l], e = offs[l + 1];
	const size_t max_svcs = null_slot;		// the null slot is the index past the last one: the ring planes hold max_svcs slots
	auto ring = [&](int lv, int k, uint32_t s) -> const HistCell & {
		return st.hist_ring[(((size_t)lv * NSLOTS + k) * max_svcs + s) * HIST_CELLS + cell];
	};

	if (cell < HIST_MAX_CELL) {
		HistCell a[NLEVELS] {};
		for (uint32_t m = b; m < e; ++m) {
			const uint32_t s = members[m];
			if (s == null_slot) continue;
#pragma unroll
			for (int lv = 0; lv < NLEVELS; ++lv) {
				const uint32_t live = lv ? live1 : live0;
#pragma unroll
				for (int k = 0; k < NSLOTS; ++k) {
					if (!((live >> k) & 1u)) continue;
					const HistCell x = ring(lv, k, s);
					a[lv].count += x.count; a[lv].sum += x.sum;
				}
			}
		}
		for (int lv = 0; lv < NLEVELS; ++lv) l_lvl[((size_t)lv * nl + l) * HIST_CELLS + cell] = a[lv];
	}
	else {
		long long mx[NLEVELS] = {LLONG_MIN, LLONG_MIN};
		unsigned long long ac = 0, ak = 0, ce = 0, se = 0;
		uint32_t rtt = 0;
		for (uint32_t m = b; m < e; ++m) {
			const uint32_t s = members[m];
			if (s == null_slot) continue;
			for (int lv = 0; lv < NLEVELS; ++lv) {
				const uint32_t live = lv ? live1 : live0;
				for (int k = 0; k < NSLOTS; ++k) if ((live >> k) & 1u) mx[lv] = max(mx[lv], ring(lv, k, s).sum);
			}
			const SlotAux x = st.slot_aux[s];
			ac += (uint32_t)x.act_last; ak += x.act_last >> 32; ce += (uint32_t)x.err_last; se += x.err_last >> 32;
			rtt = max(rtt, x.rtt_last);
		}
		for (int lv = 0; lv < NLEVELS; ++lv) { l_lvl[((size_t)lv * nl + l) * HIST_CELLS + cell] = HistCell {0, 0}; l_lvl_max[2 * l + lv] = mx[lv]; }
		l_aux[4 * l] = ac; l_aux[4 * l + 1] = ak; l_aux[4 * l + 2] = ce; l_aux[4 * l + 3] = se;
		l_rtt[l] = rtt;
	}
}

// one thread per (logical, 4 registers): per-byte max over the member services
__global__ void fold_hll_kernel(DevState st, const uint32_t *__restrict__ offs, const uint32_t *__restrict__ members, uint32_t nl, uint32_t null_slot,
		uint32_t *__restrict__ l_hll)
{
	const uint32_t words = 1u << (st.hll_p - 2);
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= (uint64_t)nl * words) return;
	const uint32_t l = (uint32_t)(i / words), w = (uint32_t)(i % words);
	uint32_t acc = 0;

	for (uint32_t m = offs[l]; m < offs[l + 1]; ++m) {
		if (members[m] == null_slot) continue;
		acc = __vmaxu4(acc, reinterpret_cast<const uint32_t *>(st.hll + ((size_t)members[m] << st.hll_p))[w]);
	}
	l_hll[i] = acc;
}

static constexpr int MG_WARPS = 2;		// 2 x 17.8 KB of scratch: static shared memory

// one warp per logical service: fold member digests one after the other (member order = the order of the map call's list)
__global__ void __launch_bounds__(MG_WARPS * 32) fold_td_kernel(DevState st, const uint32_t *__restrict__ offs, const uint32_t *__restrict__ members,
		uint32_t nl, uint32_t null_slot, SlabEntry *__restrict__ slab)
{
	__shared__ TdScratch scratch[MG_WARPS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	TdScratch &S = scratch[wid];

	for (uint32_t l = blockIdx.x * MG_WARPS + wid; l < nl; l += gridDim.x * MG_WARPS) {
		uint32_t nacc = 0;
		unsigned long long total = 0;
		double mn = INFINITY, mx = -INFINITY;

		for (uint32_t m = offs[l]; m < offs[l + 1]; ++m) {
			const uint32_t s = members[m];
			if (s == null_slot) continue;
			const TdHead h = st.td_head[s];
			if (!h.n) continue;
			nacc = warp_merge_compress(S, S.newc, nacc, st.td_cent + (size_t)s * TD_CAP, h.n, S.newc, st.td);
			total += h.total; mn = fmin(mn, h.minv); mx = fmax(mx, h.maxv);
		}
		for (uint32_t c = lane; c < TD_CAP; c += 32) slab[l].cent[c] = c < nacc ? S.newc[c] : Centroid {0.0, 0};
		if (lane == 0) { TdHead h; h.total = total; h.minv = mn; h.maxv = mx; h.n = nacc; h.pad = 0; slab[l].head = h; }
		__syncwarp();
	}
}

// one warp per logical service over the all-gathered slabs [world][nl]
__global__ void __launch_bounds__(MG_WARPS * 32) finish_td_kernel(const SlabEntry *__restrict__ gathered, uint32_t world, uint32_t nl,
		SlabEntry *__restrict__ out, TdParams P)
{
	__shared__ TdScratch scratch[MG_WARPS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	TdScratch &S = scratch[wid];

	for (uint32_t l = blockIdx.x * MG_WARPS + wid; l < nl; l += gridDim.x * MG_WARPS) {
		uint32_t nacc = 0;
		unsigned long long total = 0;
		double mn = INFINITY, mx = -INFINITY;

		for (uint32_t r = 0; r < world; ++r) {			// fixed rank-ascending order => deterministic result
			const SlabEntry &e = gathered[(size_t)r * nl + l];
			if (!e.head.n) continue;
			nacc = warp_merge_compress(S, S.newc, nacc, e.cent, e.head.n, S.newc, P);
			total += e.head.total; mn = fmin(mn, e.head.minv); mx = fmax(mx, e.head.maxv);
		}
		for (uint32_t c = lane; c < TD_CAP; c += 32) out[l].cent[c] = c < nacc ? S.newc[c] : Centroid {0.0, 0};
		if (lane == 0) { TdHead h; h.total = total; h.minv = mn; h.maxv = mx; h.n = nacc; h.pad = 0; out[l].head = h; }
		__syncwarp();
	}
}

// the merged rolling levels and aux words (GYSK_FLAG_MERGE_LEVELS; lvl == nullptr without it)
struct LevelArrays { const HistCell *lvl; const unsigned long long *aux; const long long *lvl_max, *rtt; uint32_t nl; };

// read side: one warp per logical service, its merged arrays into a shared-memory SvcRaw, then the row of summarize_warp (the
// summary of gysk_query_svcs). The merge folds neither the current window, the connection bitmaps nor the per-slot state / qps /
// active-connection words: they are zero; so are the rolling levels and the aux words unless the engine merges them (lv.lvl).
// glob_id is left 0 for the host to fill in.
static constexpr int LG_WARPS = 4;
__global__ void __launch_bounds__(LG_WARPS * 32) logical_summary_kernel(const int32_t *__restrict__ lidx, uint32_t n, uint32_t hll_p,
		const HistCell *__restrict__ l_last, const HistCell *__restrict__ l_all, const unsigned long long *__restrict__ l_conn,
		const long long *__restrict__ l_hmax, const uint8_t *__restrict__ l_hll, const SlabEntry *__restrict__ slab, LevelArrays lv,
		gysk_svc_summary *__restrict__ out)
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
			HistCell a = l_last[(size_t)l * HIST_CELLS + lane], b = l_all[(size_t)l * HIST_CELLS + lane];
			if (lane == HIST_MAX_CELL) { a.sum = l_hmax[2 * l]; b.sum = l_hmax[2 * l + 1]; }
			r.last[lane] = a; r.all[lane] = b; r.cur[lane] = HistCell {0, 0};
			for (int k = 0; k < NLEVELS; ++k) {
				HistCell c {0, 0};
				if (lv.lvl) {
					c = lv.lvl[((size_t)k * lv.nl + l) * HIST_CELLS + lane];
					if (lane == HIST_MAX_CELL) c.sum = lv.lvl_max[2 * l + k];
				}
				r.lvl[k][lane] = c;
			}
			r.bm_cur[lane] = 0; r.bm_last[lane] = 0;
			r.qps[lane] = HistCell {0, 0}; r.act[lane] = HistCell {0, 0};
		}
		if (lane == 0) {
			r.conn_cur = 0;
			r.conn_last = (l_conn[4 * l] & 0xFFFFFFFFull) | (l_conn[4 * l + 1] << 32);
			r.conn_all_cnt = l_conn[4 * l + 2]; r.conn_all_kb = l_conn[4 * l + 3];
			r.td = slab[l].head;
			r.aux = SlotAux {0, 0, 0, 0, 0, 0};
			if (lv.lvl) {
				const unsigned long long *a = lv.aux + 4 * (size_t)l;
				r.aux.act_last = (a[0] & 0xFFFFFFFFull) | (a[1] << 32);
				r.aux.err_last = (a[2] & 0xFFFFFFFFull) | (a[3] << 32);
				r.aux.rtt_last = (uint32_t)lv.rtt[l];
			}
			r.sst = SlotState {0, 0, 0, 0, 0};
		}
		for (int i = lane; i < TD_CAP; i += 32) r.cent[i] = slab[l].cent[i];
		hll_hist_warp(l_hll + ((size_t)l << hll_p), hll_p, r.hll_hist, lane);
	}
	summarize_warp(r, 0, hll_p, summ[wid], out + q, lane);
}

} // namespace gysk

namespace {

inline uint32_t div_up(uint64_t a, uint64_t b) { return (uint32_t)((a + b - 1) / b); }
inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

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


extern "C" {

int gysk_set_logical_map(gysk_engine *e, const uint64_t *glob_ids, const uint64_t *logical_ids, uint32_t n)
{
	CHECK_ENGINE(e);
	if ((!glob_ids || !logical_ids) && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Sync);

	MergeState &mg = e->mg;

	// dense logical index in order of first appearance: identical on every rank when the same list is passed
	mg.index.clear(); mg.logical_ids.clear();
	std::vector<uint32_t> lidx(n);
	for (uint32_t i = 0; i < n; ++i) {
		auto it = mg.index.find(logical_ids[i]);
		if (it == mg.index.end()) {
			it = mg.index.emplace(logical_ids[i], (uint32_t)mg.logical_ids.size()).first;
			mg.logical_ids.push_back(logical_ids[i]);
		}
		lidx[i] = it->second;
	}
	const uint32_t nl = (uint32_t)mg.logical_ids.size();

	// CSR logical -> every {glob_id} mapped to it, in map order; the slots are looked up at merge time (resolve_members_kernel)
	std::vector<uint32_t> offs(nl + 1, 0), members(n, e->cfg.max_svcs);
	std::vector<uint64_t> member_ids(n);
	for (uint32_t i = 0; i < n; ++i) offs[lidx[i] + 1]++;
	for (uint32_t l = 0; l < nl; ++l) offs[l + 1] += offs[l];
	{
		std::vector<uint32_t> cur(offs.begin(), offs.end() - 1);
		for (uint32_t i = 0; i < n; ++i) member_ids[cur[lidx[i]]++] = glob_ids[i];
	}

	// (re)allocate the arena
	auto dfree = [&](void *p) { if (p) { cudaFree(p); e->dallocs.erase(std::remove(e->dallocs.begin(), e->dallocs.end(), p), e->dallocs.end()); } };
	dfree(mg.d_offsets); dfree(mg.d_members); dfree(mg.d_member_ids); dfree(mg.arena); dfree(mg.slab); dfree(mg.final_slab);
	{
		std::vector<uint64_t> ids_keep(std::move(mg.logical_ids));
		std::unordered_map<uint64_t, uint32_t> idx_keep(std::move(mg.index));
		mg = MergeState {};
		mg.logical_ids = std::move(ids_keep); mg.index = std::move(idx_keep);
	}
	mg.nlogical = nl;

	const size_t ncms = (size_t)e->cfg.cms_depth << e->cfg.cms_log2_width;
	const size_t b_cms = ncms * 8, b_hist = (size_t)nl * HIST_CELLS * sizeof(HistCell), b_conn = (size_t)nl * 4 * 8;
	size_t off = 0;
	mg.off_sum = off;
	const size_t o_cms_cur = off; off += align256(b_cms);
	const size_t o_cms_last = off; off += align256(b_cms);
	const size_t o_hl = off; off += align256(b_hist);
	const size_t o_ha = off; off += align256(b_hist);
	const size_t o_conn = off; off += align256(b_conn);
	// GYSK_FLAG_MERGE_LEVELS appends its arrays to the ends of the SUM and i64 MAX regions: still three regions, three collectives
	const bool levels = e->cfg.flags & GYSK_FLAG_MERGE_LEVELS;
	size_t o_lvl = 0, o_aux = 0, o_lmax = 0, o_rtt = 0, o_flush = 0;
	if (levels) {
		o_lvl = off; off += align256((size_t)NLEVELS * b_hist);
		o_aux = off; off += align256((size_t)nl * 4 * 8);
	}
	mg.bytes_sum = off - mg.off_sum;
	mg.off_maxi64 = off; const size_t o_hmax = off; off += align256((size_t)nl * 2 * 8);
	if (levels) {
		o_lmax = off; off += align256((size_t)nl * NLEVELS * 8);
		o_rtt = off; off += align256((size_t)nl * 8);
		o_flush = off; off += align256(2 * 8);
	}
	mg.bytes_maxi64 = off - mg.off_maxi64;
	mg.off_maxu8 = off; const size_t o_hll = off; off += align256((size_t)nl << e->cfg.hll_p); mg.bytes_maxu8 = off - mg.off_maxu8;
	mg.arena_bytes = off;

	int rc = dalloc(e, &mg.arena, mg.arena_bytes);
	if (rc) return rc;
	mg.g_cms_cur = reinterpret_cast<unsigned long long *>(mg.arena + o_cms_cur);
	mg.g_cms_last = reinterpret_cast<unsigned long long *>(mg.arena + o_cms_last);
	mg.l_hist_last = reinterpret_cast<HistCell *>(mg.arena + o_hl);
	mg.l_hist_all = reinterpret_cast<HistCell *>(mg.arena + o_ha);
	mg.l_conn = reinterpret_cast<unsigned long long *>(mg.arena + o_conn);
	mg.l_hmax = reinterpret_cast<long long *>(mg.arena + o_hmax);
	mg.l_hll = mg.arena + o_hll;
	if (levels) {
		mg.l_lvl = reinterpret_cast<HistCell *>(mg.arena + o_lvl);
		mg.l_aux = reinterpret_cast<unsigned long long *>(mg.arena + o_aux);
		mg.l_lvl_max = reinterpret_cast<long long *>(mg.arena + o_lmax);
		mg.l_rtt = reinterpret_cast<long long *>(mg.arena + o_rtt);
		mg.l_flush = reinterpret_cast<long long *>(mg.arena + o_flush);
	}
	mg.slab_bytes = (size_t)(nl ? nl : 1) * sizeof(SlabEntry);
	if ((rc = dalloc(e, &mg.slab, mg.slab_bytes))) return rc;
	if ((rc = dalloc(e, &mg.final_slab, mg.slab_bytes))) return rc;
	if ((rc = dalloc(e, &mg.d_offsets, (size_t)nl + 1))) return rc;
	if ((rc = dalloc(e, &mg.d_members, members.size() + 1))) return rc;
	if ((rc = dalloc(e, &mg.d_member_ids, member_ids.size() + 1))) return rc;
	mg.nmembers = (uint32_t)members.size();
	if (!member_ids.empty()) CU(e, cudaMemcpyAsync(mg.d_member_ids, member_ids.data(), member_ids.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, e->stream));
	CU(e, cudaMemcpyAsync(mg.d_offsets, offs.data(), ((size_t)nl + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
	if (!members.empty()) CU(e, cudaMemcpyAsync(mg.d_members, members.data(), members.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	return post_launch(e, "set_logical_map");
}

int gysk_merge_prepare(gysk_engine *e)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Submit);
	MergeState &mg = e->mg;
	if (!mg.arena) return fail(e, GYSK_ERR_INVAL, "gysk_merge_prepare: call gysk_set_logical_map first");

	const size_t b_cms = ((size_t)e->cfg.cms_depth << e->cfg.cms_log2_width) * 8;
	const uint32_t nl = mg.nlogical;

	CU(e, cudaMemcpyAsync(mg.g_cms_cur, e->st.cms_cur, b_cms, cudaMemcpyDeviceToDevice, e->stream));
	CU(e, cudaMemcpyAsync(mg.g_cms_last, e->st.cms_last, b_cms, cudaMemcpyDeviceToDevice, e->stream));
	if (nl) {
		const uint32_t null_slot = e->cfg.max_svcs;
		if (mg.nmembers) {
			resolve_members_kernel<<<div_up(mg.nmembers, 256), 256, 0, e->stream>>>(e->st, mg.d_member_ids, mg.nmembers, mg.d_members, null_slot);
			e->kernel_launches++;
		}
		fold_hist_kernel<<<div_up((uint64_t)nl * HIST_CELLS, 256), 256, 0, e->stream>>>(e->st, mg.d_offsets, mg.d_members, nl, null_slot,
				mg.l_hist_last, mg.l_hist_all, mg.l_conn, mg.l_hmax);
		fold_hll_kernel<<<div_up((uint64_t)nl << (e->cfg.hll_p - 2), 256), 256, 0, e->stream>>>(e->st, mg.d_offsets, mg.d_members, nl, null_slot,
				reinterpret_cast<uint32_t *>(mg.l_hll));
		fold_td_kernel<<<std::min<uint32_t>(div_up(nl, MG_WARPS), 132 * 8), MG_WARPS * 32, 0, e->stream>>>(e->st, mg.d_offsets, mg.d_members, nl, null_slot,
				reinterpret_cast<SlabEntry *>(mg.slab));
		e->kernel_launches += 3;
	}
	if (mg.l_lvl) {		// GYSK_FLAG_MERGE_LEVELS: also with no logical service, for the flush tsec pair
		fold_levels_kernel<<<std::max<uint32_t>(div_up((uint64_t)nl * HIST_CELLS, 256), 1), 256, 0, e->stream>>>(e->st, mg.d_offsets, mg.d_members,
				nl, e->cfg.max_svcs, live_mask(e, 0), live_mask(e, 1), (long long)e->last_flush_tsec, mg.l_lvl, mg.l_aux, mg.l_lvl_max, mg.l_rtt,
				mg.l_flush);
		e->kernel_launches++;
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
	const bool lv = mg.l_lvl != nullptr;
	out[0] = gysk_buffer_desc {lv ? "sum_u64: cms_cur|cms_last|hist_last|hist_all|conn|levels|aux" : "sum_u64: cms_cur|cms_last|hist_last|hist_all|conn",
			mg.arena + mg.off_sum, mg.bytes_sum, GYSK_RED_SUM_U64, 0};
	out[1] = gysk_buffer_desc {lv ? "max_i64: hist max_val_seen|level max_val_seen|rtt|flush tsec" : "max_i64: hist max_val_seen",
			mg.arena + mg.off_maxi64, mg.bytes_maxi64, GYSK_RED_MAX_I64, 0};
	out[2] = gysk_buffer_desc {"max_u8: hll registers", mg.arena + mg.off_maxu8, mg.bytes_maxu8, GYSK_RED_MAX_U8, 0};
	*n = 3;
	return GYSK_OK;
}

int gysk_merge_tdigest_slab(gysk_engine *e, void **dptr, uint64_t *nbytes)
{
	CHECK_ENGINE(e);
	if (!dptr || !nbytes) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	if (!e->mg.slab) return fail(e, GYSK_ERR_INVAL, "gysk_merge_tdigest_slab: call gysk_set_logical_map first");
	*dptr = e->mg.slab; *nbytes = (uint64_t)e->mg.nlogical * sizeof(SlabEntry);
	return GYSK_OK;
}

int gysk_merge_finish(gysk_engine *e, const void *d_gathered, uint32_t world)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.prepared) return fail(e, GYSK_ERR_INVAL, "gysk_merge_finish: call gysk_merge_prepare first");
	if (!world) world = 1;
	const SlabEntry *src = d_gathered ? static_cast<const SlabEntry *>(d_gathered) : reinterpret_cast<const SlabEntry *>(mg.slab);
	if (!d_gathered) world = 1;
	if (mg.nlogical) {
		finish_td_kernel<<<std::min<uint32_t>(div_up(mg.nlogical, MG_WARPS), 132 * 8), MG_WARPS * 32, 0, e->stream>>>(src, world, mg.nlogical,
				reinterpret_cast<SlabEntry *>(mg.final_slab), e->st.td);
		e->kernel_launches++;
	}
	mg.finished = true;			// stream-ordered; the query calls synchronise
	return post_launch(e, "merge_finish");
}

int gysk_query_logical(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_svc_summary *out)
{
	CHECK_ENGINE(e);
	if ((!logical_ids || !out) && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, "gysk_query_logical: no finished merge");

	std::vector<int32_t> lidx(n);		// dense logical index, -1 for an id the map does not have
	for (uint32_t i = 0; i < n; ++i) {
		auto it = mg.index.find(logical_ids[i]);
		lidx[i] = it == mg.index.end() ? -1 : (int32_t)it->second;
	}
	const SvcRows rows {e->cfg.hll_p, out};
	const LevelArrays lv {mg.l_lvl, mg.l_aux, mg.l_lvl_max, mg.l_rtt, mg.nlogical};
	return staged_read(e, lidx.data(), n, QCHUNK, sizeof(gysk_svc_summary), "query_logical", [&](const unsigned long long *d_l, uint32_t, uint32_t m) {
		logical_summary_kernel<<<div_up(m, LG_WARPS), LG_WARPS * 32, 0, e->stream>>>(reinterpret_cast<const int32_t *>(d_l), m, e->cfg.hll_p,
				mg.l_hist_last, mg.l_hist_all, mg.l_conn, mg.l_hmax, mg.l_hll, reinterpret_cast<const SlabEntry *>(mg.final_slab), lv,
				reinterpret_cast<gysk_svc_summary *>(e->d_wstage));
		return 1;
	}, [&](const uint8_t *h_rows, uint32_t off, uint32_t m) {
		rows(h_rows, off, m);
		for (uint32_t i = 0; i < m; ++i) out[off + i].glob_id = logical_ids[off + i];
	});
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
	const auto it = mg.index.find(logical_id);
	if (it == mg.index.end()) return GYSK_ERR_NOENT;
	const uint32_t l = it->second;
	const HistCell *cells;
	const long long *mx;
	if (level) {
		const int k = which - GYSK_HIST_RESP_5MIN;
		cells = mg.l_lvl + ((size_t)k * mg.nlogical + l) * HIST_CELLS; mx = mg.l_lvl_max + 2 * (size_t)l + k;
	}
	else {
		const int k = which == GYSK_HIST_RESP_ALL;
		cells = (k ? mg.l_hist_all : mg.l_hist_last) + (size_t)l * HIST_CELLS; mx = mg.l_hmax + 2 * (size_t)l + k;
	}
	// the 15 cells, then max_val_seen_ into cell 15 (stream order: behind the merge that wrote them)
	HistCell *h = reinterpret_cast<HistCell *>(e->h_wstage);
	CU(e, cudaMemcpyAsync(h, cells, HIST_CELLS * sizeof(HistCell), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaMemcpyAsync(&h[HIST_MAX_CELL].sum, mx, sizeof(long long), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	hist_from_cells(h, 15, out, total, maxv, false);
	if (level && *total == 0) *maxv = INT64_MIN;		// as gysk_export_hist answers an empty level
	return GYSK_OK;
}

int gysk_merge_flush_range(gysk_engine *e, uint32_t *min_tsec, uint32_t *max_tsec)
{
	CHECK_ENGINE(e);
	if (!min_tsec || !max_tsec) return GYSK_ERR_INVAL;
	if (!(e->cfg.flags & GYSK_FLAG_MERGE_LEVELS)) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.finished) return fail(e, GYSK_ERR_INVAL, "gysk_merge_flush_range: no finished merge");
	long long *h = reinterpret_cast<long long *>(e->h_wstage);
	CU(e, cudaMemcpyAsync(h, mg.l_flush, 2 * sizeof(long long), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	*max_tsec = (uint32_t)h[0]; *min_tsec = (uint32_t)-h[1];
	return GYSK_OK;
}

// global count-min point query on the merged table
int gysk_query_flows_global(gysk_engine *e, const uint64_t *keys, uint32_t n, int last_window, gysk_flow_est *out)
{
	CHECK_ENGINE(e);
	if ((!keys || !out) && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	MergeState &mg = e->mg;
	if (!mg.prepared) return fail(e, GYSK_ERR_INVAL, "gysk_query_flows_global: no merge");
	DevState st = e->st;
	st.cms_cur = mg.g_cms_cur; st.cms_last = mg.g_cms_last;
	return staged_read(e, keys, n, QCHUNK, sizeof(gysk_flow_est), "query_flows_global", [&](const unsigned long long *d_keys, uint32_t, uint32_t m) {
		return launch_query_flows(st, d_keys, m, last_window, reinterpret_cast<gysk_flow_est *>(e->d_wstage), e->stream);
	}, CopyRows<gysk_flow_est> {out});
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
			if (mg.gathered) { cudaFree(mg.gathered); e->dallocs.erase(std::remove(e->dallocs.begin(), e->dallocs.end(), (void *)mg.gathered), e->dallocs.end()); mg.gathered = nullptr; }
			if ((rc = dalloc(e, &mg.gathered, mg.slab_bytes * (size_t)world, false))) return rc;
			mg.gathered_world = (uint32_t)world;
		}
		const size_t slab = (size_t)mg.nlogical * sizeof(SlabEntry);
		NC(e, a->GroupStart());
		NC(e, a->AllReduce(mg.arena + mg.off_sum, mg.arena + mg.off_sum, mg.bytes_sum / 8, ncclUint64, ncclSum, c, e->stream));
		NC(e, a->AllReduce(mg.arena + mg.off_maxi64, mg.arena + mg.off_maxi64, mg.bytes_maxi64 / 8, ncclInt64, ncclMax, c, e->stream));
		NC(e, a->AllReduce(mg.arena + mg.off_maxu8, mg.arena + mg.off_maxu8, mg.bytes_maxu8, ncclUint8, ncclMax, c, e->stream));
		if (slab) NC(e, a->AllGather(mg.slab, mg.gathered, slab, ncclUint8, c, e->stream));
		NC(e, a->GroupEnd());
		e->merges++;
	}
	return gysk_merge_finish(e, e->mg.nlogical ? e->mg.gathered : nullptr, (uint32_t)world);
}

} // extern "C"
