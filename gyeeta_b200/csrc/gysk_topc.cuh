// gysk_topc.cuh — the merge of GYSK_FLAG_SVC_TOP_CLIENTS' summaries, one warp at a time: weighted Misra-Gries in its mergeable form
// (DESIGN.md §2). gysk_kernels.cu merges each service's batches and ring slots with it, gysk_merge.cu the members of each logical
// service and the ranks.
#pragma once

#include "gysk_kernels.cuh"

namespace gysk {

// the merge's order: kbytes descending, then flow key ascending
__device__ __forceinline__ bool topc_better(const TopcCand &a, const TopcCand &b) { return a.kb > b.kb || (a.kb == b.kb && a.key < b.key); }

// The K + 1 best candidates offered so far, in order, in a warp's shared list l, n of them (warp-uniform). Every lane calls with one
// candidate or none (valid false); the flow keys offered to one list are distinct. A round that beats nothing costs one ballot.
__device__ __forceinline__ void topc_offer(TopcCand *l, uint32_t &n, const TopcCand &c, bool valid, int lane)
{
	constexpr uint32_t K1 = TOPC_K + 1;
	const bool beat = valid && (n < K1 || topc_better(c, l[K1 - 1]));
	const unsigned m = __ballot_sync(0xffffffffu, beat);
	if (!m) return;
	const TopcCand mine = (uint32_t)lane < n ? l[lane] : TopcCand {0ull, 0ull, 0ull};
	uint32_t rl = (uint32_t)lane, rc = 0;		// ranks in the union of the list and this round's winners
	for (unsigned b = m; b; b &= b - 1) {
		const int j = __ffs(b) - 1;
		const TopcCand o {__shfl_sync(0xffffffffu, c.key, j), __shfl_sync(0xffffffffu, c.kb, j), __shfl_sync(0xffffffffu, c.conns, j)};
		if ((uint32_t)lane < n && topc_better(o, mine)) ++rl;
		if (beat && j != lane && topc_better(o, c)) ++rc;
	}
	if (beat) for (uint32_t i = 0; i < n; ++i) rc += topc_better(l[i], c);
	__syncwarp();
	if ((uint32_t)lane < n && rl < K1) l[rl] = mine;
	if (beat && rc < K1) l[rc] = c;
	n = min(n + (uint32_t)__popc(m), K1);
	__syncwarp();
}

// the merge's last steps from the K + 1 best groups l[0, n): c = the (K + 1)-th kbytes (0 with at most K groups), the groups above c
// kept as kbytes - c, in order, saturated at 2^32 - 1, the rest of the entries zero; delta = delta_in + c
__device__ __forceinline__ void topc_store(const TopcCand *l, uint32_t n, unsigned long long delta_in, TopcSet *out, int lane)
{
	const unsigned long long c = n > TOPC_K ? l[TOPC_K].kb : 0ull;
	if ((uint32_t)lane < TOPC_K) {
		gysk_topc_entry e {0ull, 0u, 0u};
		if ((uint32_t)lane < n && l[lane].kb > c) {
			e.flow_key = l[lane].key;
			e.kbytes = (uint32_t)min(l[lane].kb - c, 0xFFFFFFFFull);
			e.conns = (uint32_t)min(l[lane].conns, 0xFFFFFFFFull);
		}
		out->ent[lane] = e;
	}
	if (lane == 0) out->delta = delta_in + c;
	__syncwarp();
}

// the held entries of summary s (a prefix: kbytes > 0) into buf[m ..]; returns m + their number
__device__ __forceinline__ uint32_t topc_gather(const TopcSet *s, TopcCand *buf, uint32_t m, int lane)
{
	uint32_t kb = 0;
	if ((uint32_t)lane < TOPC_K) {
		const gysk_topc_entry e = s->ent[lane];
		kb = e.kbytes;
		if (kb) buf[m + lane] = TopcCand {e.flow_key, e.kbytes, e.conns};
	}
	const uint32_t k = (uint32_t)__popc(__ballot_sync(0xffffffffu, kb != 0));
	__syncwarp();
	return m + k;
}

// the groups of buf[0, m) by flow key (kbytes and conns summed, a group with 0 kbytes dropped) offered to the list
__device__ __forceinline__ void topc_offer_groups(const TopcCand *buf, uint32_t m, TopcCand *l, uint32_t &n, int lane)
{
	for (uint32_t i0 = 0; i0 < m; i0 += 32) {
		const uint32_t i = i0 + (uint32_t)lane;
		TopcCand c {0ull, 0ull, 0ull};
		bool first = i < m;
		if (first) {
			c = buf[i];
			for (uint32_t j = 0; j < m; ++j) {
				if (j == i || buf[j].key != c.key) continue;
				if (j < i) { first = false; break; }
				c.kb += buf[j].kb; c.conns += buf[j].conns;
			}
		}
		topc_offer(l, n, c, first && c.kb != 0, lane);
	}
}

} // namespace gysk
