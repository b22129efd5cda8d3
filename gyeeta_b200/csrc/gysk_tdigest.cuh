// gysk_tdigest.cuh — warp-level building blocks of the batched merging t-digest (shared by the ingest-side update
// kernel and the multi-GPU merge kernels). Definitions: DESIGN.md §2; CPU statement: oracle/gysk_oracle.c.
#pragma once

#include "gysk_device.cuh"

namespace gysk {

// K_1 scale function of the merging t-digest (Dunning), k spanning [-delta/2, delta/2]: k(q) = delta/pi asin(2q - 1). The compress
// step works on the FIXED unit grid of k: cell j = [q_j, q_j+1) with q_j = q(k = -delta/2 + j) = (sin(pi (j/delta - 1/2)) + 1)/2. In
// weight units cell j starts at T_j = (uint64) (q_j * W) (W = total weight, one double multiply, truncated), and an item of the
// merged list (sorted by mean, exclusive weight prefix P_i, weight w_i) belongs to the cell that holds its weight CENTRE:
// T_j <= P_i + w_i / 2 < T_j+1. All items of one cell become one cluster: at most delta clusters, each reaching past its cell by at
// most half of its first and half of its last item — the t-digest size bound — with no data-dependent chain: the first item of
// cell j is the first i with 2 P_i + w_i >= 2 T_j, i.e. (integers) with C_i = P_i + floor(w_i / 2) >= T_j — C grows with i and
// never exceeds the total, so no sum overflows — delta independent binary searches over C, which is what makes the step parallel. The centre and not the start: old centroids are items of every later compress, and a start-rule cluster takes its
// whole last item, so a digest fed through many batches widened with each one and kept far fewer than delta centroids (DESIGN.md
// §2). q_j is computed once on the host (libm sin, same expression in oracle/gysk_oracle.c) so that device, host and oracle use
// identical doubles.
struct TdParams { const double *qtab; uint32_t delta; uint32_t pad; };		// qtab[0 .. delta], device memory

template <int NMAX_>
struct TdWorkT				// per warp; NMAX = 2 x TD_CAP: 13.8 KB
{
	static constexpr int NMAX = NMAX_;			// capacity of the merged list
	double			mean[NMAX];			// merged list: means ...
	unsigned long long	pref[NMAX + 1];			// ... and exclusive weight prefix: weight of item i = pref[i+1] - pref[i]
	uint16_t		bounds[TD_CAP + 2];
	uint16_t		nxt[NMAX];
	double			src[NMAX];			// the means of both input lists, staged for the merge
};
using TdWork = TdWorkT<2 * TD_CAP>;			// shared memory (13.8 KB): two lists of together up to 2 x TD_CAP centroids
using TdWorkBig = TdWorkT<1120>;			// global scratch: TD_CAP old centroids + up to NBINS (848) items of a batch
struct TdScratch : TdWork		// + an accumulator list for the folds of the merge step: 14.3 KB
{
	Centroid		newc[TD_CAP];
};

// Stable merge by mean of two mean-sorted centroid lists (`a` first on ties), then the greedy K_1 pass; one warp.
// Both inputs are fully consumed into S.mean / S.pref before `out` is written, so `out` may alias `a` or `b`.
// B_STAGED: the caller has put b's means at S.src[na, na + nb) and its weights (< 2^16 each) at S.nxt[0, nb), and `b` is unused
// (warp_merge_compress_staged); otherwise a and b may live in shared or global memory. Returns the number of centroids written to
// out (<= TD_CAP).
template <bool B_STAGED, typename Work>
__device__ __forceinline__ uint32_t td_merge_compress(Work &S, const Centroid *a, uint32_t na, const Centroid *b, uint32_t nb,
		Centroid *out, const TdParams &P)
{
	const int lane = threadIdx.x & 31;
	const uint32_t nm = na + nb;

	// The means of both lists are staged in S.src (one coalesced read per list), then the warp merges them by MERGE PATH: lane l
	// produces the outputs [l * per, (l + 1) * per) of the merged list. One binary search along its diagonal tells the lane how many
	// entries of each list lie in front of its first output; from there it is a plain two-finger merge. Order = stable merge by mean,
	// `a` first on equal means — the same list a rank-by-binary-search of every entry gives, at ~1/4 of the instructions.
	double *am = S.src, *bm = S.src + na;
	for (uint32_t j0 = 0; j0 < na; j0 += 32 * 4) {		// the loads of 4 rounds in flight together (`a` is the L2-resident digest)
		double v[4];
#pragma unroll
		for (int q = 0; q < 4; ++q) { const uint32_t j = j0 + q * 32 + lane; v[q] = j < na ? a[j].mean : 0.0; }
#pragma unroll
		for (int q = 0; q < 4; ++q) { const uint32_t j = j0 + q * 32 + lane; if (j < na) am[j] = v[q]; }
	}
	if (!B_STAGED) for (uint32_t j = lane; j < nb; j += 32) bm[j] = b[j].mean;
	__syncwarp();
	const uint32_t per = (nm + 31u) >> 5;
	const uint32_t d0 = lane * per < nm ? lane * per : nm, d1 = d0 + per < nm ? d0 + per : nm;
	unsigned long long tot = 0;
	if (d0 < d1) {
		uint32_t lo = d0 > nb ? d0 - nb : 0u, hi = d0 < na ? d0 : na;		// entries of `a` in front of output d0
		while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (am[mid] <= bm[d0 - 1u - mid]) lo = mid + 1; else hi = mid; }
		uint32_t i = lo, k = d0 - lo;
		double av = i < na ? am[i] : 0.0, bv = k < nb ? bm[k] : 0.0;
		// the two-finger walk touches shared memory only: it notes where every output comes from (S.nxt is free until the cell
		// search) and the weights — which the walk does not need — are fetched afterwards, all loads of a lane in flight together
		// (a weight load inside the walk put an L2 round trip into every step). With b staged, S.nxt holds b's weights: the walk
		// copies a b weight into S.pref[pos + 1] as it takes the item and leaves the index of an `a` item there, flagged, for the
		// fetch (S.pref is free until then)
		constexpr unsigned long long FROM_A = 1ull << 63;
		for (uint32_t pos = d0; pos < d1; ++pos) {
			const bool ta = i < na && (k >= nb || av <= bv);
			S.mean[pos] = ta ? av : bv;
			if (B_STAGED) S.pref[pos + 1] = ta ? (FROM_A | i) : (unsigned long long)S.nxt[k];
			else S.nxt[pos] = (uint16_t)(ta ? i : (0x8000u | k));
			if (ta) { ++i; av = i < na ? am[i] : 0.0; }
			else { ++k; bv = k < nb ? bm[k] : 0.0; }
		}
		for (uint32_t p0 = d0; p0 < d1; p0 += 4) {		// 4 positions at a time: their weight loads in flight together
			unsigned long long w[4];
#pragma unroll
			for (int q = 0; q < 4; ++q) {
				const uint32_t pos = p0 + q < d1 ? p0 + q : d1 - 1u;
				if (B_STAGED) { const unsigned long long f = S.pref[pos + 1]; w[q] = (f & FROM_A) ? a[(uint32_t)f].weight : f; }
				else { const uint32_t from = S.nxt[pos]; w[q] = (from & 0x8000u) ? b[from & 0x7FFFu].weight : a[from].weight; }
			}
#pragma unroll
			for (int q = 0; q < 4; ++q) if (p0 + q < d1) { S.pref[p0 + q + 1] = w[q]; tot += w[q]; }
		}
	}
	// in-place weight prefix: pref[i+1] holds w_i on entry and sum(w_0..w_i) on exit; every lane scans the outputs it produced
	{
		unsigned long long incl = tot;
#pragma unroll
		for (int off = 1; off < 32; off <<= 1) {
			const unsigned long long tt = __shfl_up_sync(0xffffffffu, incl, off);
			if (lane >= off) incl += tt;
		}
		unsigned long long run = incl - tot;
		for (uint32_t pos = d0; pos < d1; ++pos) { run += S.pref[pos + 1]; S.pref[pos + 1] = run; }
		if (lane == 0) S.pref[0] = 0;
	}
	__syncwarp();
	// the cell-search key of item i, its weight centre rounded down: C_i = P_i + floor(w_i / 2)
	auto ckey = [&S](uint32_t i) { const unsigned long long p = S.pref[i]; return p + ((S.pref[i + 1] - p) >> 1); };

	// first item of every cell: the first item whose weight centre is at or past the cell's start; empty cells drop out
	uint32_t nout = 0;
	if (nm) {
		const unsigned long long Wt = S.pref[nm];
		const double W = (double)Wt;
		// lane l owns the consecutive cells [l * cj, (l + 1) * cj): the cell starts T_j grow with j, so after one binary search for
		// its first cell a lane walks forward from the previous answer (a cell holds nm / delta items on average)
		const uint32_t cj = (P.delta + 32u) >> 5;				// ceil((delta + 1) / 32)
		uint32_t lo = 0;
		for (uint32_t j = lane * cj, jn = 0; jn < cj && j <= P.delta; ++j, ++jn) {
			const unsigned long long T = j == P.delta ? Wt : (unsigned long long)__dmul_rn(__ldg(P.qtab + j), W);
			// first i in [0, nm) with ckey(i) >= T (its weight centre at or past T), nm if none
			uint32_t steps = jn ? 0u : 8u;
			while (steps < 8u && lo < nm && ckey(lo) < T) { ++lo; ++steps; }
			if (steps == 8u) {
				uint32_t hi = nm;
				while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (ckey(mid) < T) lo = mid + 1; else hi = mid; }
			}
			S.nxt[j] = (uint16_t)lo;
		}
		__syncwarp();
		for (uint32_t j0 = 0; j0 < P.delta; j0 += 32) {
			const uint32_t j = j0 + lane;
			const bool ne = j < P.delta && S.nxt[j + 1] > S.nxt[j];
			const uint32_t m = __ballot_sync(0xffffffffu, ne);
			if (ne) S.bounds[nout + __popc(m & ((1u << lane) - 1u))] = S.nxt[j];
			nout += __popc(m);
		}
		if (lane == 0) S.bounds[nout] = (uint16_t)nm;
		__syncwarp();
	}

	for (uint32_t c = lane; c < nout; c += 32) {
		double csum = 0.0;
		const uint32_t lo = S.bounds[c], hi = S.bounds[c + 1];
		for (uint32_t i = lo; i < hi; ++i) {
			csum = __dadd_rn(csum, __dmul_rn(S.mean[i], (double)(S.pref[i + 1] - S.pref[i])));
		}
		const unsigned long long cw = S.pref[hi] - S.pref[lo];
		Centroid o; o.mean = __ddiv_rn(csum, (double)cw); o.weight = cw;
		out[c] = o;
	}
	__syncwarp();
	return nout;
}

template <typename Work>
__device__ __forceinline__ uint32_t warp_merge_compress(Work &S, const Centroid *a, uint32_t na, const Centroid *b, uint32_t nb,
		Centroid *out, const TdParams &P)
{
	return td_merge_compress<false>(S, a, na, b, nb, out, P);
}

// b already in the work area: means at S.src[na, na + nb), weights at S.nxt[0, nb); na + nb <= Work::NMAX
template <typename Work>
__device__ __forceinline__ uint32_t warp_merge_compress_staged(Work &S, const Centroid *a, uint32_t na, uint32_t nb, Centroid *out,
		const TdParams &P)
{
	return td_merge_compress<true>(S, a, na, nullptr, nb, out, P);
}

} // namespace gysk
