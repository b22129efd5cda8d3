// gysk_summary.cuh — the arithmetic of one service's / one process's summary, host + device.
//
// Every service row (gysk_query_svcs, gysk_query_window, gysk_query_logical) is summarised on the device, one warp per row
// (summarize_warp); every process row too (summarize_task). The host keeps td_quantile and hll_estimate_from_hist for the public
// gysk_tdigest_quantile / gysk_hll_estimate / gysk_query_quantiles, which answer from a service's exported sketches what its row
// holds. What keeps the two sides equal:
//   * the percentile rule is GY_HISTOGRAM::get_percentiles (common/gy_statistics.h:707-791) through hist_pct_bucket (gysk_state.cuh);
//   * t-digest quantiles: while the cumulative weights stay below 2^53 they are exact in any order, so the device's uint64 warp
//     prefix gives the doubles of the host's running sum; a heavier digest runs the host's loop on the device (td_quantile_warp).
//     The arithmetic is written with explicit round-to-nearest operations on the device so that nvcc does not contract it into a
//     fused multiply-add;
//   * HLL: the raw sum keeps the host's order (r = 63 down to 0). The linear-counting branch needs log(), which neither CUDA nor
//     glibc rounds correctly, so the device hands back -(zero registers) and the host finishes with hll_finish().
#pragma once

#include <cmath>
#include <cstring>

#include "gysk_kernels.cuh"
#include "gysk_state.cuh"

#ifdef __CUDA_ARCH__
#define GYSK_DADD(a, b) __dadd_rn((a), (b))
#define GYSK_DMUL(a, b) __dmul_rn((a), (b))
#define GYSK_DDIV(a, b) __ddiv_rn((a), (b))
#else
#define GYSK_DADD(a, b) ((a) + (b))
#define GYSK_DMUL(a, b) ((a) * (b))
#define GYSK_DDIV(a, b) ((a) / (b))
#endif

namespace gysk {

// bucket thresholds of the histogram classes, common/gy_statistics.h:1624-2063 (GYSK_CLS_* order)
struct ClsDesc { int nthr; int64_t thr[16]; int64_t minv, maxv; bool trunc_int; int fixed_diff; };

#define GYSK_CLS_TABLE { \
	{13, {1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000}, 0, 15001, false, 0},		/* RESP_TIME_HASH    :1677 */ \
	{12, {1, 10, 100, 500, 1000, 5000, 25000, 50000, 100000, 300000, 1000000, 5000000}, 0, 5000001, true, 0},	/* SEMI_LOG_HASH     :1732 */ \
	{13, {1, 10, 50, 200, 500, 1000, 3000, 6000, 10000, 15000, 25000, 60000, 150000}, 0, 150001, true, 0},	/* SEMI_LOG_HASH_LO  :1785 */ \
	{13, {1, 10, 25, 50, 125, 400, 1000, 3000, 6000, 10000, 25000, 40000, 65000}, 0, 65001, true, 0},	/* DURATION_HASH     :1838 */ \
	{12, {10, 25, 50, 75, 100, 150, 300, 500, 800, 1000, 2000, 5000}, 0, 5001, true, 0},			/* HASH_10_5000      :1911 */ \
	{10, {5, 10, 20, 40, 60, 80, 100, 140, 200, 250}, 0, 251, true, 0},					/* HASH_5_250        :1963 */ \
	{12, {1, 5, 10, 25, 50, 75, 100, 150, 300, 500, 1000, 3000}, 0, 3001, true, 0},				/* HASH_1_3000       :2016 */ \
	{11, {9, 19, 29, 39, 49, 59, 69, 79, 89, 99, 100}, 0, 101, false, 10},					/* PERCENT_HASH      :1624 */ \
}
static const ClsDesc g_cls[8] = GYSK_CLS_TABLE;
#ifdef __CUDACC__
static __constant__ ClsDesc g_cls_dev[8] = GYSK_CLS_TABLE;
#endif
#undef GYSK_CLS_TABLE

GYSK_HD const ClsDesc &cls_desc(int cls)
{
#ifdef __CUDA_ARCH__
	return g_cls_dev[cls];
#else
	return g_cls[cls];
#endif
}

// get_bucket_max_threshold<HashClass, T>, gy_statistics.h:500-515
GYSK_HD int64_t bucket_max_threshold(const ClsDesc &d, bool t_is_int, int id)
{
	const int maxb = d.nthr + 2;

	if (id == 0) return d.minv - 1;
	if (id >= maxb - 1) {
		const int64_t maxt = t_is_int ? INT32_MAX : INT64_MAX;
		const int64_t lesst = d.maxv >= INT32_MAX ? INT64_MAX : (d.maxv > (INT16_MAX >> 1) ? INT32_MAX : INT16_MAX);
		return maxt < lesst ? maxt : lesst;
	}
	return d.thr[id - 1];
}

// GY_HISTOGRAM<T, cls>::get_percentiles of one percentile: the first bucket whose cumulative count reaches the cut-off, answered with
// that bucket's upper threshold cast to T (-1 for an empty histogram: min_value - 1)
GYSK_HD int64_t hist_percentile(int cls, bool t_is_int, const uint64_t *counts, uint64_t total_count, float pct)
{
	const ClsDesc &d = cls_desc(cls);
	const int nb = d.nthr + 2;
	const int i = hist_pct_bucket(counts, nb, total_count, pct);
	const int64_t v = bucket_max_threshold(d, t_is_int, i < nb ? i : (total_count > 0 ? nb : 0));
	return t_is_int ? (int64_t)(int32_t)v : v;
}

// ---- t-digest quantile (the interpolation of tdigest_percentile between centroid centres) ----

// centre of a centroid of weight w after `cum` weight
GYSK_HD double td_center(double cum, uint64_t w) { return GYSK_DADD(cum, (double)w / 2.0); }

// between the centre of the previous centroid (prev_center, prev_mean) and the next point (center, next)
GYSK_HD double td_interp(double prev_mean, double next, double target, double prev_center, double center)
{
	const double span = GYSK_DADD(center, -prev_center);
	if (!(span > 0)) return next;
	return GYSK_DADD(prev_mean, GYSK_DMUL(GYSK_DADD(next, -prev_mean), GYSK_DDIV(GYSK_DADD(target, -prev_center), span)));
}

// the centroids td_quantile_seq reads: separate mean / weight arrays (the public API) or an array of Centroid (a row's digest)
struct TdArrays
{
	const double *means; const uint64_t *weights;
	GYSK_HD double mean(uint32_t i) const { return means[i]; }
	GYSK_HD uint64_t weight(uint32_t i) const { return weights[i]; }
};
struct TdCentroids
{
	const Centroid *c;
	GYSK_HD double mean(uint32_t i) const { return c[i].mean; }
	GYSK_HD uint64_t weight(uint32_t i) const { return c[i].weight; }
};

template <typename D>
GYSK_HD double td_quantile_seq(const D &d, uint32_t n, double minv, double maxv, double q)
{
	if (!n) return NAN;
	double total = 0;
	for (uint32_t i = 0; i < n; ++i) total = GYSK_DADD(total, (double)d.weight(i));
	if (q <= 0) return minv;
	if (q >= 1) return maxv;

	const double target = GYSK_DMUL(q, total);
	double cum = 0, prev_center = 0, prev_mean = minv;

	for (uint32_t i = 0; i < n; ++i) {
		const double center = td_center(cum, d.weight(i));
		if (target < center) return td_interp(prev_mean, d.mean(i), target, prev_center, center);
		prev_center = center; prev_mean = d.mean(i);
		cum = GYSK_DADD(cum, (double)d.weight(i));
	}
	return td_interp(prev_mean, maxv, target, prev_center, total);
}

inline double td_quantile(const double *means, const uint64_t *weights, uint32_t n, double minv, double maxv, double q)
{
	return td_quantile_seq(TdArrays {means, weights}, n, minv, maxv, q);
}

// ---- HLL estimate from the register histogram (hist64[r] = registers holding r, r clamped to 63) ----

// the raw estimate, or -(zero registers) when the linear-counting branch applies (hll_finish completes it)
GYSK_HD double hll_pending(const uint32_t *hist64, uint32_t p)
{
	const uint32_t m = 1u << p;
	double sum = 0, alpha;

	for (int r = 63; r >= 0; --r) sum = GYSK_DADD(sum, GYSK_DMUL((double)hist64[r], ldexp(1.0, -r)));
	if (m == 16) alpha = 0.673; else if (m == 32) alpha = 0.697; else if (m == 64) alpha = 0.709;
	else alpha = GYSK_DDIV(0.7213, GYSK_DADD(1.0, GYSK_DDIV(1.079, (double)m)));
	const double est = GYSK_DDIV(GYSK_DMUL(GYSK_DMUL(alpha, (double)m), (double)m), sum);
	if (est <= 2.5 * (double)m && hist64[0]) return -(double)hist64[0];
	return est;
}

inline double hll_finish(double v, uint32_t p)
{
	const double m = (double)(1u << p);
	return v < 0 ? m * log(m / -v) : v;
}

inline double hll_estimate_from_hist(const uint32_t *hist64, uint32_t p) { return hll_finish(hll_pending(hist64, p), p); }

// ---- per-service summary: SvcRaw -> the fields SvcStateFields exposes (server/gy_mfields.h:1383-1412) ----

GYSK_HD uint64_t cells_total(const HistCell *c, int nb, uint64_t *counts)
{
	uint64_t t = 0;
	for (int i = 0; i < nb; ++i) { counts[i] = c[i].count; t += c[i].count; }
	return t;
}

// everything but distinct_clients and the three t-digest quantiles (left NaN), which summarize_warp adds
GYSK_HD void summarize_fields(const SvcRaw &r, uint64_t id, gysk_svc_summary &o)
{
	memset(&o, 0, sizeof(o));
	o.glob_id = id;
	o.found = r.found;
	o.td_p50_us = o.td_p95_us = o.td_p99_us = NAN;
	if (!r.found) return;

	uint64_t counts[15], total;

	total = cells_total(r.last, 15, counts);
	o.nqrys_5s = (uint32_t)total;
	for (int b = 0; b < 15; ++b) o.total_resp_5sec += (uint64_t)r.last[b].sum;
	o.p95_5s_resp_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 95.0f);
	o.p99_5s_resp_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 99.0f);
	o.p25_5s_resp_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 25.0f);

	total = cells_total(r.lvl[0], 15, counts);
	o.p95_5min_resp_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 95.0f);
	o.p99_5min_resp_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 99.0f);
	o.nqrys_5min = total;
	total = cells_total(r.lvl[1], 15, counts);
	o.p95_5day_resp_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 95.0f);
	o.nqrys_5day = total;

	total = cells_total(r.all, 15, counts);
	o.p95_all_resp_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 95.0f);
	o.p99_all_resp_ms = hist_percentile(GYSK_CLS_RESP_TIME, false, counts, total, 99.0f);
	o.nqrys_all = total; o.max_resp_ms = r.all[HIST_MAX_CELL].sum;

	o.nconns_5s = (uint32_t)r.conn_last; o.kbytes_5s = (uint32_t)(r.conn_last >> 32);
	o.nconns_all = r.conn_all_cnt; o.kbytes_all = r.conn_all_kb;
	o.nconns_active = (uint32_t)r.aux.act_last; o.active_kbytes = (uint32_t)(r.aux.act_last >> 32);
	memcpy(&o.max_rtt_msec, &r.aux.rtt_last, 4);
	o.cli_errors = (uint32_t)r.aux.err_last; o.ser_errors = (uint32_t)(r.aux.err_last >> 32);
	o.curr_state = r.sst.state; o.curr_issue = r.sst.issue; o.issue_bit_hist = r.sst.issue_bits; o.high_resp_bit_hist = r.sst.high_bits;
	o.td_count = r.td.total;
}

#ifdef __CUDACC__
// the heavy digests' case of td_quantile_warp, one out-of-line copy instead of three inlined ones: no real stream reaches it
static __device__ __noinline__ double td_quantile_heavy(const Centroid *c, uint32_t n, double minv, double maxv, double q)
{
	return td_quantile_seq(TdCentroids {c}, n, minv, maxv, q);
}

// td_quantile of the digest in shared memory (n <= TD_CAP centroids), by one warp: each lane takes a run of centroids, a uint64 prefix
// over the warp gives every centroid the cumulative weight the host loop reaches, a ballot finds the first centre above the target.
// That holds while the weights stay below 2^45: no sum of TD_CAP of them reaches 2^53. A heavier digest takes the host's loop itself,
// whose running double sum rounds.
__device__ inline double td_quantile_warp(const Centroid *c, uint32_t n, double minv, double maxv, double q, int lane)
{
	const uint32_t per = (n + 31) >> 5, b = min(n, lane * per), e = min(n, b + per);
	unsigned long long s = 0, bits = 0;
	for (uint32_t i = b; i < e; ++i) { s += c[i].weight; bits |= c[i].weight; }
	static_assert(TD_CAP <= 256, "TD_CAP weights below 2^45 sum below 2^53");
	if (__any_sync(0xffffffffu, bits >> 45)) return td_quantile_heavy(c, n, minv, maxv, q);
	unsigned long long incl = s;
	for (int o = 1; o < 32; o <<= 1) {
		const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
		if (lane >= o) incl += t;
	}
	const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
	if (q <= 0) return minv;
	if (q >= 1) return maxv;
	const double target = __dmul_rn(q, (double)total);
	unsigned long long cum = incl - s;
	int hit = -1;
	for (uint32_t i = b; i < e; ++i) {
		if (target < td_center((double)cum, c[i].weight)) { hit = (int)i; break; }
		cum += c[i].weight;
	}
	const unsigned mask = __ballot_sync(0xffffffffu, hit >= 0);
	if (!mask) {
		const Centroid l = c[n - 1];
		return td_interp(l.mean, maxv, target, td_center((double)(total - l.weight), l.weight), (double)total);
	}
	const int src = __ffs(mask) - 1;
	const int i = __shfl_sync(0xffffffffu, hit, src);
	const unsigned long long cb = __shfl_sync(0xffffffffu, cum, src);
	const double center = td_center((double)cb, c[i].weight);
	if (i == 0) return td_interp(minv, c[0].mean, target, 0.0, center);
	const Centroid p = c[i - 1];
	return td_interp(p.mean, c[i].mean, target, td_center((double)(cb - p.weight), p.weight), center);
}

// the HLL register histogram of 2^p registers (p >= 4, 16-byte aligned) by one warp, into hist64 in shared memory; four registers per
// load, as each lane's loads are serialised by the atomics behind them
__device__ inline void hll_hist_warp(const uint8_t *regs, uint32_t p, uint32_t *hist64, int lane)
{
	hist64[lane] = 0; hist64[lane + 32] = 0;
	__syncwarp();
	const uint32_t *words = reinterpret_cast<const uint32_t *>(regs);
	for (uint32_t i = lane; i < (1u << p) / 4u; i += 32) {
		const uint32_t w = words[i];
		for (int k = 0; k < 32; k += 8) atomicAdd(&hist64[min((w >> k) & 0xFFu, 63u)], 1u);
	}
	__syncwarp();
}

// the row of r by one warp: r in shared memory (hll_hist included when found), summ the warp's sizeof(gysk_svc_summary) bytes of
// shared scratch, out the row in global memory. distinct_clients may come out as -(zero registers): the host finishes it with
// hll_finish.
__device__ inline void summarize_warp(const SvcRaw &r, uint64_t id, uint32_t hll_p, unsigned long long *summ, gysk_svc_summary *out, int lane)
{
	gysk_svc_summary &o = *reinterpret_cast<gysk_svc_summary *>(summ);
	__syncwarp();
	if (lane == 0) {
		summarize_fields(r, id, o);
		if (r.found) o.distinct_clients = hll_pending(r.hll_hist, hll_p);
	}
	const uint32_t nc = r.found ? min(r.td.n, (uint32_t)TD_CAP) : 0u;
	if (nc) {
		const double p50 = td_quantile_warp(r.cent, nc, r.td.minv, r.td.maxv, 0.50, lane);
		const double p95 = td_quantile_warp(r.cent, nc, r.td.minv, r.td.maxv, 0.95, lane);
		const double p99 = td_quantile_warp(r.cent, nc, r.td.minv, r.td.maxv, 0.99, lane);
		if (lane == 0) { o.td_p50_us = p50; o.td_p95_us = p95; o.td_p99_us = p99; }
	}
	__syncwarp();
	unsigned long long *dst = reinterpret_cast<unsigned long long *>(out);
	if (lane < (int)(sizeof(gysk_svc_summary) / 8)) dst[lane] = summ[lane];
}
#endif

// ---- per-process summary: the three MTASK_HIST p95 of AGGR_TASK_HIST_STATS (server/gy_mconnhdlr.cc:14648-14706) ----

// h: the task's three histograms {cpu %, cpu delay, blkio delay} x 16 cells; last: task_last of the slot
GYSK_HD void summarize_task(const HistCell *h, const HistCell *last, uint64_t id, uint32_t host_idx, gysk_task_summary &o)
{
	int32_t p95[3];
	uint64_t counts[15], total[3];

	memset(&o, 0, sizeof(o));
	o.aggr_task_id = id; o.found = 1; o.host_idx = host_idx;
	for (int k = 0; k < 3; ++k) {
		const int cls = k ? GYSK_CLS_DURATION : GYSK_CLS_HASH_1_3000;		// MTASK_HIST, server/gy_msocket.h:707
		total[k] = cells_total(h + k * HIST_CELLS, cls_desc(cls).nthr + 2, counts);
		p95[k] = (int32_t)hist_percentile(cls, true, counts, total[k], 95.0f);
		o.last_count[k] = last[k].count; o.last_sum[k] = last[k].sum;
	}
	o.p95_cpu_pct = p95[0]; o.p95_cpu_delay_ms = p95[1]; o.p95_blkio_delay_ms = p95[2];
	o.nsamples = total[0];
}

} // namespace gysk
