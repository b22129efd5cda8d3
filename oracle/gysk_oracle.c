/*
 * gysk_oracle.c — TEST INFRASTRUCTURE ONLY (see gysk_oracle.h). Plain-C CPU restatement of the hot path.
 * Each function cites the reference file:line (relative to the reference tree) whose behaviour it restates.
 *
 * PARITY STATUS: histogram/jhash parts are pinned (tests/test_oracle_pinning.py: the asserted values of
 * test/test_histogram.cc and the outputs of the reference compiled into oracle/_ref). Count-min, HyperLogLog
 * and t-digest are PARITY UNPINNED: the reference holds no implementation or vector for them.
 */
#include "gysk_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <limits.h>
#include <math.h>
#include <time.h>
#include <pthread.h>

/* ------------------------------------------------------------------------------------------------
 * jhash: Bob Jenkins' lookup2 (public domain, 1996) in the word-oriented form the reference uses.
 * common/jhash.h:22-35 (mix), :86-113 (jhash2), :121-140 (n-words), :44-84 (bytes)
 * ------------------------------------------------------------------------------------------------ */
#define GOLDEN		0x9e3779b9u
#define GY_SEED		0xceedfeadu	/* common/gy_common_inc.h:1112-1122 */

static inline void mix3(uint32_t *pa, uint32_t *pb, uint32_t *pc)
{
	uint32_t a = *pa, b = *pb, c = *pc;

	a -= b; a -= c; a ^= (c >> 13);
	b -= c; b -= a; b ^= (a << 8);
	c -= a; c -= b; c ^= (b >> 13);
	a -= b; a -= c; a ^= (c >> 12);
	b -= c; b -= a; b ^= (a << 16);
	c -= a; c -= b; c ^= (b >> 5);
	a -= b; a -= c; a ^= (c >> 3);
	b -= c; b -= a; b ^= (a << 10);
	c -= a; c -= b; c ^= (b >> 15);

	*pa = a; *pb = b; *pc = c;
}

uint32_t gyo_jhash_3words(uint32_t a, uint32_t b, uint32_t c, uint32_t initval)
{
	a += GOLDEN; b += GOLDEN; c += initval;
	mix3(&a, &b, &c);
	return c;
}

uint32_t gyo_jhash_2words(uint32_t a, uint32_t b, uint32_t initval)
{
	return gyo_jhash_3words(a, b, 0, initval);
}

uint32_t gyo_jhash2(const uint32_t *k, uint32_t length, uint32_t initval)
{
	uint32_t a = GOLDEN, b = GOLDEN, c = initval, len = length;

	while (len >= 3) {
		a += k[0]; b += k[1]; c += k[2];
		mix3(&a, &b, &c);
		k += 3; len -= 3;
	}
	c += length * 4;
	if (len == 2) { b += k[1]; a += k[0]; }
	else if (len == 1) { a += k[0]; }
	mix3(&a, &b, &c);
	return c;
}

uint32_t gyo_jhash(const void *key, uint32_t length, uint32_t initval)
{
	const uint8_t *k = (const uint8_t *)key;
	uint32_t a = GOLDEN, b = GOLDEN, c = initval, len = length;

	while (len >= 12) {
		a += (k[0] + ((uint32_t)k[1] << 8) + ((uint32_t)k[2] << 16) + ((uint32_t)k[3] << 24));
		b += (k[4] + ((uint32_t)k[5] << 8) + ((uint32_t)k[6] << 16) + ((uint32_t)k[7] << 24));
		c += (k[8] + ((uint32_t)k[9] << 8) + ((uint32_t)k[10] << 16) + ((uint32_t)k[11] << 24));
		mix3(&a, &b, &c);
		k += 12; len -= 12;
	}
	c += length;
	/* tail bytes: byte i of the tail lands in word i/4 (a, b) or, from the 9th on, one byte higher in c */
	for (uint32_t i = 0; i < len; ++i) {
		uint32_t v = k[i];
		if (i < 4) a += v << (8 * i);
		else if (i < 8) b += v << (8 * (i - 4));
		else c += v << (8 * (i - 8 + 1));
	}
	mix3(&a, &b, &c);
	return c;
}

uint32_t gyo_uint64_hash(uint64_t key)
{
	return gyo_jhash_2words((uint32_t)(key & 0xFFFFFFFFu), (uint32_t)(key >> 32), GY_SEED);
}

/* ------------------------------------------------------------------------------------------------
 * bucket hash classes, common/gy_statistics.h:1584-2063
 * ------------------------------------------------------------------------------------------------ */
typedef struct cls_desc
{
	int		nthr;
	int64_t		thr[16];
	int64_t		min_value, max_value;
	int		trunc_int;	/* operator()(int data): the value is narrowed to int before bucketing (:1748,:1801,...) */
	int		fixed_diff;	/* FIXED_DIFF_HASH: bucket = 1 + (data - min)/diff (:1611-1621) */
} cls_desc;

static const cls_desc g_cls[GYO_CLS_MAX] = {
	[GYO_CLS_RESP_TIME]	= { 13, {1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000}, 0, 15001, 0, 0 },		/* :1677 */
	[GYO_CLS_SEMI_LOG]	= { 12, {1, 10, 100, 500, 1000, 5000, 25000, 50000, 100000, 300000, 1000000, 5000000}, 0, 5000001, 1, 0 },	/* :1732 */
	[GYO_CLS_SEMI_LOG_LO]	= { 13, {1, 10, 50, 200, 500, 1000, 3000, 6000, 10000, 15000, 25000, 60000, 150000}, 0, 150001, 1, 0 },	/* :1785 */
	[GYO_CLS_DURATION]	= { 13, {1, 10, 25, 50, 125, 400, 1000, 3000, 6000, 10000, 25000, 40000, 65000}, 0, 65001, 1, 0 },	/* :1838 */
	[GYO_CLS_HASH_10_5000]	= { 12, {10, 25, 50, 75, 100, 150, 300, 500, 800, 1000, 2000, 5000}, 0, 5001, 1, 0 },			/* :1911 */
	[GYO_CLS_HASH_5_250]	= { 10, {5, 10, 20, 40, 60, 80, 100, 140, 200, 250}, 0, 251, 1, 0 },					/* :1963 */
	[GYO_CLS_HASH_1_3000]	= { 12, {1, 5, 10, 25, 50, 75, 100, 150, 300, 500, 1000, 3000}, 0, 3001, 1, 0 },			/* :2016 */
	/* FIXED_DIFF_HASH<int64_t,0,100,10>: thresholds tmin + (i+1)*diff - 1, last = tmax (:1570-1582) */
	[GYO_CLS_PERCENT]	= { 11, {9, 19, 29, 39, 49, 59, 69, 79, 89, 99, 100}, 0, 101, 0, 10 },					/* :1624 */
	[GYO_CLS_FD_I8_9_26_5]	= { 4, {13, 18, 23, 26}, 9, 27, 0, 5 },			/* test/test_histogram.cc:17 */
	[GYO_CLS_FD_INT_M15_M3_4] = { 4, {-12, -8, -4, -3}, -15, -2, 0, 4 },		/* test/test_histogram.cc:92 */
};

int gyo_nbuckets(int cls)
{
	if (cls < 0 || cls >= GYO_CLS_MAX) return -1;
	return g_cls[cls].nthr + 2;
}

int gyo_bucket(int cls, int64_t value)
{
	const cls_desc *d = &g_cls[cls];
	int64_t data = value;

	if (d->trunc_int) data = (int64_t)(int)value;

	if (data < d->min_value) return 0;
	if (data >= d->max_value) return d->nthr + 1;

	if (d->fixed_diff) return (int)(1 + (data - d->min_value) / d->fixed_diff);

	/* the mid-slot shortcut (:1711-1716) only changes where the scan starts, never its result */
	for (int nb = 0; nb < d->nthr; ++nb) {
		if (data <= d->thr[nb]) return nb + 1;
	}
	return d->nthr + 1;
}

/* get_bucket_max_threshold<HashClass, T>, common/gy_statistics.h:500-515 */
int64_t gyo_bucket_max_threshold(int cls, int tkind, size_t id)
{
	const cls_desc *d = &g_cls[cls];
	size_t maxb = (size_t)d->nthr + 2;

	if (id == 0) return d->min_value - 1;

	if (id >= maxb - 1) {
		int64_t maxt = (tkind == GYO_T_INT64) ? INT64_MAX : (tkind == GYO_T_INT ? INT_MAX : SCHAR_MAX);
		int64_t lesst = d->max_value >= INT_MAX ? LONG_MAX : (d->max_value > (SHRT_MAX >> 1) ? INT_MAX : SHRT_MAX);

		return lesst < maxt ? lesst : maxt;
	}
	return d->thr[id - 1];
}

static inline int64_t t_min(int tkind)
{
	return tkind == GYO_T_INT64 ? INT64_MIN : (tkind == GYO_T_INT ? INT_MIN : SCHAR_MIN);
}

static inline int64_t t_cast(int tkind, int64_t v)
{
	return tkind == GYO_T_INT64 ? v : (tkind == GYO_T_INT ? (int64_t)(int)v : (int64_t)(int8_t)v);
}

void gyo_hist_init(gyo_hist *h, int cls, int tkind)
{
	memset(h, 0, sizeof(*h));
	h->cls = cls; h->tkind = tkind;
	h->max_val = t_min(tkind);		/* max_val_seen_{numeric_limits<T>::min()} :560 */
}

/* GY_HISTOGRAM::add_data :596-623 — `T data` narrows first, then hash_(data), sum += data, count++, total++, max */
int gyo_hist_add(gyo_hist *h, int64_t value)
{
	int64_t data = t_cast(h->tkind, value);
	int b = gyo_bucket(h->cls, data);

	h->stats[b].sum += data;
	h->stats[b].count++;
	h->total_count++;
	if (h->max_val < data) h->max_val = data;
	return b;
}

/* update_from_serialized :625-650 (clock fields not modelled) */
void gyo_hist_merge(gyo_hist *dst, const gyo_hist *src)
{
	int nb = gyo_nbuckets(dst->cls);

	for (int i = 0; i < nb; ++i) {
		dst->stats[i].count += src->stats[i].count;
		dst->stats[i].sum += src->stats[i].sum;
	}
	dst->total_count += src->total_count;
	if (dst->max_val < src->max_val) dst->max_val = src->max_val;
}

/* get_percentiles :707-791. Note the float multiplier and the size_t * float product (:753-754) */
void gyo_hist_percentiles(const gyo_hist *h, const float *pcts, size_t npct, int64_t *out, float *avg)
{
	const size_t	nb = (size_t)gyo_nbuckets(h->cls);
	const size_t	total_count = h->total_count;

	if (avg) {
		int64_t total_sum = 0, cnt = total_count ? (int64_t)total_count : 1;

		for (size_t i = 0; i < nb; ++i) total_sum += h->stats[i].sum;
		*avg = (total_sum * 1.0f) / cnt;
	}

	for (size_t n = 0; n < npct; ++n) {
		float		multiplier = pcts[n] / 100.0;
		const size_t	ncutoff = total_count * multiplier;
		size_t		i, total = 0;

		for (i = 0; i < nb; ++i) {
			total += h->stats[i].count;
			if (total >= ncutoff) {
				out[n] = t_cast(h->tkind, gyo_bucket_max_threshold(h->cls, h->tkind, i));
				break;
			}
		}
		if (i < nb) continue;

		if (total_count > 0) out[n] = t_cast(h->tkind, gyo_bucket_max_threshold(h->cls, h->tkind, nb));
		else out[n] = t_cast(h->tkind, gyo_bucket_max_threshold(h->cls, h->tkind, 0));
	}
}

int gyo_hist_run(int cls, int tkind, const int64_t *vals, size_t n, const float *pcts, size_t npct,
		gyo_serial *out_stats, uint64_t *out_total, int64_t *out_max, int64_t *out_pct, int64_t *out_bucket_ids, float *out_avg)
{
	gyo_hist h;
	int nb = gyo_nbuckets(cls);

	if (nb < 0) return -1;
	gyo_hist_init(&h, cls, tkind);
	for (size_t i = 0; i < n; ++i) {
		int b = gyo_hist_add(&h, vals[i]);
		if (out_bucket_ids) out_bucket_ids[i] = b;
	}
	if (out_stats) memcpy(out_stats, h.stats, sizeof(gyo_serial) * (size_t)nb);
	if (out_total) *out_total = h.total_count;
	if (out_max) *out_max = h.max_val;
	if (npct) gyo_hist_percentiles(&h, pcts, npct, out_pct, out_avg);
	return nb;
}

/* ------------------------------------------------------------------------------------------------
 * count-min and HyperLogLog definitions (ours; PARITY UNPINNED — no reference implementation exists)
 * hash family: the reference's jhash_2words over the two halves of the key with row-salted initval
 * ------------------------------------------------------------------------------------------------ */
#define FLOW_SEED_A	GY_SEED
#define FLOW_SEED_B	(GY_SEED ^ 0x5bd1e995u)

/* Two lookup2 words per flow key: h1 = jhash_2words(lo, hi, SEED_A), h2 = jhash_2words(lo, hi, SEED_B). Count-min row r indexes
 * (h1 + r * (h2 | 1)) & (width - 1) (Kirsch & Mitzenmacher double hashing: the d row hashes of a sketch may be linear
 * combinations of two independent hashes without changing the error bound); HyperLogLog takes the 64-bit word h2:h1. */
void gyo_flow_hashes(uint64_t flow_key, uint32_t *h1, uint32_t *h2)
{
	uint32_t lo = (uint32_t)flow_key, hi = (uint32_t)(flow_key >> 32);

	*h1 = gyo_jhash_2words(lo, hi, FLOW_SEED_A);
	*h2 = gyo_jhash_2words(lo, hi, FLOW_SEED_B);
}

uint32_t gyo_cms_index(uint64_t flow_key, uint32_t row, uint32_t log2_width)
{
	uint32_t h1, h2;

	gyo_flow_hashes(flow_key, &h1, &h2);
	return (h1 + row * (h2 | 1u)) & ((1u << log2_width) - 1);
}

/* one 64-bit cell = {count: low 32, kbytes: high 32}; a single 64-bit add updates both. The count half
 * would have to exceed 2^32 events on one cell inside one window before it could carry into kbytes. */
uint64_t gyo_cms_increment(uint32_t bytes)
{
	return 1ull | ((uint64_t)(bytes >> 10) << 32);
}

/* murmur3's 64-bit finalizer over h2:h1: the register index is the top p bits of the word, and the two one-round lookup2
 * words leave those bits poorly mixed on structured keys ((client ip << 32) | port undercounted by up to 65 %). */
uint64_t gyo_hll_hash(uint64_t flow_key)
{
	uint32_t h1, h2;
	uint64_t h;

	gyo_flow_hashes(flow_key, &h1, &h2);
	h = ((uint64_t)h2 << 32) | h1;
	h ^= h >> 33; h *= 0xff51afd7ed558ccdull;
	h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull;
	h ^= h >> 33;
	return h;
}

void gyo_hll_idx_rank(uint64_t flow_key, uint32_t p, uint32_t *idx, uint8_t *rank)
{
	uint64_t h = gyo_hll_hash(flow_key);
	uint64_t w = h << p;

	*idx = (uint32_t)(h >> (64 - p));
	*rank = (uint8_t)(w ? (uint32_t)(__builtin_clzll(w) + 1) : (64u - p + 1u));
}

/* raise the 1 << p registers regs with n keys (registers are not cleared first, so sets can be added in several calls) */
void gyo_hll_registers(const uint64_t *keys, uint64_t n, uint32_t p, uint8_t *regs)
{
	for (uint64_t i = 0; i < n; ++i) {
		uint32_t idx; uint8_t rank;

		gyo_hll_idx_rank(keys[i], p, &idx, &rank);
		if (regs[idx] < rank) regs[idx] = rank;
	}
}

/* Flajolet et al. 2007 raw estimator + linear counting for the small range; 64-bit hash => no large-range
 * correction. Computed from the register-value histogram in a fixed order so that every implementation
 * (this file, the host side of libgysketch.so) produces the identical double. */
double gyo_hll_estimate(const uint8_t *regs, uint32_t p)
{
	const uint32_t	m = 1u << p;
	uint32_t	hist[66] = {0};
	double		sum = 0, alpha, e;

	for (uint32_t i = 0; i < m; ++i) hist[regs[i] > 65 ? 65 : regs[i]]++;
	for (int r = 65; r >= 0; --r) sum += (double)hist[r] * ldexp(1.0, -r);

	if (m == 16) alpha = 0.673; else if (m == 32) alpha = 0.697; else if (m == 64) alpha = 0.709;
	else alpha = 0.7213 / (1.0 + 1.079 / (double)m);

	e = alpha * (double)m * (double)m / sum;
	if (e <= 2.5 * (double)m && hist[0]) e = (double)m * log((double)m / (double)hist[0]);
	return e;
}

/* ------------------------------------------------------------------------------------------------
 * t-digest (PARITY UNPINNED). Published algorithm: T. Dunning, "The t-digest: efficient estimates of
 * distributions" — merging variant, scale function K_1 normalised so that k spans [-delta/2, delta/2]:
 * k(q) = delta/pi asin(2q - 1), i.e. delta ... 1.3 delta centroids. The reference's two t-digest users pin "100"
 * (Postgres public.tdigest(x, 100), common/gy_query_common.cc:1855; folly::TDigest(100) behind
 * SlidingWindowQuantileEstimator, test/test_quantiles.cc:32); the engine keeps delta = 200 internally (capacity 256)
 * because SURVEY.md §8c-4 asks for p99 within 1 % of the EXACT quantile on sigma 1.2-1.5 log-normal streams, which a
 * 100-centroid K_1 digest misses by 1-3 % (interpolation error ~ 1/delta^2), and recompresses to 100 on export.
 * ------------------------------------------------------------------------------------------------ */
/* Upper end q1 of the unit-k interval that starts at q0: q1 = q(k(q0) + 1) with k(q) = delta/pi asin(2q - 1), written without
 * inverse trig: with theta = asin(2 q0 - 1), sin(theta + pi/delta) = (2 q0 - 1) cos(pi/delta) + 2 sqrt(q0 (1 - q0)) sin(pi/delta).
 * Only IEEE +,-,*,/ and sqrt, each rounded on its own, in this order — the CUDA path performs the identical sequence, so both
 * produce the same bits. */
/* The compress step works on the FIXED unit grid of k: cell j = [q_j, q_j+1), q_j = q(k = -delta/2 + j) = (sin(pi (j/delta - 1/2)) + 1)/2.
 * In weight units cell j starts at T_j = (uint64) (q_j * W); an item of the merged list (sorted by mean; exclusive weight prefix
 * P_i, weight w_i, total W) belongs to the cell that holds its weight centre: T_j <= P_i + w_i / 2 < T_j+1; all items of one cell
 * become one cluster: at most delta clusters, each reaching past its cell by at most half of its first and half of its last item
 * (the t-digest size bound), and no data-dependent chain — every item finds its cell on its own. The centre, not the start: once
 * old centroids are items of the next compress, a start-rule cluster grows by its whole last item at every merge, so a digest fed
 * through many batches widens and loses centroids; with the centre an old centroid that fits a cell stays in it. The table is
 * computed with libm by this expression here and in gyeeta_b200/csrc/gysk_engine.cu (same host, same bits). */
#define GYO_TD_MAX_DELTA	256
static void td_qtab(double delta, double *qtab /* [delta + 1] */)
{
	const uint32_t d = (uint32_t)delta;

	for (uint32_t j = 0; j <= d; ++j) qtab[j] = 0.5 * (sin(M_PI * ((double)j / (double)d - 0.5)) + 1.0);
	qtab[0] = 0.0; qtab[d] = 1.0;
}

void gyo_td_init(gyo_tdigest *t)
{
	memset(t, 0, sizeof(*t));
	t->minv = INFINITY; t->maxv = -INFINITY;
}

/* cell j starts at weight T_j = (uint64) (q_j * W); an item belongs to the cell that holds its weight centre P_i + w_i / 2;
 * cluster mean = sum(mean * weight) / sum(weight), accumulated in double in input order */
uint32_t gyo_td_compress(const gyo_centroid *in, uint32_t n, double delta, gyo_centroid *out, uint32_t cap)
{
	double		qtab[GYO_TD_MAX_DELTA + 1];
	const uint32_t	d = (uint32_t)delta;
	uint64_t	W = 0, pref = 0, cw = 0;
	uint32_t	nout = 0, cell = 0;
	double		csum = 0.0;

	if (!n) return 0;
	td_qtab(delta, qtab);
	for (uint32_t i = 0; i < n; ++i) W += in[i].weight;

	for (uint32_t i = 0; i < n; ++i) {
		uint32_t c = cell;

		/* advance to the cell that holds the item's centre: T_c <= pref + w / 2 < T_c+1 (T_d = W). For integers 2 pref + w >= 2 T
		 * iff pref + floor(w / 2) >= T, a key that never exceeds W (2 T would overflow near the largest totals) */
		const uint64_t ckey = pref + in[i].weight / 2;

		while (c + 1 < d && (uint64_t)(qtab[c + 1] * (double)W) <= ckey) ++c;
		if (i && c != cell) {
			if (nout < cap) { out[nout].mean = csum / (double)cw; out[nout].weight = cw; }
			nout++;
			cw = 0; csum = 0.0;
		}
		cell = c;
		csum += in[i].mean * (double)in[i].weight;
		cw += in[i].weight;
		pref += in[i].weight;
	}
	if (nout < cap) { out[nout].mean = csum / (double)cw; out[nout].weight = cw; }
	nout++;
	return nout;
}

static int cmp_u32(const void *a, const void *b)
{
	uint32_t x = *(const uint32_t *)a, y = *(const uint32_t *)b;
	return x < y ? -1 : (x > y);
}

/* stable merge of two mean-sorted centroid lists; on equal means the `a` list goes first */
static uint32_t merge_sorted(const gyo_centroid *a, uint32_t na, const gyo_centroid *b, uint32_t nb, gyo_centroid *out)
{
	uint32_t i = 0, j = 0, k = 0;

	while (i < na && j < nb) out[k++] = (b[j].mean < a[i].mean) ? b[j++] : a[i++];
	while (i < na) out[k++] = a[i++];
	while (j < nb) out[k++] = b[j++];
	return k;
}

/* Log-linear value code: 32 bins per octave (5 mantissa bits), exact below 32. Monotone in v; < 1024 for v < 2^30.
 * The CUDA path sorts a batch's samples by (service, code) only — 27 instead of 47 significant key bits — so the samples
 * inside one bin arrive in no particular order and a bin is the unit the batch clustering works with. */
uint32_t gyo_td_code(uint32_t v)
{
	if (v < 32u) return v;
	uint32_t sh = (31u - (uint32_t)__builtin_clz(v)) - 5u;

	return ((sh + 1u) << 5) | ((v >> sh) & 31u);
}

/* What the CUDA path does for one device batch and service: the batch's samples fall into value bins — bin index =
 * gyo_td_code(usec) + RESP_TIME_HASH bucket of usec / 1000, monotone in usec, so no bin straddles a histogram bucket — and
 * every non-empty bin becomes ONE item {mean = exact usec sum / samples, weight = samples}. The items, in bin order, are merged
 * with the old centroids (old first on equal means) and one greedy pass (with the ladder) cuts the list to <= GYO_TD_CAP. */
#define GYO_NBINS	848

static uint32_t td_bin_index(uint32_t usec)
{
	return gyo_td_code(usec) + (uint32_t)gyo_bucket(GYO_CLS_RESP_TIME, (int64_t)(usec / 1000u));
}

void gyo_td_add_batch(gyo_tdigest *t, const uint32_t *vals, uint32_t n, double delta)
{
	if (!n) return;

	static __thread uint64_t	bcnt[GYO_NBINS], bsum[GYO_NBINS];
	gyo_centroid	items[GYO_NBINS], merged[GYO_NBINS + GYO_TD_CAP], outc[GYO_TD_CAP + 1];
	uint32_t	nitems = 0, vmin = vals[0], vmax = vals[0];

	memset(bcnt, 0, sizeof(bcnt)); memset(bsum, 0, sizeof(bsum));
	for (uint32_t i = 0; i < n; ++i) {
		uint32_t b = td_bin_index(vals[i]);

		bcnt[b]++; bsum[b] += vals[i];
		if (vals[i] < vmin) vmin = vals[i];
		if (vals[i] > vmax) vmax = vals[i];
	}
	for (uint32_t b = 0; b < GYO_NBINS; ++b) {
		if (!bcnt[b]) continue;
		items[nitems].mean = (double)bsum[b] / (double)bcnt[b]; items[nitems].weight = bcnt[b];
		nitems++;
	}
	if ((double)vmin < t->minv) t->minv = (double)vmin;
	if ((double)vmax > t->maxv) t->maxv = (double)vmax;

	uint32_t nm = merge_sorted(t->c, t->n, items, nitems, merged);
	uint32_t no = gyo_td_compress(merged, nm, delta, outc, GYO_TD_CAP);

	if (no > GYO_TD_CAP) no = GYO_TD_CAP;
	memcpy(t->c, outc, sizeof(gyo_centroid) * no);
	t->n = no;
	t->total += n;
}

/* classic MergingDigest: buffer 5*delta raw points, then sort buffer, merge with centroids, compress */
void gyo_td_add_classic(gyo_tdigest *t, const uint32_t *vals, uint32_t n, double delta)
{
	uint32_t bufcap = (uint32_t)(5 * delta);
	gyo_centroid *buf = (gyo_centroid *)malloc(sizeof(gyo_centroid) * (bufcap + 2 * GYO_TD_CAP));
	gyo_centroid *tmp = (gyo_centroid *)malloc(sizeof(gyo_centroid) * (bufcap + 2 * GYO_TD_CAP));
	uint32_t *chunk = (uint32_t *)malloc(sizeof(uint32_t) * bufcap);
	gyo_centroid outc[GYO_TD_CAP + 1];

	for (uint32_t off = 0; off < n; off += bufcap) {
		uint32_t m = n - off < bufcap ? n - off : bufcap;

		memcpy(chunk, vals + off, sizeof(uint32_t) * m);
		qsort(chunk, m, sizeof(uint32_t), cmp_u32);
		for (uint32_t i = 0; i < m; ++i) { buf[i].mean = (double)chunk[i]; buf[i].weight = 1; }
		if ((double)chunk[0] < t->minv) t->minv = (double)chunk[0];
		if ((double)chunk[m - 1] > t->maxv) t->maxv = (double)chunk[m - 1];

		uint32_t nm = merge_sorted(t->c, t->n, buf, m, tmp);
		uint32_t no = gyo_td_compress(tmp, nm, delta, outc, GYO_TD_CAP);

		if (no > GYO_TD_CAP) no = GYO_TD_CAP;
		memcpy(t->c, outc, sizeof(gyo_centroid) * no);
		t->n = no;
		t->total += m;
	}
	free(buf); free(tmp); free(chunk);
}

/* quantile by linear interpolation between centroid centres (centre of centroid i sits at cumulative weight
 * W_{i-1} + w_i/2); the two ends interpolate towards the tracked min / max. */
double gyo_td_quantile(const gyo_centroid *c, uint32_t n, double minv, double maxv, double q)
{
	double total = 0, target, cum = 0, prev_center, prev_mean;

	if (!n) return NAN;
	for (uint32_t i = 0; i < n; ++i) total += (double)c[i].weight;
	if (q <= 0) return minv;
	if (q >= 1) return maxv;
	target = q * total;

	prev_center = 0; prev_mean = minv;
	for (uint32_t i = 0; i < n; ++i) {
		double center = cum + (double)c[i].weight / 2.0;

		if (target < center) {
			double span = center - prev_center;
			return span > 0 ? prev_mean + (c[i].mean - prev_mean) * ((target - prev_center) / span) : c[i].mean;
		}
		prev_center = center; prev_mean = c[i].mean;
		cum += (double)c[i].weight;
	}
	{
		double span = total - prev_center;
		return span > 0 ? prev_mean + (maxv - prev_mean) * ((target - prev_center) / span) : maxv;
	}
}

double gyo_td_quantile_f(const float *means, const float *weights, uint32_t n, float minv, float maxv, double q)
{
	gyo_centroid c[2 * GYO_TD_CAP];

	if (n > 2 * GYO_TD_CAP) n = 2 * GYO_TD_CAP;
	for (uint32_t i = 0; i < n; ++i) { c[i].mean = means[i]; c[i].weight = (uint64_t)weights[i]; }
	return gyo_td_quantile(c, n, minv, maxv, q);
}

/* ------------------------------------------------------------------------------------------------
 * engine-level oracle: sequential fold of the 32-byte event stream into the same state the CUDA engine keeps.
 * Semantics per event type are those of include/gysketch.h; each follows the reference code cited there.
 * ------------------------------------------------------------------------------------------------ */
typedef struct svc_state
{
	uint64_t	id;
	gyo_hist	cur, last, all;		/* RESP_TIME_HASH, T = int64 */
	gyo_hist	ring[GYO_NLEVELS][GYO_NSLOTS];	/* 300 s and 432000 s levels, 10 slots each */
	uint64_t	conn_cur, conn_last;	/* packed {count, kbytes} like a CMS cell */
	uint32_t	bm_cur[16], bm_last[16];	/* CONN_BITMAP transposed: per response bucket a mask over (client port & 31) */
	uint64_t	conn_all_cnt, conn_all_kb;
	uint8_t		*hll;
	gyo_tdigest	td;
	uint32_t	*pend;			/* RESP samples (usec) of the batch being ingested */
	uint32_t	npend, cappend;
	uint32_t	first_seen, last_active;	/* tsec of the first flush that saw the service / of the last window with events */
	uint64_t	act_cur, act_last;	/* ACTIVE_CONN_STATS roll-up {active conns : 32 | kbytes : 32} */
	uint64_t	err_cur, err_last;	/* API_TRAN error counters {client : 32 | server : 32} */
	uint32_t	rtt_cur, rtt_last;	/* max of max_rtt_msec_ (float bits; non-negative floats order like their bits) */
	gyo_hist	qps_hist, act_hist;	/* TCP_LISTENER::qps_hist_ (SEMI_LOG_HASH_LO, int) / active_conn_hist_ (HASH_1_3000, int), gy_socket_stat.h:548-549 */
	uint8_t		state, issue, issue_bits, high_bits;	/* curr_state_, curr_issue_, issue_bit_hist_, high_resp_bit_hist_ (gy_socket_stat.h:654-657) */
	uint32_t	nconn_active;		/* last reported active connection count (kept between ACTIVE_CONN_STATS reports) */
} svc_state;

typedef struct task_state
{
	uint64_t	id;
	gyo_hist	cpu_pct, cpu_delay, blkio_delay;	/* MTASK_HIST, server/gy_msocket.h:704-718 */
	uint64_t	prev[3][2], last[3][2];			/* {count, sum} totals at the last flush / of the last closed window */
} task_state;

typedef struct idmap { uint64_t *keys; uint32_t *vals; uint32_t cap, n; uint32_t *freed; uint32_t nfreed; } idmap;
#define GYO_TOMBSTONE	(~0ull)		/* key of a deleted entry: never matches, never ends a probe chain */

struct gyo_engine
{
	uint32_t	max_svcs, max_tasks, depth, log2w, hll_p, flags, rank, world;
	double		delta;
	idmap		smap, tmap;
	svc_state	*svcs;
	task_state	*tasks;
	uint64_t	*cms_cur, *cms_last;
	uint64_t	n_in, n_drop, n_resp, n_tcp, n_task, n_foreign;
	uint64_t	ring_epoch[GYO_NLEVELS][GYO_NSLOTS];
	uint32_t	last_flush_tsec;
	uint32_t	*touched;		/* slots with pending RESP samples in the batch being ingested */
	uint32_t	ntouched;
	uint32_t	idle_evict_secs;	/* 0 = never */
	uint64_t	*evicted;		/* ids evicted by the last flush */
	uint32_t	nevicted;
	uint64_t	evicted_total;
};

static uint32_t pow2_at_least(uint32_t v) { uint32_t p = 16; while (p < v) p <<= 1; return p; }

static void idmap_init(idmap *m, uint32_t maxn)
{
	m->cap = pow2_at_least(maxn * 2);
	m->keys = (uint64_t *)calloc(m->cap, sizeof(uint64_t));
	m->vals = (uint32_t *)calloc(m->cap, sizeof(uint32_t));
	m->freed = (uint32_t *)calloc(maxn ? maxn : 1, sizeof(uint32_t));
	m->n = 0; m->nfreed = 0;
}

/* open addressing keyed by get_uint64_hash (how the reference keys listen_tbl_, gy_mconnhdlr.cc:11183) */
static int idmap_find(idmap *m, uint64_t key, int insert, uint32_t maxn)
{
	uint32_t pos = gyo_uint64_hash(key) & (m->cap - 1);

	if (key == GYO_TOMBSTONE) return -1;
	for (;;) {
		if (m->keys[pos] == key) return (int)m->vals[pos];
		if (m->keys[pos] == 0) {
			if (!insert || key == GYO_TOMBSTONE) return -1;
			if (m->nfreed) { m->keys[pos] = key; m->vals[pos] = m->freed[--m->nfreed]; return (int)m->vals[pos]; }	/* recycled slot */
			if (m->n >= maxn) return -1;
			m->keys[pos] = key; m->vals[pos] = m->n;
			return (int)m->n++;
		}
		pos = (pos + 1) & (m->cap - 1);
	}
}

gyo_engine *gyo_create(uint32_t max_svcs, uint32_t max_tasks, uint32_t cms_depth, uint32_t cms_log2_width, uint32_t hll_p,
		uint32_t td_compression, uint32_t flags, uint32_t rank, uint32_t world)
{
	gyo_engine *e = (gyo_engine *)calloc(1, sizeof(*e));

	e->max_svcs = max_svcs; e->max_tasks = max_tasks; e->depth = cms_depth; e->log2w = cms_log2_width;
	e->hll_p = hll_p; e->delta = td_compression; e->flags = flags; e->rank = rank; e->world = world ? world : 1;
	idmap_init(&e->smap, max_svcs);
	idmap_init(&e->tmap, max_tasks ? max_tasks : 1);
	e->svcs = (svc_state *)calloc(max_svcs, sizeof(svc_state));
	e->tasks = (task_state *)calloc(max_tasks ? max_tasks : 1, sizeof(task_state));
	e->cms_cur = (uint64_t *)calloc((size_t)cms_depth << cms_log2_width, sizeof(uint64_t));
	e->cms_last = (uint64_t *)calloc((size_t)cms_depth << cms_log2_width, sizeof(uint64_t));
	e->touched = (uint32_t *)malloc(sizeof(uint32_t) * max_svcs);
	e->evicted = (uint64_t *)malloc(sizeof(uint64_t) * max_svcs);
	memset(e->ring_epoch, 0xFF, sizeof(e->ring_epoch));
	return e;
}

void gyo_destroy(gyo_engine *e)
{
	if (!e) return;
	for (uint32_t i = 0; i < e->smap.n; ++i) { free(e->svcs[i].hll); free(e->svcs[i].pend); }
	free(e->svcs); free(e->tasks); free(e->cms_cur); free(e->cms_last); free(e->touched); free(e->evicted);
	free(e->smap.keys); free(e->smap.vals); free(e->tmap.keys); free(e->tmap.vals); free(e->smap.freed); free(e->tmap.freed);
	free(e);
}

static svc_state *get_svc(gyo_engine *e, uint64_t id, int insert)
{
	int slot = idmap_find(&e->smap, id, insert, e->max_svcs);

	if (slot < 0) return NULL;
	svc_state *s = &e->svcs[slot];
	if (s->id != id) {			/* fresh or recycled slot */
		free(s->hll); free(s->pend);
		memset(s, 0, sizeof(*s));
		s->id = id;
		gyo_hist_init(&s->cur, GYO_CLS_RESP_TIME, GYO_T_INT64);
		gyo_hist_init(&s->last, GYO_CLS_RESP_TIME, GYO_T_INT64);
		gyo_hist_init(&s->all, GYO_CLS_RESP_TIME, GYO_T_INT64);
		for (int l = 0; l < GYO_NLEVELS; ++l) for (int k = 0; k < GYO_NSLOTS; ++k) gyo_hist_init(&s->ring[l][k], GYO_CLS_RESP_TIME, GYO_T_INT64);
		gyo_hist_init(&s->qps_hist, GYO_CLS_SEMI_LOG_LO, GYO_T_INT);
		gyo_hist_init(&s->act_hist, GYO_CLS_HASH_1_3000, GYO_T_INT);
		s->state = GYO_STATE_OK; s->issue = 0; s->issue_bits = 0; s->high_bits = 0; s->nconn_active = 0;
		s->hll = (uint8_t *)calloc(1u << e->hll_p, 1);
		gyo_td_init(&s->td);
	}
	return s;
}

static task_state *get_task(gyo_engine *e, uint64_t id, int insert)
{
	uint32_t before = e->tmap.n;
	int slot = idmap_find(&e->tmap, id, insert, e->max_tasks);

	if (slot < 0) return NULL;
	task_state *t = &e->tasks[slot];
	if ((uint32_t)slot >= before) {
		t->id = id;
		gyo_hist_init(&t->cpu_pct, GYO_CLS_HASH_1_3000, GYO_T_INT);
		gyo_hist_init(&t->cpu_delay, GYO_CLS_DURATION, GYO_T_INT);
		gyo_hist_init(&t->blkio_delay, GYO_CLS_DURATION, GYO_T_INT);
	}
	return t;
}

int gyo_register_ids(gyo_engine *e, const uint64_t *ids, uint32_t n, int is_task)
{
	for (uint32_t i = 0; i < n; ++i) {
		if (!ids[i]) continue;
		if (is_task ? !get_task(e, ids[i], 1) : !get_svc(e, ids[i], 1)) return -28;
	}
	return 0;
}

int gyo_ingest(gyo_engine *e, const gyo_event *ev, uint64_t n)
{
	const int autoreg = (int)(e->flags & 1u);
	const uint32_t wmask = (1u << e->log2w) - 1;

	for (uint64_t i = 0; i < n; ++i) {
		const gyo_event *p = &ev[i];

		if (e->world > 1 && (p->host_idx % e->world) != e->rank) { e->n_foreign++; continue; }
		e->n_in++;
		if (p->svc_id == 0) { e->n_drop++; continue; }

		switch (p->type) {

		case 5 : {	/* RESP: SVC_INFO_CAP::upd_stats_on_req gy_proto_parser.cc:2678 (usec/1000 -> resp_cache_.add_cache);
				   validity rule of handle_ipv4_resp_event gy_socket_stat.cc:1519-1524 (drop > 1 000 000 msec) */
			uint32_t ms = p->value / 1000u;
			if (ms > 1000000u) { e->n_drop++; break; }
			svc_state *s = get_svc(e, p->svc_id, autoreg);
			if (!s) { e->n_drop++; break; }
			{
				/* TCP_LISTENER::CONN_BITMAP::add_response, common/gy_socket_stat.h:403-410: respmap_[cli_port & 0x1F].set(bucket) */
				int b = gyo_hist_add(&s->cur, (int64_t)ms);
				s->bm_cur[b] |= 1u << (uint32_t)(p->flow_key & 0x1F);
			}
			/* SVC_INFO_CAP::upd_stats_on_req, gy_proto_parser.cc:2685-2692: stats_.ncli_errors_++ / nser_errors_++ */
			if (p->flags & 3u) s->err_cur += (uint64_t)(p->flags & 1u) | ((uint64_t)((p->flags >> 1) & 1u) << 32);
			if (s->npend == 0) e->touched[e->ntouched++] = (uint32_t)(s - e->svcs);
			if (s->npend == s->cappend) {
				s->cappend = s->cappend ? s->cappend * 2 : 16;
				s->pend = (uint32_t *)realloc(s->pend, sizeof(uint32_t) * s->cappend);
			}
			s->pend[s->npend++] = p->value;
			e->n_resp++;
			break;
		}

		case 1 : case 2 : case 3 : case 4 : {	/* TCP connect/accept/close: group-by of partha_tcp_conn_info gy_mconnhdlr.cc:9245-9311
							   approximated by CMS(flow) + HLL(svc) + an exact per-service cell */
			svc_state *s = get_svc(e, p->svc_id, autoreg);
			if (!s) { e->n_drop++; break; }
			uint64_t inc = gyo_cms_increment(p->value);
			for (uint32_t r = 0; r < e->depth; ++r) {
				e->cms_cur[((size_t)r << e->log2w) + (gyo_cms_index(p->flow_key, r, e->log2w) & wmask)] += inc;
			}
			uint32_t idx; uint8_t rank;
			gyo_hll_idx_rank(p->flow_key, e->hll_p, &idx, &rank);
			if (s->hll[idx] < rank) s->hll[idx] = rank;
			s->conn_cur += inc;
			e->n_tcp++;
			break;
		}

		case 7 : {	/* ACTIVE: one ACTIVE_CONN_STATS record = the 15-s inet_diag group-by {ser_glob_id, cli_task_aggr_id} of
				   upd_conn_from_diag (common/gy_socket_stat.cc:6156-6194: bytes +=, active conns +=, max rtt) as madhava
				   receives it (handle_partha_active_conns, server/gy_mconnhdlr.cc:7705). value = kbytes, flags = active_conns_,
				   tsec = float bits of max_rtt_msec_. Flow sketch: conns and kbytes of the flow; service: totals of the window */
			svc_state *s = get_svc(e, p->svc_id, autoreg);
			if (!s) { e->n_drop++; break; }
			uint64_t inc = (uint64_t)p->flags | ((uint64_t)p->value << 32);
			for (uint32_t r = 0; r < e->depth; ++r) {
				e->cms_cur[((size_t)r << e->log2w) + (gyo_cms_index(p->flow_key, r, e->log2w) & wmask)] += inc;
			}
			uint32_t idx; uint8_t rank;
			gyo_hll_idx_rank(p->flow_key, e->hll_p, &idx, &rank);
			if (s->hll[idx] < rank) s->hll[idx] = rank;
			s->act_cur += inc;
			if (p->tsec > s->rtt_cur) s->rtt_cur = p->tsec;
			e->n_tcp++;
			break;
		}

		case 6 : {	/* TASK: MAGGR_TASK::set_local_task_state server/gy_msocket.h:1009-1018 */
			task_state *t = get_task(e, p->svc_id, autoreg);
			if (!t) { e->n_drop++; break; }
			gyo_hist_add(&t->cpu_pct, (int64_t)(int)p->value);
			gyo_hist_add(&t->cpu_delay, (int64_t)(int)(uint32_t)(p->flow_key & 0xFFFFFFFFu));
			gyo_hist_add(&t->blkio_delay, (int64_t)(int)(uint32_t)(p->flow_key >> 32));
			e->n_task++;
			break;
		}

		default :
			e->n_drop++;
			break;
		}
	}

	/* end of device batch: batched t-digest update per touched service */
	for (uint32_t i = 0; i < e->ntouched; ++i) {
		svc_state *s = &e->svcs[e->touched[i]];

		gyo_td_add_batch(&s->td, s->pend, s->npend, e->delta);
		s->npend = 0;
	}
	e->ntouched = 0;
	return 0;
}

/* 5-second roll: listener_stats_update gy_socket_stat.cc:3898 reads the window that just closed, then the window restarts.
 * Levels follow Level_5s_5min_5days_all (gy_statistics.h:1545-1551) with 10 slots per level (:1105). folly's
 * MultiLevelTimeSeries is un-vendored, so the slot rule is OUR definition: level with duration D has 10 slots of width D/10;
 * a window closing at tsec is added to slot (tsec / width) % 10 after that slot is cleared if it still holds an older epoch;
 * a level's answer = sum of the slots whose epoch lies within the last 10 epochs. The 5-s level is the window itself. */
static const uint32_t g_level_width[GYO_NLEVELS] = { 30, 43200 };

static void level_sum(const gyo_engine *e, const svc_state *s, int l, gyo_hist *out);

/* ---- listener state ---------------------------------------------------------------------------------------------------------
 * TCP_LISTENER::get_curr_state, common/gy_socket_stat.cc:2020-2875, without the sentence it formats. Statement order and operand
 * types as in the reference (ser_errors uint32, curr_qps int, data_value int64, mean_val_ double, 0.8f / 1.1f / 1.2f float
 * constants). Line numbers cite the condition each rule restates. */
static int resp_bucketid(int64_t thr)		/* get_bucketid_from_threshold<RESP_TIME_HASH>, common/gy_statistics.h:517-531 */
{
	const int64_t *t = g_cls[GYO_CLS_RESP_TIME].thr;
	for (int i = 0; i < 13; ++i) if (thr == t[i]) return i + 1;
	if (thr < 0) return 0;
	return 14;
}

#define OUT(st_, is_)	do { *state = (uint8_t)(st_); *issue = (uint8_t)(is_); return; } while (0)
#define OK_OR_ERRORS()	OUT(GYO_STATE_OK, ser ? GYO_ISSUE_SERVER_ERRORS : GYO_ISSUE_NONE)

void gyo_listener_state(const gyo_state_in *in, uint8_t *high, uint8_t *state, uint8_t *issue)
{
	const uint32_t	ser = in->ser_errors;
	const size_t	nq = (size_t)in->nqrys_5s;
	const int	tissue = in->task_issue, severe = in->task_severe, delay = in->task_delay;
	const int	nbad = in->ntasks_issue, ngood = in->ntasks_noissue;
	const int	b5 = resp_bucketid(in->r5p95), b300 = resp_bucketid(in->r300p95), b5d = resp_bucketid(in->r5dp95);	/* :2094-2096 */
	int		qps = (int)(in->nqrys_5s / 5);
	if (in->last_qps_count > qps) qps = in->last_qps_count;						/* :2092 */
	const int	worse = (b5 > b5d + 2) && (b5 > b300);

	*high = (uint8_t)(*high << 1);										/* :2120 */

	if (qps == 0 && (!tissue || !severe || !ser)) OUT(GYO_STATE_IDLE, GYO_ISSUE_NONE);			/* :2122-2136 */

	if (b5 == 1 || in->r5p95 < in->r5dp95) {								/* :2139 */
		if (qps <= in->qps_p25 && in->qps_p25 < in->qps_p95) {						/* :2143 */
			if (!tissue) {
				if (!ser) OUT(GYO_STATE_IDLE, GYO_ISSUE_NONE);					/* :2145 */
				if ((size_t)(uint32_t)(ser * 2u) > nq) OUT(GYO_STATE_SEVERE, GYO_ISSUE_SERVER_ERRORS);	/* :2154 */
				if ((size_t)(uint32_t)(ser * 5u) > nq) OUT(GYO_STATE_BAD, GYO_ISSUE_SERVER_ERRORS);	/* :2162 */
				if (ser < nq * 0.1) OUT(GYO_STATE_OK, GYO_ISSUE_SERVER_ERRORS);			/* :2170 */
			}
			else {
				if ((size_t)(uint32_t)(ser * 2u) > nq) OUT(GYO_STATE_SEVERE, GYO_ISSUE_SERVER_ERRORS);	/* :2181 */
				if ((size_t)(uint32_t)(ser * 5u) > nq) OUT(GYO_STATE_BAD, GYO_ISSUE_SERVER_ERRORS);	/* :2189 */
				if (ser) OUT(GYO_STATE_BAD, GYO_ISSUE_TASKS);						/* :2197 */
				if (severe && nbad > 0 && ngood == 0) OUT(GYO_STATE_BAD, GYO_ISSUE_TASKS);		/* :2206 */
				if (in->nconn > in->act_p25) OUT(GYO_STATE_OK, GYO_ISSUE_TASKS);			/* :2216 */
			}
		}
		if (ser) {											/* :2229 */
			if ((size_t)(uint32_t)(ser * 2u) > nq) OUT(GYO_STATE_SEVERE, GYO_ISSUE_SERVER_ERRORS);
			if ((size_t)(uint32_t)(ser * 5u) > nq) OUT(GYO_STATE_BAD, GYO_ISSUE_SERVER_ERRORS);
		}
		if (tissue && severe && nbad > 0 && ngood == 0) OUT(GYO_STATE_BAD, GYO_ISSUE_TASKS);		/* :2260 */
		if (ser) OUT(GYO_STATE_OK, GYO_ISSUE_SERVER_ERRORS);						/* :2294 */
		if (qps <= in->qps_p95 || b5 + 2 <= b5d) OUT(GYO_STATE_GOOD, GYO_ISSUE_NONE);			/* :2276 */
		OUT(GYO_STATE_OK, GYO_ISSUE_QPS_HIGH);								/* :2287 */
	}

	if (in->r5p95 == in->r5dp95) {										/* :2307 */
		if (ser) {
			if ((size_t)(uint32_t)(ser * 2u) > nq) OUT(GYO_STATE_SEVERE, GYO_ISSUE_SERVER_ERRORS);
			if ((size_t)(uint32_t)(ser * 5u) > nq) OUT(GYO_STATE_BAD, GYO_ISSUE_SERVER_ERRORS);
		}
		if (in->mean5 <= in->mean5d * 0.8f) {								/* :2340 */
			if (qps <= in->qps_p25) {								/* :2342 */
				if (ser) OUT(GYO_STATE_BAD, GYO_ISSUE_SERVER_ERRORS);
				if (!tissue) OUT(GYO_STATE_IDLE, GYO_ISSUE_NONE);
				if (nbad > 0 && ngood == 0) OUT(GYO_STATE_BAD, GYO_ISSUE_TASKS);
				if (nbad > 0 && in->tasks_delay_msec >= 1000) OUT(GYO_STATE_BAD, GYO_ISSUE_TASKS);
			}
			if (!tissue && !ser) OUT(GYO_STATE_GOOD, GYO_ISSUE_NONE);				/* :2386 */
			if (ser && tissue) OUT(GYO_STATE_BAD, GYO_ISSUE_TASKS);					/* :2394-2395 */
			/* :2402-2415: the {SERVER_ERRORS, OK} assignment for errors without a process issue has no return and is overwritten */
			OUT(GYO_STATE_OK, GYO_ISSUE_TASKS);
		}
		if (in->mean5 <= in->mean5d * 1.2f) OUT(GYO_STATE_OK, GYO_ISSUE_NONE);				/* :2419 */
	}

	*high |= 1;												/* :2430 */

	if (ser) {
		if ((size_t)(uint32_t)(ser * 2u) > nq) OUT(GYO_STATE_SEVERE, GYO_ISSUE_SERVER_ERRORS);		/* :2433 */
		if ((size_t)(uint32_t)(ser * 5u) > nq) OUT(GYO_STATE_BAD, GYO_ISSUE_SERVER_ERRORS);
	}
	if (qps > in->qps_p95 && qps - in->qps_p95 > 5 && qps > in->qps_p95 * 1.1f)				/* :2464 */
		OUT(worse ? GYO_STATE_SEVERE : GYO_STATE_BAD, GYO_ISSUE_QPS_HIGH);
	if (tissue || (delay && nbad + ngood > 2 && in->tasks_delay_msec * 4 > in->total_resp_msec))		/* :2494 */
		OUT(worse ? GYO_STATE_SEVERE : GYO_STATE_BAD, GYO_ISSUE_TASKS);
	if (in->curr_active_conn > in->act_p95 && in->curr_active_conn - in->act_p95 > 1)			/* :2525 */
		OUT(worse && in->curr_active_conn > 10 ? GYO_STATE_SEVERE : GYO_STATE_BAD, GYO_ISSUE_ACTIVE_CONN_HIGH);
	if (in->r5p95 == in->r5dp95 && in->r5p99 > in->r5dp99) OK_OR_ERRORS();					/* :2552-2554 */
	if (qps <= in->qps_p25 && in->nconn <= in->act_p25) {							/* :2576 */
		if (delay && in->cpu_issue && in->mem_issue) OUT(GYO_STATE_BAD, GYO_ISSUE_TASKS);
		if (delay && (in->cpu_issue || in->mem_issue) && in->tasks_delay_msec * 4 > in->total_resp_msec) OUT(GYO_STATE_BAD, GYO_ISSUE_TASKS);
		OK_OR_ERRORS();
	}
	{
		const int avg5d = (int)((int64_t)in->tcount_5d / (in->secs_5d > 0 ? in->secs_5d : 1));	/* :2638 */
		if (avg5d < (qps >> 1) && in->r5p95 <= in->rallp95 && in->mean5 <= in->meanall * 1.1f) OK_OR_ERRORS();
	}
	if (qps <= in->qps_p25 && in->curr_active_conn <= in->act_p25 && b5 <= b5d + 1) OK_OR_ERRORS();	/* :2661 */
	if (b5 <= b5d + 1 && b300 == b5d && in->mean5 > in->mean300 && in->mean300 < in->mean5d * 1.1f) OK_OR_ERRORS();	/* :2684-2685 */
	if (in->curr_active_conn >= 15 && b5 == b5d + 1) {							/* :2710 */
		int b = b5;
		while (b < 15 && in->nactive_conn_arr[b] <= 3) b++;
		if (b > b5) OK_OR_ERRORS();
	}
	if (__builtin_popcount(*high) < 5) OK_OR_ERRORS();							/* :2748-2749 */
	{
		const int st = worse ? GYO_STATE_SEVERE : GYO_STATE_BAD;					/* :2774 */
		if (in->tasks_delay_msec * 4 > in->total_resp_msec && st == GYO_STATE_BAD) OUT(st, GYO_ISSUE_TASKS);	/* :2791 */
		if (in->nserdepends > 0) OUT(st, GYO_ISSUE_DEPENDENT);						/* :2825 */
		if (in->tasks_delay_msec * 10 > in->total_resp_msec) OUT(st, GYO_ISSUE_TASKS);			/* :2829 */
		OUT(st, ser ? GYO_ISSUE_SERVER_ERRORS : GYO_ISSUE_UNKNOWN);					/* :2855-2860 */
	}
}
#undef OUT
#undef OK_OR_ERRORS

/* statistics of one response level as TIME_HISTOGRAM::get_stats hands them out (common/gy_statistics.h:1333-1362; percentile rule:
 * GY_HISTOGRAM::get_percentiles — folly's level percentile is un-vendored, see DESIGN.md §5) */
static void level_stats(const gyo_hist *h, int64_t *p95, int64_t *p99, int64_t *p25, uint64_t *cnt, uint64_t *sum, double *mean)
{
	const float pcts[3] = {95, 99, 25};
	int64_t v[3];
	uint64_t c = 0, sm = 0;

	gyo_hist_percentiles(h, pcts, 3, v, NULL);
	for (int b = 0; b < 15; ++b) { c += h->stats[b].count; sm += (uint64_t)h->stats[b].sum; }
	for (int k = 0; k < 3; ++k) if (v[k] < 0) v[k] = 0;
	*p95 = v[0]; *p99 = v[1]; if (p25) *p25 = v[2];
	*cnt = c; *sum = sm; *mean = (double)(int64_t)sm / (double)(c ? (int64_t)c : 1);
}

/* the part of listener_stats_update (common/gy_socket_stat.cc:4045-4272) around the state decision, for one service whose closing
 * window was not stale: qps / active-connection samples (:4111-4130), the connection counts (:4158-4173), get_curr_state (:4233),
 * issue_bit_hist_ and the young-listener override (:4242-4272). Called by gyo_flush after the window has rolled. */
static void svc_update_state(const gyo_engine *e, svc_state *s, uint32_t tsec)
{
	gyo_state_in in;
	gyo_hist l300, l5d;
	uint64_t c, sm;
	const float pq[2] = {95, 25};
	int64_t v[2];

	memset(&in, 0, sizeof(in));
	level_stats(&s->last, &in.r5p95, &in.r5p99, NULL, &in.nqrys_5s, &in.total_resp_msec, &in.mean5);
	level_sum(e, s, 0, &l300); level_sum(e, s, 1, &l5d);
	level_stats(&l300, &in.r300p95, &in.r300p99, NULL, &c, &sm, &in.mean300);
	level_stats(&l5d, &in.r5dp95, &in.r5dp99, &in.r5dp25, &in.tcount_5d, &sm, &in.mean5d);
	level_stats(&s->all, &in.rallp95, &in.rallp99, NULL, &c, &sm, &in.meanall);

	in.last_qps_count = (int32_t)(in.nqrys_5s / 5);
	gyo_hist_add(&s->qps_hist, in.last_qps_count);								/* :4113 */
	if ((uint32_t)s->act_last) s->nconn_active = (uint32_t)s->act_last;					/* a report arrived in this window */
	gyo_hist_add(&s->act_hist, (int64_t)(int32_t)s->nconn_active);					/* :4128 */
	gyo_hist_percentiles(&s->qps_hist, pq, 2, v, NULL); in.qps_p95 = v[0]; in.qps_p25 = v[1];
	gyo_hist_percentiles(&s->act_hist, pq, 2, v, NULL); in.act_p95 = v[0]; in.act_p25 = v[1];

	in.nconn = (int32_t)s->nconn_active;
	in.curr_active_conn = in.nconn;
	for (int b = 0; b < 15; ++b) {										/* :4160-4168 */
		in.nactive_conn_arr[b] = (uint8_t)__builtin_popcount(s->bm_last[b]);
		if (in.curr_active_conn < in.nactive_conn_arr[b]) in.curr_active_conn = in.nactive_conn_arr[b];
	}
	in.ser_errors = (uint32_t)(s->err_last >> 32);
	const uint32_t age = tsec > s->first_seen ? tsec - s->first_seen : 0;
	in.secs_5d = age + 1 < 432000 ? age + 1 : 432000;							/* :2033-2034, :2067-2074 */

	gyo_listener_state(&in, &s->high_bits, &s->state, &s->issue);
	if (age > 100 || in.ser_errors) {									/* :4242 */
		s->issue_bits = (uint8_t)(s->issue_bits << 1);
		if (s->state >= GYO_STATE_BAD) s->issue_bits |= 1;
	}
	else { s->issue_bits = 0; s->issue = GYO_ISSUE_NONE; s->state = GYO_STATE_OK; }			/* :4262-4270 */
}

int gyo_export_state(gyo_engine *e, uint64_t id, uint32_t out[5])
{
	int slot = idmap_find(&e->smap, id, 0, 0);
	if (slot < 0) return -2;
	const svc_state *s = &e->svcs[slot];
	out[0] = s->state; out[1] = s->issue; out[2] = s->issue_bits; out[3] = s->high_bits; out[4] = s->nconn_active;
	return 0;
}

void gyo_flush(gyo_engine *e, uint32_t tsec)
{
	int clear[GYO_NLEVELS], slot[GYO_NLEVELS];

	for (int l = 0; l < GYO_NLEVELS; ++l) {
		uint64_t epoch = tsec / g_level_width[l];
		slot[l] = (int)(epoch % GYO_NSLOTS);
		clear[l] = e->ring_epoch[l][slot[l]] != epoch;
		e->ring_epoch[l][slot[l]] = epoch;
	}
	e->last_flush_tsec = tsec;

	e->nevicted = 0;
	for (uint32_t i = 0; i < e->smap.n; ++i) {
		svc_state *s = &e->svcs[i];

		if (!s->id) continue;		/* evicted, slot waiting for reuse */
		/* idle-service rule (ours, after common/gy_socket_stat.cc:3968-3982: tclock != 0, tclock + 300 s < now, tstart + 600 s < now) */
		int active = (uint32_t)s->conn_cur != 0 || (s->conn_cur >> 32) != 0 || s->act_cur != 0 || s->err_cur != 0;
		for (int b = 0; b < 15 && !active; ++b) active = s->cur.stats[b].count != 0;
		if (!s->first_seen) s->first_seen = tsec ? tsec : 1u;
		if (active) s->last_active = tsec ? tsec : 1u;

		s->last = s->cur;
		gyo_hist_merge(&s->all, &s->cur);
		for (int l = 0; l < GYO_NLEVELS; ++l) {
			if (clear[l]) gyo_hist_init(&s->ring[l][slot[l]], GYO_CLS_RESP_TIME, GYO_T_INT64);
			gyo_hist_merge(&s->ring[l][slot[l]], &s->cur);
		}
		gyo_hist_init(&s->cur, GYO_CLS_RESP_TIME, GYO_T_INT64);
		memcpy(s->bm_last, s->bm_cur, sizeof(s->bm_cur)); memset(s->bm_cur, 0, sizeof(s->bm_cur));	/* CONN_BITMAP::clear every 5 s, :436 */
		s->conn_last = s->conn_cur;
		s->conn_all_cnt += (uint32_t)s->conn_cur;
		s->conn_all_kb += s->conn_cur >> 32;
		s->conn_cur = 0;
		s->act_last = s->act_cur; s->act_cur = 0; s->err_last = s->err_cur; s->err_cur = 0; s->rtt_last = s->rtt_cur; s->rtt_cur = 0;
		/* a window without any event of the service is "stale" (:4098-4107): the reference leaves the listener's state as it is */
		if (active) svc_update_state(e, s, tsec);

		if (e->idle_evict_secs && s->last_active && (uint64_t)s->last_active + e->idle_evict_secs < tsec &&
				(uint64_t)s->first_seen + 2ull * e->idle_evict_secs < tsec) {
			/* delete: table entry -> tombstone, slot number recycled, state gone */
			uint32_t pos = gyo_uint64_hash(s->id) & (e->smap.cap - 1);
			while (e->smap.keys[pos] != s->id && e->smap.keys[pos] != 0) pos = (pos + 1) & (e->smap.cap - 1);
			if (e->smap.keys[pos] == s->id) e->smap.keys[pos] = GYO_TOMBSTONE;
			e->evicted[e->nevicted++] = s->id; e->evicted_total++;
			e->smap.freed[e->smap.nfreed++] = i;
			free(s->hll); free(s->pend);
			memset(s, 0, sizeof(*s));
		}
	}
	/* per-task window of the three histograms = totals now - totals at the previous flush (feeds the task top-N) */
	for (uint32_t i = 0; i < e->tmap.n; ++i) {
		task_state *ts = &e->tasks[i];
		const gyo_hist *hh[3] = { &ts->cpu_pct, &ts->cpu_delay, &ts->blkio_delay };
		for (int h = 0; h < 3; ++h) {
			uint64_t cnt = 0, sum = 0;
			for (int b = 0; b < 15; ++b) { cnt += hh[h]->stats[b].count; sum += (uint64_t)hh[h]->stats[b].sum; }
			ts->last[h][0] = cnt - ts->prev[h][0]; ts->last[h][1] = sum - ts->prev[h][1];
			ts->prev[h][0] = cnt; ts->prev[h][1] = sum;
		}
	}
	uint64_t *t = e->cms_last; e->cms_last = e->cms_cur; e->cms_cur = t;
	memset(e->cms_cur, 0, sizeof(uint64_t) * ((size_t)e->depth << e->log2w));
}

/* last closed window of a task: out[h*2] = samples, out[h*2+1] = sum, h = cpu_pct, cpu_delay, blkio_delay */
int gyo_task_last(gyo_engine *e, uint64_t id, uint64_t out[6])
{
	task_state *t = get_task(e, id, 0);
	if (!t) return -2;
	for (int h = 0; h < 3; ++h) { out[2 * h] = t->last[h][0]; out[2 * h + 1] = t->last[h][1]; }
	return 0;
}

void gyo_set_idle_evict(gyo_engine *e, uint32_t secs) { e->idle_evict_secs = secs; }

uint32_t gyo_evicted(gyo_engine *e, uint64_t *out, uint32_t cap, uint64_t *total)
{
	for (uint32_t i = 0; i < e->nevicted && i < cap; ++i) out[i] = e->evicted[i];
	if (total) *total = e->evicted_total;
	return e->nevicted;
}

uint32_t gyo_nsvcs(gyo_engine *e) { return e->smap.n - e->smap.nfreed; }

static void level_sum(const gyo_engine *e, const svc_state *s, int l, gyo_hist *out)
{
	const uint64_t now_epoch = e->last_flush_tsec / g_level_width[l];

	gyo_hist_init(out, GYO_CLS_RESP_TIME, GYO_T_INT64);
	for (int k = 0; k < GYO_NSLOTS; ++k) {
		const uint64_t ep = e->ring_epoch[l][k];
		if (ep != UINT64_MAX && ep + GYO_NSLOTS > now_epoch && ep <= now_epoch) gyo_hist_merge(out, &s->ring[l][k]);
	}
}

int gyo_export_hist(gyo_engine *e, uint64_t id, int which, gyo_serial *out15, uint64_t *total, int64_t *maxv)
{
	const gyo_hist *h = NULL;

	gyo_hist lvl;

	if (which <= 2) {
		int slot = idmap_find(&e->smap, id, 0, 0);
		if (slot < 0) return -2;
		h = which == 0 ? &e->svcs[slot].cur : (which == 1 ? &e->svcs[slot].last : &e->svcs[slot].all);
	}
	else if (which == 6 || which == 7) {
		int slot = idmap_find(&e->smap, id, 0, 0);
		if (slot < 0) return -2;
		level_sum(e, &e->svcs[slot], which - 6, &lvl);
		h = &lvl;
	}
	else if (which == 8 || which == 9) {
		int slot = idmap_find(&e->smap, id, 0, 0);
		if (slot < 0) return -2;
		h = which == 8 ? &e->svcs[slot].qps_hist : &e->svcs[slot].act_hist;
	}
	else {
		int slot = idmap_find(&e->tmap, id, 0, 0);
		if (slot < 0) return -2;
		h = which == 3 ? &e->tasks[slot].cpu_pct : (which == 4 ? &e->tasks[slot].cpu_delay : &e->tasks[slot].blkio_delay);
	}
	memset(out15, 0, sizeof(gyo_serial) * 15);
	memcpy(out15, h->stats, sizeof(gyo_serial) * (size_t)gyo_nbuckets(h->cls));
	*total = h->total_count; *maxv = h->max_val;
	return 0;
}

int gyo_export_hll(gyo_engine *e, uint64_t id, uint8_t *regs)
{
	int slot = idmap_find(&e->smap, id, 0, 0);
	if (slot < 0) return -2;
	memcpy(regs, e->svcs[slot].hll, 1u << e->hll_p);
	return 0;
}

int gyo_export_tdigest(gyo_engine *e, uint64_t id, gyo_tdigest *out)
{
	int slot = idmap_find(&e->smap, id, 0, 0);
	if (slot < 0) return -2;
	*out = e->svcs[slot].td;
	return 0;
}

int gyo_export_conn(gyo_engine *e, uint64_t id, uint64_t *cur, uint64_t *last, uint64_t *all_cnt, uint64_t *all_kb)
{
	int slot = idmap_find(&e->smap, id, 0, 0);
	if (slot < 0) return -2;
	*cur = e->svcs[slot].conn_cur; *last = e->svcs[slot].conn_last;
	*all_cnt = e->svcs[slot].conn_all_cnt; *all_kb = e->svcs[slot].conn_all_kb;
	return 0;
}

/* out[0..5] = act_cur, act_last, err_cur, err_last, rtt_cur (float bits), rtt_last */
int gyo_export_aux(gyo_engine *e, uint64_t id, uint64_t out[6])
{
	int slot = idmap_find(&e->smap, id, 0, 0);
	if (slot < 0) return -2;
	const svc_state *s = &e->svcs[slot];
	out[0] = s->act_cur; out[1] = s->act_last; out[2] = s->err_cur; out[3] = s->err_last; out[4] = s->rtt_cur; out[5] = s->rtt_last;
	return 0;
}

/* CONN_BITMAP::get_conn_breakup, common/gy_socket_stat.h:412-433: per bucket the number of port-hash slots that saw it */
int gyo_export_conn_bitmap(gyo_engine *e, uint64_t id, int last_window, uint32_t *masks15, uint8_t *nconn15)
{
	int slot = idmap_find(&e->smap, id, 0, 0);
	if (slot < 0) return -2;
	const uint32_t *bm = last_window ? e->svcs[slot].bm_last : e->svcs[slot].bm_cur;
	for (int j = 0; j < 15; ++j) { masks15[j] = bm[j]; nconn15[j] = (uint8_t)__builtin_popcount(bm[j]); }
	return 0;
}

const uint64_t *gyo_cms_table(gyo_engine *e, int last_window)
{
	return last_window ? e->cms_last : e->cms_cur;
}

void gyo_counters(gyo_engine *e, uint64_t out[8])
{
	out[0] = e->n_in; out[1] = e->n_drop; out[2] = e->n_resp; out[3] = e->n_tcp; out[4] = e->n_task;
	out[5] = e->smap.n - e->smap.nfreed; out[6] = e->tmap.n; out[7] = e->n_foreign;
}

/* additive merge of a peer shard: histogram sums (update_from_serialized), CMS sums, HLL max — the CPU statement
 * of the NCCL merge step; mirrors STATE_ONE::add_stats common/gy_comm_proto.h:3199-3214 */
void gyo_merge_from(gyo_engine *dst, const gyo_engine *src)
{
	size_t ncell = (size_t)dst->depth << dst->log2w;

	for (size_t i = 0; i < ncell; ++i) { dst->cms_cur[i] += src->cms_cur[i]; dst->cms_last[i] += src->cms_last[i]; }

	for (uint32_t i = 0; i < src->smap.n; ++i) {
		const svc_state *s = &src->svcs[i];
		if (!s->id) continue;		/* evicted */
		svc_state *d = get_svc(dst, s->id, 1);
		if (!d) continue;
		gyo_hist_merge(&d->cur, &s->cur); gyo_hist_merge(&d->last, &s->last); gyo_hist_merge(&d->all, &s->all);
		d->conn_cur += s->conn_cur; d->conn_last += s->conn_last;
		d->conn_all_cnt += s->conn_all_cnt; d->conn_all_kb += s->conn_all_kb;
		for (uint32_t r = 0; r < (1u << dst->hll_p); ++r) if (d->hll[r] < s->hll[r]) d->hll[r] = s->hll[r];
		/* t-digest: rank-ascending merge = concatenate sorted centroid lists, compress */
		gyo_centroid merged[2 * GYO_TD_CAP], outc[GYO_TD_CAP + 1];
		uint32_t nm = merge_sorted(d->td.c, d->td.n, s->td.c, s->td.n, merged);
		uint32_t no = gyo_td_compress(merged, nm, dst->delta, outc, GYO_TD_CAP);
		if (no > GYO_TD_CAP) no = GYO_TD_CAP;
		memcpy(d->td.c, outc, sizeof(gyo_centroid) * no);
		d->td.n = no; d->td.total += s->td.total;
		if (s->td.minv < d->td.minv) d->td.minv = s->td.minv;
		if (s->td.maxv > d->td.maxv) d->td.maxv = s->td.maxv;
	}
	for (uint32_t i = 0; i < src->tmap.n; ++i) {
		const task_state *s = &src->tasks[i];
		task_state *d = get_task(dst, s->id, 1);
		if (!d) continue;
		gyo_hist_merge(&d->cpu_pct, &s->cpu_pct); gyo_hist_merge(&d->cpu_delay, &s->cpu_delay);
		gyo_hist_merge(&d->blkio_delay, &s->blkio_delay);
	}
}

/* ---- CPU baseline: one engine + one pre-sharded event array per thread, no shared state ---- */
typedef struct bench_arg { gyo_engine *e; const gyo_event *ev; uint64_t n, batch; } bench_arg;

static void *bench_thread(void *p)
{
	bench_arg *a = (bench_arg *)p;

	for (uint64_t off = 0; off < a->n; off += a->batch) {
		uint64_t m = a->n - off < a->batch ? a->n - off : a->batch;
		gyo_ingest(a->e, a->ev + off, m);
	}
	return NULL;
}

double gyo_bench_ingest(gyo_engine **engines, const gyo_event **shards, const uint64_t *counts, int nthreads, uint64_t batch)
{
	pthread_t	*th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
	bench_arg	*args = (bench_arg *)malloc(sizeof(bench_arg) * (size_t)nthreads);
	struct timespec	t0, t1;

	clock_gettime(CLOCK_MONOTONIC, &t0);
	for (int t = 0; t < nthreads; ++t) {
		args[t].e = engines[t]; args[t].ev = shards[t]; args[t].n = counts[t]; args[t].batch = batch ? batch : counts[t] + 1;
		pthread_create(&th[t], NULL, bench_thread, &args[t]);
	}
	for (int t = 0; t < nthreads; ++t) pthread_join(th[t], NULL);
	clock_gettime(CLOCK_MONOTONIC, &t1);
	free(th); free(args);
	return (double)(t1.tv_sec - t0.tv_sec) + (double)(t1.tv_nsec - t0.tv_nsec) * 1e-9;
}


/* ---- a15b ------------------------------------------------------------------------------------------------------------------ */
typedef struct aggr_rec			/* comm::AGGR_TASK_STATE_NOTIFY, common/gy_comm_proto.h:2114-2170 */
{
	uint64_t	aggr_task_id;
	char		onecomm[16];
	int32_t		pid_arr[2];
	uint32_t	tcp_kbytes, tcp_conns;
	float		total_cpu_pct;
	uint32_t	rss_mb, cpu_delay_msec, vm_delay_msec, blkio_delay_msec;
	uint16_t	ntasks_total, ntasks_issue;
	uint8_t		curr_state, curr_issue, issue_bit_hist, severe_issue_bit_hist, issue_string_len, padding_len, pad[2];
} aggr_rec;

uint32_t gyo_task_groupby(const gyo_proc_sample *recs, uint64_t n, void *out72, uint32_t cap)
{
	_Static_assert(sizeof(aggr_rec) == 72 && sizeof(gyo_proc_sample) == 64, "wire sizes");
	uint64_t	tcap = 16;
	while (tcap < 2 * n + 2) tcap <<= 1;
	uint64_t	*keys = (uint64_t *)calloc(tcap, 8);
	uint32_t	*vals = (uint32_t *)calloc(tcap, 4);
	aggr_rec	*grp = (aggr_rec *)calloc(n ? n : 1, sizeof(aggr_rec));
	uint32_t	ng = 0;

	for (uint64_t i = 0; i < n; ++i) {
		const gyo_proc_sample *p = &recs[i];
		uint64_t pos = (p->aggr_task_id * 0x9E3779B97F4A7C15ull) >> 20 & (tcap - 1);
		int fresh = 0;
		while (keys[pos] != p->aggr_task_id || !vals[pos]) {
			if (!vals[pos]) { keys[pos] = p->aggr_task_id; vals[pos] = ++ng; fresh = 1; break; }
			pos = (pos + 1) & (tcap - 1);
		}
		aggr_rec *a = &grp[vals[pos] - 1];

		if (p->is_issue) {								/* :763-788 */
			if (a->ntasks_issue < 2) a->pid_arr[a->ntasks_issue] = p->pid;
			a->ntasks_issue++;
			a->curr_issue = p->issue;
			a->issue_bit_hist |= p->issue_bit_hist;
			a->severe_issue_bit_hist |= p->severe_issue_bit_hist;
		}
		if (a->curr_state < p->state) a->curr_state = p->state;				/* :790 */
		a->tcp_kbytes += p->tcp_kbytes; a->tcp_conns += p->tcp_conns;			/* :803-804 */
		a->total_cpu_pct += p->cpu_pct;							/* :839: float accumulate in walk order */
		a->rss_mb += p->rss_mb;								/* :840 */
		a->cpu_delay_msec += p->cpu_delay_msec; a->vm_delay_msec += p->vm_delay_msec; a->blkio_delay_msec += p->blkio_delay_msec;	/* :858-860 */
		a->ntasks_total++;								/* :862 */
		if (a->ntasks_total == 2) a->pid_arr[1] = p->pid;				/* :864 */
		if (fresh) {									/* :868-872 */
			a->aggr_task_id = p->aggr_task_id;
			memcpy(a->onecomm, p->comm, sizeof(a->onecomm));
			a->pid_arr[0] = p->pid;
		}
	}
	memcpy(out72, grp, sizeof(aggr_rec) * (ng < cap ? ng : cap));
	free(keys); free(vals); free(grp);
	return ng;
}
