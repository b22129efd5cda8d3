/*
 * gysk_oracle.h — TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement (plain C) of the algorithms on the hot path of include/gysketch.h. Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this library;
 * the product (libgysketch.so) never links, loads or calls it.
 *
 * Pinning (see oracle/README.md):
 *   - jhash, bucket hashes, GY_HISTOGRAM add/merge/percentiles: pinned against the reference's own asserted
 *     fixture test/test_histogram.cc:29-147 and against outputs of the reference compiled here (oracle/_ref).
 *   - count-min, HyperLogLog, t-digest: the reference has no implementation and no test vector for them
 *     (SURVEY.md §0.1, §8c)  =>  PARITY UNPINNED for these three; they are definitions, stated here, that the
 *     CUDA path must reproduce bit-exactly (CMS cells, HLL registers) or within epsilon (t-digest quantiles).
 */
#ifndef GYSK_ORACLE_H
#define GYSK_ORACLE_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* histogram classes: ids 0..7 equal GYSK_CLS_* of include/gysketch.h; 8,9 are the two FIXED_DIFF_HASH
 * instantiations asserted in test/test_histogram.cc */
enum {
	GYO_CLS_RESP_TIME = 0, GYO_CLS_SEMI_LOG, GYO_CLS_SEMI_LOG_LO, GYO_CLS_DURATION, GYO_CLS_HASH_10_5000,
	GYO_CLS_HASH_5_250, GYO_CLS_HASH_1_3000, GYO_CLS_PERCENT, GYO_CLS_FD_I8_9_26_5, GYO_CLS_FD_INT_M15_M3_4, GYO_CLS_MAX
};

/* value type T of GY_HISTOGRAM<T, Hash> */
enum { GYO_T_INT64 = 0, GYO_T_INT = 1, GYO_T_INT8 = 2 };

#define GYO_MAX_BUCKETS		16
#define GYO_NLEVELS		2	/* rolling levels beyond the 5-s window: 300 s and 432000 s */
#define GYO_NSLOTS		10	/* slots per level, common/gy_statistics.h:1105 */

typedef struct gyo_serial { uint64_t count; int64_t sum; } gyo_serial;	/* == HIST_SERIAL */

typedef struct gyo_hist
{
	gyo_serial	stats[GYO_MAX_BUCKETS];
	uint64_t	total_count;
	int64_t		max_val;
	int32_t		cls, tkind;
} gyo_hist;

typedef struct gyo_event		/* == gysk_event */
{
	uint64_t	svc_id, flow_key;
	uint32_t	value, host_idx, tsec;
	uint16_t	type, flags;
} gyo_event;

typedef struct gyo_centroid { double mean; uint64_t weight; } gyo_centroid;

#define GYO_TD_CAP		256

typedef struct gyo_tdigest
{
	gyo_centroid	c[GYO_TD_CAP];
	uint32_t	n;
	uint64_t	total;
	double		minv, maxv;
} gyo_tdigest;

/* ---- jhash (Bob Jenkins lookup2 as used by the reference, common/jhash.h:22-140) ---- */
uint32_t gyo_jhash_3words(uint32_t a, uint32_t b, uint32_t c, uint32_t initval);
uint32_t gyo_jhash_2words(uint32_t a, uint32_t b, uint32_t initval);
uint32_t gyo_jhash2(const uint32_t *k, uint32_t length, uint32_t initval);
uint32_t gyo_jhash(const void *key, uint32_t length, uint32_t initval);
uint32_t gyo_uint64_hash(uint64_t key);			/* common/gy_common_inc.h:1120 */

/* ---- bucket hashes + GY_HISTOGRAM (common/gy_statistics.h:455-894, 1565-2063) ---- */
int	gyo_nbuckets(int cls);
int	gyo_bucket(int cls, int64_t value);		/* HashClass::operator() incl. the (int) truncation of :1748 etc. */
int64_t	gyo_bucket_max_threshold(int cls, int tkind, size_t id);	/* :500-515 */
void	gyo_hist_init(gyo_hist *h, int cls, int tkind);
int	gyo_hist_add(gyo_hist *h, int64_t value);	/* add_data :596-623, returns bucket */
void	gyo_hist_merge(gyo_hist *dst, const gyo_hist *src);	/* update_from_serialized :625-650 */
void	gyo_hist_percentiles(const gyo_hist *h, const float *pcts, size_t npct, int64_t *out, float *avg);	/* :707-791 */
/* convenience: run a fresh histogram over vals */
int	gyo_hist_run(int cls, int tkind, const int64_t *vals, size_t n, const float *pcts, size_t npct,
		gyo_serial *out_stats, uint64_t *out_total, int64_t *out_max, int64_t *out_pct, int64_t *out_bucket_ids, float *out_avg);

/* ---- sketch definitions (ours; parity unpinned) ---- */
uint32_t gyo_cms_index(uint64_t flow_key, uint32_t row, uint32_t log2_width);
uint64_t gyo_cms_increment(uint32_t bytes);		/* 1 | (bytes >> 10) << 32 */
void	gyo_flow_hashes(uint64_t flow_key, uint32_t *h1, uint32_t *h2);
uint64_t gyo_hll_hash(uint64_t flow_key);	/* fmix64(h2:h1) */
uint32_t gyo_td_code(uint32_t usec);	/* log-linear bin of a response time, 32 bins per octave */
void	gyo_hll_idx_rank(uint64_t flow_key, uint32_t p, uint32_t *idx, uint8_t *rank);
void	gyo_hll_registers(const uint64_t *keys, uint64_t n, uint32_t p, uint8_t *regs);	/* regs[idx] = max(regs[idx], rank) per key */
double	gyo_hll_estimate(const uint8_t *regs, uint32_t p);

void	gyo_td_init(gyo_tdigest *t);
/* Dunning's merging t-digest, K_1 scale k(q) = delta/(2 pi) asin(2q-1): greedy single pass over sorted centroids */
uint32_t gyo_td_compress(const gyo_centroid *sorted_in, uint32_t n, double delta, gyo_centroid *out, uint32_t cap);
/* batched update = what the CUDA path does per device batch: cluster the batch's sorted samples, then merge
 * the new clusters with the old centroids */
void	gyo_td_add_batch(gyo_tdigest *t, const uint32_t *vals, uint32_t n, double delta);
/* classic buffered MergingDigest (buffer of 5*delta points) — the "reference CPU path" for epsilon parity */
void	gyo_td_add_classic(gyo_tdigest *t, const uint32_t *vals, uint32_t n, double delta);
double	gyo_td_quantile(const gyo_centroid *c, uint32_t n, double minv, double maxv, double q);
double	gyo_td_quantile_f(const float *means, const float *weights, uint32_t n, float minv, float maxv, double q);

/* ---- engine-level oracle over the 32-byte event stream ---- */
typedef struct gyo_engine gyo_engine;

gyo_engine *gyo_create(uint32_t max_svcs, uint32_t max_tasks, uint32_t cms_depth, uint32_t cms_log2_width, uint32_t hll_p,
		uint32_t td_compression, uint32_t flags, uint32_t rank, uint32_t world);
void	gyo_destroy(gyo_engine *e);
int	gyo_register_ids(gyo_engine *e, const uint64_t *ids, uint32_t n, int is_task);
int	gyo_ingest(gyo_engine *e, const gyo_event *ev, uint64_t n);	/* one device batch */
void	gyo_flush(gyo_engine *e, uint32_t tsec);
/* idle-service eviction at flush (rule of common/gy_socket_stat.cc:3968-3982); 0 = never */
int	gyo_task_last(gyo_engine *e, uint64_t id, uint64_t out[6]);
void	gyo_set_idle_evict(gyo_engine *e, uint32_t secs);
uint32_t gyo_evicted(gyo_engine *e, uint64_t *out, uint32_t cap, uint64_t *total);	/* ids evicted by the last flush */
uint32_t gyo_nsvcs(gyo_engine *e);
int	gyo_export_hist(gyo_engine *e, uint64_t id, int which, gyo_serial *out15, uint64_t *total, int64_t *maxv);
int	gyo_export_hll(gyo_engine *e, uint64_t id, uint8_t *regs);
int	gyo_export_tdigest(gyo_engine *e, uint64_t id, gyo_tdigest *out);
int	gyo_export_conn(gyo_engine *e, uint64_t id, uint64_t *cur, uint64_t *last, uint64_t *all_cnt, uint64_t *all_kb);
int	gyo_export_aux(gyo_engine *e, uint64_t id, uint64_t out[6]);	/* ACTIVE_CONN_STATS roll-up, API_TRAN error counters, max rtt */
int	gyo_export_conn_bitmap(gyo_engine *e, uint64_t id, int last_window, uint32_t *masks15, uint8_t *nconn15);
const uint64_t *gyo_cms_table(gyo_engine *e, int last_window);
void	gyo_counters(gyo_engine *e, uint64_t out[8]);	/* in, dropped, resp, tcp, task, nsvcs, ntasks, foreign */
void	gyo_merge_from(gyo_engine *dst, const gyo_engine *src);	/* additive roll-up of a peer shard (hist sum, cms sum, hll max) */

/* CPU baseline: nthreads engines each ingest their own pre-sharded event array; returns wall seconds */
double	gyo_bench_ingest(gyo_engine **engines, const gyo_event **shards, const uint64_t *counts, int nthreads, uint64_t batch);

/* ---- listener state: TCP_LISTENER::get_curr_state, common/gy_socket_stat.cc:2020-2875 (OBJ_STATE_E / LISTENER_ISSUE_SRC,
 * common/gy_json_field_maps.h:242-250, :419-435) ---- */
enum { GYO_STATE_IDLE = 0, GYO_STATE_GOOD, GYO_STATE_OK, GYO_STATE_BAD, GYO_STATE_SEVERE, GYO_STATE_DOWN };
enum { GYO_ISSUE_NONE = 0, GYO_ISSUE_TASKS, GYO_ISSUE_QPS_HIGH, GYO_ISSUE_ACTIVE_CONN_HIGH, GYO_ISSUE_SERVER_ERRORS, GYO_ISSUE_OS_CPU,
       GYO_ISSUE_OS_MEMORY, GYO_ISSUE_DEPENDENT, GYO_ISSUE_UNKNOWN };
typedef struct gyo_state_in		/* same layout as gysk_listener_state_in (include/gysketch.h) */
{
	int64_t		r5p95, r5p99, r300p95, r300p99, r5dp95, r5dp99, r5dp25, rallp95, rallp99;
	uint64_t	nqrys_5s, total_resp_msec, tcount_5d;
	double		mean5, mean300, mean5d, meanall;
	int64_t		qps_p95, qps_p25, act_p95, act_p25, secs_5d;
	int32_t		last_qps_count, nconn, curr_active_conn;
	uint32_t	ser_errors;
	uint8_t		nactive_conn_arr[16];
	uint8_t		task_issue, task_severe, task_delay, cpu_issue, mem_issue, pad0[3];
	int32_t		ntasks_issue, ntasks_noissue;
	uint64_t	tasks_delay_msec;
	uint32_t	nserdepends, pad1;
} gyo_state_in;
void	gyo_listener_state(const gyo_state_in *in, uint8_t *high_resp_bit_hist, uint8_t *state, uint8_t *issue);
/* what the flush derived for a service: out = {state, issue, issue_bit_hist, high_resp_bit_hist, nconn_active} */
int	gyo_export_state(gyo_engine *e, uint64_t id, uint32_t out[5]);

/* ---- a15b: the per-process -> per-aggregate-process group-by of TASK_HANDLER's 5-s tick, common/gy_task_handler.cc:752-880:
 * aggrnotmap.try_emplace(aggr_task_id) per process, in the order the processes are walked ---- */
typedef struct gyo_proc_sample		/* same layout as gysk_proc_sample (include/gysketch.h), 64 bytes */
{
	uint64_t	aggr_task_id;
	int32_t		pid;
	float		cpu_pct;		/* avg_cpu_pct / npct, :826-839 */
	uint32_t	rss_mb;
	uint32_t	cpu_delay_msec, vm_delay_msec, blkio_delay_msec;	/* nsec / GY_NSEC_PER_MSEC per process, :858-860 */
	uint32_t	tcp_kbytes, tcp_conns;	/* non-zero only in the 15-s network ticks, :791-813 */
	uint8_t		state, issue, issue_bit_hist, severe_issue_bit_hist, is_issue, pad[3];
	char		comm[16];
} gyo_proc_sample;
/* out: AGGR_TASK_STATE_NOTIFY records (72 bytes each, common/gy_comm_proto.h:2114-2170), groups in order of first appearance;
 * returns the number of groups (records beyond cap are not written) */
uint32_t gyo_task_groupby(const gyo_proc_sample *recs, uint64_t n, void *out72, uint32_t cap);

#ifdef __cplusplus
}
#endif
#endif
