// gysk_state.cuh — the listener state classifier of the 5-s reducer (SURVEY.md §8 row a10), host + device.
//
// What it restates: TCP_LISTENER::get_curr_state, common/gy_socket_stat.cc:2020-2875 — the decision the reference's
// listener_stats_update (:4233) takes once per listener and 5-s window from
//   * the response histogram's statistics of four levels (5 s, 300 s, 5 days, all-time): p95 / p99 (/ p25), count, sum, mean (:2078-2091),
//   * the p95 / p25 of the listener's qps_hist_ and active_conn_hist_ (:2097-2098; GY_HISTOGRAM<int, SEMI_LOG_HASH_LO> /
//     GY_HISTOGRAM<int, HASH_1_3000>, common/gy_socket_stat.h:548-549, fed at :4111-4126),
//   * the window's query rate, connection counts, server errors, the per-bucket active connection counts of CONN_BITMAP,
//   * the status of the listener's processes, host cpu / memory issue flags and the number of listeners it depends on — inputs that
//     come from outside this path (task handler, host state, dependency graph): the engine passes "no issue" for them, a caller that
//     has them uses gysk_classify_listener() directly,
// and the listener's high_resp_bit_hist_ (one bit per window, shifted in here, :2120 / :2430).
// Outputs are OBJ_STATE_E / LISTENER_ISSUE_SRC (common/gy_json_field_maps.h:242-250, :419-435). The reference also formats a
// sentence per outcome; the sentence is not produced here (the encoder sends an empty issue string).
// Arithmetic follows the reference's types: `x * 0.8f` with a double x is a double product by the float constant, `v * 1.1f` with an
// integer v is a float product, ser_errors is a uint32 (so `ser_errors * 2` wraps like the reference's).
#pragma once

#include <cstdint>

#include "../../include/gysketch.h"

#if defined(__CUDACC__)
#define GYSK_HD __host__ __device__ __forceinline__
#else
#define GYSK_HD inline
#endif

namespace gysk {

// get_bucketid_from_threshold<RESP_TIME_HASH>, common/gy_statistics.h:517-531: the bucket whose upper threshold equals the value;
// anything else (incl. 0, the clamp of an empty level) that is not below min_value maps to the last bucket
GYSK_HD int resp_bucketid_from_threshold(int64_t thr)
{
	const int64_t t[13] = {1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000};
	for (int i = 0; i < 13; ++i) if (thr == t[i]) return i + 1;
	return thr < 0 ? 0 : 14;
}

// GY_HISTOGRAM::get_percentiles (common/gy_statistics.h:707-791) on 15 bucket counts: index of the first bucket whose cumulative count
// reaches size_t(float(total) * float(pct / 100.0)); `nb` (= one past the last bucket) when none does
GYSK_HD int hist_pct_bucket(const uint64_t *counts, int nb, uint64_t total_count, float pct)
{
	const float multiplier = (float)((double)pct / 100.0);
	const uint64_t ncutoff = (uint64_t)((float)total_count * multiplier);
	uint64_t total = 0;
	for (int i = 0; i < nb; ++i) {
		total += counts[i];
		if (total >= ncutoff) return i;
	}
	return nb;
}

// get_bucket_max_threshold<HashClass, T> (common/gy_statistics.h:500-515) for the three classes the classifier reads, then the
// `if (data_value < 0) data_value = 0` of TIME_HISTOGRAM::get_stats (:1352) for the response levels
GYSK_HD int64_t resp_bucket_value(int b, uint64_t total_count)
{
	const int64_t t[13] = {1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000};
	if (b >= 15) b = total_count > 0 ? 15 : 0;
	if (b == 0) return 0;				// min_value - 1 = -1, clamped
	if (b >= 14) return 32767;			// max_value 15001 <= INT16_MAX / 2: INT16_MAX
	return t[b - 1];
}
GYSK_HD int64_t qps_bucket_value(int b, uint64_t total_count)		// SEMI_LOG_HASH_LO :1785, T = int
{
	const int64_t t[13] = {1, 10, 50, 200, 500, 1000, 3000, 6000, 10000, 15000, 25000, 60000, 150000};
	if (b >= 15) b = total_count > 0 ? 15 : 0;
	if (b == 0) return -1;
	if (b >= 14) return 2147483647;			// max_value 150001 > INT16_MAX / 2: INT32_MAX
	return t[b - 1];
}
GYSK_HD int64_t act_bucket_value(int b, uint64_t total_count)		// HASH_1_3000 :2016, T = int
{
	const int64_t t[12] = {1, 5, 10, 25, 50, 75, 100, 150, 300, 500, 1000, 3000};
	if (b >= 14) b = total_count > 0 ? 14 : 0;
	if (b == 0) return -1;
	if (b >= 13) return 32767;			// max_value 3001 <= INT16_MAX / 2: INT16_MAX
	return t[b - 1];
}
GYSK_HD int bucket_semi_log_lo(int data)				// SEMI_LOG_HASH_LO::get_bucket_from_data :1803
{
	const int t[13] = {1, 10, 50, 200, 500, 1000, 3000, 6000, 10000, 15000, 25000, 60000, 150000};
	if (data < 0) return 0;
	if (data >= 150001) return 14;
	int b = 1;
	for (int i = 0; i < 13; ++i) b += (data > t[i]);
	return b;
}

GYSK_HD void classify_listener(const gysk_listener_state_in &in, uint8_t &high_resp_bit_hist, uint8_t &state, uint8_t &issue)
{
	const uint32_t ser = in.ser_errors;
	const uint64_t n5 = in.nqrys_5s;
	const bool task_issue = !!in.task_issue, is_severe = !!in.task_severe, is_delay = !!in.task_delay;
	const bool cpu_issue = !!in.cpu_issue, mem_issue = !!in.mem_issue;
	const int nti = in.ntasks_issue, ntn = in.ntasks_noissue;
	const int b5 = resp_bucketid_from_threshold(in.r5p95), b300 = resp_bucketid_from_threshold(in.r300p95),
			b5day = resp_bucketid_from_threshold(in.r5dp95);						// :2094-2096
	const int tcnt5 = (int)(n5 / 5);
	const int curr_qps = in.last_qps_count > tcnt5 ? in.last_qps_count : tcnt5;					// :2092
	const uint32_t ser2 = ser * 2u, ser5 = ser * 5u;								// uint32 products, as `ser_errors * 2`
	const bool much_worse = (b5 > b5day + 2) && (b5 > b300);							// the SEVERE rule (:2467, :2497, :2774)

#define GYSK_RET(st_, is_) do { state = (uint8_t)(st_); issue = (uint8_t)(is_); return; } while (0)
	high_resp_bit_hist = (uint8_t)(high_resp_bit_hist << 1);							// :2120

	if (curr_qps == 0) {												// :2122
		if (!task_issue || !is_severe || !ser) GYSK_RET(GYSK_STATE_IDLE, GYSK_ISSUE_NONE);
	}

	if (b5 == 1 || in.r5p95 < in.r5dp95) {										// :2139: 5-s p95 <= 1 msec or below the 5-day p95
		if ((int64_t)curr_qps <= in.qps_p25 && in.qps_p25 < in.qps_p95) {					// :2143 QPS too low
			if (!task_issue && !ser) GYSK_RET(GYSK_STATE_IDLE, GYSK_ISSUE_NONE);				// :2145
			else if (!task_issue && ser) {									// :2153
				if ((uint64_t)ser2 > n5) GYSK_RET(GYSK_STATE_SEVERE, GYSK_ISSUE_SERVER_ERRORS);
				else if ((uint64_t)ser5 > n5) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_SERVER_ERRORS);
				else if ((double)ser < (double)n5 * 0.1) GYSK_RET(GYSK_STATE_OK, GYSK_ISSUE_SERVER_ERRORS);
			}
			else {												// :2180 a process issue
				if ((uint64_t)ser2 > n5) GYSK_RET(GYSK_STATE_SEVERE, GYSK_ISSUE_SERVER_ERRORS);
				else if ((uint64_t)ser5 > n5) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_SERVER_ERRORS);
				else if (ser) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_LISTENER_TASKS);
				if (is_severe && nti > 0 && ntn == 0) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_LISTENER_TASKS);	// :2206
				if ((int64_t)in.nconn > in.act_p25) GYSK_RET(GYSK_STATE_OK, GYSK_ISSUE_LISTENER_TASKS);	// :2216
			}
		}
		if (ser) {												// :2228 ff.
			if ((uint64_t)ser2 > n5) GYSK_RET(GYSK_STATE_SEVERE, GYSK_ISSUE_SERVER_ERRORS);
			else if ((uint64_t)ser5 > n5) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_SERVER_ERRORS);
		}
		if (task_issue && is_severe && nti > 0 && ntn == 0) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_LISTENER_TASKS);	// :2260
		if (!ser) {												// :2275
			if ((int64_t)curr_qps <= in.qps_p95 || b5 + 2 <= b5day) GYSK_RET(GYSK_STATE_GOOD, GYSK_ISSUE_NONE);
			GYSK_RET(GYSK_STATE_OK, GYSK_ISSUE_QPS_HIGH);							// :2287 (curr_qps > p95 is what is left)
		}
		GYSK_RET(GYSK_STATE_OK, GYSK_ISSUE_SERVER_ERRORS);							// :2295
	}

	if (in.r5p95 == in.r5dp95) {											// :2307
		if (ser) {
			if ((uint64_t)ser2 > n5) GYSK_RET(GYSK_STATE_SEVERE, GYSK_ISSUE_SERVER_ERRORS);
			else if ((uint64_t)ser5 > n5) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_SERVER_ERRORS);
		}
		if (in.mean5 <= in.mean5d * 0.8f) {									// :2340
			if ((int64_t)curr_qps <= in.qps_p25) {								// :2342
				if (ser) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_SERVER_ERRORS);
				else if (!task_issue) GYSK_RET(GYSK_STATE_IDLE, GYSK_ISSUE_NONE);
				else if (nti > 0 && ntn == 0) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_LISTENER_TASKS);
				else if (nti > 0 && in.tasks_delay_msec >= 1000) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_LISTENER_TASKS);
			}
			if (!task_issue && !ser) GYSK_RET(GYSK_STATE_GOOD, GYSK_ISSUE_NONE);				// :2386
			else if (ser && task_issue) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_LISTENER_TASKS);		// :2394
			// :2402-2415: server errors without a process issue set {SERVER_ERRORS, OK} but do NOT return; the statement that
			// follows overwrites both — reproduced as the reference executes it
			GYSK_RET(GYSK_STATE_OK, GYSK_ISSUE_LISTENER_TASKS);
		}
		if (in.mean5 <= in.mean5d * 1.2f) GYSK_RET(GYSK_STATE_OK, GYSK_ISSUE_NONE);				// :2419
	}

	high_resp_bit_hist |= 1;											// :2430 the response IS high this window

	if (ser) {													// :2432
		if ((uint64_t)ser2 > n5) GYSK_RET(GYSK_STATE_SEVERE, GYSK_ISSUE_SERVER_ERRORS);
		else if ((uint64_t)ser5 > n5) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_SERVER_ERRORS);
	}
	// :2464 QPS well above its p95
	if ((int64_t)curr_qps > in.qps_p95 && (int64_t)curr_qps - in.qps_p95 > 5 && (float)curr_qps > (float)in.qps_p95 * 1.1f)
		GYSK_RET(much_worse ? GYSK_STATE_SEVERE : GYSK_STATE_BAD, GYSK_ISSUE_QPS_HIGH);
	// :2494 processes flagged, or their delays make up a quarter of the response time
	if (task_issue || (is_delay && nti + ntn > 2 && in.tasks_delay_msec * 4 > in.total_resp_msec))
		GYSK_RET(much_worse ? GYSK_STATE_SEVERE : GYSK_STATE_BAD, GYSK_ISSUE_LISTENER_TASKS);
	// :2525 active connections above their p95
	if ((int64_t)in.curr_active_conn > in.act_p95 && (int64_t)in.curr_active_conn - in.act_p95 > 1)
		GYSK_RET((much_worse && in.curr_active_conn > 10) ? GYSK_STATE_SEVERE : GYSK_STATE_BAD, GYSK_ISSUE_ACTIVE_CONN_HIGH);
	// :2552 same p95 bucket as the 5-day level but a worse p99: outliers
	if (in.r5p95 == in.r5dp95 && in.r5p99 > in.r5dp99) GYSK_RET(GYSK_STATE_OK, ser ? GYSK_ISSUE_SERVER_ERRORS : GYSK_ISSUE_NONE);
	// :2576 low QPS and few connections
	if ((int64_t)curr_qps <= in.qps_p25 && (int64_t)in.nconn <= in.act_p25) {
		if (is_delay && cpu_issue && mem_issue) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_LISTENER_TASKS);
		else if (is_delay && (cpu_issue || mem_issue) && in.tasks_delay_msec * 4 > in.total_resp_msec) GYSK_RET(GYSK_STATE_BAD, GYSK_ISSUE_LISTENER_TASKS);
		GYSK_RET(GYSK_STATE_OK, ser ? GYSK_ISSUE_SERVER_ERRORS : GYSK_ISSUE_NONE);
	}
	// :2638 the 5-day average QPS is below half of the current one and the response is no worse than the all-time one
	{
		const int avg_5day_qps = (int)((int64_t)in.tcount_5d / (in.secs_5d > 0 ? in.secs_5d : 1));
		if (avg_5day_qps < (curr_qps >> 1) && in.r5p95 <= in.rallp95 && in.mean5 <= in.meanall * 1.1f)
			GYSK_RET(GYSK_STATE_OK, ser ? GYSK_ISSUE_SERVER_ERRORS : GYSK_ISSUE_NONE);
	}
	// :2661 few active connections, low QPS, at most one bucket worse
	if ((int64_t)curr_qps <= in.qps_p25 && (int64_t)in.curr_active_conn <= in.act_p25 && b5 <= b5day + 1)
		GYSK_RET(GYSK_STATE_OK, ser ? GYSK_ISSUE_SERVER_ERRORS : GYSK_ISSUE_NONE);
	// :2684 only the 5-s level is up, the 300-s level is where the 5-day level is: transient
	if (b5 <= b5day + 1 && b300 == b5day && in.mean5 > in.mean300 && in.mean300 < in.mean5d * 1.1f)
		GYSK_RET(GYSK_STATE_OK, ser ? GYSK_ISSUE_SERVER_ERRORS : GYSK_ISSUE_NONE);
	// :2710 the slow responses sit on at most 3 connections per bucket (CONN_BITMAP counts): a local effect
	if (in.curr_active_conn >= 15 && b5 == b5day + 1) {
		int b = b5;
		for (; b < 15; ++b) if (in.nactive_conn_arr[b] > 3) break;
		if (b > b5) GYSK_RET(GYSK_STATE_OK, ser ? GYSK_ISSUE_SERVER_ERRORS : GYSK_ISSUE_NONE);
	}
	// :2748 high in fewer than 5 of the last 8 windows
	{
		int nhigh = 0;
		for (uint32_t v = high_resp_bit_hist; v; v &= v - 1) nhigh++;
		if (nhigh < 5) GYSK_RET(GYSK_STATE_OK, ser ? GYSK_ISSUE_SERVER_ERRORS : GYSK_ISSUE_NONE);
	}
	// :2771 nothing explains it away
	const uint8_t st = much_worse ? GYSK_STATE_SEVERE : GYSK_STATE_BAD;
	if (in.tasks_delay_msec * 4 > in.total_resp_msec && st == GYSK_STATE_BAD) GYSK_RET(st, GYSK_ISSUE_LISTENER_TASKS);	// :2791
	if (in.nserdepends > 0) GYSK_RET(st, GYSK_ISSUE_DEPENDENT_SERVER_LISTENER);					// :2825
	if (in.tasks_delay_msec * 10 > in.total_resp_msec) GYSK_RET(st, GYSK_ISSUE_LISTENER_TASKS);			// :2829
	GYSK_RET(st, ser ? GYSK_ISSUE_SERVER_ERRORS : GYSK_ISSUE_SRC_UNKNOWN);					// :2855-2860
#undef GYSK_RET
}

// issue_bit_hist_ and the "just started" override of listener_stats_update, common/gy_socket_stat.cc:4242-4272: a listener younger
// than 100 s without server errors reports {OK, NONE} and clears its issue history
GYSK_HD void apply_issue_history(uint32_t age_secs, uint32_t ser_errors, uint8_t &state, uint8_t &issue, uint8_t &issue_bit_hist)
{
	if (age_secs > 100u || ser_errors) {
		issue_bit_hist = (uint8_t)(issue_bit_hist << 1);
		if (state >= GYSK_STATE_BAD) issue_bit_hist |= 1;
	}
	else { issue_bit_hist = 0; issue = GYSK_ISSUE_NONE; state = GYSK_STATE_OK; }
}

// TCP_SOCK_HANDLER::host_status_update's state rule, common/gy_socket_stat.cc:4455-4528, in its statement order
inline uint8_t classify_host(const gysk_host_state_in &in)
{
	const bool cpu = !!in.cpu_issue, mem = !!in.mem_issue, scpu = !!in.severe_cpu_issue, smem = !!in.severe_mem_issue;
	const uint32_t nti = in.ntasks_issue, nts = in.ntasks_severe, nli = in.nlisten_issue, nls = in.nlisten_severe;

	if ((nts || nls) && (scpu || smem)) return GYSK_STATE_SEVERE;					// :4462
	if (!cpu && !mem && !nti && !nli) return in.cpu_idle ? GYSK_STATE_IDLE : GYSK_STATE_GOOD;		// :4467
	if ((nti || nli) && (cpu || mem)) return (nti > 5 || nli > 5) ? GYSK_STATE_SEVERE : GYSK_STATE_BAD;	// :4479
	if (cpu || mem) return (scpu || smem) ? GYSK_STATE_BAD : GYSK_STATE_OK;				// :4488
	if (nli) {												// :4498
		if (nls || nti) return nli > 5 ? GYSK_STATE_SEVERE : GYSK_STATE_BAD;
		return nli > 2 ? GYSK_STATE_BAD : GYSK_STATE_OK;
	}
	if (nti && (nts || nti > 5)) return GYSK_STATE_BAD;						// :4518
	return GYSK_STATE_OK;
}

} // namespace gysk
