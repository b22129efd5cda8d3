// gysk_groupby.cu — SURVEY.md §8 row a15b: the per-process -> per-aggregate-process group-by in front of partha_aggr_task_state.
//
// Reference: TASK_HANDLER's 5-s tick walks every process and folds it into aggrnotmap.try_emplace(aggr_task_id)
// (common/gy_task_handler.cc:752-880): sums of tcp kbytes / conns (:803-804), a FLOAT sum of the per-process cpu percentages in walk
// order (:839), rss, the three delay sums in msec (:858-860), process counts, the worst state, the issue of the last process that has
// one, the OR of the issue bit histories and up to two pids (:763-788, :862-872). The result is the AGGR_TASK_STATE_NOTIFY batch
// partha sends (common/gy_comm_proto.h:2114-2170), i.e. the input of row a15.
//
// Here: one thread per sample inserts its aggr_task_id into a scratch open-addressing table and obtains a dense group number; the
// samples' {group : 32 | arrival index : 32} keys go through the engine's stable radix sort on the group bits; one thread per group
// then folds the group's samples IN ARRIVAL ORDER with the reference's statement order — the float accumulator sees the same sequence
// of additions as the reference's walk, so the sum is the same float. Groups leave in order of first appearance (a second sort of
// {first arrival index | group}). Everything but the two copies runs on the engine's stream.
#include <algorithm>
#include <cstring>

#include "gysk_engine.h"
#include "gysk_wire.h"

namespace gysk {

static_assert(sizeof(gysk_proc_sample) == 64, "gysk_proc_sample");
static_assert(sizeof(wire::AGGR_TASK_STATE_NOTIFY) == 72, "AGGR_TASK_STATE_NOTIFY");

static constexpr unsigned long long GB_EMPTY = ~0ull;

// group number of every sample's id (first come, first numbered: the numbers only group, the output order comes from the arrival index)
__global__ void __launch_bounds__(256) gb_insert_kernel(const gysk_proc_sample *__restrict__ recs, uint32_t n, unsigned long long *__restrict__ tkeys,
		uint32_t *__restrict__ tvals, uint32_t tmask, unsigned long long *__restrict__ keys, unsigned long long *__restrict__ counters /* [0] groups, [1] n */)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i == 0) counters[1] = n;
	if (i >= n) return;
	const unsigned long long id = recs[i].aggr_task_id;
	uint32_t pos = (uint32_t)((id * 0x9E3779B97F4A7C15ull) >> 32) & tmask;
	uint32_t g1 = 0;
	for (;;) {
		unsigned long long k = tkeys[pos];
		if (k == GB_EMPTY) {
			k = atomicCAS(&tkeys[pos], GB_EMPTY, id);
			if (k == GB_EMPTY) {					// this thread owns the entry: number the group, publish the number
				g1 = (uint32_t)atomicAdd(&counters[0], 1ull) + 1u;
				__threadfence();
				atomicExch(&tvals[pos], g1);
				break;
			}
		}
		if (k == id) {
			while ((g1 = *(volatile uint32_t *)&tvals[pos]) == 0) __nanosleep(20);	// the owner is a few instructions from publishing
			break;
		}
		pos = (pos + 1) & tmask;
	}
	keys[i] = ((unsigned long long)(g1 - 1u) << 32) | i;
}

// one thread per sorted key; the thread at the head of a group folds it (common/gy_task_handler.cc:763-872, same statement order)
__global__ void __launch_bounds__(128) gb_fold_kernel(const unsigned long long *__restrict__ sorted, const gysk_proc_sample *__restrict__ recs, uint32_t n,
		wire::AGGR_TASK_STATE_NOTIFY *__restrict__ groups, unsigned long long *__restrict__ gkeys)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const unsigned long long k0 = sorted[i];
	const uint32_t g = (uint32_t)(k0 >> 32);
	if (i && (uint32_t)(sorted[i - 1] >> 32) == g) return;

	wire::AGGR_TASK_STATE_NOTIFY a;
	memset(&a, 0, sizeof(a));
	for (uint32_t j = i; j < n; ++j) {
		const unsigned long long k = sorted[j];
		if ((uint32_t)(k >> 32) != g) break;
		const gysk_proc_sample p = recs[(uint32_t)k];
		if (p.is_issue) {
			if (a.ntasks_issue_ < 2) a.pid_arr_[a.ntasks_issue_] = p.pid;
			a.ntasks_issue_++;
			a.curr_issue_ = p.issue;
			a.issue_bit_hist_ |= p.issue_bit_hist;
			a.severe_issue_bit_hist_ |= p.severe_issue_bit_hist;
		}
		if (a.curr_state_ < p.state) a.curr_state_ = p.state;
		a.tcp_kbytes_ += p.tcp_kbytes; a.tcp_conns_ += p.tcp_conns;
		a.total_cpu_pct_ = __fadd_rn(a.total_cpu_pct_, p.cpu_pct);		// float, arrival order, no contraction
		a.rss_mb_ += p.rss_mb;
		a.cpu_delay_msec_ += p.cpu_delay_msec; a.vm_delay_msec_ += p.vm_delay_msec; a.blkio_delay_msec_ += p.blkio_delay_msec;
		a.ntasks_total_++;
		if (a.ntasks_total_ == 2) a.pid_arr_[1] = p.pid;
		if (j == i) {
			a.aggr_task_id_ = p.aggr_task_id;
			memcpy(a.onecomm_, p.comm, sizeof(a.onecomm_));
			a.pid_arr_[0] = p.pid;
		}
	}
	groups[g] = a;
	gkeys[g] = ((unsigned long long)(uint32_t)k0 << 32) | g;			// {arrival index of the group's first sample | group}
}

__global__ void __launch_bounds__(128) gb_emit_kernel(const unsigned long long *__restrict__ sorted_groups, const unsigned long long *__restrict__ ngroups_p,
		const wire::AGGR_TASK_STATE_NOTIFY *__restrict__ groups, wire::AGGR_TASK_STATE_NOTIFY *__restrict__ out, uint32_t cap)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t ng = (uint32_t)*ngroups_p;
	if (i >= ng || i >= cap) return;
	out[i] = groups[(uint32_t)sorted_groups[i]];
}

} // namespace gysk

using namespace gysk;

extern "C" int gysk_task_groupby(gysk_engine *e, const gysk_proc_sample *samples, uint32_t n, void *out_records, uint32_t cap, uint32_t *ngroups)
{
	CHECK_ENGINE(e);
	if ((!samples && n) || (!out_records && cap) || !ngroups) return GYSK_ERR_INVAL;
	*ngroups = 0;
	if (!n) return GYSK_OK;
	if (n > e->cfg.max_batch) return fail(e, GYSK_ERR_INVAL, "gysk_task_groupby: more samples than max_batch (the sort buffers' size)");
	GYSK_ENTER(e, Sync);					// the sort buffers are shared with the batch kernels

	uint32_t tcap = 1024;
	while (tcap < 2ull * n) tcap <<= 1;
	gysk_proc_sample *d_recs = nullptr;
	unsigned long long *d_tkeys = nullptr, *d_cnt = nullptr;
	uint32_t *d_tvals = nullptr;
	wire::AGGR_TASK_STATE_NOTIFY *d_groups = nullptr, *d_out = nullptr;
	auto release = [&]() { cudaFree(d_recs); cudaFree(d_tkeys); cudaFree(d_tvals); cudaFree(d_groups); cudaFree(d_out); cudaFree(d_cnt); };
#define GB(call) do { cudaError_t ce__ = (call); if (ce__ != cudaSuccess) { release(); return fail(e, GYSK_ERR_CUDA, #call, ce__); } } while (0)
	GB(cudaMalloc(&d_recs, (size_t)n * sizeof(gysk_proc_sample)));
	GB(cudaMalloc(&d_tkeys, (size_t)tcap * 8)); GB(cudaMalloc(&d_tvals, (size_t)tcap * 4));
	GB(cudaMalloc(&d_groups, (size_t)n * sizeof(wire::AGGR_TASK_STATE_NOTIFY)));
	GB(cudaMalloc(&d_out, (size_t)std::min(n, std::max(cap, 1u)) * sizeof(wire::AGGR_TASK_STATE_NOTIFY)));
	GB(cudaMalloc(&d_cnt, 16));
	GB(cudaMemcpyAsync(d_recs, samples, (size_t)n * sizeof(gysk_proc_sample), cudaMemcpyHostToDevice, e->stream));
	GB(cudaMemsetAsync(d_tkeys, 0xFF, (size_t)tcap * 8, e->stream));
	GB(cudaMemsetAsync(d_tvals, 0, (size_t)tcap * 4, e->stream));
	GB(cudaMemsetAsync(d_cnt, 0, 16, e->stream));

	gb_insert_kernel<<<(n + 255) / 256, 256, 0, e->stream>>>(d_recs, n, d_tkeys, d_tvals, tcap - 1, e->tmp.keys_a, d_cnt);
	int which = 0, bits = 1;
	while (bits < 32 && (1ull << bits) < n) bits++;			// group numbers are < n
	int nl = launch_radix_sort(e->tmp, d_cnt + 1, n, 32, 32 + bits, &which, e->stream);
	if (nl < 0) { release(); return fail(e, GYSK_ERR_INVAL, "gysk_task_groupby: sort plan"); }
	e->kernel_launches += 1 + nl;
	// the fold reads the sorted keys from one buffer and leaves the groups' {first index | group} keys in keys_a for the second sort
	unsigned long long *sorted = which ? e->tmp.keys_b : e->tmp.keys_a;
	unsigned long long *gkeys = which ? e->tmp.keys_a : nullptr;
	unsigned long long *d_gtmp = nullptr;
	if (!gkeys) { GB(cudaMalloc(&d_gtmp, (size_t)n * 8)); gkeys = d_gtmp; }
	gb_fold_kernel<<<(n + 127) / 128, 128, 0, e->stream>>>(sorted, d_recs, n, d_groups, gkeys);
	if (d_gtmp) GB(cudaMemcpyAsync(e->tmp.keys_a, d_gtmp, (size_t)n * 8, cudaMemcpyDeviceToDevice, e->stream));
	nl = launch_radix_sort(e->tmp, d_cnt, n, 32, 32 + bits, &which, e->stream);
	if (nl < 0) { release(); cudaFree(d_gtmp); return fail(e, GYSK_ERR_INVAL, "gysk_task_groupby: sort plan"); }
	gb_emit_kernel<<<(n + 127) / 128, 128, 0, e->stream>>>(which ? e->tmp.keys_b : e->tmp.keys_a, d_cnt, d_groups, d_out, cap);
	e->kernel_launches += 2 + nl;

	unsigned long long h_cnt[2] = {0, 0};
	GB(cudaMemcpyAsync(h_cnt, d_cnt, 16, cudaMemcpyDeviceToHost, e->stream));
	GB(cudaStreamSynchronize(e->stream));
	const uint32_t ng = (uint32_t)h_cnt[0];
	if (ng && cap) GB(cudaMemcpy(out_records, d_out, (size_t)std::min(ng, cap) * sizeof(wire::AGGR_TASK_STATE_NOTIFY), cudaMemcpyDeviceToHost));
	release();
	cudaFree(d_gtmp);
#undef GB
	*ngroups = ng;
	return post_launch(e, "task group-by");
}
