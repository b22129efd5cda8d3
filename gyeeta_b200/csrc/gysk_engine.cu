// gysk_engine.cu — host runtime of libgysketch.so and the C ABI declared in include/gysketch.h.
//
// One engine = one GPU. Ingest calls are serialised by a mutex, copy their input into page-locked staging (the
// reference's handlers never retain caller buffers: DB_WRITE_ARR frees them when the L2 loop iteration ends,
// server/gy_mconnhdlr.h:424-431) and hand full batches to the device: H2D on a copy stream, kernels on the compute
// stream, two device event buffers so the copy of batch k+1 overlaps the kernels of batch k.
#include "gysk_engine.h"
#include "gysk_state.cuh"
#include "gysk_summary.cuh"
#include "gysk_wire.h"

using namespace gysk;

namespace {

thread_local std::string g_create_error;
std::atomic<uint64_t> g_engine_uid {1};

} // namespace

namespace gysk {

int fail(gysk_engine *e, int code, const char *what, cudaError_t ce)
{
	char buf[512];

	if (ce != cudaSuccess) snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(ce));
	else snprintf(buf, sizeof(buf), "%s", what);
	if (e) {
		e->err = buf;
		if (code == GYSK_ERR_CUDA) e->sticky = true;
	}
	else g_create_error = buf;
	return code;
}

int post_launch(gysk_engine *e, const char *what)
{
	cudaError_t ce = cudaGetLastError();
	if (ce != cudaSuccess) return fail(e, GYSK_ERR_CUDA, what, ce);
	return 0;
}

} // namespace gysk

namespace {

uint32_t pow2_at_least(uint64_t v) { uint32_t p = 16; while (p < v) p <<= 1; return p; }

// the values the slot field of a batch's sort keys takes: the service slots, and with trace rows the null slot and one pseudo-slot per row
uint32_t key_slots(const gysk_engine *e) { return e->cfg.max_svcs + (e->st.trace.rows ? 1u + e->st.trace.rows : 0u); }

// one device batch: ingest kernel, the TCP and TASK drain passes over the records it queued, then the sort + t-digest chain over
// the keys it emitted. `consumed` (optional) is recorded once the ingest kernel has read the events: the event buffer may be refilled
// from there on, so that the next H2D copy overlaps the drain and merge kernels.
int process_device_batch(gysk_engine *e, const gysk_event *d_ev, uint64_t n, cudaEvent_t consumed)
{
	if (!n) return 0;
	if (n >= (1ull << BIN_CNT_BITS)) return fail(e, GYSK_ERR_INVAL, "device batch holds 2^27 or more events");
	cudaEvent_t *pe = nullptr;
	if (e->profiling) {
		if (e->prof_used + 3 > e->prof_events.size()) {
			for (int i = 0; i < 3; ++i) {
				cudaEvent_t ev;
				CU(e, cudaEventCreate(&ev));
				e->prof_events.push_back(ev);
			}
		}
		pe = &e->prof_events[e->prof_used];
		e->prof_used += 3;
		CU(e, cudaEventRecord(pe[0], e->stream));
	}
	RecRegions rr;
	const int li = launch_ingest(e->st, e->tmp, d_ev, n, key_slots(e), rr, e->stream);
	if (li < 0) return fail(e, GYSK_ERR_INVAL, "ingest launch: no sort plan, or record regions beyond the record queue");
	e->kernel_launches += li;
	if (consumed) CU(e, cudaEventRecord(consumed, e->stream));
	e->kernel_launches += launch_drains(e->st, e->tmp, rr, n, e->stream);
	if (pe) CU(e, cudaEventRecord(pe[1], e->stream));
	// No number travels back to the host inside a batch: the list of touched services and its length stay in device memory.
	e->kernel_launches += launch_batch_merge(e->st, e->tmp, n, key_slots(e), e->stream);
	if (pe) CU(e, cudaEventRecord(pe[2], e->stream));
	e->batches++;
	return post_launch(e, "ingest batch");
}

// pick up the eviction list of the last flush, once its copy has landed
int collect_evicted(gysk_engine *e)
{
	if (!e->evict_pending) return 0;
	CU(e, cudaEventSynchronize(e->ev_evict));
	const uint64_t cnt = std::min<uint64_t>(e->h_evict[0], e->cfg.max_svcs);
	e->h_evict_fail = e->h_evict[e->cfg.max_svcs + 1];
	e->evicted_ids.assign(e->h_evict + 1, e->h_evict + 1 + cnt);
	e->tombstones += cnt; e->evicted_total += cnt;
	if (e->h_tevict) {
		const uint64_t tcnt = std::min<uint64_t>(e->h_tevict[0], e->cfg.max_tasks);
		e->evicted_task_ids.assign(e->h_tevict + 1, e->h_tevict + 1 + tcnt);
		std::sort(e->evicted_task_ids.begin(), e->evicted_task_ids.end());		// the list's order depends on the device's atomics
		e->task_tombstones += tcnt; e->task_evicted_total += tcnt;
	}
	e->evict_pending = false;
	return 0;
}

} // namespace

// ---- staging: per-thread page-locked buffers -> device event buffer -> kernels -------------------------------------
//
// Up to 16 handle_l2_misc threads call gysk_ingest concurrently (server/gy_mconnhdlr.h:53-63, routing :16252). Each calling
// thread owns a ThreadStage: two page-locked chunks it fills WITHOUT the engine mutex — validation, record walk and compaction of
// the wire records run in parallel across threads. Only a full chunk takes the engine mutex, for as long as it takes to enqueue
// one asynchronous H2D copy into the current device event buffer (and, when that buffer is full, the batch's kernel launches).
// Readers (sync, flush, queries) first drain every thread's partial chunk, so "all events handed in before the call are applied".
// Lock order: ThreadStage::m, then gysk_engine::mtx; drain_all takes tstage_mtx, then each ThreadStage::m in turn.

// device event buffer k holds stage_fill events whose copies are enqueued on copy_stream: run the batch
int gysk::submit_stage(gysk_engine *e)
{
	const int k = e->stage_cur;
	const uint32_t n = e->stage_fill;

	if (!n) return 0;
	CU(e, cudaEventRecord(e->ev_copied[k], e->copy_stream));
	CU(e, cudaStreamWaitEvent(e->stream, e->ev_copied[k], 0));
	int rc = process_device_batch(e, e->d_events[k], n, e->ev_done[k]);
	if (rc) return rc;
	e->stage_cur = (k + 1) % NBUF;
	e->stage_fill = 0;
	return 0;
}

namespace {

// Place n events behind what the current device buffer already holds, buffer after buffer (engine mutex held). For each part,
// write(dst, off, m) enqueues on copy_stream whatever writes events [off, off + m) of the n at dst; a full buffer runs its batch.
template <typename Write>
int place_events(gysk_engine *e, uint64_t n, Write write)
{
	for (uint64_t off = 0; off < n; ) {
		const int k = e->stage_cur;
		const uint32_t m = (uint32_t)std::min<uint64_t>(e->cfg.stage_batch - e->stage_fill, n - off);

		if (e->stage_fill == 0) CU(e, cudaStreamWaitEvent(e->copy_stream, e->ev_done[k], 0));	// the kernels that last read buffer k have run
		int rc = write(e->d_events[k] + e->stage_fill, off, m);
		if (rc) return rc;
		e->stage_fill += m; off += m;
		if (e->stage_fill == e->cfg.stage_batch && (rc = submit_stage(e))) return rc;
	}
	return 0;
}

// the copy of n events from page-locked host memory (engine mutex held)
int append_chunk(gysk_engine *e, const gysk_event *src, uint64_t n)
{
	return place_events(e, n, [&](gysk_event *dst, uint64_t off, uint32_t m) {
		CU(e, cudaMemcpyAsync(dst, src + off, (size_t)m * sizeof(gysk_event), cudaMemcpyHostToDevice, e->copy_stream));
		return 0;
	});
}

} // namespace

int gysk::sync_locked(gysk_engine *e)
{
	int rc = submit_stage(e);
	if (rc) return rc;
	CU(e, cudaStreamSynchronize(e->copy_stream));
	CU(e, cudaStreamSynchronize(e->stream));
	return 0;
}

namespace {

// engines alive (uid): a thread that exits hands its stages back to the engines that still exist
std::mutex g_live_mtx;
std::vector<uint64_t> g_live;

struct TlsStages
{
	std::vector<std::pair<uint64_t, ThreadStage *>> v;
	~TlsStages()
	{
		std::lock_guard<std::mutex> lk(g_live_mtx);
		for (auto &kv : v) if (std::find(g_live.begin(), g_live.end(), kv.first) != g_live.end()) kv.second->orphan.store(true, std::memory_order_release);
	}
};
thread_local TlsStages tls_stages_holder;
#define tls_stages tls_stages_holder.v

// the calling thread's stage of this engine: its own, else one whose thread is gone (madhava's handler threads live as long as the
// process, but a pool that recycles threads must not pay two cudaHostAlloc calls per new thread), else a new one
ThreadStage *get_stage(gysk_engine *e)
{
	for (auto &kv : tls_stages) if (kv.first == e->uid) return kv.second;
	std::lock_guard<std::mutex> lk(e->tstage_mtx);
	for (auto &old : e->tstages) {
		bool want = true;
		if (old->orphan.compare_exchange_strong(want, false, std::memory_order_acq_rel)) {
			if (tls_stages.size() > 64) tls_stages.erase(tls_stages.begin());
			tls_stages.emplace_back(e->uid, old.get());
			return old.get();
		}
	}
	auto ts = std::make_unique<ThreadStage>();
	ts->cap = std::min<uint32_t>(e->cfg.stage_batch, THREAD_STAGE_EVENTS);
	if (cudaSetDevice(e->dev) != cudaSuccess) return nullptr;
	for (int i = 0; i < 2; ++i) {
		if (cudaHostAlloc((void **)&ts->buf[i], (size_t)ts->cap * sizeof(gysk_event), cudaHostAllocDefault) != cudaSuccess) return nullptr;
		if (cudaEventCreateWithFlags(&ts->copied[i], cudaEventDisableTiming) != cudaSuccess) return nullptr;
	}
	ThreadStage *raw = ts.get();
	e->tstages.push_back(std::move(ts));
	if (tls_stages.size() > 64) tls_stages.erase(tls_stages.begin());		// engines long gone
	tls_stages.emplace_back(e->uid, raw);
	return raw;
}

// hand the filled part of the thread's current chunk to the device (ThreadStage::m held by the caller)
int flush_stage(gysk_engine *e, ThreadStage *ts)
{
	if (!ts->fill) return 0;
	{
		std::lock_guard<std::mutex> lk(e->mtx);
		CU(e, cudaSetDevice(e->dev));
		int rc = append_chunk(e, ts->buf[ts->cur], ts->fill);
		if (rc) return rc;
		CU(e, cudaEventRecord(ts->copied[ts->cur], e->copy_stream));
	}
	ts->cur ^= 1; ts->fill = 0;
	CU(e, cudaEventSynchronize(ts->copied[ts->cur]));		// the other chunk's copy (issued a whole chunk ago) has left the host
	return 0;
}

inline gysk_event *stage_slot(gysk_engine *e, ThreadStage *ts, int *rc)
{
	if (ts->fill == ts->cap) { *rc = flush_stage(e, ts); if (*rc) return nullptr; }
	return ts->buf[ts->cur] + ts->fill++;
}

int stage_events(gysk_engine *e, ThreadStage *ts, const gysk_event *ev, uint64_t n)
{
	while (n) {
		if (ts->fill == ts->cap) { int rc = flush_stage(e, ts); if (rc) return rc; }
		const uint32_t m = (uint32_t)std::min<uint64_t>(ts->cap - ts->fill, n);
		memcpy(ts->buf[ts->cur] + ts->fill, ev, (size_t)m * sizeof(gysk_event));
		ts->fill += m; ev += m; n -= m;
	}
	return 0;
}

} // namespace

// every thread's partial chunk goes to the device (called by readers BEFORE they take the engine mutex)
int gysk::drain_all(gysk_engine *e)
{
	std::lock_guard<std::mutex> lk(e->tstage_mtx);
	for (auto &ts : e->tstages) {
		std::lock_guard<std::mutex> l2(ts->m);
		int rc = flush_stage(e, ts.get());
		if (rc) return rc;
	}
	return 0;
}

namespace gysk {

// ---- pure host helpers: the reference's percentile rule and the estimators -------------------------------

void hist_from_cells(const HistCell *cells, int nb, gysk_hist_serial *out, uint64_t *total, int64_t *maxv, bool t_is_int)
{
	uint64_t t = 0;

	for (int i = 0; i < GYSK_HIST_MAX_BUCKETS; ++i) {
		if (i < nb) { out[i].count = cells[i].count; out[i].sum = cells[i].sum; t += cells[i].count; }
		else { out[i].count = 0; out[i].sum = 0; }
	}
	*total = t;			// total_count_ always equals the sum of the bucket counts (add_data bumps both)
	int64_t m = cells[HIST_MAX_CELL].sum;
	if (t_is_int && m == INT64_MIN) m = INT32_MIN;		// numeric_limits<int>::min() for GY_HISTOGRAM<int, ...>
	*maxv = m;
}

void level_from_cells(const HistCell *cells, gysk_hist_serial *out, uint64_t *total, int64_t *maxv)
{
	hist_from_cells(cells, 15, out, total, maxv, false);
	if (*total == 0) *maxv = INT64_MIN;
}

int tdigest_out(const TdHead &head, const Centroid *cent, double *means, uint64_t *weights, uint32_t cap, uint32_t *n, double *minv, double *maxv)
{
	const uint32_t nc = std::min<uint32_t>(std::min<uint32_t>(head.n, TD_CAP), cap);
	for (uint32_t c = 0; c < nc; ++c) { means[c] = cent[c].mean; weights[c] = cent[c].weight; }
	*n = nc;
	if (minv) *minv = head.minv;
	if (maxv) *maxv = head.maxv;
	return head.n > cap ? GYSK_ERR_NOSPC : GYSK_OK;
}

int query_flows_in(gysk_engine *e, const unsigned long long *tbl, const uint64_t *keys, uint32_t n, gysk_flow_est *out, const char *what)
{
	DevState st = e->st;
	st.cms_cur = const_cast<unsigned long long *>(tbl);
	return staged_read(e, keys, n, QCHUNK, sizeof(gysk_flow_est), what, [&](const unsigned long long *d_keys, uint32_t, uint32_t m) {
		return launch_query_flows(st, d_keys, m, 0, reinterpret_cast<gysk_flow_est *>(e->d_wstage), e->stream);
	}, CopyRows<gysk_flow_est> {out});
}

} // namespace gysk

namespace {

// the unit grid of the K_1 scale: q_j = (sin(pi (j/delta - 1/2)) + 1)/2 — libm on the host, the same expression as the oracle. The
// device's grid and the pgtext export's compress both come from here.
std::vector<double> k1_grid(uint32_t delta)
{
	std::vector<double> q(delta + 1);
	for (uint32_t j = 0; j <= delta; ++j) q[j] = 0.5 * (sin(M_PI * ((double)j / (double)delta - 0.5)) + 1.0);
	q[0] = 0.0; q[delta] = 1.0;
	return q;
}

// the single-id reads: one piece of one id, whose raw state (`bytes` of it) the caller reads from the head of h_wstage
template <typename Launch>
int stage_one(gysk_engine *e, uint64_t id, size_t bytes, const char *what, Launch launch)
{
	return staged_read(e, &id, 1, 1, bytes, what, launch, RowsStay {});
}

int stage_svc_raw(gysk_engine *e, uint64_t id)
{
	return stage_one(e, id, sizeof(SvcRaw), "gather_svcs", [&](const unsigned long long *d_ids, uint32_t, uint32_t m) {
		return launch_gather_svcs(e->st, d_ids, m, reinterpret_cast<SvcRaw *>(e->d_wstage), e->stream);
	});
}

// the two summary rows, by id (d_ids) or by slot (d_slots), into the stage
int launch_rows(gysk_engine *e, const unsigned long long *d_ids, const unsigned long long *d_slots, uint32_t m, gysk_svc_summary *)
{
	return launch_svc_summaries(e->st, d_ids, d_slots, m, reinterpret_cast<gysk_svc_summary *>(e->d_wstage), e->stream);
}
int launch_rows(gysk_engine *e, const unsigned long long *d_ids, const unsigned long long *d_slots, uint32_t m, gysk_task_summary *)
{
	return launch_task_summaries(e->st, d_ids, d_slots, m, reinterpret_cast<gysk_task_summary *>(e->d_wstage), e->stream);
}
int launch_rows(gysk_engine *e, const unsigned long long *, const unsigned long long *d_slots, uint32_t m, gysk_listener_day_stats *)
{
	return launch_day_stats(e->st, d_slots, m, reinterpret_cast<gysk_listener_day_stats *>(e->d_wstage), e->stream);
}
// The rolling levels at the flush of tsec: the closing window goes to ring slot (tsec / width) % NSLOTS of each level, and a slot
// still holding an older epoch is cleared first (LevelRing::fresh records it). Then the live slots, whose epochs lie in the level's
// last NSLOTS: what every reader of the levels sums until the next flush. GYSK_FLAG_FLOW_LEVEL's count-min ring takes level 0's
// decision as it is (launch_cms_level_roll). Slot widths: Level_5s_5min_5days_all durations {300 s, 432000 s} / 10 slots
// (gy_statistics.h:1548, :1105).
int roll_levels(gysk_engine *e, uint32_t tsec)
{
	static constexpr uint32_t width[NLEVELS] = {30, 43200};
	LevelRing &lv = e->st.levels;

	lv.fresh = 0;
	for (int l = 0; l < NLEVELS; ++l) {
		const uint64_t epoch = tsec / width[l];
		const uint32_t k = (uint32_t)(epoch % NSLOTS);
		if (e->ring_epoch[l][k] != epoch) {
			CU(e, cudaMemsetAsync(lv.row(l, k, 0), 0, (size_t)lv.stride * HIST_CELLS * sizeof(HistCell), e->stream));
			e->ring_epoch[l][k] = epoch;
			lv.fresh |= 1u << l;
		}
		lv.cur[l] = k;
		lv.live[l] = 0;
		for (int j = 0; j < NSLOTS; ++j) {
			const uint64_t ep = e->ring_epoch[l][j];
			if (ep != ~0ull && ep + NSLOTS > epoch && ep <= epoch) lv.live[l] |= 1u << j;
		}
	}
	return 0;
}

// ---- capacity: the per-slot arrays --------------------------------------------------------------------------------
//
// Every device array indexed by service or process slot, with its elements per slot: f(pointer, elements per slot, kind). Svc arrays
// hold max_svcs + 1 slots (slot max_svcs is the null slot), the level ring max_svcs rows in each of its NLEVELS x NSLOTS planes
// (LevelRing::stride), Task arrays max_tasks slots. gysk_create allocates exactly these, gysk_grow moves them, slot_bytes sums them.
// The process eviction's arrays exist only with task_idle_evict_secs (task_evict). The batch's segment arrays (Seg) are indexed by the
// slot field of the sort keys: max_svcs + 1 entries, and one more per trace row (max_trace_svcs) beyond the null slot.
enum class SlotKind { Svc, Ring, Task, Seg };

template <typename F>
void each_slot_array(DevState &st, SortTemp &tmp, uint32_t hll_p, bool task_evict, F f)
{
	f(st.slot_id, 1, SlotKind::Svc); f(st.slot_host, 1, SlotKind::Svc);
	f(st.slot_first_seen, 1, SlotKind::Svc); f(st.slot_last_active, 1, SlotKind::Svc);
	f(st.evict_list, 1, SlotKind::Svc); f(st.evict_ids, 1, SlotKind::Svc); f(st.svc_tbl.free_slots, 1, SlotKind::Svc);
	f(st.hist_cur, HIST_CELLS, SlotKind::Svc); f(st.hist_last, HIST_CELLS, SlotKind::Svc); f(st.hist_all, HIST_CELLS, SlotKind::Svc);
	f(st.levels.ring, (size_t)NLEVELS * NSLOTS * HIST_CELLS, SlotKind::Ring);
	f(st.conn_cur, 1, SlotKind::Svc); f(st.conn_last, 1, SlotKind::Svc); f(st.conn_all_cnt, 1, SlotKind::Svc); f(st.conn_all_kb, 1, SlotKind::Svc);
	f(st.bm_cur, HIST_CELLS, SlotKind::Svc); f(st.bm_last, HIST_CELLS, SlotKind::Svc);
	f(st.hll, (size_t)1 << hll_p, SlotKind::Svc);
	f(st.td_cent, TD_CAP, SlotKind::Svc); f(st.td_head, 1, SlotKind::Svc);
	f(st.slot_batch, 1, SlotKind::Svc); f(st.slot_aux, 1, SlotKind::Svc);
	f(st.qps_hist, HIST_CELLS, SlotKind::Svc); f(st.act_hist, HIST_CELLS, SlotKind::Svc); f(st.slot_state, 1, SlotKind::Svc);
	f(tmp.touched, 1, SlotKind::Seg); f(tmp.segs, 1, SlotKind::Seg);
	f(st.task_hist, 3 * HIST_CELLS, SlotKind::Task); f(st.task_prev, 3, SlotKind::Task); f(st.task_last, 3, SlotKind::Task);
	f(st.task_slot_id, 1, SlotKind::Task); f(st.task_slot_host, 1, SlotKind::Task);
	if (task_evict) {
		f(st.task_last_active, 1, SlotKind::Task); f(st.task_evict_list, 1, SlotKind::Task); f(st.task_evict_ids, 1, SlotKind::Task);
		f(st.task_tbl.free_slots, 1, SlotKind::Task);
	}
}

// device bytes of one service slot (its ring rows included) and of one process slot: the sums of each_slot_array
void slot_bytes(uint32_t hll_p, bool task_evict, uint64_t *svc, uint64_t *task)
{
	DevState st {};
	SortTemp tmp {};
	uint64_t b[4] = {0, 0, 0, 0};
	each_slot_array(st, tmp, hll_p, task_evict, [&](auto *&p, size_t k, SlotKind kind) { b[(int)kind] += k * sizeof(*p); });
	*svc = b[(int)SlotKind::Svc] + b[(int)SlotKind::Ring] + b[(int)SlotKind::Seg];
	*task = b[(int)SlotKind::Task];
}

size_t slots_of(SlotKind kind, uint32_t max_svcs, uint32_t max_tasks, uint32_t max_trace)
{
	return kind == SlotKind::Svc ? (size_t)max_svcs + 1 : kind == SlotKind::Ring ? (size_t)max_svcs :
			kind == SlotKind::Seg ? (size_t)max_svcs + 1 + max_trace : (size_t)max_tasks;
}

// the arrays sized by capacity beside the per-slot ones: an id table's entries, the sort buffers' keys and look-back tiles, the batch
// rows of the long key segments
uint32_t table_cap(uint32_t slots) { return pow2_at_least((uint64_t)slots * 2); }
size_t sort_keys(const gysk_config &cfg)
{
	return std::max<size_t>(std::max<size_t>(std::max<size_t>((size_t)cfg.max_svcs + 1, cfg.max_tasks) + 1, cfg.max_batch), (size_t)cfg.max_trace_svcs + 1);
}
uint32_t sort_tiles(size_t nkeys) { return (uint32_t)((nkeys + SORT_TILE - 1) / SORT_TILE); }
size_t batch_rows(const gysk_config &cfg) { return std::min<size_t>((size_t)cfg.max_svcs + 1 + cfg.max_trace_svcs, ((size_t)cfg.max_batch + LONG_SEG - 1) / LONG_SEG); }
// trace rows fit the 24-bit slot field of the sort keys as pseudo-slots max_svcs + 1 .. max_svcs + max_trace_svcs
bool trace_fits(uint32_t max_svcs, uint32_t max_trace) { return !max_trace || (uint64_t)max_svcs + 1 + max_trace <= (1ull << 24); }

SvcRows finish_rows(const gysk_engine *e, gysk_svc_summary *out) { return SvcRows {e->cfg.hll_p, out}; }
CopyRows<gysk_task_summary> finish_rows(const gysk_engine *, gysk_task_summary *out) { return CopyRows<gysk_task_summary> {out}; }
CopyRows<gysk_listener_day_stats> finish_rows(const gysk_engine *, gysk_listener_day_stats *out) { return CopyRows<gysk_listener_day_stats> {out}; }

} // namespace

// the linear-counting branch of the HLL estimate needs log(), which neither CUDA nor glibc rounds correctly: the host takes it
void gysk::SvcRows::operator()(const uint8_t *rows, uint32_t off, uint32_t m) const
{
	const gysk_svc_summary *r = reinterpret_cast<const gysk_svc_summary *>(rows);
	for (uint32_t i = 0; i < m; ++i) {
		out[off + i] = r[i];
		out[off + i].distinct_clients = hll_finish(r[i].distinct_clients, hll_p);
	}
}

// ============================================================================================================
// C ABI
// ============================================================================================================
extern "C" {

int gysk_abi_version(void) { return GYSK_ABI_VERSION; }

void gysk_config_default(gysk_config *cfg)
{
	if (!cfg) return;
	memset(cfg, 0, sizeof(*cfg));
	cfg->struct_size = sizeof(*cfg);
	cfg->device = 0;
	cfg->max_svcs = 1u << 17;
	cfg->max_tasks = 1u << 16;
	cfg->cms_depth = 4;
	cfg->cms_log2_width = 20;
	cfg->hll_p = 12;
	cfg->td_compression = 200;
	cfg->max_batch = 1u << 22;
	cfg->stage_batch = 0;
	cfg->flags = GYSK_FLAG_AUTO_REGISTER;
	cfg->rank = 0; cfg->world = 1;
}

const char *gysk_last_error(gysk_engine *e)
{
	return e ? e->err.c_str() : g_create_error.c_str();
}

void gysk_destroy(gysk_engine *e)
{
	if (!e) return;
	{ std::lock_guard<std::mutex> lk(g_live_mtx); g_live.erase(std::remove(g_live.begin(), g_live.end(), e->uid), g_live.end()); }
	cudaSetDevice(e->dev);
	if (e->stream) cudaStreamSynchronize(e->stream);
	if (e->copy_stream) cudaStreamSynchronize(e->copy_stream);
	merge_release(e);
	for (int k = 0; k < NBUF; ++k) {
		if (e->ev_copied[k]) cudaEventDestroy(e->ev_copied[k]);
		if (e->ev_done[k]) cudaEventDestroy(e->ev_done[k]);
		if (e->ev_raw_done[k]) cudaEventDestroy(e->ev_raw_done[k]);
	}
	for (auto &ts : e->tstages) {
		for (int i = 0; i < 2; ++i) { if (ts->buf[i]) cudaFreeHost(ts->buf[i]); if (ts->copied[i]) cudaEventDestroy(ts->copied[i]); }
	}
	for (cudaEvent_t ev : e->prof_events) cudaEventDestroy(ev);
	if (e->ev_evict) cudaEventDestroy(e->ev_evict);
	if (e->ev_used) cudaEventDestroy(e->ev_used);
	for (auto &a : e->dallocs) cudaFree(a.first);
	for (void *p : e->hallocs) cudaFreeHost(p);
	if (e->stream) cudaStreamDestroy(e->stream);
	if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
	delete e;
}

int gysk_create(const gysk_config *ucfg, gysk_engine **out)
{
	if (!out) return GYSK_ERR_INVAL;
	*out = nullptr;

	gysk_config cfg;
	gysk_config_default(&cfg);
	if (ucfg) {
		if (ucfg->struct_size != sizeof(gysk_config)) return fail(nullptr, GYSK_ERR_INVAL, "gysk_config.struct_size mismatch");
		cfg = *ucfg;
	}
	if (!cfg.world) cfg.world = 1;
	if (!cfg.stage_batch || cfg.stage_batch > cfg.max_batch) cfg.stage_batch = std::min<uint32_t>(cfg.max_batch, 1u << 22);
	if (cfg.max_svcs < 1 || cfg.max_svcs > (1u << 24) || cfg.max_tasks < 1 || cfg.max_tasks > (1u << 24) || cfg.cms_depth < 1 ||
			cfg.cms_depth > 8 || cfg.cms_log2_width < 4 || cfg.cms_log2_width > 28 || cfg.hll_p < 4 || cfg.hll_p > 16 ||
			cfg.td_compression < 10 || cfg.td_compression > (uint32_t)TD_CAP || cfg.max_batch < 1024 || cfg.max_batch >= (1u << 27) ||
			cfg.rank >= cfg.world || !trace_fits(cfg.max_svcs, cfg.max_trace_svcs))
		return fail(nullptr, GYSK_ERR_INVAL, "gysk_config out of range");
	if ((cfg.flags & GYSK_FLAG_MERGE_TRACES) && !cfg.max_trace_svcs)
		return fail(nullptr, GYSK_ERR_INVAL, "GYSK_FLAG_MERGE_TRACES needs trace rows (gysk_config.max_trace_svcs > 0)");

	int ndev = 0;
	cudaError_t ce = cudaGetDeviceCount(&ndev);
	if (ce != cudaSuccess || ndev <= 0 || cfg.device < 0 || cfg.device >= ndev)
		return fail(nullptr, GYSK_ERR_NODEV, "no usable CUDA device (libgysketch has no CPU fallback)", ce);

	cudaDeviceProp prop;
	if ((ce = cudaGetDeviceProperties(&prop, cfg.device)) != cudaSuccess) return fail(nullptr, GYSK_ERR_NODEV, "cudaGetDeviceProperties", ce);
	if (prop.major != 9 || prop.minor != 0) return fail(nullptr, GYSK_ERR_NODEV, "device is not sm_90 (kernels are built for sm_90a only)");

	gysk_engine *e = new (std::nothrow) gysk_engine;
	if (!e) return fail(nullptr, GYSK_ERR_NOMEM, "new gysk_engine");
	e->cfg = cfg; e->dev = cfg.device; e->uid = g_engine_uid.fetch_add(1);
	{ std::lock_guard<std::mutex> lk(g_live_mtx); g_live.push_back(e->uid); }
	memset(e->ring_epoch, 0xFF, sizeof(e->ring_epoch));

	int rc = 0;
	auto bail = [&](int code) { g_create_error = e->err; gysk_destroy(e); return code; };

	if ((ce = cudaSetDevice(e->dev)) != cudaSuccess) { fail(e, GYSK_ERR_CUDA, "cudaSetDevice", ce); return bail(GYSK_ERR_CUDA); }
	if ((ce = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)) != cudaSuccess ||
			(ce = cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking)) != cudaSuccess) {
		fail(e, GYSK_ERR_CUDA, "cudaStreamCreate", ce); return bail(GYSK_ERR_CUDA);
	}

	DevState &st = e->st;
	const size_t ns = (size_t)cfg.max_svcs + 1;		// slot max_svcs = the null slot: never handed out, always pristine
	const uint32_t scap = table_cap(cfg.max_svcs + 1), tcap = table_cap(cfg.max_tasks);

#define A(call) do { if ((rc = (call)) != 0) return bail(rc); } while (0)
	A(dalloc(e, &st.counters, (size_t)CTR_MAX));
	A(dalloc(e, &st.svc_tbl.ent, scap)); st.svc_tbl.mask = scap - 1; st.svc_tbl.max_slots = cfg.max_svcs;
	A(dalloc(e, &st.svc_tbl.count, 1));
	A(dalloc(e, &st.svc_tbl.free_n, 1));
	A(dalloc(e, &st.task_tbl.ent, tcap)); st.task_tbl.mask = tcap - 1; st.task_tbl.max_slots = cfg.max_tasks;
	A(dalloc(e, &st.task_tbl.count, 1));
	if (cfg.task_idle_evict_secs) A(dalloc(e, &st.task_tbl.free_n, 1));		// without it the process table has no free stack
	SortTemp &tmp = e->tmp;
	each_slot_array(st, tmp, cfg.hll_p, cfg.task_idle_evict_secs, [&](auto *&p, size_t k, SlotKind kind) { if (!rc) rc = dalloc(e, &p, slots_of(kind, cfg.max_svcs, cfg.max_tasks, cfg.max_trace_svcs) * k); });
	if (rc) return bail(rc);
	st.levels.stride = cfg.max_svcs;
	st.svc_tbl.slot_id = st.slot_id; st.svc_tbl.slot_host = st.slot_host;
	st.task_tbl.slot_id = st.task_slot_id; st.task_tbl.slot_host = st.task_slot_host;
	A(halloc(e, &e->h_evict, ns + 2));
	e->h_evict[0] = 0; e->h_evict[cfg.max_svcs + 1] = 0;
	if ((ce = cudaEventCreateWithFlags(&e->ev_evict, cudaEventDisableTiming)) != cudaSuccess) { fail(e, GYSK_ERR_CUDA, "cudaEventCreate", ce); return bail(GYSK_ERR_CUDA); }
	if (cfg.task_idle_evict_secs) {
		A(halloc(e, &e->h_tevict, (size_t)cfg.max_tasks + 1, cudaHostAllocMapped));
		e->h_tevict[0] = 0;
		if ((ce = cudaHostGetDevicePointer((void **)&e->d_tevict, e->h_tevict, 0)) != cudaSuccess) { fail(e, GYSK_ERR_CUDA, "cudaHostGetDevicePointer", ce); return bail(GYSK_ERR_CUDA); }
	}
	A(halloc(e, &e->h_used, 4));
	e->h_used[3] = 0;		// processes on the free stack: stays 0 without process eviction
	if ((ce = cudaEventCreateWithFlags(&e->ev_used, cudaEventDisableTiming)) != cudaSuccess) { fail(e, GYSK_ERR_CUDA, "cudaEventCreate", ce); return bail(GYSK_ERR_CUDA); }
	A(dalloc(e, &st.cms_cur, (size_t)cfg.cms_depth << cfg.cms_log2_width)); A(dalloc(e, &st.cms_last, (size_t)cfg.cms_depth << cfg.cms_log2_width));
	if (cfg.flags & GYSK_FLAG_FLOW_LEVEL) {
		// not per slot: outside each_slot_array, so gysk_grow leaves them; device_bytes counts them
		A(dalloc(e, &st.cms_ring, (size_t)NSLOTS * ((size_t)cfg.cms_depth << cfg.cms_log2_width)));
		A(dalloc(e, &st.cms_5min, (size_t)cfg.cms_depth << cfg.cms_log2_width));
	}
	st.cms_depth = cfg.cms_depth; st.cms_log2w = cfg.cms_log2_width; st.cms_wmask = (1u << cfg.cms_log2_width) - 1; st.hll_p = cfg.hll_p;
	st.rank = cfg.rank; st.world = cfg.world; st.auto_register = (cfg.flags & GYSK_FLAG_AUTO_REGISTER) ? 1 : 0;
	st.td_delta = (double)cfg.td_compression;
	{
		const std::vector<double> qtab = k1_grid(cfg.td_compression);
		double *d_q = nullptr;
		A(dalloc(e, &d_q, qtab.size(), false));
		if ((ce = cudaMemcpy(d_q, qtab.data(), qtab.size() * sizeof(double), cudaMemcpyHostToDevice)) != cudaSuccess) { fail(e, GYSK_ERR_CUDA, "qtab", ce); return bail(GYSK_ERR_CUDA); }
		st.td.qtab = d_q; st.td.delta = cfg.td_compression; st.td.pad = 0;
	}
	{
		// dense value bins of the hot services (DESIGN.md §4): GYSK_HOT_ROWS rows of 16 KB (default 2048, 0 switches the path off); a
		// service turns hot with GYSK_HOT_MIN (default 4096) .. GYSK_HOT_MAX samples in one batch unless its fullest bin holds more
		// than GYSK_HOT_BIN_MAX (default 131072) of them. Routing only: results do not depend on any of these.
		auto envl = [](const char *name, long dflt) { const char *v = getenv(name); return v ? atol(v) : dflt; };
		long rows = envl("GYSK_HOT_ROWS", 2048);
		if (rows < 0) rows = 0;
		if (rows > 65536) rows = 65536;
		if ((size_t)rows > ns) rows = (long)ns;
		st.hot_cap = (uint32_t)rows;
		st.hot_min = (uint32_t)std::max(1l, envl("GYSK_HOT_MIN", 4096));
		st.hot_max = (uint32_t)std::min<long>(0xFFFFFFFFl, std::max(1l, envl("GYSK_HOT_MAX", 0xFFFFFFFFl)));
		st.hot_bin_max = (uint32_t)std::min<long>(0xFFFFFFFFl, std::max(1l, envl("GYSK_HOT_BIN_MAX", 131072)));
		st.hot_rows = nullptr; st.hot_slot = nullptr;
		if (rows) { A(dalloc(e, &st.hot_rows, (size_t)rows * HOT_ROW_WORDS)); A(dalloc(e, &st.hot_slot, (size_t)rows)); }
	}
	const size_t nsort = sort_keys(cfg);		// RESP keys of a batch; the top-N sorts rank services / tasks
	tmp.nkeys = nsort;
	tmp.max_tiles = sort_tiles(nsort);
	A(dalloc(e, &tmp.keys_a, nsort, false)); A(dalloc(e, &tmp.keys_b, nsort, false));
	A(dalloc(e, &tmp.tile_status, (size_t)RADIX_MAX * tmp.max_tiles));
	tmp.epoch = &e->sort_epoch;
	A(dalloc(e, &tmp.os_ghist, (size_t)OS_GHIST_WORDS));
	{
		const size_t nmw = (size_t)TD_MERGE_MAX_SMS * TD_MERGE_CTAS_PER_SM * 4;		// warps of bins_merge_kernel
		// a batch has fewer than max_batch / LONG_SEG segments of more than LONG_SEG keys, and no more than one per service. The
		// rows start at zero and bins_merge_kernel leaves them so.
		const size_t nbrows = batch_rows(cfg);
		A(dalloc(e, &tmp.long_slot, nbrows, false)); A(dalloc(e, &tmp.batch_rows, nbrows * HOT_ROW_WORDS));
		A(dalloc(e, &tmp.items_scratch, nmw * NBINS, false)); A(dalloc(e, &tmp.big_scratch, nmw, false));
		// the batch's connection / process record queue: one region per ingest warp (SortTemp::recq)
		const uint32_t nsm = (uint32_t)prop.multiProcessorCount;
		tmp.rec_cnt_cap = nsm * IngestShape::WARPS * IngestShape::MIN_CTAS;
		tmp.recq_cap = (uint64_t)cfg.max_batch + (uint64_t)tmp.rec_cnt_cap * IngestShape::CHUNK;
		A(dalloc(e, &tmp.recq, (size_t)tmp.recq_cap, false)); A(dalloc(e, &tmp.rec_cnt, (size_t)tmp.rec_cnt_cap, false));
		// the batch's flow table (FlowTable): zero here, and the TASK drain pass leaves it so after every batch. Not per slot: outside
		// each_slot_array, so gysk_grow leaves it
		tmp.flow_cap = std::min<uint32_t>(FLOW_ENT_MAX, pow2_at_least(2ull * cfg.max_batch));
		A(dalloc(e, &tmp.flow, (size_t)tmp.flow_cap));
	}
	st.svc_tbl.insert_fail = st.counters + CTR_INSERT_FAIL; st.task_tbl.insert_fail = nullptr;
	if (cfg.max_trace_svcs) {
		// trace rows (TraceTable): not per service slot but per row, so gysk_slot_bytes leaves them out and device_bytes counts them; only
		// the slot -> row map grows with the service table
		TraceTable &tr = st.trace;
		const size_t nr = cfg.max_trace_svcs;
		tr.rows = cfg.max_trace_svcs; tr.par = 0; tr.base = cfg.max_svcs + 1;
		A(dalloc(e, &tr.row_of, ns)); A(dalloc(e, &tr.row_slot, nr, false)); A(dalloc(e, &tr.free_rows, nr, false));
		A(dalloc(e, &tr.cnt, 2 * nr * TRACE_WORDS)); A(dalloc(e, &tr.head, 2 * nr)); A(dalloc(e, &tr.cent, 2 * nr * TRACE_TD_CAP));
		A(dalloc(e, &tr.count, 1)); A(dalloc(e, &tr.free_n, 1)); A(dalloc(e, &tr.dropped, 1));
		if ((ce = cudaMemsetAsync(tr.row_slot, 0xFF, nr * sizeof(uint32_t), e->stream)) != cudaSuccess) { fail(e, GYSK_ERR_CUDA, "trace rows", ce); return bail(GYSK_ERR_CUDA); }
		const std::vector<double> qtab = k1_grid(TRACE_TD_DELTA);
		double *d_q = nullptr;
		A(dalloc(e, &d_q, qtab.size(), false));
		if ((ce = cudaMemcpy(d_q, qtab.data(), qtab.size() * sizeof(double), cudaMemcpyHostToDevice)) != cudaSuccess) { fail(e, GYSK_ERR_CUDA, "trace qtab", ce); return bail(GYSK_ERR_CUDA); }
		tr.td.qtab = d_q; tr.td.delta = TRACE_TD_DELTA; tr.td.pad = 0;
	}

	for (int k = 0; k < NBUF; ++k) {
		A(dalloc(e, &e->d_events[k], (size_t)cfg.stage_batch, false));
		e->raw_bytes = (size_t)cfg.stage_batch * 32;
		A(dalloc(e, &e->d_raw[k], e->raw_bytes, false));
		if ((ce = cudaEventCreateWithFlags(&e->ev_copied[k], cudaEventDisableTiming)) != cudaSuccess ||
				(ce = cudaEventCreateWithFlags(&e->ev_raw_done[k], cudaEventDisableTiming)) != cudaSuccess ||
				(ce = cudaEventCreateWithFlags(&e->ev_done[k], cudaEventDisableTiming)) != cudaSuccess) {
			fail(e, GYSK_ERR_CUDA, "cudaEventCreate", ce); return bail(GYSK_ERR_CUDA);
		}
	}
	A(dalloc(e, &e->d_qids, (size_t)QCHUNK)); A(halloc(e, &e->h_qids, (size_t)QCHUNK));
	A(halloc(e, &e->h_counters, (size_t)CTR_MAX + 2));
	A(dalloc(e, &e->d_wstage, STAGE_BYTES, false)); A(halloc(e, &e->h_wstage, STAGE_BYTES));
#undef A

	e->kernel_launches += launch_init_slots(st, 0, cfg.max_svcs + 1, 0, cfg.max_tasks, e->stream);
	if ((ce = cudaStreamSynchronize(e->stream)) != cudaSuccess || (ce = cudaGetLastError()) != cudaSuccess) {
		fail(e, GYSK_ERR_CUDA, "engine init", ce); return bail(GYSK_ERR_CUDA);
	}
	*out = e;
	return GYSK_OK;
}

void *gysk_stream(gysk_engine *e) { return e ? (void *)e->stream : nullptr; }

int gysk_profile_enable(gysk_engine *e, int on)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Sync);
	e->profiling = !!on;
	e->prof_used = 0;
	return GYSK_OK;
}

int gysk_profile_read(gysk_engine *e, double *ms_ingest, double *ms_tdigest, uint64_t *nbatches)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Sync);
	double a = 0, b = 0;
	for (size_t i = 0; i + 3 <= e->prof_used; i += 3) {
		float t1 = 0, t2 = 0;
		CU(e, cudaEventElapsedTime(&t1, e->prof_events[i], e->prof_events[i + 1]));
		CU(e, cudaEventElapsedTime(&t2, e->prof_events[i + 1], e->prof_events[i + 2]));
		a += t1; b += t2;
	}
	if (ms_ingest) *ms_ingest = a;
	if (ms_tdigest) *ms_tdigest = b;
	if (nbatches) *nbatches = e->prof_used / 3;
	e->prof_used = 0;
	return GYSK_OK;
}

int gysk_get_stats(gysk_engine *e, gysk_stats *out)
{
	CHECK_ENGINE(e);
	if (!out) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Sync);
	CU(e, cudaMemcpyAsync(e->h_counters, e->st.counters, sizeof(unsigned long long) * CTR_MAX, cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaMemcpyAsync(e->h_counters + CTR_MAX, e->st.svc_tbl.count, sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaMemcpyAsync(e->h_counters + CTR_MAX + 1, e->st.task_tbl.count, sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	memset(out, 0, sizeof(*out));
	out->events_in = e->h_counters[CTR_IN]; out->events_dropped = e->h_counters[CTR_DROPPED];
	out->events_resp = e->h_counters[CTR_RESP]; out->events_tcp = e->h_counters[CTR_TCP]; out->events_task = e->h_counters[CTR_TASK];
	if (int rc = collect_evicted(e)) return rc;
	int32_t nfree = 0;
	CU(e, cudaMemcpy(&nfree, e->st.svc_tbl.free_n, sizeof(nfree), cudaMemcpyDeviceToHost));
	out->nsvcs = std::min<uint64_t>((uint32_t)e->h_counters[CTR_MAX], e->cfg.max_svcs) - (uint64_t)std::max(nfree, 0);
	out->svcs_evicted = e->evicted_total;
	int32_t tfree = 0;
	if (e->st.task_tbl.free_n) CU(e, cudaMemcpy(&tfree, e->st.task_tbl.free_n, sizeof(tfree), cudaMemcpyDeviceToHost));
	out->ntasks = std::min<uint64_t>((uint32_t)e->h_counters[CTR_MAX + 1], e->cfg.max_tasks) - (uint64_t)std::max(tfree, 0);
	out->batches = e->batches; out->kernel_launches = e->kernel_launches;
	out->wire_msgs_ok = e->wire_ok; out->wire_msgs_bad = e->wire_bad;
	return GYSK_OK;
}

// diagnostic: rows of dense value bins handed out to hot services so far (results never depend on it)
int64_t gysk_hot_rows_in_use(gysk_engine *e)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Sync);
	if (!e->st.hot_rows) return 0;
	unsigned long long n = 0;
	CU(e, cudaMemcpy(&n, e->st.counters + CTR_NHOT_NEXT, sizeof(n), cudaMemcpyDeviceToHost));
	return (int64_t)n;
}

// introspection (no device needed): word of value bin `bin` inside a hot row's {samples | remainders} half; the usec sum of the bin
// lies GYSK_HOT_ROW_BINS words further on. ~0 for a bin the engine does not have.
uint32_t gysk_hot_row_word(uint32_t bin)
{
	return bin < (uint32_t)NBINS ? hot_word(bin) : 0xFFFFFFFFu;
}

// diagnostic: response samples of the last device batch that travelled as sort keys (the others went to hot rows)
int64_t gysk_last_batch_keys(gysk_engine *e)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Sync);
	unsigned long long n = 0;
	CU(e, cudaMemcpy(&n, e->st.counters + CTR_NKEYS, sizeof(n), cudaMemcpyDeviceToHost));
	return (int64_t)n;
}

// diagnostic: connection records of the last device batch whose count-min update bypassed the flow table
int64_t gysk_last_batch_flow_direct(gysk_engine *e)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Sync);
	unsigned long long n = 0;
	CU(e, cudaMemcpy(&n, e->st.counters + CTR_FLOW_DIRECT, sizeof(n), cudaMemcpyDeviceToHost));
	return (int64_t)n;
}

// diagnostic: entries of the flow table that are not zero (a key or a sum left behind); 0 whenever no batch is in flight
int64_t gysk_flow_table_used(gysk_engine *e)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Sync);
	std::vector<FlowEnt> t(e->tmp.flow_cap);
	CU(e, cudaMemcpy(t.data(), e->tmp.flow, t.size() * sizeof(FlowEnt), cudaMemcpyDeviceToHost));
	return (int64_t)std::count_if(t.begin(), t.end(), [](const FlowEnt &f) { return f.key || f.inc; });
}

int gysk_register_ids(gysk_engine *e, const uint64_t *ids, uint32_t n, int is_task)
{
	CHECK_ENGINE(e);
	if (!ids && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	return staged_read(e, ids, n, QCHUNK, 0, "register",
			[&](const unsigned long long *d_ids, uint32_t, uint32_t m) { return launch_register(e->st, d_ids, m, is_task, e->stream); }, RowsStay {});
}

// ---- ingest -----------------------------------------------------------------------------------------------

int gysk_ingest_device(gysk_engine *e, const gysk_event *d_events, uint64_t n)
{
	CHECK_ENGINE(e);
	if (!d_events && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);					// keep arrival order
	for (uint64_t off = 0; off < n; off += e->cfg.max_batch) {
		const uint64_t m = std::min<uint64_t>(e->cfg.max_batch, n - off);
		if (int rc = process_device_batch(e, d_events + off, m, nullptr)) return rc;
	}
	return GYSK_OK;
}

int gysk_ingest_pinned(gysk_engine *e, const gysk_event *pinned, uint64_t n)
{
	CHECK_ENGINE(e);
	if (!pinned && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	// zero copy on the host: the H2D copies read the caller's page-locked buffer directly, chunk by chunk into the two device
	// event buffers; the copy of chunk c+1 is enqueued as soon as the ingest kernel of chunk c is, so the link never idles
	return append_chunk(e, pinned, n);
}

} // extern "C"

// ---- raw records: decoded into the canonical 32-byte event — by the same inline functions on the host (a few records: the
// calling thread's stage) and on the device (bulk: the raw bytes cross the link, a kernel expands them; SURVEY.md §8f-2) ----------
namespace gysk {

__host__ __device__ inline uint32_t bswap16(uint32_t v) { return ((v & 0xFFu) << 8) | ((v >> 8) & 0xFFu); }
__host__ __device__ inline uint32_t clamp32(uint64_t v) { return v > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)v; }

// listener id of a raw eBPF record: the reference keys listeners by NS_IP_PORT {ip, port, netns} (gy_socket_stat.cc:1529) and
// derives glob_id_ with CityHash (:1824); the id is opaque to the engine, so any deterministic 64-bit fold of the same triple
// serves: two lookup2 words. IPv6 addresses are folded to 32 bits first.
__host__ __device__ inline uint64_t raw_svc_id(uint32_t ip, uint32_t netns, uint32_t port)
{
	uint64_t id = ((uint64_t)jhash_2words(ip, netns, GY_SEED) << 32) | jhash_2words(port, netns, GY_SEED ^ ip);
	return id ? id : 1;
}
__host__ __device__ inline uint32_t fold_ip6(const uint32_t w[4]) { return jhash_2words(w[2], w[3], jhash_2words(w[0], w[1], GY_SEED)); }

__host__ __device__ inline void ev_pad(gysk_event &o) { o.svc_id = 0; o.flow_key = 0; o.value = 0; o.host_idx = 0; o.tsec = 0; o.type = 0xFFFF; o.flags = 0; }

// TCP_SOCK_HANDLER::handle_ipv4_resp_event / handle_ipv6_resp_event, common/gy_socket_stat.cc:1517-1552: tresp = lsndtime - lrcvtime
// (msec), dropped when (uint32_t)tresp > 1 000 000; ports arrive in network byte order (ntohs :1526-1527); the client port keys
// CONN_BITMAP (gy_socket_stat.h:403-410)
__host__ __device__ inline void decode_resp(uint32_t sip, uint32_t cip, uint32_t netns, uint32_t sport_be, uint32_t dport_be, uint32_t lsnd, uint32_t lrcv,
		uint32_t host_idx, gysk_event &o)
{
	const uint32_t tresp = lsnd - lrcv;
	if (tresp > 1000000u) { ev_pad(o); return; }
	const uint32_t sport = bswap16(sport_be), dport = bswap16(dport_be);
	o.svc_id = raw_svc_id(sip, netns, sport);
	o.flow_key = ((uint64_t)cip << 32) | dport;
	o.value = tresp * 1000u; o.host_idx = host_idx; o.tsec = 0; o.type = GYSK_EV_RESP; o.flags = 0;
}

// TCP_SOCK_HANDLER::handle_ipv4_conn_event / handle_ipv6_conn_event, common/gy_socket_stat.cc:241-294: type 1..4; on close the
// byte counters are added to the listener totals (handle_bpf_close_ser :850)
__host__ __device__ inline void decode_conn(uint32_t saddr, uint32_t daddr, uint32_t netns, uint32_t sport_be, uint32_t dport_be, uint32_t type,
		uint64_t bytes, uint64_t ts_ns, uint32_t host_idx, gysk_event &o)
{
	if (type < GYSK_EV_CONNECT || type > GYSK_EV_CLOSE_SER) { ev_pad(o); return; }
	const bool ser_side = (type == GYSK_EV_ACCEPT || type == GYSK_EV_CLOSE_SER);
	const uint32_t hs = bswap16(sport_be), hd = bswap16(dport_be);
	const uint32_t sip = ser_side ? saddr : daddr, sport = ser_side ? hs : hd;
	const uint32_t cip = ser_side ? daddr : saddr, cport = ser_side ? hd : hs;
	o.svc_id = raw_svc_id(sip, netns, sport);
	o.flow_key = ((uint64_t)cip << 32) | cport;
	o.value = clamp32(bytes);
	o.host_idx = host_idx; o.tsec = (uint32_t)(ts_ns / 1000000000ull); o.type = (uint16_t)type; o.flags = 0;
}

__host__ __device__ inline uint32_t raw_stride(uint32_t kind)
{
	switch (kind) {
	case GYSK_RAW_EVENT32 : return 32;
	case GYSK_RAW_TCP_IPV4_EVENT : return sizeof(wire::tcp_ipv4_event_t);
	case GYSK_RAW_TCP_IPV4_RESP : return sizeof(wire::tcp_ipv4_resp_event_t);
	case GYSK_RAW_TCP_IPV6_EVENT : return sizeof(wire::tcp_ipv6_event_t);
	case GYSK_RAW_TCP_IPV6_RESP : return sizeof(wire::tcp_ipv6_resp_event_t);
	case GYSK_RAW_RESP16 : return sizeof(gysk_resp16);
	case GYSK_RAW_TCP24 : return sizeof(gysk_tcp24);
	case GYSK_RAW_TASK24 : return sizeof(gysk_task24);
	default : return 0;
	}
}

__host__ __device__ inline void decode_raw(uint32_t kind, const void *rec, uint32_t host_idx, gysk_event &o)
{
	switch (kind) {
	case GYSK_RAW_TCP_IPV4_RESP : {
		const wire::tcp_ipv4_resp_event_t &p = *static_cast<const wire::tcp_ipv4_resp_event_t *>(rec);
		decode_resp(p.saddr, p.daddr, p.netns, p.sport, p.dport, p.lsndtime, p.lrcvtime, host_idx, o);
		break;
	}
	case GYSK_RAW_TCP_IPV6_RESP : {
		const wire::tcp_ipv6_resp_event_t &p = *static_cast<const wire::tcp_ipv6_resp_event_t *>(rec);
		decode_resp(fold_ip6(p.saddr), fold_ip6(p.daddr), p.netns, p.sport, p.dport, p.lsndtime, p.lrcvtime, host_idx, o);
		break;
	}
	case GYSK_RAW_TCP_IPV4_EVENT : {
		const wire::tcp_ipv4_event_t &p = *static_cast<const wire::tcp_ipv4_event_t *>(rec);
		decode_conn(p.saddr, p.daddr, p.netns, p.sport, p.dport, p.type, p.bytes_received + p.bytes_acked, p.ts_ns, host_idx, o);
		break;
	}
	case GYSK_RAW_TCP_IPV6_EVENT : {
		const wire::tcp_ipv6_event_t &p = *static_cast<const wire::tcp_ipv6_event_t *>(rec);
		decode_conn(fold_ip6(p.saddr), fold_ip6(p.daddr), p.netns, p.sport, p.dport, p.type, p.bytes_received + p.bytes_acked, p.ts_ns, host_idx, o);
		break;
	}
	case GYSK_RAW_RESP16 : {
		const gysk_resp16 &p = *static_cast<const gysk_resp16 *>(rec);
		o.svc_id = p.svc_id; o.flow_key = p.cli_port; o.value = p.usec; o.host_idx = p.host_idx; o.tsec = 0; o.type = GYSK_EV_RESP; o.flags = p.flags;
		break;
	}
	case GYSK_RAW_TCP24 : {
		const gysk_tcp24 &p = *static_cast<const gysk_tcp24 *>(rec);
		o.svc_id = p.svc_id; o.flow_key = p.flow_key; o.value = p.bytes; o.host_idx = p.host_idx; o.tsec = 0; o.type = p.type; o.flags = 0;
		break;
	}
	case GYSK_RAW_TASK24 : {
		const gysk_task24 &p = *static_cast<const gysk_task24 *>(rec);
		o.svc_id = p.aggr_task_id; o.flow_key = (uint64_t)p.cpu_delay_msec | ((uint64_t)p.blkio_delay_msec << 32); o.value = p.cpu_pct;
		o.host_idx = p.host_idx; o.tsec = 0; o.type = GYSK_EV_TASK; o.flags = 0;
		break;
	}
	default : ev_pad(o); break;
	}
}

// one thread per raw record: 16-byte stores of the expanded event
__global__ void __launch_bounds__(256) decode_raw_kernel(uint32_t kind, const uint8_t *__restrict__ raw, uint32_t n, uint32_t host_idx, gysk_event *__restrict__ out)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	gysk_event o;
	decode_raw(kind, raw + (size_t)i * raw_stride(kind), host_idx, o);
	uint4 *d = reinterpret_cast<uint4 *>(out + i);
	d[0] = make_uint4((uint32_t)o.svc_id, (uint32_t)(o.svc_id >> 32), (uint32_t)o.flow_key, (uint32_t)(o.flow_key >> 32));
	d[1] = make_uint4(o.value, o.host_idx, o.tsec, (uint32_t)o.type | ((uint32_t)o.flags << 16));
}

// ---- wire records: one decoder per kind, record -> event; false for a record the reference skips -------------------------------

// partha_tcp_conn_info (gy_mconnhdlr.cc:9130)
inline bool decode_wire(const wire::TCP_CONN_NOTIFY &r, uint32_t host_idx, gysk_event &o)
{
	if (!r.ser_glob_id_ || !r.cli_task_aggr_id_) return false;		// :9143 guard of the group-by
	const bool closed = !!r.tusec_close_;
	if (r.is_tcp_accept_event_) o.type = closed ? GYSK_EV_CLOSE_SER : GYSK_EV_ACCEPT;
	else if (r.is_tcp_connect_event_) o.type = closed ? GYSK_EV_CLOSE_CLI : GYSK_EV_CONNECT;
	else return false;
	o.svc_id = r.ser_glob_id_; o.flow_key = r.cli_task_aggr_id_;
	o.value = closed ? clamp32(r.bytes_sent_ + r.bytes_rcvd_) : 0;
	o.host_idx = host_idx; o.tsec = (uint32_t)((closed ? r.tusec_close_ : r.tusec_start_) / 1000000ull); o.flags = 0;
	return true;
}

// partha_aggr_task_state (gy_mconnhdlr.cc:9959) -> MAGGR_TASK::set_local_task_state (gy_msocket.h:1009)
inline bool decode_wire(const wire::AGGR_TASK_STATE_NOTIFY &r, uint32_t host_idx, gysk_event &o)
{
	if (!r.aggr_task_id_) return false;
	o.svc_id = r.aggr_task_id_;
	o.flow_key = (uint64_t)r.cpu_delay_msec_ | ((uint64_t)r.blkio_delay_msec_ << 32);
	o.value = (uint32_t)(int)r.total_cpu_pct_;				// (int)ptask->total_cpu_pct_ , gy_msocket.h:1014
	o.host_idx = host_idx; o.tsec = 0; o.type = GYSK_EV_TASK; o.flags = 0;
	return true;
}

// handle_partha_active_conns (gy_mconnhdlr.cc:7705) -> insert_active_conns (:7788): one record per {listener, client process}
inline bool decode_wire(const wire::ACTIVE_CONN_STATS &r, uint32_t host_idx, gysk_event &o)
{
	if (!r.listener_glob_id_) return false;
	o.svc_id = r.listener_glob_id_; o.flow_key = r.cli_aggr_task_id_;
	o.value = clamp32((r.bytes_sent_ + r.bytes_received_) >> 10);
	o.host_idx = host_idx;
	const float rtt = r.max_rtt_msec_ > 0 ? r.max_rtt_msec_ : 0.0f;
	memcpy(&o.tsec, &rtt, 4);
	o.type = GYSK_EV_ACTIVE; o.flags = r.active_conns_;
	return true;
}

// API_TRAN, common/gy_proto_common.h:140-204, read at the offsets of wire::API_TRAN_OFF.
// SVC_INFO_CAP::upd_stats_on_req (gy_proto_parser.cc:2678-2694): nrequests_++, resp_cache_.add_cache(response_usec_ / 1000),
// error counters. is_error / is_serv_err are the parser's verdict; the record carries errorcode_: != 0 is an error, >= 500 a
// server error (HTTP status convention of the reference's http parser).
struct ApiTran
{
	using O = wire::API_TRAN_OFF;
	const uint8_t *p;
	template <typename T> T at(size_t off) const { T v; memcpy(&v, p + off, sizeof(T)); return v; }
	size_t get_elem_size() const { return O::SIZE + at<uint16_t>(O::REQUEST_LEN) + at<uint16_t>(O::LENEXT) + p[O::PADLEN]; }
};
inline bool decode_wire(const ApiTran &r, uint32_t host_idx, gysk_event &o)
{
	using O = ApiTran::O;
	const int32_t err = r.at<int32_t>(O::ERRORCODE);
	o.svc_id = r.at<uint64_t>(O::GLOB_ID);
	o.flow_key = r.at<uint16_t>(O::CLIPORT);				// cliport_ (host order): CONN_BITMAP index
	o.value = clamp32(r.at<uint64_t>(O::RESPONSE_USEC));			// beyond 1 000 000 msec: dropped by the validity rule on the device
	o.host_idx = host_idx; o.tsec = (uint32_t)(r.at<uint64_t>(O::TUPD_USEC) / 1000000ull);
	o.type = GYSK_EV_RESP;
	o.flags = err == 0 ? 0 : (err >= 500 ? GYSK_EVF_SER_ERROR : GYSK_EVF_CLI_ERROR);
	return true;
}
// the record's GYSK_EV_TRACE (engines with trace rows): bytes in / out from reqlen_ / reslen_, a new connection when reqnum_ is 0
inline bool decode_trace(const ApiTran &r, uint32_t host_idx, gysk_event &o)
{
	using O = ApiTran::O;
	const int32_t err = r.at<int32_t>(O::ERRORCODE);
	o.svc_id = r.at<uint64_t>(O::GLOB_ID);
	o.flow_key = (uint64_t)clamp32(r.at<uint64_t>(O::REQLEN)) | ((uint64_t)clamp32(r.at<uint64_t>(O::RESLEN)) << 32);
	o.value = clamp32(r.at<uint64_t>(O::RESPONSE_USEC));
	o.host_idx = host_idx; o.tsec = (uint32_t)(r.at<uint64_t>(O::TUPD_USEC) / 1000000ull);
	o.type = GYSK_EV_TRACE;
	o.flags = (err != 0 ? GYSK_EVF_TRACE_ERROR : 0u) | (r.at<uint64_t>(O::REQNUM) == 0 ? GYSK_EVF_TRACE_NEWCONN : 0u);
	return true;
}

} // namespace gysk

namespace {

// the record walk of the partha_* handlers (partha_tcp_conn_info, gy_mconnhdlr.cc:9130): i < nevents && ptr < pendptr, stride
// get_elem_size(); a non-zero f(record) ends the walk and is returned
template <typename T, typename F>
int walk(const T *p, uint32_t n, const uint8_t *pend, F f)
{
	for (uint32_t i = 0; i < n && (const uint8_t *)p < pend; ++i, p = (const T *)((const uint8_t *)p + p->get_elem_size()))
		if (int rc = f(*p)) return rc;
	return 0;
}

// records expanded on the calling thread: decode(event) of each record, the events it keeps into the thread's stage in order
template <typename Decode>
inline int stage_record(gysk_engine *e, ThreadStage *ts, Decode decode)
{
	gysk_event ev;
	if (!decode(ev)) return 0;
	int rc = 0;
	if (gysk_event *o = stage_slot(e, ts, &rc)) *o = ev;
	return rc;
}

template <typename T>
int stage_walk(gysk_engine *e, ThreadStage *ts, const T *p, uint32_t n, const uint8_t *pend, uint32_t host_idx)
{
	return walk(p, n, pend, [&](const T &r) { return stage_record(e, ts, [&](gysk_event &o) { return decode_wire(r, host_idx, o); }); });
}

int wire_reject(gysk_engine *e, const char *what)
{
	e->wire_bad++;
	return fail(e, GYSK_ERR_INVAL, what);
}

// Bulk path of a fixed-stride raw kind: the raw bytes go H2D once per piece (straight from the caller's buffer when that is
// page-locked, else through the thread's chunk), and decode_raw_kernel expands them into the device event buffers. A piece holds
// at most one device buffer of events, so that each copy is followed by a batch as soon as it lands; it also fits one raw buffer
// and, from pageable memory, one thread chunk. It may straddle two device buffers.
int ingest_raw_bulk(gysk_engine *e, ThreadStage *ts, uint32_t kind, uint32_t host_idx, const uint8_t *src, uint64_t n)
{
	const uint32_t stride = raw_stride(kind);
	cudaPointerAttributes pa {};
	const bool pinned = cudaPointerGetAttributes(&pa, src) == cudaSuccess && pa.type == cudaMemoryTypeHost;
	cudaGetLastError();
	// Pageable input bounces through the thread's chunk: hand over what it holds first. Page-locked input does not touch the chunk,
	// so its records may reach the device ahead of records this thread staged before the call.
	int rc = pinned ? 0 : flush_stage(e, ts);
	if (rc) return rc;
	const uint64_t piece = std::min<uint64_t>(e->cfg.stage_batch, (pinned ? e->raw_bytes : (size_t)ts->cap * sizeof(gysk_event)) / stride);
	while (n) {
		const uint64_t m = std::min(piece, n);
		const uint8_t *hsrc = src;
		if (!pinned) {
			CU(e, cudaEventSynchronize(ts->copied[ts->cur]));		// this chunk's last copy has left the host
			memcpy(ts->buf[ts->cur], src, (size_t)m * stride);
			hsrc = reinterpret_cast<const uint8_t *>(ts->buf[ts->cur]);
		}
		std::lock_guard<std::mutex> lk(e->mtx);
		CU(e, cudaSetDevice(e->dev));
		const int r = e->raw_cur;
		CU(e, cudaStreamWaitEvent(e->copy_stream, e->ev_raw_done[r], 0));		// the decode kernels that last read raw buffer r have run
		CU(e, cudaMemcpyAsync(e->d_raw[r], hsrc, (size_t)m * stride, cudaMemcpyHostToDevice, e->copy_stream));
		if (!pinned) { CU(e, cudaEventRecord(ts->copied[ts->cur], e->copy_stream)); ts->cur ^= 1; }
		// the expansion runs on the copy stream too: a buffer's events are complete in copy-stream order, as append_chunk's are
		rc = place_events(e, m, [&](gysk_event *dst, uint64_t off, uint32_t k) {
			decode_raw_kernel<<<(k + 255) / 256, 256, 0, e->copy_stream>>>(kind, e->d_raw[r] + off * stride, k, host_idx, dst);
			e->kernel_launches++;
			return 0;
		});
		if (rc) return rc;
		CU(e, cudaEventRecord(e->ev_raw_done[r], e->copy_stream));
		e->raw_cur = (r + 1) % NBUF;
		src += m * stride; n -= m;
	}
	return post_launch(e, "raw decode");
}

} // namespace

extern "C" {

int gysk_ingest_raw(gysk_engine *e, const uint8_t host_id[16], uint32_t host_idx, uint32_t kind, const void *events, uint32_t n)
{
	CHECK_ENGINE(e);
	(void)host_id;
	if (!events && n) return GYSK_ERR_INVAL;
	ThreadStage *ts = get_stage(e);
	if (!ts) return fail(e, GYSK_ERR_NOMEM, "thread stage");
	std::lock_guard<std::mutex> tl(ts->m);
	const uint8_t *p = static_cast<const uint8_t *>(events);

	if (kind == GYSK_RAW_EVENT32) return stage_events(e, ts, static_cast<const gysk_event *>(events), n);
	if (kind == GYSK_RAW_API_TRAN) {
		const bool trace = e->cfg.max_trace_svcs != 0;
		for (ApiTran r {p}; n; --n, r.p += r.get_elem_size()) {
			if (int rc = stage_record(e, ts, [&](gysk_event &o) { return decode_wire(r, host_idx, o); })) return rc;
			if (trace) if (int rc = stage_record(e, ts, [&](gysk_event &o) { return decode_trace(r, host_idx, o); })) return rc;
		}
		return GYSK_OK;
	}
	const uint32_t stride = raw_stride(kind);
	if (!stride) return fail(e, GYSK_ERR_INVAL, "gysk_ingest_raw: unknown kind");
	if (n >= RAW_BULK_MIN) return ingest_raw_bulk(e, ts, kind, host_idx, p, n);
	// a handful of records (one perf-buffer wake-up): expanded by the calling thread, dropped records skipped
	for (; n; --n, p += stride)
		if (int rc = stage_record(e, ts, [&](gysk_event &o) { decode_raw(kind, p, host_idx, o); return o.type != 0xFFFF; })) return rc;
	return GYSK_OK;
}

// One wire message body, exactly the arguments handle_l2_misc hands to partha_<kind>() (gy_mconnhdlr.cc:4745-4800).
int gysk_ingest(gysk_engine *e, const uint8_t host_id[16], uint32_t host_idx, uint32_t subtype, void *recs, uint32_t nevents, const void *endptr)
{
	CHECK_ENGINE(e);
	(void)host_id;
	if (!recs || !endptr || (const uint8_t *)endptr < (const uint8_t *)recs) return GYSK_ERR_INVAL;
	ThreadStage *ts = get_stage(e);
	if (!ts) return fail(e, GYSK_ERR_NOMEM, "thread stage");
	std::lock_guard<std::mutex> tl(ts->m);
	const uint8_t *pend = static_cast<const uint8_t *>(endptr);
	int rc = 0;

	switch (subtype) {

	case GYSK_NOTIFY_TCP_CONN : {
		using T = wire::TCP_CONN_NOTIFY;
		T *pone = static_cast<T *>(recs);
		if (!wire::validate_batch<T>(pone, nevents, pend, T::MAX_NUM_CONNS, [](const T & t) -> size_t { return t.cli_cmdline_len_; }))
			return wire_reject(e, "TCP_CONN_NOTIFY::validate failed");
		rc = stage_walk(e, ts, pone, nevents, pend, host_idx);
		break;
	}

	case GYSK_NOTIFY_AGGR_TASK_STATE : {
		using T = wire::AGGR_TASK_STATE_NOTIFY;
		T *pone = static_cast<T *>(recs);
		if (!wire::validate_batch<T>(pone, nevents, pend, T::MAX_NUM_TASKS, [](const T & t) -> size_t { return t.issue_string_len_; }))
			return wire_reject(e, "AGGR_TASK_STATE_NOTIFY::validate failed");
		HostTaskTopn tt;						// the seven per-host rankings of :10012-10079
		walk(pone, nevents, pend, [&](const T &t) { tt.offer(t); return 0; });
		{
			std::lock_guard<std::mutex> lk(e->host_mtx);
			e->host_task_topn[host_idx] = std::move(tt);
		}
		rc = stage_walk(e, ts, pone, nevents, pend, host_idx);
		break;
	}

	case GYSK_NOTIFY_ACTIVE_CONN_STATS : {
		// ACTIVE_CONN_STATS::validate (common/gy_comm_proto.h:2806): fixed stride, nevents <= MAX_NUM_CONNS, all records inside the message
		using T = wire::ACTIVE_CONN_STATS;
		const T *pone = static_cast<const T *>(recs);
		if (nevents > T::MAX_NUM_CONNS || (const uint8_t *)(pone + nevents) > pend) return wire_reject(e, "ACTIVE_CONN_STATS::validate failed");
		rc = stage_walk(e, ts, pone, nevents, pend, host_idx);
		break;
	}

	case GYSK_NOTIFY_LISTENER_STATE : {
		using T = wire::LISTENER_STATE_NOTIFY;
		T *pone = static_cast<T *>(recs);
		if (!wire::validate_batch<T>(pone, nevents, pend, T::MAX_NUM_LISTENERS, [](const T & t) -> size_t { return t.issue_string_len_; }))
			return wire_reject(e, "LISTENER_STATE_NOTIFY::validate failed");
		// Pre-aggregated 5-s listener state. With the per-sample reduction lifted onto the GPU the per-listener fields are
		// derived by the engine itself; what these records still feed is the per-host roll-up of partha_listener_state
		// (gy_mconnhdlr.cc:11175-11251): summstats.update(*pone) per record == LISTEN_SUMM_STATS::update, gy_msocket.h:854-866,
		// and the per-host top-N queues (:11262-11304). <= 512 records per host per 5 s: host-side integer work.
		gysk_host_summary hs;
		memset(&hs, 0, sizeof(hs));
		HostTopn topn;
		walk(pone, nevents, pend, [&](const T &l) {
			// gy_mconnhdlr.cc:11183-11251: LISTEN_FLAG_DELETE records only delete the listener, records with
			// curr_state_ > STATE_DOWN count as errors; neither reaches summstats.update()
			if (l.query_flags_ == wire::LISTEN_FLAG_DELETE || l.curr_state_ > wire::STATE_DOWN) return 0;
			hs.nstates[l.curr_state_]++;
			hs.tot_qps += (int32_t)(l.nqrys_5s_ / 5);
			hs.tot_act_conn += (int32_t)l.nconns_active_;
			hs.tot_kb_inbound += (int32_t)l.curr_kbytes_inbound_;
			hs.tot_kb_outbound += (int32_t)l.curr_kbytes_outbound_;
			hs.tot_ser_errors += (int32_t)l.ser_errors_;
			hs.nlisteners++;
			hs.nactive += !!l.nqrys_5s_;
			topn.offer(l);
			return 0;
		});
		std::lock_guard<std::mutex> lk(e->host_mtx);
		e->host_summ[host_idx] = hs;
		e->host_topn[host_idx] = topn;
		break;
	}

	default :
		return fail(e, GYSK_ERR_NOTSUP, "gysk_ingest: subtype not on the hot path");
	}
	if (rc) return rc;
	e->wire_ok++;
	return GYSK_OK;
}

// Whole message: COMM_HEADER + EVENT_NOTIFY + records, the pointer arithmetic of handle_l2_misc (gy_mconnhdlr.cc:4745-4760)
int gysk_ingest_msg(gysk_engine *e, const uint8_t host_id[16], uint32_t host_idx, void *msg, uint32_t msglen)
{
	CHECK_ENGINE(e);
	if (!msg || msglen < sizeof(wire::COMM_HEADER) + sizeof(wire::EVENT_NOTIFY)) return GYSK_ERR_INVAL;
	wire::COMM_HEADER *phdr = static_cast<wire::COMM_HEADER *>(msg);

	if (phdr->magic_ != wire::PM_HDR_MAGIC || phdr->data_type_ != wire::COMM_EVENT_NOTIFY || phdr->total_sz_ > msglen ||
			phdr->total_sz_ >= wire::MAX_COMM_DATA_SZ || phdr->padding_sz_ > phdr->total_sz_ ||
			phdr->get_act_len() < sizeof(wire::COMM_HEADER) + sizeof(wire::EVENT_NOTIFY))
		return wire_reject(e, "COMM_HEADER::validate failed");
	uint8_t *pendptr = static_cast<uint8_t *>(msg) + phdr->get_act_len();
	wire::EVENT_NOTIFY *pevtnot = reinterpret_cast<wire::EVENT_NOTIFY *>(phdr + 1);

	return gysk_ingest(e, host_id, host_idx, pevtnot->subtype_, pevtnot + 1, pevtnot->nevents_, pendptr);
}

int gysk_sync(gysk_engine *e)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Sync);
	return GYSK_OK;
}

} // extern "C"

// ---- capacity growth ------------------------------------------------------------------------------------------------
namespace {

// bytes of device buffer p (0: none)
size_t dsize(const gysk_engine *e, const void *p)
{
	for (const auto &a : e->dallocs) if (a.first == p) return a.second;
	return 0;
}

// the copies of the slot -> id / host arrays an IdTable carries
void link_tables(DevState &st)
{
	st.svc_tbl.slot_id = st.slot_id; st.svc_tbl.slot_host = st.slot_host;
	st.task_tbl.slot_id = st.task_slot_id; st.task_tbl.slot_host = st.task_slot_host;
}

// Moves one device array whose first old_n elements are valid into a new one of new_n: the prefix copied, the tail zeroed, the old
// array freed before the caller moves on to the next one (the peak is the new footprint plus the largest old array). An array that
// already holds new_n elements (moved by an earlier growth that stopped half way; its tail is still zero: nothing at the old capacity
// writes there) stays. A failed allocation leaves p as it was. Stream synchronised on return.
template <typename T>
int regrow(gysk_engine *e, T *&p, size_t old_n, size_t new_n)
{
	if (dsize(e, p) >= new_n * sizeof(T)) return 0;
	T *q = nullptr;
	if (int rc = dalloc(e, &q, new_n, false)) return rc;
	if (old_n) CU(e, cudaMemcpyAsync(q, p, old_n * sizeof(T), cudaMemcpyDeviceToDevice, e->stream));
	CU(e, cudaMemsetAsync(q + old_n, 0, (new_n - old_n) * sizeof(T), e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	dfree(e, p);
	p = q;
	return 0;
}

// The level ring [NLEVELS][NSLOTS][stride][16] at the stride new_ms: each of its NLEVELS x NSLOTS planes (stride rows, contiguous)
// moves with one copy to the head of its new plane, the rows behind it zeroed. The source pitch is the ring's own stride, which an
// earlier growth that stopped half way may already have raised.
int regrow_ring(gysk_engine *e, uint32_t new_ms)
{
	LevelRing &lv = e->st.levels;
	if (lv.stride >= new_ms) return 0;
	const size_t row = (size_t)HIST_CELLS * sizeof(HistCell), planes = (size_t)NLEVELS * NSLOTS;
	HistCell *q = nullptr;
	if (int rc = dalloc(e, &q, planes * new_ms * HIST_CELLS)) return rc;
	for (size_t k = 0; k < planes; ++k)
		CU(e, cudaMemcpyAsync(q + k * new_ms * HIST_CELLS, lv.ring + k * lv.stride * HIST_CELLS, lv.stride * row, cudaMemcpyDeviceToDevice, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	dfree(e, lv.ring);
	lv.ring = q;
	lv.stride = new_ms;
	return 0;
}

// The device bytes gysk_grow adds to the engine going from cfg to (ms, mt), the largest array it frees on the way (held beside the
// new one while it is copied), and the allocations it makes (each may be rounded up to the allocator's 2 MiB granularity)
void grow_bytes(const gysk_engine *e, uint32_t ms, uint32_t mt, size_t *add, size_t *largest_old, size_t *nalloc)
{
	const gysk_config &cfg = e->cfg;
	gysk_config to = cfg;
	to.max_svcs = ms; to.max_tasks = mt;
	DevState st {};
	SortTemp tmp {};
	size_t a = 0, big = 0, n = 0;
	auto move = [&](size_t elem, size_t old_n, size_t new_n) {
		if (new_n <= old_n) return;
		a += (new_n - old_n) * elem;
		big = std::max(big, old_n * elem);
		n++;
	};
	each_slot_array(st, tmp, cfg.hll_p, cfg.task_idle_evict_secs, [&](auto *&p, size_t k, SlotKind kind) {
		move(k * sizeof(*p), slots_of(kind, cfg.max_svcs, cfg.max_tasks, cfg.max_trace_svcs), slots_of(kind, ms, mt, cfg.max_trace_svcs));
	});
	if (cfg.max_trace_svcs) move(sizeof(uint32_t), (size_t)cfg.max_svcs + 1, (size_t)ms + 1);		// TraceTable::row_of
	if (ms != cfg.max_svcs) move(sizeof(TblEntry), table_cap(cfg.max_svcs + 1), table_cap(ms + 1));
	if (mt != cfg.max_tasks) move(sizeof(TblEntry), table_cap(cfg.max_tasks), table_cap(mt));
	const size_t k0 = sort_keys(cfg), k1 = sort_keys(to);
	move(sizeof(unsigned long long), k0, k1); move(sizeof(unsigned long long), k0, k1);
	move((size_t)RADIX_MAX * sizeof(unsigned long long), sort_tiles(k0), sort_tiles(k1));
	move(sizeof(uint32_t), batch_rows(cfg), batch_rows(to)); move((size_t)HOT_ROW_WORDS * sizeof(unsigned long long), batch_rows(cfg), batch_rows(to));
	*add = a; *largest_old = big; *nalloc = n;
}

// gysk_grow, engine held and both streams idle.
// Phase 1 moves the per-slot arrays, the sort buffers and the batch rows one by one. The engine stays at its old capacity throughout:
// a moved array is only longer, its valid prefix unchanged and its tail zero, and the IdTable copies of the slot arrays follow each
// move. A cudaMalloc that fails there (the pre-check passed, but another tenant of the device took the memory since) ends the growth
// with GYSK_ERR_NOMEM and an engine that answers as before at its old capacity; a later gysk_grow finds the arrays already moved.
// Phase 2 allocates the new id tables and the eviction buffer while the old ones still serve (a failure: the same). Phase 3 commits
// the new capacity and allocates nothing.
int grow_locked(gysk_engine *e, uint32_t ms, uint32_t mt)
{
	gysk_config &cfg = e->cfg;
	if (ms < cfg.max_svcs || mt < cfg.max_tasks || ms > (1u << 24) || mt > (1u << 24)) return fail(e, GYSK_ERR_INVAL, "gysk_grow: shrink or beyond 1 << 24");
	if (!trace_fits(ms, cfg.max_trace_svcs)) return fail(e, GYSK_ERR_INVAL, "gysk_grow: max_svcs + 1 + max_trace_svcs beyond 1 << 24");
	if (ms == cfg.max_svcs && mt == cfg.max_tasks) return GYSK_OK;
	size_t add = 0, big = 0, nalloc = 0, nfree = 0, ntotal = 0;
	grow_bytes(e, ms, mt, &add, &big, &nalloc);
	CU(e, cudaMemGetInfo(&nfree, &ntotal));
	if (add + big + nalloc * (2u << 20) > nfree) return fail(e, GYSK_ERR_NOMEM, "gysk_grow: the new arrays do not fit the device's free memory");

	if (int rc = collect_evicted(e)) return rc;		// h_evict moves: nothing may still be on its way into it
	const uint32_t os = cfg.max_svcs, ot = cfg.max_tasks;
	DevState &st = e->st;
	SortTemp &tmp = e->tmp;
	gysk_config to = cfg;
	to.max_svcs = ms; to.max_tasks = mt;
	int rc = 0;
	// phase 1
	each_slot_array(st, tmp, cfg.hll_p, cfg.task_idle_evict_secs, [&](auto *&p, size_t k, SlotKind kind) {
		if (rc) return;
		if (kind == SlotKind::Ring) rc = regrow_ring(e, ms);
		else rc = regrow(e, p, slots_of(kind, os, ot, cfg.max_trace_svcs) * k, slots_of(kind, ms, mt, cfg.max_trace_svcs) * k);
		link_tables(st);
	});
	if (!rc && st.trace.rows) rc = regrow(e, st.trace.row_of, (size_t)os + 1, (size_t)ms + 1);
	const size_t k0 = sort_keys(cfg), k1 = sort_keys(to), b0 = batch_rows(cfg), b1 = batch_rows(to);
	if (!rc && !(rc = regrow(e, tmp.keys_a, k0, k1)) && !(rc = regrow(e, tmp.keys_b, k0, k1)) &&
			!(rc = regrow(e, tmp.tile_status, (size_t)RADIX_MAX * sort_tiles(k0), (size_t)RADIX_MAX * sort_tiles(k1)))) {
		tmp.nkeys = std::max(tmp.nkeys, k1); tmp.max_tiles = std::max(tmp.max_tiles, sort_tiles(k1));
	}
	if (!rc && !(rc = regrow(e, tmp.long_slot, b0, b1))) rc = regrow(e, tmp.batch_rows, b0 * HOT_ROW_WORDS, b1 * HOT_ROW_WORDS);
	if (rc) return rc;
	// phase 2
	TblEntry *sent = nullptr, *tent = nullptr;
	unsigned long long *hev = nullptr, *htev = nullptr, *dtev = nullptr;
	if ((ms != os && (rc = dalloc(e, &sent, table_cap(ms + 1), false))) || (mt != ot && (rc = dalloc(e, &tent, table_cap(mt), false))) ||
			(ms != os && (rc = halloc(e, &hev, (size_t)ms + 3))) ||
			(mt != ot && e->h_tevict && (rc = halloc(e, &htev, (size_t)mt + 1, cudaHostAllocMapped)))) {
		dfree(e, sent); dfree(e, tent); hfree(e, hev);
		return rc;
	}
	if (htev) {
		const cudaError_t ce = cudaHostGetDevicePointer((void **)&dtev, htev, 0);
		if (ce != cudaSuccess) { dfree(e, sent); dfree(e, tent); hfree(e, hev); hfree(e, htev); return fail(e, GYSK_ERR_CUDA, "cudaHostGetDevicePointer", ce); }
	}
	// phase 3: the old null slot and every new slot in their just-created state (the new null slot is the last one), then both id
	// tables rebuilt at their new capacity: slot numbers, hot rows (SlotBatch::hot of the slot) and the free stack stay. A rebuild
	// also drops tombstones and the dead entries of lost insert races, as gysk_flush's does.
	cfg = to;
	e->kernel_launches += launch_init_slots(st, os, ms + 1, ot, mt, e->stream);
	auto swap_table = [&](IdTable &t, TblEntry *ent, uint32_t slots, uint32_t max_slots) {
		TblEntry *old = t.ent;
		t.ent = ent; t.mask = table_cap(slots) - 1; t.max_slots = max_slots;
		e->kernel_launches += launch_rebuild_table(t, max_slots, e->stream);
		dfree(e, old);
	};
	if (ms != os) {
		hev[0] = 0; hev[ms + 1] = e->h_evict[os + 1];		// the insert-fail word of h_evict sits at [max_svcs + 1]
		hfree(e, e->h_evict);
		e->h_evict = hev;
		swap_table(st.svc_tbl, sent, ms + 1, ms);
		unsigned long long fails = 0;
		CU(e, cudaMemcpyAsync(&fails, st.counters + CTR_INSERT_FAIL, sizeof(fails), cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaStreamSynchronize(e->stream));
		e->tombstones = 0; e->insert_fail_seen = fails;
	}
	if (mt != ot) {
		if (htev) {
			htev[0] = 0;
			hfree(e, e->h_tevict);
			e->h_tevict = htev; e->d_tevict = dtev;
		}
		swap_table(st.task_tbl, tent, mt, mt);
		e->task_tombstones = 0;
	}
	e->mg.members.null_slot = ms;			// the member slots are resolved again at every gysk_merge_prepare
	if (st.trace.rows) st.trace.base = ms + 1;	// the pseudo-slots of the next batch's trace keys
	e->ngrows++;
	CU(e, cudaStreamSynchronize(e->stream));
	return post_launch(e, "grow");
}

// Auto-grow at gysk_flush: each table whose slots in use as of the previous flush reached half its capacity doubles, up to its
// limit. The counts were copied behind that flush's kernels, a window ago: the event wait finds them long landed.
int auto_grow(gysk_engine *e)
{
	if (!e->used_pending) return 0;
	CU(e, cudaEventSynchronize(e->ev_used));
	e->used_pending = false;
	const uint32_t ms = e->cfg.max_svcs, mt = e->cfg.max_tasks;
	const uint64_t svcs = (uint64_t)std::min(e->h_used[0], ms) - (uint64_t)std::max((int32_t)e->h_used[1], 0);
	const uint64_t tasks = (uint64_t)std::min(e->h_used[2], mt) - (uint64_t)std::max((int32_t)e->h_used[3], 0);
	auto next = [](uint32_t cap, uint64_t used, uint32_t limit) {
		return limit > cap && 2 * used >= cap ? (uint32_t)std::min<uint64_t>(2ull * cap, limit) : cap;
	};
	const uint32_t ns = next(ms, svcs, e->grow_limit_svcs), nt = next(mt, tasks, e->grow_limit_tasks);
	if (ns == ms && nt == mt) return 0;
	if (int rc = sync_locked(e)) return rc;
	// GYSK_ERR_NOMEM leaves the engine as it was at its capacity (grow_locked): the flush goes on there, and the next one tries again
	const int rc = grow_locked(e, ns, nt);
	return rc == GYSK_ERR_NOMEM ? 0 : rc;
}

} // namespace

extern "C" {

int gysk_grow(gysk_engine *e, uint32_t max_svcs, uint32_t max_tasks)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Sync);
	return grow_locked(e, max_svcs, max_tasks);
}

int gysk_set_auto_grow(gysk_engine *e, uint32_t max_svcs_limit, uint32_t max_tasks_limit)
{
	CHECK_ENGINE(e);
	if (max_svcs_limit > (1u << 24) || max_tasks_limit > (1u << 24)) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	e->grow_limit_svcs = max_svcs_limit; e->grow_limit_tasks = max_tasks_limit;
	return GYSK_OK;
}

int gysk_capacity_info(gysk_engine *e, gysk_capacity *out)
{
	CHECK_ENGINE(e);
	if (!out) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Sync);
	uint32_t cnt[2] = {0, 0};
	int32_t nfree = 0, tfree = 0;
	CU(e, cudaMemcpy(&cnt[0], e->st.svc_tbl.count, sizeof(uint32_t), cudaMemcpyDeviceToHost));
	CU(e, cudaMemcpy(&cnt[1], e->st.task_tbl.count, sizeof(uint32_t), cudaMemcpyDeviceToHost));
	CU(e, cudaMemcpy(&nfree, e->st.svc_tbl.free_n, sizeof(nfree), cudaMemcpyDeviceToHost));
	if (e->st.task_tbl.free_n) CU(e, cudaMemcpy(&tfree, e->st.task_tbl.free_n, sizeof(tfree), cudaMemcpyDeviceToHost));
	memset(out, 0, sizeof(*out));
	out->max_svcs = e->cfg.max_svcs; out->max_tasks = e->cfg.max_tasks;
	out->svcs_in_use = std::min(cnt[0], e->cfg.max_svcs) - (uint32_t)std::max(nfree, 0);
	out->tasks_in_use = std::min(cnt[1], e->cfg.max_tasks) - (uint32_t)std::max(tfree, 0);
	out->ngrows = e->ngrows;
	out->device_bytes = e->dbytes;
	return GYSK_OK;
}

int gysk_slot_bytes(const gysk_config *cfg, uint64_t *svc_slot_bytes, uint64_t *task_slot_bytes)
{
	if (!svc_slot_bytes || !task_slot_bytes) return GYSK_ERR_INVAL;
	gysk_config c;
	gysk_config_default(&c);
	if (cfg) {
		if (cfg->struct_size != sizeof(gysk_config)) return GYSK_ERR_INVAL;
		c = *cfg;
	}
	if (c.hll_p < 4 || c.hll_p > 16) return GYSK_ERR_INVAL;
	slot_bytes(c.hll_p, c.task_idle_evict_secs != 0, svc_slot_bytes, task_slot_bytes);
	return GYSK_OK;
}

int gysk_flush(gysk_engine *e, uint32_t tsec)
{
	CHECK_ENGINE(e);
	GYSK_ENTER(e, Submit);

	if (int rc = auto_grow(e)) return rc;
	if (int rc = roll_levels(e, tsec)) return rc;
	e->last_flush_tsec = tsec;

	if (int rc = collect_evicted(e)) return rc;		// list of the previous flush (normally long complete)
	// tombstones lengthen probe chains: once they fill an eighth of the table, rebuild it from the live slots
	const uint64_t dead = e->h_evict_fail > e->insert_fail_seen ? e->h_evict_fail - e->insert_fail_seen : 0;
	if (e->tombstones + dead > ((uint64_t)e->st.svc_tbl.mask + 1) / 8) {
		e->kernel_launches += launch_rebuild_table(e->st.svc_tbl, e->cfg.max_svcs, e->stream);
		e->tombstones = 0; e->insert_fail_seen = e->h_evict_fail;
	}
	if (e->task_tombstones > ((uint64_t)e->st.task_tbl.mask + 1) / 8) {		// the same for the process table
		e->kernel_launches += launch_rebuild_table(e->st.task_tbl, e->cfg.max_tasks, e->stream);
		e->task_tombstones = 0;
	}
	e->kernel_launches += launch_flush(e->st, e->cfg.max_svcs, tsec, e->cfg.idle_evict_secs, e->stream);
	e->kernel_launches += launch_task_flush(e->st, e->cfg.max_tasks, tsec, e->cfg.task_idle_evict_secs, e->d_tevict, e->stream);
	if (e->st.trace.rows) {
		// trace rows: the open window closes, the other half (the window before it) is cleared and opens
		const uint32_t open = e->st.trace.par ^ 1u;
		e->kernel_launches += launch_trace_roll(e->st, open, e->st.trace.rows, e->stream);
		e->st.trace.par = open;
	}
	if (e->grow_limit_svcs > e->cfg.max_svcs || e->grow_limit_tasks > e->cfg.max_tasks) {
		// auto-grow: the slot counts travel to the host behind the kernels, for the next flush's decision
		CU(e, cudaMemcpyAsync(e->h_used, e->st.svc_tbl.count, sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaMemcpyAsync(e->h_used + 1, e->st.svc_tbl.free_n, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaMemcpyAsync(e->h_used + 2, e->st.task_tbl.count, sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
		if (e->st.task_tbl.free_n) CU(e, cudaMemcpyAsync(e->h_used + 3, e->st.task_tbl.free_n, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaEventRecord(e->ev_used, e->stream));
		e->used_pending = true;
	}
	if (e->cfg.idle_evict_secs) {
		// count + ids travel to the host behind the kernels; nobody waits for them here
		CU(e, cudaMemcpyAsync(e->h_evict, e->st.counters + CTR_NEVICT, sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaMemcpyAsync(e->h_evict + e->cfg.max_svcs + 1, e->st.counters + CTR_INSERT_FAIL, sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaMemcpyAsync(e->h_evict + 1, e->st.evict_ids, (size_t)e->cfg.max_svcs * sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
	}
	if (e->cfg.idle_evict_secs || e->cfg.task_idle_evict_secs) {		// the process list is written to h_tevict by its eviction kernel
		CU(e, cudaEventRecord(e->ev_evict, e->stream));
		e->evict_pending = true;
	}
	if (e->st.cms_ring) e->kernel_launches += launch_cms_level_roll(e->st, e->stream);		// GYSK_FLAG_FLOW_LEVEL
	std::swap(e->st.cms_cur, e->st.cms_last);
	CU(e, cudaMemsetAsync(e->st.cms_cur, 0, sizeof(unsigned long long) * ((size_t)e->cfg.cms_depth << e->cfg.cms_log2_width), e->stream));
	return post_launch(e, "flush");
}

int gysk_evicted_ids(gysk_engine *e, uint64_t *out, uint32_t cap, uint32_t *n)
{
	CHECK_ENGINE(e);
	if (!n || (!out && cap)) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	if (int rc = collect_evicted(e)) return rc;
	*n = (uint32_t)e->evicted_ids.size();
	for (uint32_t i = 0; i < *n && i < cap; ++i) out[i] = e->evicted_ids[i];
	return GYSK_OK;
}

int gysk_evicted_task_ids(gysk_engine *e, uint64_t *out, uint32_t cap, uint32_t *n)
{
	CHECK_ENGINE(e);
	if (!n || (!out && cap)) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	if (int rc = collect_evicted(e)) return rc;
	*n = (uint32_t)e->evicted_task_ids.size();
	for (uint32_t i = 0; i < *n && i < cap; ++i) out[i] = e->evicted_task_ids[i];
	return GYSK_OK;
}

int gysk_task_evict_count(gysk_engine *e, uint64_t *total)
{
	CHECK_ENGINE(e);
	if (!total) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Drain);
	if (int rc = collect_evicted(e)) return rc;
	*total = e->task_evicted_total;
	return GYSK_OK;
}

} // extern "C"

// ---- queries ------------------------------------------------------------------------------------------------

namespace {

// the device half of a window read: the listed keys {host | slot} of the selection (seen_before: see launch_window_list), host-sorted
// with `order`, at *d_keys (their ids at *d_ids); *n of them
int list_slots(gysk_engine *e, int is_task, int32_t host_idx, uint32_t flags, uint32_t seen_before, bool order, const unsigned long long **d_keys,
		const unsigned long long **d_ids, uint32_t *n)
{
	uint32_t nslots = 0;
	CU(e, cudaMemcpyAsync(&nslots, is_task ? e->st.task_tbl.count : e->st.svc_tbl.count, sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	nslots = std::min(nslots, is_task ? e->cfg.max_tasks : e->cfg.max_svcs);
	unsigned long long *d_n = e->st.counters + CTR_NWINDOW;
	const int nl = launch_window_list(e->st, e->tmp, nslots, is_task, host_idx, flags & GYSK_WINDOW_ACTIVE_ONLY, active_mark(e), seen_before, d_n, order,
			d_keys, d_ids, e->stream);
	if (nl < 0) return fail(e, GYSK_ERR_INVAL, "window read: sort failed");
	e->kernel_launches += nl;
	unsigned long long cnt = 0;
	CU(e, cudaMemcpyAsync(&cnt, d_n, sizeof(cnt), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	*n = (uint32_t)cnt;
	return post_launch(e, "window list");
}

// The slots a window read returns, in its order, at tmp.keys_a[0 .. want): the live slots of the selection grouped by host (a stable
// radix sort of {host | slot} keys on the device), then by id inside each host (on the host: slot numbers depend on insertion races,
// the order must not). *n = rows that match. Stream synchronised by the caller.
int window_list(gysk_engine *e, int is_task, int32_t host_idx, uint32_t flags, uint32_t seen_before, uint32_t want, uint32_t *n)
{
	const unsigned long long *d_keys = nullptr, *d_ids = nullptr;
	int rc = list_slots(e, is_task, host_idx, flags, seen_before, want > 0, &d_keys, &d_ids, n);
	if (rc) return rc;
	const uint32_t cnt = *n;
	if (!want || !cnt) return 0;

	std::vector<uint64_t> &keys = e->win_keys, &ids = e->win_ids;
	keys.resize(cnt); ids.resize(cnt);
	CU(e, cudaMemcpyAsync(keys.data(), d_keys, cnt * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaMemcpyAsync(ids.data(), d_ids, cnt * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	// within a host, by id (ids are unique)
	std::vector<std::pair<uint64_t, uint64_t>> &rows = e->win_rows;
	rows.resize(cnt);
	for (size_t i = 0; i < cnt; ++i) rows[i] = {ids[i], keys[i] & 0xFFFFFFFFull};
	for (size_t a = 0; a < cnt && a < want; ) {
		size_t b = a + 1;
		while (b < cnt && (keys[b] >> 32) == (keys[a] >> 32)) ++b;
		std::sort(rows.begin() + a, rows.begin() + b);
		a = b;
	}
	for (size_t i = 0; i < cnt && i < want; ++i) ids[i] = rows[i].second;
	CU(e, cudaMemcpyAsync(e->tmp.keys_a, ids.data(), (size_t)std::min<uint64_t>(want, cnt) * sizeof(uint64_t), cudaMemcpyHostToDevice, e->stream));
	return 0;
}

// gysk_query_svcs / gysk_query_tasks: the rows of n ids, in QCHUNK pieces
template <typename Row>
int query_rows(gysk_engine *e, const uint64_t *ids, uint32_t n, Row *out, const char *what)
{
	CHECK_ENGINE(e);
	if ((!ids || !out) && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);
	return staged_read(e, ids, n, QCHUNK, sizeof(Row), what,
			[&](const unsigned long long *d_ids, uint32_t, uint32_t m) { return launch_rows(e, d_ids, nullptr, m, out); }, finish_rows(e, out));
}

// gysk_query_window_hosts / gysk_query_task_window: the slots of window_list, summarised in WIN_ROWS pieces; hosts (optional) from
// the same snapshot
template <typename Row>
int window_rows(gysk_engine *e, int32_t host_idx, uint32_t flags, Row *out, uint32_t *hosts, uint32_t cap, uint32_t *n, const char *what)
{
	CHECK_ENGINE(e);
	if (!n || (!out && cap) || (flags & ~GYSK_WINDOW_ACTIVE_ONLY)) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Sync);
	// day stats: only services first seen more than 15 minutes before the last flush (tcur > tstart + 15 * 60, gy_socket_stat.cc:2102)
	const uint32_t seen_before = !std::is_same<Row, gysk_listener_day_stats>::value ? ~0u : e->last_flush_tsec > 900u ? e->last_flush_tsec - 900u : 0u;
	uint32_t total = 0;
	int rc = window_list(e, std::is_same<Row, gysk_task_summary>::value, host_idx, flags, seen_before, cap, &total);
	if (rc) return rc;
	const uint32_t m = std::min(cap, total);
	rc = staged_read<uint64_t>(e, nullptr, m, WIN_ROWS, sizeof(Row), what,
			[&](const unsigned long long *, uint32_t off, uint32_t k) { return launch_rows(e, nullptr, e->tmp.keys_a + off, k, out); }, finish_rows(e, out));
	if (rc) return rc;
	// the within-host reorder of window_list leaves every position in its host's run
	if (hosts) for (uint32_t i = 0; i < m; ++i) hosts[i] = (uint32_t)(e->win_keys[i] >> 32);
	*n = total;
	return GYSK_OK;
}

// gysk_topn_svcs / gysk_topn_tasks: the n best of nslots by one metric, the non-zero entries kept
int topn_rows(gysk_engine *e, int is_task, int metric, int32_t host_idx, uint32_t n, gysk_topn_entry *out, uint32_t *nout, const char *what)
{
	GYSK_ENTER(e, Sync);
	uint32_t nslots = 0;
	CU(e, cudaMemcpy(&nslots, is_task ? e->st.task_tbl.count : e->st.svc_tbl.count, sizeof(uint32_t), cudaMemcpyDeviceToHost));
	nslots = std::min(nslots, is_task ? e->cfg.max_tasks : e->cfg.max_svcs);
	gysk_topn_entry *d_out = reinterpret_cast<gysk_topn_entry *>(e->d_wstage);
	const gysk_topn_entry *h_out = reinterpret_cast<const gysk_topn_entry *>(e->h_wstage);
	CU(e, cudaMemsetAsync(d_out, 0, sizeof(gysk_topn_entry) * n, e->stream));
	const int nl = launch_topn(e->st, e->tmp, nslots, is_task, metric, host_idx, n, d_out, e->stream);
	if (nl < 0) return fail(e, GYSK_ERR_INVAL, (std::string(what) + ": sort failed").c_str());
	e->kernel_launches += nl;
	CU(e, cudaMemcpyAsync(e->h_wstage, d_out, sizeof(gysk_topn_entry) * n, cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	if (int rc = post_launch(e, what)) return rc;
	uint32_t k = 0;
	for (uint32_t i = 0; i < n; ++i) if (h_out[i].glob_id && h_out[i].score) out[k++] = h_out[i];
	*nout = k;
	return GYSK_OK;
}

} // namespace

extern "C" {

int gysk_query_svcs(gysk_engine *e, const uint64_t *ids, uint32_t n, gysk_svc_summary *out)
{
	return query_rows(e, ids, n, out, "svc_summaries");
}

int gysk_query_window(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_svc_summary *out, uint32_t cap, uint32_t *n)
{
	return gysk_query_window_hosts(e, host_idx, flags, out, nullptr, cap, n);
}

int gysk_query_window_hosts(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_svc_summary *out, uint32_t *hosts, uint32_t cap, uint32_t *n)
{
	return window_rows(e, host_idx, flags, out, hosts, cap, n, "query_window");
}

int gysk_query_day_stats(gysk_engine *e, int32_t host_idx, gysk_listener_day_stats *out, uint32_t *hosts, uint32_t cap, uint32_t *n)
{
	return window_rows(e, host_idx, 0, out, hosts, cap, n, "day_stats");
}

// the host-sorted keys of every live service, the per-run counts beside them in the other sort buffer, then the host rows in stage-sized
// pieces by rank
int gysk_query_host_listen(gysk_engine *e, gysk_host_listen *out, uint32_t cap, uint32_t *n)
{
	CHECK_ENGINE(e);
	if (!n || (!out && cap)) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Sync);
	const unsigned long long *d_keys = nullptr, *d_ids = nullptr;
	uint32_t nkeys = 0;
	int rc = list_slots(e, 0, -1, 0, ~0u, true, &d_keys, &d_ids, &nkeys);
	if (rc) return rc;
	if (!nkeys) { *n = 0; return GYSK_OK; }
	unsigned long long *acc = const_cast<unsigned long long *>(d_ids), *d_rows = e->st.counters + CTR_NHOSTS;
	const unsigned long long *d_n = e->st.counters + CTR_NWINDOW;
	gysk_host_listen *d_out = reinterpret_cast<gysk_host_listen *>(e->d_wstage);
	constexpr uint32_t piece = (uint32_t)(STAGE_BYTES / sizeof(gysk_host_listen));
	e->kernel_launches += launch_host_listen_count(e->st, d_keys, d_n, nkeys, active_mark(e), acc, e->stream);
	e->kernel_launches += launch_host_listen_rows(d_keys, d_n, acc, 0, std::min(cap, piece), d_out, d_rows, e->stream);
	unsigned long long nrows = 0;
	CU(e, cudaMemcpyAsync(&nrows, d_rows, sizeof(nrows), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	if ((rc = post_launch(e, "host_listen"))) return rc;
	*n = (uint32_t)nrows;
	// the first piece is in the stage already; more than `piece` hosts take one more pass over the keys per piece
	return staged_read<uint64_t>(e, nullptr, std::min(cap, *n), piece, sizeof(gysk_host_listen), "host_listen",
			[&](const unsigned long long *, uint32_t off, uint32_t m) {
				return off ? launch_host_listen_rows(d_keys, d_n, acc, off, m, d_out, d_rows, e->stream) : 0;
			}, CopyRows<gysk_host_listen> {out});
}

int gysk_query_tasks(gysk_engine *e, const uint64_t *ids, uint32_t n, gysk_task_summary *out)
{
	return query_rows(e, ids, n, out, "task_summaries");
}

int gysk_query_task_window(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_task_summary *out, uint32_t cap, uint32_t *n)
{
	return window_rows(e, host_idx, flags, out, nullptr, cap, n, "task_window");
}

int gysk_export_hist(gysk_engine *e, uint64_t id, int which, gysk_hist_serial out[GYSK_HIST_MAX_BUCKETS], uint64_t *total, int64_t *maxv)
{
	CHECK_ENGINE(e);
	if (!out || !total || !maxv) return GYSK_ERR_INVAL;
	if (which >= GYSK_HIST_TASK_CPU_PCT && which <= GYSK_HIST_TASK_BLKIO_DELAY) return gysk_export_task_hist(e, id, which, out, total, maxv);
	if (which > GYSK_HIST_ACTIVE_CONN) return GYSK_ERR_INVAL;
	if (which < 0) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);
	if (int rc = stage_svc_raw(e, id)) return rc;
	const SvcRaw &r = *reinterpret_cast<const SvcRaw *>(e->h_wstage);
	if (!r.found) return GYSK_ERR_NOENT;
	if (which == GYSK_HIST_RESP_5MIN || which == GYSK_HIST_RESP_5DAY) { level_from_cells(r.lvl[which - GYSK_HIST_RESP_5MIN], out, total, maxv); return GYSK_OK; }
	if (which == GYSK_HIST_QPS) { hist_from_cells(r.qps, 15, out, total, maxv, true); return GYSK_OK; }
	if (which == GYSK_HIST_ACTIVE_CONN) { hist_from_cells(r.act, 14, out, total, maxv, true); return GYSK_OK; }
	hist_from_cells(which == GYSK_HIST_RESP_CUR ? r.cur : (which == GYSK_HIST_RESP_LAST ? r.last : r.all), 15, out, total, maxv, false);
	return GYSK_OK;
}

int gysk_export_task_hist(gysk_engine *e, uint64_t id, int which, gysk_hist_serial out[GYSK_HIST_MAX_BUCKETS], uint64_t *total, int64_t *maxv)
{
	CHECK_ENGINE(e);
	if (!out || !total || !maxv || which < GYSK_HIST_TASK_CPU_PCT || which > GYSK_HIST_TASK_BLKIO_DELAY) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);
	int rc = stage_one(e, id, sizeof(TaskRaw), "gather_tasks", [&](const unsigned long long *d_ids, uint32_t, uint32_t m) {
		return launch_gather_tasks(e->st, d_ids, m, reinterpret_cast<TaskRaw *>(e->d_wstage), e->stream);
	});
	if (rc) return rc;
	const TaskRaw &r = *reinterpret_cast<const TaskRaw *>(e->h_wstage);
	if (!r.found) return GYSK_ERR_NOENT;
	const int h = which - GYSK_HIST_TASK_CPU_PCT;
	hist_from_cells(r.h[h], h == 0 ? 14 : 15, out, total, maxv, true);
	return GYSK_OK;
}

// CONN_BITMAP::get_conn_breakup (common/gy_socket_stat.h:412-433): per response bucket the number of (client port & 31) slots seen
int gysk_export_conn_bitmap(gysk_engine *e, uint64_t id, int last_window, uint32_t masks[GYSK_HIST_MAX_BUCKETS], uint8_t nconn_arr[GYSK_HIST_MAX_BUCKETS])
{
	CHECK_ENGINE(e);
	if (!masks || !nconn_arr) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);
	if (int rc = stage_svc_raw(e, id)) return rc;
	const SvcRaw &r = *reinterpret_cast<const SvcRaw *>(e->h_wstage);
	if (!r.found) return GYSK_ERR_NOENT;
	const uint32_t *bm = last_window ? r.bm_last : r.bm_cur;
	for (int j = 0; j < GYSK_HIST_MAX_BUCKETS; ++j) { masks[j] = bm[j]; nconn_arr[j] = (uint8_t)__builtin_popcount(bm[j]); }
	return GYSK_OK;
}

int gysk_export_hll(gysk_engine *e, uint64_t id, uint8_t *regs)
{
	CHECK_ENGINE(e);
	if (!regs) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);
	int rc = stage_one(e, id, HLL_STAGE_REGS + ((size_t)1 << e->cfg.hll_p), "gather_hll", [&](const unsigned long long *d_ids, uint32_t, uint32_t) {
		return launch_gather_hll(e->st, d_ids, reinterpret_cast<int32_t *>(e->d_wstage), e->d_wstage + HLL_STAGE_REGS, e->stream);
	});
	if (rc) return rc;
	if (!*reinterpret_cast<const int32_t *>(e->h_wstage)) return GYSK_ERR_NOENT;
	memcpy(regs, e->h_wstage + HLL_STAGE_REGS, (size_t)1 << e->cfg.hll_p);
	return GYSK_OK;
}

int gysk_export_tdigest(gysk_engine *e, uint64_t id, double *means, uint64_t *weights, uint32_t cap, uint32_t *n, double *minv, double *maxv)
{
	CHECK_ENGINE(e);
	if (!means || !weights || !n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);
	if (int rc = stage_svc_raw(e, id)) return rc;
	const SvcRaw &r = *reinterpret_cast<const SvcRaw *>(e->h_wstage);
	if (!r.found) return GYSK_ERR_NOENT;
	return tdigest_out(r.td, r.cent, means, weights, cap, n, minv, maxv);
}

// Summary encoder (SURVEY §8f-2, output side): per-service summaries -> one NOTIFY_LISTENER_STATE message body, i.e. the records
// MTCP_LISTENER::set_state / the listener-state DB insert read (LISTENER_STATE_NOTIFY, common/gy_comm_proto.h:2183-2254; consumer
// partha_listener_state, server/gy_mconnhdlr.cc:11175-11251). Fields the engine computes are filled (nqrys_5s_, total_resp_5sec_,
// p95_5s_resp_ms_, p95_5min_resp_ms_, nconns_ = TCP events of the window, curr_kbytes_inbound_ = their kbytes); what only the host
// agent knows (task counters, errors, http flag) is zero; curr_state_ is STATE_IDLE (0) without queries, else STATE_OK (2) — the
// state classifier is out of scope. No issue string: every record is sizeof(LISTENER_STATE_NOTIFY) = 88 bytes, 8-byte aligned.
int gysk_encode_listener_state(const gysk_svc_summary *sums, uint32_t n, void *buf, uint32_t cap, uint32_t *nrecs, uint32_t *nbytes)
{
	if ((!sums && n) || !buf || !nrecs || !nbytes) return GYSK_ERR_INVAL;
	auto clamp32 = [](uint64_t v) -> uint32_t { return v > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)v; };
	auto clampms = [](int64_t v) -> uint32_t { return v < 0 ? 0u : (v > 0xFFFFFFFFll ? 0xFFFFFFFFu : (uint32_t)v); };
	uint8_t *p = static_cast<uint8_t *>(buf);
	uint32_t k = 0;

	for (uint32_t i = 0; i < n; ++i) {
		if (!sums[i].found) continue;
		if (k >= wire::LISTENER_STATE_NOTIFY::MAX_NUM_LISTENERS) break;			// one message holds at most 512 records (:2222)
		if ((size_t)(k + 1) * sizeof(wire::LISTENER_STATE_NOTIFY) > cap) return GYSK_ERR_NOSPC;
		wire::LISTENER_STATE_NOTIFY r;
		memset(&r, 0, sizeof(r));
		r.glob_id_ = sums[i].glob_id;
		r.nqrys_5s_ = sums[i].nqrys_5s;
		r.total_resp_5sec_ = clamp32(sums[i].total_resp_5sec);
		r.p95_5s_resp_ms_ = clampms(sums[i].p95_5s_resp_ms);
		r.p95_5min_resp_ms_ = clampms(sums[i].p95_5min_resp_ms);
		r.nconns_ = sums[i].nconns_5s;
		r.nconns_active_ = sums[i].nconns_active;
		r.ser_errors_ = sums[i].ser_errors; r.cli_errors_ = sums[i].cli_errors;
		r.curr_kbytes_inbound_ = sums[i].kbytes_5s;
		r.curr_state_ = sums[i].curr_state; r.curr_issue_ = sums[i].curr_issue;		// the device-side get_curr_state of the window
		r.issue_bit_hist_ = sums[i].issue_bit_hist; r.high_resp_bit_hist_ = sums[i].high_resp_bit_hist;
		memcpy(p + (size_t)k * sizeof(r), &r, sizeof(r));
		k++;
	}
	*nrecs = k; *nbytes = k * (uint32_t)sizeof(wire::LISTENER_STATE_NOTIFY);
	return GYSK_OK;
}

// Text form of the Postgres `tdigest` type (extension tvondra/tdigest, loaded by the reference with `create extension if not
// exists tdigest`, common/gy_query_common.cc:3385-3387; version unpinned there). tdigest_out prints
//   "flags %d count %ld compression %d centroids %d" followed by " (%lf, %ld)" per centroid, flags = 1 (TDIGEST_STORES_MEAN),
// and tdigest_in parses the same with sscanf: a row built from this string answers tdigest_percentile(col, p) like the rows the
// reference aggregates with public.tdigest(expr, 100) (gy_query_common.cc:1805-1858). Means are printed with 17 significant
// digits (sscanf %lf reads them back exactly). Returns the string length (without NUL), or GYSK_ERR_NOSPC.
int gysk_tdigest_to_pgtext(const double *means, const uint64_t *weights, uint32_t n, uint32_t compression, char *buf, uint32_t cap)
{
	if ((!means || !weights) && n) return GYSK_ERR_INVAL;
	if (!buf || !cap) return GYSK_ERR_INVAL;
	uint64_t total = 0;
	for (uint32_t i = 0; i < n; ++i) total += weights[i];
	int off = snprintf(buf, cap, "flags 1 count %llu compression %u centroids %u", (unsigned long long)total, compression, n);
	if (off < 0 || (uint32_t)off >= cap) return GYSK_ERR_NOSPC;
	for (uint32_t i = 0; i < n; ++i) {
		const int k = snprintf(buf + off, cap - off, " (%.17g, %llu)", means[i], (unsigned long long)weights[i]);
		if (k < 0 || (uint32_t)(off + k) >= cap) return GYSK_ERR_NOSPC;
		off += k;
	}
	return off;
}

// The engine keeps delta = 200 internally; the Postgres side of the reference aggregates with public.tdigest(expr, 100)
// (common/gy_query_common.cc:1855) and the extension refuses to combine digests of different compression, so the export is one
// more fixed-grid K_1 compress at compression 100 (host side). Each centroid goes to the cell that holds its start: the export
// compresses a finished digest once, and a cluster widened by one last item (a delta = 200 centroid, half a cell here) stays
// within the accuracy the export is tested to (tests/test_gpu_td_accuracy.py). The device's centre rule (gysk_tdigest.cuh) is
// there for the repeated merges, where the start rule's widening compounds.
static uint32_t host_td_compress(const double *means, const uint64_t *w, uint32_t n, uint32_t delta, double *om, uint64_t *ow)
{
	if (!n) return 0;
	const std::vector<double> qtab = k1_grid(delta);
	uint64_t W = 0, pref = 0, cw = 0;
	for (uint32_t i = 0; i < n; ++i) W += w[i];
	uint32_t nout = 0, cur = 0;
	double csum = 0.0;
	for (uint32_t i = 0; i < n; ++i) {
		uint32_t lo = cur;
		while (lo + 1 < delta && (uint64_t)(qtab[lo + 1] * (double)W) <= pref) ++lo;		// cell j starts at weight (uint64) (q_j W)
		if (i && lo != cur) { om[nout] = csum / (double)cw; ow[nout++] = cw; cw = 0; csum = 0.0; }
		cur = lo;
		csum += means[i] * (double)w[i]; cw += w[i]; pref += w[i];
	}
	om[nout] = csum / (double)cw; ow[nout++] = cw;
	return nout;
}

} // extern "C"

int gysk::tdigest_pgtext(gysk_engine *e, uint64_t id, ExportTd export_td, char *buf, uint32_t cap)
{
	double means[TD_CAP], minv = 0, maxv = 0, om[TD_CAP];
	uint64_t w[TD_CAP], ow[TD_CAP];
	uint32_t n = 0;
	int rc = export_td(e, id, means, w, TD_CAP, &n, &minv, &maxv);
	if (rc) return rc;
	const uint32_t no = host_td_compress(means, w, n, 100, om, ow);
	return gysk_tdigest_to_pgtext(om, ow, no, 100, buf, cap);
}

int gysk::tdigest_quantiles(gysk_engine *e, uint64_t id, ExportTd export_td, const double *qs, uint32_t nq, double *out)
{
	double means[TD_CAP], minv = 0, maxv = 0;
	uint64_t w[TD_CAP];
	uint32_t n = 0;
	int rc = export_td(e, id, means, w, TD_CAP, &n, &minv, &maxv);

	if (rc) return rc;
	if ((!qs || !out) && nq) return GYSK_ERR_INVAL;
	for (uint32_t i = 0; i < nq; ++i) out[i] = td_quantile(means, w, n, minv, maxv, qs[i]);
	return GYSK_OK;
}

extern "C" {

int gysk_export_tdigest_pgtext(gysk_engine *e, uint64_t id, char *buf, uint32_t cap)
{
	return tdigest_pgtext(e, id, gysk_export_tdigest, buf, cap);
}

int gysk_query_quantiles(gysk_engine *e, uint64_t id, const double *qs, uint32_t nq, double *out)
{
	return tdigest_quantiles(e, id, gysk_export_tdigest, qs, nq, out);
}

int gysk_query_flows(gysk_engine *e, const uint64_t *keys, uint32_t n, int last_window, gysk_flow_est *out)
{
	CHECK_ENGINE(e);
	if ((!keys || !out) && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);
	return query_flows_in(e, last_window ? e->st.cms_last : e->st.cms_cur, keys, n, out, "query_flows");
}

int gysk_query_flows_5min(gysk_engine *e, const uint64_t *keys, uint32_t n, gysk_flow_est *out)
{
	CHECK_ENGINE(e);
	if ((!keys || !out) && n) return GYSK_ERR_INVAL;
	if (!(e->cfg.flags & GYSK_FLAG_FLOW_LEVEL)) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Submit);
	return query_flows_in(e, e->st.cms_5min, keys, n, out, "query_flows_5min");
}

int gysk_topn_svcs(gysk_engine *e, int metric, int32_t host_idx, uint32_t n, gysk_topn_entry *out, uint32_t *nout)
{
	CHECK_ENGINE(e);
	if (!out || !nout || n == 0 || n > 64 || metric < GYSK_TOPN_QPS || metric > GYSK_TOPN_ISSUE) return GYSK_ERR_INVAL;
	return topn_rows(e, 0, metric, host_idx, n, out, nout, "gysk_topn_svcs");
}

int gysk_topn_tasks(gysk_engine *e, int metric, uint32_t n, gysk_topn_entry *out, uint32_t *nout)
{
	CHECK_ENGINE(e);
	if (!out || !nout || n == 0 || n > 64 || metric < GYSK_TOPN_TASK_CPU || metric > GYSK_TOPN_TASK_BLKIO_DELAY) return GYSK_ERR_INVAL;
	return topn_rows(e, 1, metric, -1, n, out, nout, "gysk_topn_tasks");
}

int gysk_query_host_summary(gysk_engine *e, uint32_t host_idx, gysk_host_summary *out)
{
	CHECK_ENGINE(e);
	if (!out) return GYSK_ERR_INVAL;
	std::lock_guard<std::mutex> lk(e->host_mtx);
	auto it = e->host_summ.find(host_idx);
	if (it == e->host_summ.end()) return GYSK_ERR_NOENT;
	*out = it->second;
	return GYSK_OK;
}

int gysk_query_cluster_state(gysk_engine *e, const uint32_t *host_idxs, uint32_t n, gysk_cluster_state *out)
{
	CHECK_ENGINE(e);
	if (!out || (!host_idxs && n)) return GYSK_ERR_INVAL;
	std::lock_guard<std::mutex> lk(e->host_mtx);
	memset(out, 0, sizeof(*out));
	auto add = [&](const gysk_host_summary & hs) {
		const uint32_t issues = (uint32_t)(hs.nstates[3] + hs.nstates[4] + hs.nstates[5]);	// STATE_BAD, STATE_SEVERE, STATE_DOWN
		out->nhosts++;
		out->nsvc_issue += issues; out->nsvcissue_hosts += !!issues;
		out->nsvc += (uint32_t)hs.nlisteners;
		out->total_qps += (uint32_t)hs.tot_qps;
		out->svc_net_mb += (uint32_t)((hs.tot_kb_inbound + hs.tot_kb_outbound) / 1024);
	};
	if (!host_idxs) { for (const auto & kv : e->host_summ) add(kv.second); }
	else {
		for (uint32_t i = 0; i < n; ++i) {
			auto it = e->host_summ.find(host_idxs[i]);
			if (it != e->host_summ.end()) add(it->second);
		}
	}
	return GYSK_OK;
}

// the per-host rankings the reference keeps in PARTHA_INFO (BOUNDED_PRIO_QUEUE, 10 entries per host, gy_mconnhdlr.h:961,975), as
// of each host's last NOTIFY_LISTENER_STATE / NOTIFY_AGGR_TASK_STATE message; host_idx < 0 merges the hosts of this engine
int gysk_topn_host(gysk_engine *e, int what, int32_t host_idx, uint32_t n, gysk_topn_entry *out, uint32_t *nout)
{
	CHECK_ENGINE(e);
	if (!out || !nout || !n || n > 64 || what < 0 || what > GYSK_HOSTTOP_TASK_BLKIO_DELAY) return GYSK_ERR_INVAL;
	std::lock_guard<std::mutex> lk(e->host_mtx);
	std::vector<gysk_topn_entry> all;
	auto take = [&](uint32_t h, const TopQueue &q) { for (const TopEntry &t : q.v) all.push_back(gysk_topn_entry {t.id, t.score, h, 0}); };
	if (what <= GYSK_HOSTTOP_SVC_NET) {
		for (const auto &kv : e->host_topn) if (host_idx < 0 || kv.first == (uint32_t)host_idx) take(kv.first, kv.second.q[what]);
	}
	else {
		for (const auto &kv : e->host_task_topn) if (host_idx < 0 || kv.first == (uint32_t)host_idx) take(kv.first, kv.second.q[what - GYSK_HOSTTOP_TASK_ISSUE]);
	}
	std::sort(all.begin(), all.end(), [](const gysk_topn_entry &a, const gysk_topn_entry &b) { return a.score != b.score ? a.score > b.score : a.glob_id < b.glob_id; });
	*nout = (uint32_t)std::min<size_t>(all.size(), n);
	for (uint32_t i = 0; i < *nout; ++i) out[i] = all[i];
	return GYSK_OK;
}

int gysk_export_cms(gysk_engine *e, int last_window, uint64_t *cells)
{
	CHECK_ENGINE(e);
	if (!cells) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Sync);
	CU(e, cudaMemcpy(cells, last_window ? e->st.cms_last : e->st.cms_cur, sizeof(uint64_t) * ((size_t)e->cfg.cms_depth << e->cfg.cms_log2_width),
			cudaMemcpyDeviceToHost));
	return GYSK_OK;
}

int gysk_export_cms_5min(gysk_engine *e, uint64_t *cells)
{
	CHECK_ENGINE(e);
	if (!cells) return GYSK_ERR_INVAL;
	if (!(e->cfg.flags & GYSK_FLAG_FLOW_LEVEL)) return GYSK_ERR_NOTSUP;
	GYSK_ENTER(e, Sync);
	CU(e, cudaMemcpy(cells, e->st.cms_5min, sizeof(uint64_t) * ((size_t)e->cfg.cms_depth << e->cfg.cms_log2_width), cudaMemcpyDeviceToHost));
	return GYSK_OK;
}

// ---- pure helpers ------------------------------------------------------------------------------------------------

int gysk_hist_nbuckets(int cls)
{
	if (cls < 0 || cls > GYSK_CLS_PERCENT) return GYSK_ERR_INVAL;
	return g_cls[cls].nthr + 2;
}

int gysk_hist_bucket(int cls, int64_t value)
{
	if (cls < 0 || cls > GYSK_CLS_PERCENT) return GYSK_ERR_INVAL;
	const ClsDesc &d = g_cls[cls];
	int64_t data = d.trunc_int ? (int64_t)(int32_t)value : value;

	if (data < d.minv) return 0;
	if (data >= d.maxv) return d.nthr + 1;
	if (d.fixed_diff) return (int)(1 + (data - d.minv) / d.fixed_diff);
	int b = 1;
	for (int i = 0; i < d.nthr; ++i) b += (data > d.thr[i]);
	return b;
}

// GY_HISTOGRAM::get_percentiles, common/gy_statistics.h:707-791: float multiplier, size_t * float cut-off,
// first bucket whose cumulative count reaches it, answer = that bucket's upper threshold cast to T
int gysk_hist_percentiles(int cls, int t_is_int, const gysk_hist_serial *stats, uint64_t total_count, const float *pcts, uint32_t npct, int64_t *out)
{
	if (cls < 0 || cls > GYSK_CLS_PERCENT || !stats || (!pcts && npct) || (!out && npct)) return GYSK_ERR_INVAL;
	uint64_t counts[GYSK_HIST_MAX_BUCKETS];
	for (int i = 0; i < g_cls[cls].nthr + 2; ++i) counts[i] = stats[i].count;
	for (uint32_t n = 0; n < npct; ++n) out[n] = hist_percentile(cls, !!t_is_int, counts, total_count, pcts[n]);
	return GYSK_OK;
}

// TCP_LISTENER::get_curr_state for a caller that has the inputs from outside the path (process status, host state, dependencies)
int gysk_classify_listener(const gysk_listener_state_in *in, uint8_t *high_resp_bit_hist, uint8_t *state, uint8_t *issue)
{
	if (!in || !high_resp_bit_hist || !state || !issue) return GYSK_ERR_INVAL;
	classify_listener(*in, *high_resp_bit_hist, *state, *issue);
	return GYSK_OK;
}

int gysk_classify_host(const gysk_host_state_in *in, uint8_t *state)
{
	if (!in || !state) return GYSK_ERR_INVAL;
	*state = classify_host(*in);
	return GYSK_OK;
}

double gysk_hll_estimate(const uint8_t *regs, uint32_t p)
{
	if (!regs || p < 4 || p > 16) return NAN;
	uint32_t hist[64] = {0};
	for (uint32_t i = 0; i < (1u << p); ++i) hist[regs[i] > 63 ? 63 : regs[i]]++;
	return hll_estimate_from_hist(hist, p);
}

double gysk_tdigest_quantile(const double *means, const uint64_t *weights, uint32_t n, double minv, double maxv, double q)
{
	if ((!means || !weights) && n) return NAN;
	return td_quantile(means, weights, n, minv, maxv, q);
}

uint32_t gysk_uint64_hash(uint64_t key) { return uint64_hash(key); }

// ---- multi-GPU merge: implemented in gysk_merge.cu ------------------------------------------------------------

} // extern "C"

// ---- request traces (gysk_config.max_trace_svcs) --------------------------------------------------------------

namespace {

constexpr uint32_t TRACE_WIN_ROWS = (uint32_t)(STAGE_BYTES / sizeof(gysk_trace_row));		// trace rows per window-read pass
static_assert(sizeof(gysk_trace_row) == 320 && QCHUNK <= TRACE_WIN_ROWS, "the stage holds a chunk of trace rows");
static_assert(sizeof(TraceRaw) <= STAGE_BYTES, "the stage holds one trace digest");

// rows handed out so far (engine held, stream synchronised on return)
int trace_rows_out(gysk_engine *e, uint32_t *nrows)
{
	uint32_t c = 0;
	CU(e, cudaMemcpyAsync(&c, e->st.trace.count, sizeof(c), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	*nrows = std::min(c, e->st.trace.rows);
	return 0;
}

} // namespace

extern "C" {

int gysk_query_traces(gysk_engine *e, const uint64_t *ids, uint32_t n, gysk_trace_row *out)
{
	CHECK_ENGINE(e);
	if (!e->st.trace.rows) return GYSK_ERR_NOTSUP;
	if ((!ids || !out) && n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);
	return staged_read(e, ids, n, QCHUNK, sizeof(gysk_trace_row), "trace_rows", [&](const unsigned long long *d_ids, uint32_t, uint32_t m) {
		return launch_trace_rows(e->st, d_ids, nullptr, m, reinterpret_cast<gysk_trace_row *>(e->d_wstage), e->stream);
	}, CopyRows<gysk_trace_row> {out});
}

// the rows of the selection listed on the device, ordered by id on the host, then read by row in stage-sized passes
int gysk_query_trace_window(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_trace_row *out, uint32_t cap, uint32_t *n)
{
	CHECK_ENGINE(e);
	if (!e->st.trace.rows) return GYSK_ERR_NOTSUP;
	if (!n || (!out && cap) || (flags & ~GYSK_WINDOW_ACTIVE_ONLY)) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Sync);
	uint32_t nrows = 0;
	if (int rc = trace_rows_out(e, &nrows)) return rc;
	unsigned long long *d_n = e->st.counters + CTR_NWINDOW;
	e->kernel_launches += launch_trace_list(e->st, nrows, host_idx, flags & GYSK_WINDOW_ACTIVE_ONLY, e->tmp.keys_b, e->tmp.keys_a, d_n, e->stream);
	unsigned long long cnt = 0;
	CU(e, cudaMemcpyAsync(&cnt, d_n, sizeof(cnt), cudaMemcpyDeviceToHost, e->stream));
	CU(e, cudaStreamSynchronize(e->stream));
	if (int rc = post_launch(e, "trace list")) return rc;
	const uint32_t total = (uint32_t)cnt, m = std::min(cap, total);
	if (m) {
		std::vector<uint64_t> &ids = e->win_ids, &rows = e->win_keys;
		ids.resize(total); rows.resize(total);
		CU(e, cudaMemcpyAsync(ids.data(), e->tmp.keys_b, total * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaMemcpyAsync(rows.data(), e->tmp.keys_a, total * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
		CU(e, cudaStreamSynchronize(e->stream));
		std::vector<std::pair<uint64_t, uint64_t>> &order = e->win_rows;
		order.resize(total);
		for (uint32_t i = 0; i < total; ++i) order[i] = {ids[i], rows[i]};
		std::sort(order.begin(), order.end());		// ids are unique; the list's order depends on the device's atomics
		for (uint32_t i = 0; i < m; ++i) rows[i] = order[i].second;
		CU(e, cudaMemcpyAsync(e->tmp.keys_a, rows.data(), (size_t)m * sizeof(uint64_t), cudaMemcpyHostToDevice, e->stream));
		int rc = staged_read<uint64_t>(e, nullptr, m, TRACE_WIN_ROWS, sizeof(gysk_trace_row), "trace_rows", [&](const unsigned long long *, uint32_t off, uint32_t k) {
			return launch_trace_rows(e->st, nullptr, e->tmp.keys_a + off, k, reinterpret_cast<gysk_trace_row *>(e->d_wstage), e->stream);
		}, CopyRows<gysk_trace_row> {out});
		if (rc) return rc;
	}
	*n = total;
	return GYSK_OK;
}

int gysk_export_trace_tdigest(gysk_engine *e, uint64_t id, int last_window, double *means, uint64_t *weights, uint32_t cap, uint32_t *n,
		double *minv, double *maxv)
{
	CHECK_ENGINE(e);
	if (!e->st.trace.rows) return GYSK_ERR_NOTSUP;
	if (!means || !weights || !n) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Submit);
	int rc = stage_one(e, id, sizeof(TraceRaw), "gather_trace", [&](const unsigned long long *d_ids, uint32_t, uint32_t) {
		return launch_gather_trace(e->st, d_ids, last_window, reinterpret_cast<TraceRaw *>(e->d_wstage), e->stream);
	});
	if (rc) return rc;
	const TraceRaw &r = *reinterpret_cast<const TraceRaw *>(e->h_wstage);
	if (!r.found) return GYSK_ERR_NOENT;
	TdHead h;
	h.total = r.total; h.minv = r.minv; h.maxv = r.maxv; h.n = r.n; h.pad = 0;
	return tdigest_out(h, r.cent, means, weights, cap, n, minv, maxv);
}

int gysk_export_trace_tdigest_pgtext(gysk_engine *e, uint64_t id, int last_window, char *buf, uint32_t cap)
{
	double means[TRACE_TD_CAP], mn, mx;
	uint64_t weights[TRACE_TD_CAP];
	uint32_t n = 0;
	int rc = gysk_export_trace_tdigest(e, id, last_window, means, weights, TRACE_TD_CAP, &n, &mn, &mx);
	if (rc) return rc;
	return gysk_tdigest_to_pgtext(means, weights, n, TRACE_TD_DELTA, buf, cap);		// at compression 100 already: no recompress
}

int gysk_trace_info(gysk_engine *e, uint32_t *rows_in_use, uint64_t *dropped)
{
	CHECK_ENGINE(e);
	if (!e->st.trace.rows) return GYSK_ERR_NOTSUP;
	if (!rows_in_use || !dropped) return GYSK_ERR_INVAL;
	GYSK_ENTER(e, Sync);
	int32_t nfree = 0;
	unsigned long long d = 0;
	CU(e, cudaMemcpy(&nfree, e->st.trace.free_n, sizeof(nfree), cudaMemcpyDeviceToHost));
	CU(e, cudaMemcpy(&d, e->st.trace.dropped, sizeof(d), cudaMemcpyDeviceToHost));
	uint32_t nrows = 0;
	if (int rc = trace_rows_out(e, &nrows)) return rc;
	*rows_in_use = nrows - (uint32_t)std::max(nfree, 0);
	*dropped = d;
	return GYSK_OK;
}

} // extern "C"
