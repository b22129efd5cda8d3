// The read side of the host shim (gyeeta_b200/host/gy_gysk_shim.h): window_listener_states and handle_aggr_task_hist_stats, linked
// against libgysketch.so. Without a GPU both report failure and leave the records alone. With one, services on three hosts (one of
// them with more than 512) come back as NOTIFY_LISTENER_STATE batches of at most 512 records whose concatenation is the encoding of
// the gysk_query_window rows, and the p95 fill changes exactly the records of processes the engine holds for that partha (a
// process of another host and an unknown one stay as they are).
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include "gy_gysk_shim.h"
#include "gysk_wire.h"

struct PARTHA_INFO { uint64_t machine_id_[2] {1, 2}; uint32_t gysk_host_idx_ {1}; };

int main()
{
	using namespace gysk::wire;

	gysk_config cfg;
	gysk_config_default(&cfg);
	gysk_engine *e = nullptr;
	int rc = gysk_create(&cfg, &e);
	std::printf("gysk_create rc=%d (%s)\n", rc, rc ? gysk_last_error(nullptr) : "ok");

	gysk_shim::GYSK_HANDLER h(e);
	auto partha = std::make_shared<PARTHA_INFO>();
	AGGR_TASK_HIST_STATS recs[4];
	std::memset(recs, 0, sizeof(recs));
	for (int i = 0; i < 4; ++i) {
		recs[i].aggr_task_id_ = i < 3 ? 5 + i : 99;
		recs[i].starttimeusec_ = 1000 + i; recs[i].nprocs_ = 7;
		recs[i].p95_cpu_pct_ = recs[i].p95_cpu_delay_ms_ = recs[i].p95_blkio_delay_ms_ = 0xABCDu;
	}
	AGGR_TASK_HIST_STATS before[4];
	std::memcpy(before, recs, sizeof(recs));

	if (!e) {
		int nb = 0;
		const bool win = h.window_listener_states([&](uint32_t, const void *, uint32_t, uint32_t) { ++nb; });
		const bool tasks = h.handle_aggr_task_hist_stats(partha, recs, 4);
		const bool same = 0 == std::memcmp(before, recs, sizeof(recs));
		std::printf("window: %d batches: %d tasks: %d unchanged: %d\n", win, nb, tasks, same);
		return (rc == GYSK_ERR_NODEV && !win && nb == 0 && !tasks && same) ? 0 : 1;
	}

	// services: 10 on host 0, 1200 on host 1 (three batches), 600 on host 3; processes 5 and 6 on host 1, 7 on host 2
	std::vector<gysk_event> ev;
	const uint32_t nper[4] = {10, 1200, 0, 600};
	for (uint32_t host = 0; host < 4; ++host)
		for (uint32_t i = 0; i < nper[host]; ++i) {
			gysk_event x {};
			x.svc_id = 0x100000ull * (host + 1) + 977 * (nper[host] - i); x.flow_key = i; x.value = 1000 * (1 + i % 50); x.host_idx = host;
			x.type = GYSK_EV_RESP;
			ev.push_back(x);
		}
	for (uint64_t id = 5; id <= 7; ++id)
		for (uint32_t i = 0; i < 20; ++i) {
			gysk_event x {};
			x.svc_id = id; x.flow_key = ((uint64_t)(3 * i) << 32) | (i * 7); x.value = i * (uint32_t)id; x.host_idx = id == 7 ? 2 : 1; x.type = GYSK_EV_TASK;
			ev.push_back(x);
		}
	const uint8_t mid[16] = {1};
	bool good = 0 == gysk_ingest_raw(e, mid, 0, GYSK_RAW_EVENT32, ev.data(), (uint32_t)ev.size());
	good = good && h.flush_window(5);

	std::vector<uint8_t> got;
	uint32_t nbatches = 0, maxrecs = 0, prev_host = 0, bad_order = 0;
	good = good && h.window_listener_states([&](uint32_t host, const void *p, uint32_t nrecs, uint32_t nbytes) {
		nbatches++;
		if (nrecs > maxrecs) maxrecs = nrecs;
		if (host < prev_host) bad_order++;
		prev_host = host;
		got.insert(got.end(), (const uint8_t *)p, (const uint8_t *)p + nbytes);
	});
	uint32_t n = 0;
	std::vector<gysk_svc_summary> rows(2000);
	good = good && 0 == gysk_query_window(e, -1, 0, rows.data(), (uint32_t)rows.size(), &n);
	std::vector<uint8_t> want(rows.size() * sizeof(LISTENER_STATE_NOTIFY));
	uint32_t wbytes = 0;
	for (uint32_t off = 0; good && off < n; off += 512) {
		uint32_t nrecs = 0, nbytes = 0;
		good = 0 == gysk_encode_listener_state(rows.data() + off, n - off < 512 ? n - off : 512, want.data() + wbytes, (uint32_t)want.size() - wbytes, &nrecs, &nbytes);
		wbytes += nbytes;
	}
	const bool same_bytes = good && got.size() == wbytes && 0 == std::memcmp(got.data(), want.data(), wbytes);
	std::printf("window rows: %u batches: %u max records: %u order errors: %u same bytes: %d\n", n, nbatches, maxrecs, bad_order, same_bytes);

	const bool tasks = h.handle_aggr_task_hist_stats(partha, recs, 4);
	gysk_task_summary ts[4];
	uint64_t ids[4] = {5, 6, 7, 99};
	good = good && tasks && 0 == gysk_query_tasks(e, ids, 4, ts);
	bool fill_ok = good && ts[0].found && ts[1].found && ts[2].found && ts[2].host_idx == 2 && !ts[3].found;
	for (int i = 0; fill_ok && i < 4; ++i) {
		AGGR_TASK_HIST_STATS x = before[i];
		if (i < 2) {
			x.p95_cpu_pct_ = (uint32_t)ts[i].p95_cpu_pct; x.p95_cpu_delay_ms_ = (uint32_t)ts[i].p95_cpu_delay_ms;
			x.p95_blkio_delay_ms_ = (uint32_t)ts[i].p95_blkio_delay_ms;
		}
		fill_ok = 0 == std::memcmp(&x, &recs[i], sizeof(x));
	}
	std::printf("task fill: %d p95: %d %d %d\n", fill_ok, ts[0].p95_cpu_pct, ts[0].p95_cpu_delay_ms, ts[0].p95_blkio_delay_ms);
	gysk_destroy(e);
	return (good && same_bytes && n == 1810 && nbatches == 6 && maxrecs == 512 && bad_order == 0 && fill_ok) ? 0 : 2;
}
