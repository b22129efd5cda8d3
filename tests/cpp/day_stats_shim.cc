// The listener-walk half of the host shim (gyeeta_b200/host/gy_gysk_shim.h): window_listener_day_stats and host_state, linked against
// libgysketch.so. Without a GPU both report failure and leave the message alone. With one, services on three hosts (one of them with
// more than 2048) come back after 900 s as NOTIFY_LISTENER_DAY_STATS batches of at most 2048 records, one host per batch, whose
// concatenation is the bytes of the gysk_query_day_stats rows; host_state fills the listener counts of the partha's host, recomputes the
// state with gysk_classify_host and rewrites bit 0 of issue_bit_hist_, IDLE and GOOD messages included, reading the engine once per
// flush_window however many messages arrive in between.
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
	HOST_STATE_NOTIFY msg;
	std::memset(&msg, 0, sizeof(msg));
	msg.curr_state_ = GYSK_STATE_IDLE; msg.issue_bit_hist_ = 0x6; msg.ntasks_ = 40;

	if (!e) {
		int nb = 0;
		HOST_STATE_NOTIFY before = msg;
		const bool day = h.window_listener_day_stats([&](uint32_t, const void *, uint32_t) { ++nb; });
		const bool hs = h.host_state(partha, &msg);
		const bool same = 0 == std::memcmp(&before, &msg, sizeof(msg));
		std::printf("day: %d batches: %d host_state: %d unchanged: %d\n", day, nb, hs, same);
		return (rc == GYSK_ERR_NODEV && !day && nb == 0 && !hs && same) ? 0 : 1;
	}

	// services: 10 on host 0, 2500 on host 1 (two batches), 600 on host 3
	std::vector<gysk_event> ev;
	const uint32_t nper[4] = {10, 2500, 0, 600};
	for (uint32_t host = 0; host < 4; ++host)
		for (uint32_t i = 0; i < nper[host]; ++i) {
			gysk_event x {};
			x.svc_id = 0x100000ull * (host + 1) + 977 * (nper[host] - i); x.flow_key = i; x.value = 1000 * (1 + i % 50); x.host_idx = host;
			x.type = GYSK_EV_RESP;
			ev.push_back(x);
		}
	const uint8_t mid[16] = {1};
	bool good = 0 == gysk_ingest_raw(e, mid, 0, GYSK_RAW_EVENT32, ev.data(), (uint32_t)ev.size());
	good = good && h.flush_window(5);
	int early = 0;
	good = good && h.window_listener_day_stats([&](uint32_t, const void *, uint32_t) { ++early; });
	good = good && 0 == gysk_ingest_raw(e, mid, 0, GYSK_RAW_EVENT32, ev.data(), (uint32_t)ev.size());
	good = good && h.flush_window(1000);

	std::vector<uint8_t> got;
	uint32_t nbatches = 0, maxrecs = 0, prev_host = 0, bad_order = 0;
	good = good && h.window_listener_day_stats([&](uint32_t host, const void *p, uint32_t nrecs) {
		nbatches++;
		if (nrecs > maxrecs) maxrecs = nrecs;
		if (host < prev_host) bad_order++;
		prev_host = host;
		got.insert(got.end(), (const uint8_t *)p, (const uint8_t *)p + nrecs * sizeof(LISTENER_DAY_STATS));
	});
	uint32_t n = 0;
	std::vector<gysk_listener_day_stats> rows(4000);
	good = good && 0 == gysk_query_day_stats(e, -1, rows.data(), nullptr, (uint32_t)rows.size(), &n);
	const bool same_bytes = good && got.size() == n * sizeof(LISTENER_DAY_STATS) && 0 == std::memcmp(got.data(), rows.data(), got.size());
	std::printf("day rows: %u early batches: %d batches: %u max records: %u order errors: %u same bytes: %d\n", n, early, nbatches, maxrecs, bad_order,
			same_bytes);

	// host_state on crafted messages of host 1
	gysk_host_listen hl[8];
	uint32_t nh = 0;
	good = good && 0 == gysk_query_host_listen(e, hl, 8, &nh);
	gysk_host_listen mine {1, 0, 0, 0};
	for (uint32_t i = 0; i < nh && i < 8; ++i) if (hl[i].host_idx == 1) mine = hl[i];
	struct Case { uint8_t state, cpu, mem, scpu, smem; uint32_t nti, nts; };
	const Case cases[] = { {GYSK_STATE_IDLE, 0, 0, 0, 0, 0, 0}, {GYSK_STATE_GOOD, 0, 0, 0, 0, 0, 0}, {GYSK_STATE_OK, 1, 0, 0, 0, 0, 0},
			{GYSK_STATE_BAD, 0, 1, 0, 1, 2, 0}, {GYSK_STATE_SEVERE, 1, 1, 1, 0, 7, 3} };
	int hs_ok = 0, idle_kept = 0;
	// the five messages of one window: the first reads the host rows from the engine, the other four answer from them
	gysk_stats s0 {}, s1 {}, s2 {}, s3 {}, s4 {};
	good = good && 0 == gysk_get_stats(e, &s0);
	for (const Case &c : cases) {
		if (&c == cases + 1) good = good && 0 == gysk_get_stats(e, &s1);
		HOST_STATE_NOTIFY m = msg;
		m.curr_state_ = c.state; m.cpu_issue_ = c.cpu; m.mem_issue_ = c.mem; m.severe_cpu_issue_ = c.scpu; m.severe_mem_issue_ = c.smem;
		m.ntasks_issue_ = c.nti; m.ntasks_severe_ = c.nts;
		HOST_STATE_NOTIFY want = m;
		gysk_host_state_in in {};
		in.cpu_issue = c.cpu; in.mem_issue = c.mem; in.severe_cpu_issue = c.scpu; in.severe_mem_issue = c.smem; in.cpu_idle = c.state == GYSK_STATE_IDLE;
		in.ntasks_issue = c.nti; in.ntasks_severe = c.nts; in.nlisten_issue = mine.nlisten_issue; in.nlisten_severe = mine.nlisten_severe;
		uint8_t st = 0;
		gysk_classify_host(&in, &st);
		want.nlisten_ = mine.nlisten; want.nlisten_issue_ = mine.nlisten_issue; want.nlisten_severe_ = mine.nlisten_severe;
		want.curr_state_ = st; want.issue_bit_hist_ = (uint8_t)((m.issue_bit_hist_ & ~1u) | (st >= GYSK_STATE_BAD));
		const bool ok = h.host_state(partha, &m) && 0 == std::memcmp(&m, &want, sizeof(m));
		hs_ok += ok;
		if (c.state <= GYSK_STATE_GOOD && ok && m.curr_state_ == c.state) idle_kept++;
	}
	good = good && 0 == gysk_get_stats(e, &s2);
	// the next window: one read again, and it sees the listeners created since
	std::vector<gysk_event> more(ev.begin(), ev.begin() + 10);
	for (gysk_event &x : more) { x.svc_id += 7; x.host_idx = 1; }
	good = good && 0 == gysk_ingest_raw(e, mid, 0, GYSK_RAW_EVENT32, more.data(), (uint32_t)more.size());
	good = good && h.flush_window(1005) && 0 == gysk_get_stats(e, &s3);
	HOST_STATE_NOTIFY m2 = msg;
	good = good && h.host_state(partha, &m2) && h.host_state(partha, &m2) && 0 == gysk_get_stats(e, &s4);
	const bool one_read = s1.kernel_launches > s0.kernel_launches && s2.kernel_launches == s1.kernel_launches &&
			s4.kernel_launches - s3.kernel_launches == s1.kernel_launches - s0.kernel_launches;
	std::printf("host_state: %d of 5 idle/good kept: %d nlisten: %u one read per window: %d next window nlisten: %u\n", hs_ok, idle_kept, mine.nlisten,
			one_read, m2.nlisten_);
	gysk_destroy(e);
	return (good && same_bytes && n == 3110 && early == 0 && nbatches == 4 && maxrecs == 2048 && bad_order == 0 && hs_ok == 5 && idle_kept == (mine.nlisten_issue ? 0 : 2) &&
			mine.nlisten == 2500 && one_read && m2.nlisten_ == 2510) ? 0 : 2;
}
