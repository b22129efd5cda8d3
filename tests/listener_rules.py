"""The listener state decision of every flush (state_kernel / svc_update_state: TCP_LISTENER::get_curr_state behind
listener_stats_update, common/gy_socket_stat.cc:2020-2875, :4045-4272), restated from what an engine exports, and a set of
services whose per-window recipes land on every rule exit the engine can reach.

The restatement builds gysk_listener_state_in from the exported histograms (HIST_RESP_LAST / _5MIN / _5DAY / _ALL, HIST_QPS,
HIST_ACTIVE_CONN), the last window's CONN_BITMAP, the window's row (nconns_active, ser_errors) and the flush timeline the test
drives; the percentiles come from gysk_hist_percentiles. It then applies gysk_classify_listener and the issue-history rule. The
process, cpu / memory, dependency and task-delay inputs are 0, as on the device.

`rule_exit` labels the exit of the decision tree an input takes (the reference line of the rule), and the boundary facts met on
the way, so that a test can assert which rules and which sides of each boundary a run reached."""

import numpy as np

from gyeeta_b200 import engine as ge

M32 = 0xFFFFFFFF
RESP_THR = (1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000)
CLS_RESP, CLS_SEMI_LOG_LO, CLS_HASH_1_3000 = 0, 2, 6
SECS_5D = 432000

# ------------------------------------------------------------------------------------------------------------------------------
# the restatement
# ------------------------------------------------------------------------------------------------------------------------------


def hist_pct(ser, cls, t_is_int, pcts, nb=15):
    """gysk_hist_percentiles over the first nb cells of an exported histogram, total = their counts"""
    s = np.zeros(15, dtype=ge.SERIAL_DTYPE)
    s[:nb] = ser[:nb]
    p = np.asarray(pcts, dtype=np.float32)
    out = np.zeros(len(p), dtype=np.int64)
    rc = ge.load_library().gysk_hist_percentiles(cls, t_is_int, ge._p(s), int(s["count"].sum()), ge._p(p), len(p), ge._p(out))
    assert rc == 0, rc
    return [int(v) for v in out]


def level_stats(ser):
    """TIME_HISTOGRAM::get_stats (common/gy_statistics.h:1333-1362): p95 / p99 / p25 clamped at 0, count, sum, sum / max(count, 1)"""
    p95, p99, p25 = (max(v, 0) for v in hist_pct(ser, CLS_RESP, 0, (95.0, 99.0, 25.0)))
    cnt = int(ser["count"].sum())
    tot = int(sum(int(v) % (1 << 64) for v in ser["sum"].tolist())) % (1 << 64)
    tot_i = tot - (1 << 64) if tot >> 63 else tot
    return dict(p95=p95, p99=p99, p25=p25, cnt=cnt, sum=tot, mean=float(tot_i) / float(cnt if cnt else 1))


def restate(src, id_, tsec, first, nconn):
    """gysk_listener_state_in of one service at the flush at tsec. src: hist(id, which) -> (cells, total, max), bitmap(id) ->
    per-bucket connection counts of the last window, row(id) -> (nconns_active, ser_errors). first: tsec of the first flush that saw
    the service; nconn: the active connections of the last ACTIVE_CONN_STATS report (0 when there was none)."""
    x = ge.ListenerStateIn()
    s5 = level_stats(src.hist(id_, ge.HIST_RESP_LAST)[0])
    s300 = level_stats(src.hist(id_, ge.HIST_RESP_5MIN)[0])
    s5d = level_stats(src.hist(id_, ge.HIST_RESP_5DAY)[0])
    sall = level_stats(src.hist(id_, ge.HIST_RESP_ALL)[0])
    x.r5p95, x.r5p99, x.nqrys_5s, x.total_resp_msec, x.mean5 = s5["p95"], s5["p99"], s5["cnt"], s5["sum"], s5["mean"]
    x.r300p95, x.r300p99, x.mean300 = s300["p95"], s300["p99"], s300["mean"]
    x.r5dp95, x.r5dp99, x.r5dp25, x.tcount_5d, x.mean5d = s5d["p95"], s5d["p99"], s5d["p25"], s5d["cnt"], s5d["mean"]
    x.rallp95, x.rallp99, x.meanall = sall["p95"], sall["p99"], sall["mean"]
    # qps_hist_ / active_conn_hist_ already hold this window's sample (added before the percentiles, :4111-4130); the
    # active-connection histogram has 14 buckets (HASH_1_3000)
    x.qps_p95, x.qps_p25 = hist_pct(src.hist(id_, ge.HIST_QPS)[0], CLS_SEMI_LOG_LO, 1, (95.0, 25.0))
    x.act_p95, x.act_p25 = hist_pct(src.hist(id_, ge.HIST_ACTIVE_CONN)[0], CLS_HASH_1_3000, 1, (95.0, 25.0), nb=14)
    x.last_qps_count = s5["cnt"] // 5
    x.nconn = nconn
    cnt = src.bitmap(id_)
    x.curr_active_conn = max([nconn] + [int(c) for c in cnt])
    for b in range(15):
        x.nactive_conn_arr[b] = int(cnt[b])
    x.ser_errors = src.row(id_)[1]
    age = tsec - first if tsec > first else 0
    x.secs_5d = min(age + 1, SECS_5D)
    return x, age


def issue_history(age, ser, state, issue, ibits):
    """listener_stats_update, common/gy_socket_stat.cc:4242-4272: a listener younger than 100 s without server errors reports
    {OK, NONE} and clears its issue history"""
    if age > 100 or ser:
        return state, issue, ((ibits << 1) | (state >= ge.STATE_BAD)) & 0xFF
    return ge.STATE_OK, ge.ISSUE_NONE, 0


def expected(x, age, prev):
    """(state, issue, issue_bit_hist, high_resp_bit_hist) after one evaluation, from the previous four fields"""
    st, iss, hb = ge.classify_listener(x, prev[3])
    st, iss, ib = issue_history(age, x.ser_errors, st, iss, prev[2])
    return (st, iss, ib, hb)


# ------------------------------------------------------------------------------------------------------------------------------
# which exit of the decision tree an input takes (process, cpu / memory, dependency and delay inputs 0)
# ------------------------------------------------------------------------------------------------------------------------------


def resp_bucketid(thr):
    for i, t in enumerate(RESP_THR):
        if thr == t:
            return i + 1
    return 0 if thr < 0 else 14


def f32(v):
    return float(np.float32(v))


def rule_exit(x, hb):
    """(label, state, issue, facts): the reference line of the exit get_curr_state takes for x, its outcome, and the boundary facts
    met on the way as (name, value) pairs. Mirrors gysk_state.cuh's classify_listener for inputs without process, host or dependency
    issues; the tests check it against gysk_classify_listener on every input they label."""
    assert not (x.task_issue or x.task_severe or x.task_delay or x.cpu_issue or x.mem_issue or x.ntasks_issue or x.ntasks_noissue
                or x.tasks_delay_msec or x.nserdepends)
    S, I = ge, ge
    facts = set()
    ser, n5 = x.ser_errors, x.nqrys_5s
    b5, b300, b5d = resp_bucketid(x.r5p95), resp_bucketid(x.r300p95), resp_bucketid(x.r5dp95)
    qps = max(x.last_qps_count, int(n5 // 5))
    worse = b5 > b5d + 2 and b5 > b300
    if b5 > b300 and b5 - b5d in (2, 3):
        facts.add(("worse", b5 - b5d))

    def ser_rule(tag):
        ser2, ser5 = (ser * 2) & M32, (ser * 5) & M32
        if ser2 - n5 in (0, 1):
            facts.add(("ser2", ser2 - n5))
        if ser5 - n5 in (0, 1):
            facts.add(("ser5", ser5 - n5))
        if ser2 > n5:
            return (tag + "s", S.STATE_SEVERE, I.ISSUE_SERVER_ERRORS)
        if ser5 > n5:
            return (tag + "b", S.STATE_BAD, I.ISSUE_SERVER_ERRORS)
        return None

    def ok(tag):
        return (tag, S.STATE_OK, I.ISSUE_SERVER_ERRORS if ser else I.ISSUE_NONE)

    def out(r):
        return r + (facts,)

    if qps == 0:
        return out(("2122", S.STATE_IDLE, I.ISSUE_NONE))
    if b5 == 1 or x.r5p95 < x.r5dp95:                                         # :2139 faster than the 5-day level
        if qps <= x.qps_p25 and x.qps_p25 < x.qps_p95:                          # :2143 QPS too low
            if not ser:
                return out(("2145", S.STATE_IDLE, I.ISSUE_NONE))
            r = ser_rule("2153")
            if r:
                return out(r)
            if ser < n5 * 0.1:
                return out(("2170", S.STATE_OK, I.ISSUE_SERVER_ERRORS))
        if ser:
            r = ser_rule("2228")
            if r:
                return out(r)
            return out(("2295", S.STATE_OK, I.ISSUE_SERVER_ERRORS))
        if qps <= x.qps_p95 or b5 + 2 <= b5d:
            return out(("2275", S.STATE_GOOD, I.ISSUE_NONE))
        return out(("2287", S.STATE_OK, I.ISSUE_QPS_HIGH))
    if x.r5p95 == x.r5dp95:                                                   # :2307 the 5-day level's bucket
        if ser:
            r = ser_rule("2307")
            if r:
                return out(r)
        if x.mean5 <= x.mean5d * f32(0.8):                                     # :2340
            if qps <= x.qps_p25:
                if ser:
                    return out(("2342", S.STATE_BAD, I.ISSUE_SERVER_ERRORS))
                return out(("2342i", S.STATE_IDLE, I.ISSUE_NONE))
            if not ser:
                return out(("2386", S.STATE_GOOD, I.ISSUE_NONE))
            return out(("2402", S.STATE_OK, I.ISSUE_LISTENER_TASKS))
        if x.mean5 <= x.mean5d * f32(1.2):
            return out(("2419", S.STATE_OK, I.ISSUE_NONE))
    if ser:                                                                   # :2430 the response is high
        r = ser_rule("2432")
        if r:
            return out(r)
    st = S.STATE_SEVERE if worse else S.STATE_BAD
    if qps > x.qps_p95:                                                       # :2464 QPS well above its p95
        p11 = f32(f32(x.qps_p95) * f32(1.1))
        if qps - x.qps_p95 in (5, 6) and qps > p11:
            facts.add(("qps_diff", qps - x.qps_p95))
        if qps - x.qps_p95 > 5:
            if qps <= p11 < qps + 1:
                facts.add(("qps_1.1", 0))
            elif qps - 1 <= p11 < qps:
                facts.add(("qps_1.1", 1))
        if qps - x.qps_p95 > 5 and f32(qps) > p11:
            return out(("2464", st, I.ISSUE_QPS_HIGH))
    if x.curr_active_conn > x.act_p95:                                        # :2525
        if x.curr_active_conn - x.act_p95 in (1, 2):
            facts.add(("act_diff", x.curr_active_conn - x.act_p95))
        if x.curr_active_conn - x.act_p95 > 1:
            return out(("2525", S.STATE_SEVERE if worse and x.curr_active_conn > 10 else S.STATE_BAD, I.ISSUE_ACTIVE_CONN_HIGH))
    if x.r5p95 == x.r5dp95 and x.r5p99 > x.r5dp99:
        return out(ok("2552"))
    if qps <= x.qps_p25 and x.nconn <= x.act_p25:
        return out(ok("2576"))
    avg5d = int(x.tcount_5d // (x.secs_5d if x.secs_5d > 0 else 1))
    if x.r5p95 <= x.rallp95 and x.mean5 <= x.meanall * f32(1.1) and avg5d - (qps >> 1) in (-1, 0):
        facts.add(("avg5d", avg5d - (qps >> 1), x.secs_5d == SECS_5D))
    if avg5d < (qps >> 1) and x.r5p95 <= x.rallp95 and x.mean5 <= x.meanall * f32(1.1):
        return out(ok("2638"))
    if qps <= x.qps_p25 and x.curr_active_conn <= x.act_p25 and b5 <= b5d + 1:
        return out(ok("2661"))
    if b5 <= b5d + 1 and b300 == b5d and x.mean5 > x.mean300 and x.mean300 < x.mean5d * f32(1.1):
        return out(ok("2684"))
    if b5 == b5d + 1 and x.nactive_conn_arr[b5] <= 3 and x.curr_active_conn in (14, 15):
        facts.add(("active_conn", x.curr_active_conn))
    if b5 == b5d + 1 and x.curr_active_conn >= 15 and x.nactive_conn_arr[b5] in (3, 4):
        facts.add(("bitmap_bucket", x.nactive_conn_arr[b5]))
    if x.curr_active_conn >= 15 and b5 == b5d + 1:                          # :2710 slow responses on few connections
        b = b5
        while b < 15 and x.nactive_conn_arr[b] <= 3:
            b += 1
        if b > b5:
            return out(ok("2710"))
    nhigh = bin(((hb << 1) | 1) & 0xFF).count("1")
    if nhigh in (4, 5):
        facts.add(("nhigh", nhigh))
    if nhigh < 5:
        return out(ok("2748"))
    return out(("2855", st, I.ISSUE_SERVER_ERRORS if ser else I.ISSUE_UNKNOWN))


# every (state, issue) pair the tree gives without process, host or dependency inputs, and the exits that reach them. :2661 is not
# among them: its test `curr_active_conn <= act_p25` follows :2576's `nconn <= act_p25` with the same QPS test, and
# curr_active_conn >= nconn (it is their max with the CONN_BITMAP counts), so whatever passes :2661 has already left at :2576
REACHABLE_PAIRS = {(ge.STATE_IDLE, ge.ISSUE_NONE), (ge.STATE_GOOD, ge.ISSUE_NONE), (ge.STATE_OK, ge.ISSUE_NONE),
                   (ge.STATE_OK, ge.ISSUE_QPS_HIGH), (ge.STATE_OK, ge.ISSUE_SERVER_ERRORS), (ge.STATE_OK, ge.ISSUE_LISTENER_TASKS)} | \
    {(s, i) for s in (ge.STATE_BAD, ge.STATE_SEVERE) for i in (ge.ISSUE_SERVER_ERRORS, ge.ISSUE_QPS_HIGH, ge.ISSUE_ACTIVE_CONN_HIGH,
                                                              ge.ISSUE_UNKNOWN)}
assert len(REACHABLE_PAIRS) == 14


# ------------------------------------------------------------------------------------------------------------------------------
# scenarios: one engine, many services, each with its own per-window recipe on one flush timeline
# ------------------------------------------------------------------------------------------------------------------------------

# Flush times. 1000 .. 1101: the first services are seen at 1000, so 1100 / 1101 are ages 100 / 101. From 1130 on one flush every
# 30 s: each window opens a slot of the 300-s level (10 slots of 30 s), which then holds the last 10 windows while the 5-day level
# holds them all. The last four windows jump past 5 days: they are in slot epoch 10 of the 5-day level (43 200-s slots), so the
# level holds them only, while the all-time level holds everything. For a service first seen at 1000, secs_5d = age + 1 =
# 431 061 at SECS_5D + 60 (not clamped yet) and min(433 001, 432 000) at SECS_5D + 2000 (clamped).
JUMP = 16
POST = [SECS_5D + 30, SECS_5D + 60, SECS_5D + 90, SECS_5D + 2000]
TIMES = [1000, 1030, 1060, 1090, 1100, 1101] + [1130 + 30 * k for k in range(JUMP + 1)] + POST
NWIN = len(TIMES)


def R(n, ms, ports=2, ser=0, port0=0):
    """n responses of ms msec from client ports port0 .. port0 + ports - 1 (round robin), the first `ser` flagged as server errors"""
    return ("resp", n, ms, ports, ser, port0)


def A(nconn):
    """one ACTIVE_CONN_STATS record with nconn active connections"""
    return ("active", nconn)


def T(n):
    """n connection events"""
    return ("conn", n)


def FILL(n, ms):
    """n responses of ms msec from two client ports that fill a level: a test may hand them to an engine as 32-byte events even
    where it sends a window's other responses as API_TRAN records"""
    return ("fill", n, ms)


class Svc:
    """one service: plan(w) -> the chunks of window w; probes {w: rule label} the exit its inputs must take at that flush"""

    def __init__(self, name, plan, probes, host=0):
        self.name, self.plan, self.probes, self.host = name, plan, dict(probes), host


def build_window(svcs, ids, w):
    """(EVENT_DTYPE array of window w, set of ids with events in it, mask of the FILL events)"""
    parts, active, fill = [], set(), []
    for s, id_ in zip(svcs, ids):
        for ch in s.plan(w):
            if ch[0] == "fill":
                ch = R(ch[1], ch[2]) + (True,)
            if ch[0] == "resp":
                _k, n, ms, ports, ser, port0 = ch[:6]
                ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
                ev["type"] = ge.EV_RESP
                ev["value"] = ms * 1000 + 400
                ev["flow_key"] = port0 + np.arange(n) % ports + 1024
                ev["flags"][:ser] = ge.EVF_SER_ERROR
            elif ch[0] == "active":
                ev = np.zeros(1, dtype=ge.EVENT_DTYPE)
                ev["type"], ev["flags"], ev["value"], ev["flow_key"] = ge.EV_ACTIVE, ch[1], 3, 77
            else:
                ev = np.zeros(ch[1], dtype=ge.EVENT_DTYPE)
                ev["type"], ev["value"], ev["flow_key"] = ge.EV_ACCEPT, 2048, 4000 + np.arange(ch[1])
            if len(ev):
                ev["svc_id"], ev["host_idx"] = id_, s.host
                parts.append(ev)
                fill.append(np.full(len(ev), len(ch) == 7))
                active.add(int(id_))
    if not parts:
        return np.zeros(0, dtype=ge.EVENT_DTYPE), active, np.zeros(0, dtype=bool)
    return np.concatenate(parts), active, np.concatenate(fill)


class Expect:
    """what the test knows of its own stream, and the state it expects: first flush of every id, the last reported active
    connections, the previous four state fields; `step` evaluates the restatement for the ids with events in the closed window"""

    def __init__(self):
        self.first, self.nconn, self.state = {}, {}, {}

    def forget(self, id_):
        for d in (self.first, self.nconn, self.state):
            d.pop(id_, None)

    def step(self, src, tsec, ids, active):
        """-> {id: (state fields, rule label, facts)} of the evaluated ids; stale ids keep their state"""
        out = {}
        for id_ in ids:
            id_ = int(id_)
            if id_ not in self.first and id_ in active:
                self.first[id_] = tsec
            if id_ not in active:
                continue
            nca = src.row(id_)[0]
            if nca:
                self.nconn[id_] = nca                       # a report arrived in this window; otherwise the last one stays
            x, age = restate(src, id_, tsec, self.first[id_], self.nconn.get(id_, 0))
            prev = self.state.get(id_, (ge.STATE_OK, ge.ISSUE_NONE, 0, 0))
            want = expected(x, age, prev)
            label, st, iss, facts = rule_exit(x, prev[3])
            assert (st, iss) == ge.classify_listener(x, prev[3])[:2], (label, st, iss)
            facts = set(facts)
            if age in (100, 101):
                facts.add(("age", age, bool(x.ser_errors)))
            if age <= 100 and not x.ser_errors:
                label = label + "+young"
            self.state[id_] = want
            out[id_] = (want, label, facts, x)
        return out


P = 16          # the probe window of most scenarios: t = 1430
J = TIMES.index(POST[0])            # the first window after the jump past 5 days


def base(w, ms=20, early_ms=None, lo=40, hi=400, hi_conn=20):
    """even windows: lo responses + 3 active connections; odd: 1000 (before 1190) / hi responses + hi_conn active connections.
    qps_hist: p25 10 / p95 200 (lo 40, hi 400); active_conn_hist: p25 5 / p95 25; 5-day and 300-s p95 30 msec"""
    m = early_ms if (early_ms and w < 8) else ms
    if w % 2 == 0:
        return [R(lo, m), A(3)]
    return [R(1000 if w < 8 and hi > lo else hi, m), A(hi_conn)]


def plan(probes, **bk):
    """base windows, except those listed in probes {w: chunks}"""
    return lambda w: probes[w] if w in probes else base(w, **bk)


def tail(n, nslow, ms, ser=0, **kw):
    """n responses: n - nslow at 20 msec and nslow at ms, which sets the window's p95 when nslow > 5 % of n"""
    return [R(n - nslow, 20, ser=ser, **kw), R(nslow, ms)]


SLOW_MEAN = dict(early_ms=12, ms=28)      # mean300 >= 1.1 mean5d: the transient rule :2684 cannot fire


def avg5d(at, tcount):
    """the 5-day QPS rule :2638 at window `at` (J + 1: secs_5d = age + 1 = 431 061; J + 3: secs_5d clamped at 432 000) with
    curr_qps >> 1 == 1 and tcount_5d = `tcount` samples in the 5-day level, so that avg_5day_qps = tcount_5d / secs_5d is 0 (the
    rule takes the window: OK) or 1 (it does not, and 5 high windows of the last 8 leave it BAD). Before the jump, 30 000 responses
    of 100 msec put the all-time p95 in the 100-msec bucket and four windows of 150 msec are high; after it, a FILL of the 5-day
    level at 20 msec, then at `at` 10 responses, 2 of them in the 100-msec bucket, at a mean below 1.1 of the all-time mean."""
    quiet = [R(10, 11), A(20)]                                                  # :2342 idle, not high
    probes = {8: base(8) + [R(30_000, 100)], **{w: tail(100, 10, 150) + [A(20)] for w in range(J - 4, J)},
              J: [FILL(tcount - 10 - 10 * (at - J - 1), 20), A(20)], **{w: quiet for w in range(J + 1, at)},
              at: [R(8, 11), R(2, 61), A(20)]}
    return plan(probes)


SVCS = [
    # ---- no queries: :2122
    Svc("qps0_4resp", plan({P: [R(4, 20)]}), {P: "2122"}),
    Svc("active_only", plan({P: [A(7)]}), {P: "2122"}),
    Svc("conn_only", plan({P: [T(5)]}), {P: "2122"}),
    # ---- faster than the 5-day level: :2139
    Svc("fast_lowqps", plan({P: [R(5, 5)]}), {P: "2145"}),
    Svc("fast_lowqps_ser2_eq", plan({P: [R(40, 5, ser=20)]}), {P: "2153b"}),
    Svc("fast_lowqps_ser2_gt", plan({P: [R(41, 5, ser=21)]}), {P: "2153s"}),
    Svc("fast_lowqps_ser5_eq", plan({P: [R(40, 5, ser=8)]}), {P: "2295"}),
    Svc("fast_lowqps_ser5_gt", plan({P: [R(39, 5, ser=8)]}), {P: "2153b"}),
    Svc("fast_lowqps_ser_few", plan({P: [R(50, 5, ser=4)]}), {P: "2170"}),
    Svc("fast_ser2_eq", plan({P: [R(400, 5, ser=200)]}), {P: "2228b"}),
    Svc("fast_ser2_gt", plan({P: [R(401, 5, ser=201)]}), {P: "2228s"}),
    Svc("fast_ser5_eq", plan({P: [R(400, 5, ser=80)]}), {P: "2295"}),
    Svc("fast_ser5_gt", plan({P: [R(404, 5, ser=81)]}), {P: "2228b"}),
    Svc("fast_good", plan({P: [R(400, 5)]}), {P: "2275"}),
    Svc("fast_qps_high", plan({P: [R(1105, 5)]}), {P: "2287"}),
    Svc("fastest_qps_high", plan({P: [R(1105, 1)]}), {P: "2275"}),
    # ---- the 5-day level's p95 bucket: :2307
    Svc("same_ser2", plan({P: [R(400, 20, ser=201)]}), {P: "2307s"}),
    Svc("same_ser5", plan({P: [R(400, 20, ser=100)]}), {P: "2307b"}),
    Svc("same_lowmean_lowqps_ser", plan({P: [R(40, 12, ser=2)]}), {P: "2342"}),
    Svc("same_lowmean_lowqps", plan({P: [R(40, 12)]}), {P: "2342i"}),
    Svc("same_lowmean", plan({P: [R(400, 12)]}), {P: "2386"}),
    Svc("same_lowmean_ser", plan({P: [R(400, 12, ser=10)]}), {P: "2402"}),
    Svc("same", plan({P: [R(400, 20)]}), {P: "2419"}),
    # ---- slower than the 5-day level
    Svc("slow_ser2", plan({P: tail(100, 10, 50, ser=51)}), {P: "2432s"}),
    Svc("slow_ser2_eq", plan({P: tail(100, 10, 50, ser=50)}), {P: "2432b"}),
    Svc("slow_qps_1.1_eq", plan({P: tail(1100, 105, 50)}), {P: "2684"}),
    Svc("slow_qps_1.1_gt", plan({P: tail(1105, 105, 50)}), {P: "2464"}),
    Svc("slow_qps_severe", plan({P: tail(1105, 105, 150)}), {P: "2464"}),
    Svc("slow_qps_diff5", plan({P: tail(75, 10, 50)}, lo=40, hi=40), {P: "2684"}),
    Svc("slow_qps_diff6", plan({P: tail(80, 10, 50)}, lo=40, hi=40), {P: "2464"}),
    Svc("slow_act_diff1", plan({P: tail(100, 10, 50) + [A(26)]}), {P: "2684"}),
    Svc("slow_act_diff2", plan({P: tail(100, 10, 50) + [A(27)]}), {P: "2525"}),
    Svc("slow_act_severe", plan({P: tail(100, 10, 150) + [A(27)]}), {P: "2525"}),
    Svc("slow_outlier", plan({P: [R(388, 20), R(12, 500)]}), {P: "2552"}),
    Svc("slow_lowqps", plan({P: tail(40, 5, 50) + [A(3)]}), {P: "2576"}),
    Svc("slow_transient", plan({P: tail(100, 10, 50)}), {P: "2684"}),
    Svc("slow_bitmap_nconn", plan({P: tail(100, 10, 50)}, **SLOW_MEAN), {P: "2710"}),
    # 12 reported connections, so the CONN_BITMAP counts decide curr_active_conn (14 / 15) and the slow bucket's count (3 / 4)
    Svc("slow_bitmap_15", plan({P: [R(90, 20, ports=15), R(10, 50, ports=3)]}, hi_conn=12, **SLOW_MEAN), {P: "2710"}),
    Svc("slow_bitmap_14", plan({P: [R(90, 20, ports=14), R(10, 50, ports=3)]}, hi_conn=12, **SLOW_MEAN), {P: "2855"}),
    Svc("slow_bitmap_4", plan({P: [R(90, 20, ports=15), R(10, 50, ports=4)]}, hi_conn=12, **SLOW_MEAN), {P: "2855"}),
    Svc("slow_run_bad", plan({w: tail(100, 10, 100) for w in range(P, P + 5)}), {P + 3: "2748", P + 4: "2855"}),
    Svc("slow_run_severe", plan({w: tail(100, 10, 150) for w in range(P, P + 5)}), {P + 3: "2748", P + 4: "2855"}),
    Svc("slow_run_ser", plan({w: tail(100, 10, 100, ser=1) for w in range(P, P + 5)}), {P + 3: "2748", P + 4: "2855"}),
    # ---- after the jump past 5 days: the 5-day level holds the new windows only, the all-time level everything
    Svc("slow_5day_qps", plan({**{w: base(w, ms=50) for w in range(8, J)}, J + 1: tail(400, 40, 50)}), {J + 1: "2638"}),
    # avg_5day_qps against curr_qps >> 1 on both sides, with secs_5d = age + 1 and with secs_5d clamped
    Svc("avg5d_0", avg5d(J + 1, 431_060), {J + 1: "2638"}),
    Svc("avg5d_1", avg5d(J + 1, 431_061), {J + 1: "2855"}),
    Svc("avg5d_0_clamped", avg5d(J + 3, 431_999), {J + 3: "2638"}),
    Svc("avg5d_1_clamped", avg5d(J + 3, 432_000), {J + 3: "2855"}),
    # ---- an evicted service (silent from 1250, evicted at 1610) and a new one that takes its slot after the jump
    Svc("gone", plan({**{w: tail(100, 10, 100) for w in range(6, 10)}, **{w: [] for w in range(10, NWIN)}}), {6: "2748"}),
    Svc("fresh", plan({w: [] for w in range(J)}), {J: "2419+young"}),
    # ---- 100 / 101 s after the first flush
    Svc("age_100", plan({4: [R(400, 5)], 5: [R(400, 5)]}), {4: "2275+young", 5: "2275"}),
    Svc("age_100_ser", plan({4: [R(400, 5, ser=201)], 5: [R(400, 5, ser=201)]}), {4: "2228s", 5: "2228s"}),
    # ---- a window without events: the state stays
    Svc("stale", plan({P: [], P + 1: []}), {P: "stale", P + 1: "stale"}),
]

# the exits the scenarios reach: every exit of the tree without process, host or dependency inputs except :2661 (REACHABLE_PAIRS)
NAMED_EXITS = {"2122", "2145", "2153s", "2153b", "2170", "2228s", "2228b", "2295", "2275", "2287", "2307s", "2307b", "2342", "2342i",
               "2386", "2402", "2419", "2432s", "2432b", "2464", "2525", "2552", "2576", "2638", "2684", "2710", "2748", "2855"}
# both sides of every boundary
BOUNDARY_FACTS = {("ser2", 0), ("ser2", 1), ("ser5", 0), ("ser5", 1), ("qps_diff", 5), ("qps_diff", 6), ("qps_1.1", 0), ("qps_1.1", 1),
                  ("act_diff", 1), ("act_diff", 2), ("active_conn", 14), ("active_conn", 15), ("bitmap_bucket", 3), ("bitmap_bucket", 4),
                  ("nhigh", 4), ("nhigh", 5), ("worse", 2), ("worse", 3), ("age", 100, False), ("age", 101, False), ("age", 100, True),
                  ("age", 101, True), ("avg5d", -1, False), ("avg5d", 0, False), ("avg5d", -1, True), ("avg5d", 0, True)}
for _i, _s in enumerate(SVCS):
    _s.host = _i % 3
IDLE_EVICT = 300


def run(feed, flush, src, evicted, check):
    """drive every scenario: feed(ev, fill) (fill: mask of the FILL events) and flush(tsec) the engine(s), evicted() -> ids the flush
    evicted; after every flush check(w, tsec, ids, res, state) with res = Expect.step's answer and state = the four state fields
    expected of every live service, stale ones included. Asserts every probe; returns (pairs reached, facts met)."""
    from gyeeta_b200 import synth
    ids = synth.service_ids(len(SVCS))
    ex = Expect()
    pairs, facts, exits = set(), set(), set()
    for w, t in enumerate(TIMES):
        ev, active, fill = build_window(SVCS, ids, w)
        feed(ev, fill)
        flush(t)
        gone = [int(i) for i in evicted()]
        prev = dict(ex.state)
        for i in gone:
            ex.forget(i)
        res = ex.step(src, t, [i for i in ids.tolist() if i not in gone], active)
        for s, id_ in zip(SVCS, ids.tolist()):
            if w not in s.probes:
                continue
            if s.probes[w] == "stale":
                assert id_ not in res and ex.state[id_] == prev[id_], (s.name, w)
            else:
                assert id_ in res and res[id_][1] == s.probes[w], (s.name, w, res.get(id_, (None, None))[1], s.probes[w])
                exits.add(s.probes[w].split("+")[0])
        for want, _label, f, _x in res.values():
            pairs.add(want[:2])
            facts |= f
        check(w, t, ids, res, ex.state)
    assert exits == NAMED_EXITS, sorted(NAMED_EXITS ^ exits)
    return pairs, facts, ex
