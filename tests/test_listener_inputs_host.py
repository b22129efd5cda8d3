"""The restatement of the listener state decision's inputs (tests/listener_rules.py) pinned to the CPU oracle: after every flush of
the scenarios, the classifier on inputs restated from the oracle's exports gives the oracle's own four state fields for every
service, and the scenarios reach every rule exit and both sides of every boundary they name."""
import numpy as np

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests import listener_rules as lr


class OracleSource:
    def __init__(self, orc):
        self.orc = orc

    def hist(self, id_, which):
        return self.orc.export_hist(id_, which)

    def bitmap(self, id_):
        return self.orc.export_conn_bitmap(id_, True)[1]

    def row(self, id_):
        a = self.orc.export_aux(id_)
        return a["act_last"] & lr.M32, a["err_last"] >> 32


def test_rule_exit_agrees_with_the_classifier_and_reaches_14_pairs():
    """without process, host or dependency inputs the tree gives exactly the 14 pairs of REACHABLE_PAIRS (the other four need
    those inputs), and rule_exit's outcome is gysk_classify_listener's and the oracle's on 60 000 random inputs"""
    rng = np.random.default_rng(5)
    vals = [0, 1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000, 32767]
    qv = [-1, 1, 10, 50, 200, 500, 1000, 3000, 6000, 2147483647]
    av = [-1, 1, 5, 10, 25, 50, 75, 100, 32767]
    seen, labels = set(), set()
    for _ in range(60_000):
        x = ge.ListenerStateIn()
        base = int(rng.integers(1, 13))
        for f in ("r5p95", "r5p99", "r300p95", "r300p99", "r5dp95", "r5dp99", "r5dp25", "rallp95", "rallp99"):
            setattr(x, f, vals[int(np.clip(base + rng.integers(-2, 3), 0, 14))])
        x.nqrys_5s = int(rng.choice([0, 3, 40, 500, 20_000]))
        x.total_resp_msec = int(x.nqrys_5s * rng.integers(1, 200))
        x.tcount_5d = int(rng.integers(0, 10_000_000))
        m = float(rng.integers(1, 300))
        x.mean5, x.mean300, x.mean5d, x.meanall = m, m * float(rng.choice([0.7, 0.95, 1.0, 1.3])), m * float(rng.choice([0.7, 1.0, 1.15, 1.5])), m * float(rng.choice([0.8, 1.0, 1.2]))
        q = sorted(int(v) for v in rng.choice(qv, 2)); a = sorted(int(v) for v in rng.choice(av, 2))
        x.qps_p25, x.qps_p95, x.act_p25, x.act_p95 = q[0], q[1], a[0], a[1]
        x.secs_5d = int(rng.choice([1, 300, 432000]))
        x.last_qps_count = int(rng.choice([0, 2, 45, 210, 5000]))
        x.nconn = int(rng.integers(0, 200))
        x.curr_active_conn = x.nconn + int(rng.choice([0, 0, 1, 30]))          # the engine's curr_active_conn is never below nconn
        x.ser_errors = int(rng.choice([0, 0, 0, 1, 30, 400, 0x90000000]))
        for b in range(15):
            x.nactive_conn_arr[b] = int(rng.integers(0, 6))
        hb = int(rng.integers(0, 256))
        label, st, iss, _f = lr.rule_exit(x, hb)
        g = ge.classify_listener(x, hb)
        assert (st, iss) == g[:2] == po.listener_state(x, hb)[:2], (label, st, iss, g)
        seen.add(g[:2])
        labels.add(label)
    assert seen == lr.REACHABLE_PAIRS, sorted(seen ^ lr.REACHABLE_PAIRS)
    assert "2661" not in labels


def test_restated_inputs_reproduce_the_oracle_states():
    orc = po.OracleEngine(max_svcs=len(lr.SVCS) - 1, max_tasks=16)
    orc.set_idle_evict(lr.IDLE_EVICT)
    src = OracleSource(orc)
    nchecked = [0]

    def check(w, t, ids, res, state):
        for id_, want in state.items():                     # the services evaluated at this flush and the stale ones
            assert orc.export_state(id_)[:4] == want, (w, id_, res.get(id_, (None, None))[1])
            nchecked[0] += 1
        for _want, _label, _f, x in res.values():
            assert x.curr_active_conn >= x.nconn

    pairs, facts, ex = lr.run(lambda ev, _fill: orc.ingest(ev), orc.flush, src, lambda: orc.evicted_ids()[0], check)
    assert pairs == lr.REACHABLE_PAIRS, sorted(pairs ^ lr.REACHABLE_PAIRS)
    assert lr.BOUNDARY_FACTS <= facts, sorted(lr.BOUNDARY_FACTS - facts)
    assert nchecked[0] > 1000
