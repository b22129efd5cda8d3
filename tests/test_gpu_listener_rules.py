"""The device's listener state decision (state_kernel) at every rule exit it can reach. The scenarios of tests/listener_rules.py run
through the engine and the CPU oracle; after every flush, for every service, four answers must be equal: the device row's
(curr_state, curr_issue, issue_bit_hist, high_resp_bit_hist), the oracle's, gysk_classify_listener on inputs restated from the
device's own exports, and the scenario's named rule exit where it names one. The readers of that state — the per-host issue counts
of gysk_query_host_listen, the GYSK_TOPN_ISSUE ranking and the window read — must agree with it after every flush too."""
import ctypes as C

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200.wire import API_TRAN
from tests import listener_rules as lr
from tests.util import make_pair

pytestmark = pytest.mark.gpu



def by_id_rows(eng, ids):
    ids = np.ascontiguousarray(ids, dtype=np.uint64)
    out = (ge.SvcSummary * len(ids))()
    eng._chk(eng.L.gysk_query_svcs(eng.h, ge._p(ids), len(ids), out))
    return {int(r.glob_id): r for r in out if r.found}


class EngineSource:
    """the restatement's inputs from the device's exports; rows are read once per flush"""

    def __init__(self, eng):
        self.eng, self.rows = eng, {}

    def hist(self, id_, which):
        return self.eng.export_hist(id_, which)

    def bitmap(self, id_):
        return self.eng.export_conn_bitmap(id_, True)[1]

    def row(self, id_):
        r = self.rows[id_]
        return r.nconns_active, r.ser_errors


def api_tran(ev):
    """the responses of ev as API_TRAN records (errorcode 500 for a server error, 200 otherwise)"""
    rec = np.zeros(len(ev), dtype=API_TRAN)
    rec["tupd_usec"] = 1_700_000_000_000_000 + np.arange(len(ev))
    rec["response_usec"], rec["glob_id"], rec["cliport"] = ev["value"], ev["svc_id"], ev["flow_key"]
    rec["errorcode"] = np.where(ev["flags"] & ge.EVF_SER_ERROR, 500, 200)
    return rec


@pytest.mark.parametrize("errors", ["flags", "api_tran"])
@pytest.mark.parametrize("nbatch", [1, 3])
@pytest.mark.parametrize("hot", [False, True], ids=["hot_off", "hot_rows"])
def test_device_state_equals_oracle_restatement_and_rule(monkeypatch, hot, nbatch, errors):
    monkeypatch.setenv("GYSK_HOT_ROWS", "2048" if hot else "0")
    monkeypatch.setenv("GYSK_HOT_MIN", "8" if hot else "4096")
    eng, orc = make_pair(max_svcs=len(lr.SVCS) - 1, max_tasks=16, max_batch=1 << 14, idle_evict_secs=lr.IDLE_EVICT)
    src = EngineSource(eng)
    host_of = {}
    evicted = []

    def feed(ev, fill):
        for id_, h in zip(ev["svc_id"].tolist(), ev["host_idx"].tolist()):
            host_of[id_] = h
        for part, pfill in zip(np.array_split(ev, nbatch), np.array_split(fill, nbatch)):
            if errors == "api_tran":
                resp = (part["type"] == ge.EV_RESP) & ~pfill           # the error-free FILLs of the 5-day level stay 32-byte events
                for h in np.unique(part["host_idx"][resp]).tolist():
                    rec = api_tran(part[resp & (part["host_idx"] == h)])
                    eng.ingest_raw(ge.RAW_API_TRAN, rec, len(rec), host_idx=h)
                if (~resp).any():
                    eng.ingest_events(np.ascontiguousarray(part[~resp]))
            else:
                eng.ingest_events(np.ascontiguousarray(part))
            eng.sync()
            orc.ingest(part)

    def flush(t):
        eng.flush(t)
        orc.flush(t)
        e, o = eng.evicted_ids(), orc.evicted_ids()[0]
        assert sorted(e.tolist()) == sorted(o.tolist())
        evicted[:] = e.tolist()
        for i in evicted:
            host_of.pop(i, None)
        src.rows = by_id_rows(eng, list(host_of))

    def check(w, t, ids, res, state):
        alive = [i for i in ids.tolist() if i in host_of]
        rows = src.rows
        assert sorted(rows) == sorted(alive) == sorted(state)
        # the device row, the oracle and the restatement: this flush's evaluation, or the last one for a stale service
        expect = {}
        for id_ in alive:
            r = rows[id_]
            got = (r.curr_state, r.curr_issue, r.issue_bit_hist, r.high_resp_bit_hist)
            assert got == orc.export_state(id_)[:4] == state[id_], (w, id_, res.get(id_, (None, None))[1], got, state[id_])
            expect[id_] = got
        # per host: services evaluated at this flush with issue bit 0 set, and those of them SEVERE or worse
        hl, nh = eng.query_host_listen()
        want_hl = []
        for h in sorted(set(host_of.values())):
            on = [i for i in alive if host_of[i] == h]
            iss = [i for i in on if i in res and res[i][0][2] & 1]
            want_hl.append((h, len(on), len(iss), sum(1 for i in iss if res[i][0][0] >= ge.STATE_SEVERE)))
        assert [(r.host_idx, r.nlisten, r.nlisten_issue, r.nlisten_severe) for r in hl] == want_hl and nh == len(want_hl), w
        # GYSK_TOPN_ISSUE: every service worse than OK, worst first
        top = eng.topn(ge.TOPN_ISSUE, 64)
        bad = sorted((i, s[0], host_of[i]) for i, s in expect.items() if s[0] > ge.STATE_OK)
        assert sorted(top) == bad and [sc for _i, sc, _h in top] == sorted((s for _i, s, _h in bad), reverse=True), w
        # the window read's rows are the by-id rows, byte for byte
        wrows, n = eng.query_window()
        assert n == len(alive) and sorted(r.glob_id for r in wrows) == sorted(alive)
        for r in wrows:
            assert bytes(r) == bytes(rows[r.glob_id]), (w, r.glob_id)

    pairs, facts, _ex = lr.run(feed, flush, src, lambda: evicted, check)
    assert pairs == lr.REACHABLE_PAIRS, sorted(pairs ^ lr.REACHABLE_PAIRS)
    assert lr.BOUNDARY_FACTS <= facts, sorted(lr.BOUNDARY_FACTS - facts)
