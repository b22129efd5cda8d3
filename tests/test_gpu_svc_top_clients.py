"""Each service's heaviest clients on the device (GYSK_FLAG_SVC_TOP_CLIENTS). After every device batch each service's open row, and after
every flush of the flow level's scripted sequences its last and 300-s rows, must be byte-equal to the restatement of
tests/svc_top_clients.py, the window read row for row the by-id read, and the guarantees must hold against exact per-client sums, which
add up to the service's own nconns_5s / kbytes_5s. Also every counting route (and the records that never count), the split path of a
service with 2^20 clients in one batch, 2^17 services with one client each, a batch of max_batch connection records, eviction, growth
and auto-grow, the refusals, and the flag off against on."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import svc_top_clients as tc
from tests.flow_level import SEQUENCES, flow_events
from tests.test_gpu_flow_level import _route_window, _rowbytes

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
CFG = dict(max_svcs=1024, max_tasks=64, max_batch=1 << 14, cms_log2_width=12)
WHICH = (ge.TOPC_OPEN, ge.TOPC_LAST, ge.TOPC_5MIN)


def _noise(rng, ids, n):
    """response samples with error flags, trace events and process samples: none of them counts"""
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = ids[rng.integers(0, len(ids), n)]
    ev["flow_key"] = rng.integers(1, 1 << 62, n, dtype=np.uint64)
    ev["type"] = rng.choice(np.array([ge.EV_RESP, ge.EV_TRACE, ge.EV_TASK], dtype=np.uint16), n)
    ev["value"] = rng.integers(100, 1 << 20, n)
    ev["flags"] = rng.integers(0, 4, n)
    return ev


def _body(r):
    """the bytes of a row after its id and found word"""
    return np.asarray(r["n"]).tobytes() + np.asarray(r["delta"]).tobytes() + np.asarray(r["entries"]).tobytes()


def _expect(summary):
    out = np.zeros(1, dtype=ge.SVC_TOP_CLIENTS_DTYPE)[0]
    n, delta, a = tc.row(summary)
    out["n"], out["delta"] = n, delta
    out["entries"]["flow_key"], out["entries"]["kbytes"], out["entries"]["conns"] = a[:, 0], a[:, 1], a[:, 2]
    return out


class Run:
    """one engine with the flag, the restatement and the exact sums of the open window"""

    def __init__(self, **kw):
        self.eng = ge.Engine(svc_top_clients=True, max_trace_svcs=64, **{**CFG, **kw})
        self.model = tc.TopClients()
        self.open_exact, self.last_exact = {}, {}
        self.seen = set()

    def batch(self, ev, what=None):
        """one device batch (at most max_batch events), then every seen service's open row"""
        self.eng.ingest_events(ev)
        self.eng.sync()
        self.model.batch(ev)
        for s, d in tc.batch_sums(ev).items():
            o = self.open_exact.setdefault(s, {})
            for k, (kb, c) in d.items():
                a = o.setdefault(k, [0, 0])
                a[0] += kb
                a[1] += c
        self.seen |= set(np.unique(ev["svc_id"]).tolist())
        self.check((ge.TOPC_OPEN,), what)

    def flush(self, t, what=None):
        self.eng.flush(t)
        self.model.evict(self.eng.evicted_ids())
        self.model.flush(t)
        self.last_exact, self.open_exact = self.open_exact, {}
        self.check((ge.TOPC_LAST, ge.TOPC_5MIN), what)

    def check(self, which, what=None):
        e = self.eng
        ids = np.array(sorted(self.seen | {0, 12345}), dtype=np.uint64)
        for w in which:
            rows = e.query_svc_top_clients(ids, w)
            for sid, r in zip(ids.tolist(), rows):
                want = _expect(self.model.get(w, sid))
                assert r["glob_id"] == sid
                assert _body(r) == _body(want), (what, w, sid, r, want)
            wrows, hosts, n = e.query_top_clients_window(w)
            vrows, vhosts, vn = e.query_window_hosts()
            assert n == vn and wrows["glob_id"].tolist() == [v.glob_id for v in vrows] and hosts.tolist() == vhosts.tolist(), what
            assert wrows.tobytes() == e.query_svc_top_clients(wrows["glob_id"], w).tobytes(), what
        if ge.TOPC_LAST in which:
            live = [s for s in self.seen if s in self.last_exact]
            summ = {r["glob_id"]: r for r in e.query_svcs(np.array(live, dtype=np.uint64))}
            for s in live:
                ex = self.last_exact[s]
                assert sum(v[1] for v in ex.values()) == summ[s]["nconns_5s"], (what, s)
                assert sum(v[0] for v in ex.values()) & 0xFFFFFFFF == summ[s]["kbytes_5s"], (what, s)
                tc.check_guarantees(self.model.get(ge.TOPC_LAST, s), ex)


@pytest.mark.parametrize("hot", [True, False])
@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_rows_after_every_batch_and_flush(name, hot, monkeypatch):
    if not hot:
        monkeypatch.setenv("GYSK_HOT_ROWS", "0")
    tsecs = SEQUENCES[name]
    rng = np.random.default_rng(300 + len(tsecs) + hot)
    keys = rng.integers(1, 1 << 62, 60, dtype=np.uint64)          # few clients: services hold fewer, about and more than K
    run = Run()
    for i, t in enumerate(tsecs):
        for b in range(int(rng.integers(1, 4))):
            ev = flow_events(rng, int(rng.integers(200, 5000)), keys[: int(rng.integers(5, len(keys)))], nsvc=int(rng.integers(4, 64)))
            ev = np.concatenate([ev, _noise(rng, np.unique(ev["svc_id"]), 2000)])
            run.batch(rng.permutation(ev), (name, i, b))
        run.flush(t, (name, i, t))


def test_guarantees_against_exact_over_windows():
    """the 300-s level's guarantees over the records of the windows it holds, on Zipf traffic"""
    from tests.flow_level import held_windows
    rng = np.random.default_rng(5)
    keys = rng.integers(1, 1 << 62, 4000, dtype=np.uint64)
    run = Run()
    tsecs, windows = [], []
    for t in SEQUENCES["steps_5s"][:30]:
        ev = flow_events(rng, 6000, keys[np.minimum(rng.zipf(1.2, 6000), len(keys)) - 1], nsvc=8)
        ev["flow_key"] = keys[np.minimum(rng.zipf(1.2, len(ev)), len(keys)) - 1]
        run.batch(ev)
        run.flush(t)
        tsecs.append(t)
        windows.append(ev)
        held = np.concatenate([windows[i] for i in held_windows(tsecs)])
        for s, ex in tc.batch_sums(held).items():
            tc.check_guarantees(run.model.get(ge.TOPC_5MIN, s), ex)
            r = run.eng.query_svc_top_clients(np.array([s], dtype=np.uint64), ge.TOPC_5MIN)[0]
            assert r["n"] > 0


@pytest.mark.parametrize("route", ["event32", "tcp24", "ipv4_raw", "ipv6_raw", "notify_tcp_conn", "notify_active_conn"])
def test_every_route_counts_and_the_others_never(route):
    """one window of the route: rows as the restatement of the route's events (the raw routes, whose services the host derives: the
    guarantees against each service's own kbytes_5s / nconns_5s). Then a window of response samples, trace events, process samples and
    API_TRAN records only: every last row is empty"""
    from tests.trace_agg import api_tran
    rng = np.random.default_rng(sum(map(ord, route)))
    keys = rng.integers(1, 1 << 62, 40, dtype=np.uint64)
    eng = ge.Engine(svc_top_clients=True, max_trace_svcs=64, **CFG)
    ingest, ev, nkept, _units = _route_window(rng, route, keys, host=3)
    assert ingest(eng) in (None, 0)
    eng.sync()
    eng.flush(30)
    rows, _, n = eng.query_window_hosts()
    assert n > 0 and nkept > 0
    ids = np.array([r.glob_id for r in rows], dtype=np.uint64)
    got = eng.query_svc_top_clients(ids, ge.TOPC_LAST)
    if ev is not None:
        model = tc.TopClients()
        model.batch(ev)
        model.flush(30)
        for r in got:
            want = _expect(model.get(ge.TOPC_LAST, r["glob_id"]))
            assert _body(r) == _body(want), (route, r["glob_id"])
    if route == "notify_active_conn":
        assert (got["n"] == 0).all() and (got["delta"] == 0).all()
    else:
        assert (got["n"] > 0).any()
    for r, s in zip(got, rows):
        kb = r["entries"]["kbytes"].astype(np.int64)
        assert kb.sum() + (tc.K + 1) * int(r["delta"]) <= s.kbytes_5s
        assert int(r["entries"]["conns"].sum()) <= s.nconns_5s
    rec = api_tran(ids[rng.integers(0, len(ids), 3000)], rng.integers(100, 3_000_000, 3000).astype(np.uint64), reqlen=100, reslen=200,
                   reqnum=rng.integers(0, 3, 3000), errorcode=rng.integers(0, 2, 3000) * 500, cliport=rng.integers(40000, 40100, 3000))
    eng.ingest_events(_noise(rng, ids, 4000))
    assert eng.ingest_raw(ge.RAW_API_TRAN, rec, len(rec)) in (None, 0)
    eng.sync()
    assert (eng.query_svc_top_clients(ids, ge.TOPC_OPEN)["n"] == 0).all()
    eng.flush(35)
    last = eng.query_svc_top_clients(ids, ge.TOPC_LAST)
    assert (last["n"] == 0).all() and (last["delta"] == 0).all()


def _one_service_batch(rng, sid, nclients, n):
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["type"] = sid, ge.EV_CLOSE_SER
    ev["flow_key"] = rng.permutation(nclients).astype(np.uint64)[np.arange(n) % nclients] + np.uint64(1 << 40)
    ev["value"] = (rng.zipf(1.5, n) % 5000) << 10
    return ev


def test_split_path_of_a_service_with_2_20_clients():
    """2^20 distinct clients of one service in one batch: the segment is cut into pieces; the row stays the restatement's, with old
    entries met in some pieces and not in others"""
    rng = np.random.default_rng(21)
    run = Run(max_batch=1 << 21, max_svcs=64)
    run.batch(_one_service_batch(rng, 77, 40, 400), "seed")
    ev = _one_service_batch(rng, 77, 1 << 20, (1 << 20) + 5000)
    ev["flow_key"][:20] = run.model.get(ge.TOPC_OPEN, 77)[0][0][0]      # the heaviest old client among the new ones
    run.batch(ev, "2^20")
    run.flush(5, "2^20")
    tc.check_guarantees(run.model.get(ge.TOPC_LAST, 77), run.last_exact[77])


def test_2_17_services_with_one_client_each():
    rng = np.random.default_rng(22)
    n = 1 << 17
    run = Run(max_batch=1 << 18, max_svcs=n + 16)
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = np.arange(1, n + 1, dtype=np.uint64) * np.uint64(2654435761)
    ev["flow_key"], ev["type"], ev["value"] = rng.integers(1, 1 << 62, n, dtype=np.uint64), ge.EV_CONNECT, rng.integers(0, 1 << 22, n)
    run.batch(ev)
    run.flush(5)


def test_a_batch_of_max_batch_connection_records():
    rng = np.random.default_rng(23)
    mb = 1 << 20
    run = Run(max_batch=mb, max_svcs=4096)
    keys = rng.integers(1, 1 << 62, 1 << 16, dtype=np.uint64)
    ev = flow_events(rng, mb, keys, nsvc=3000)
    ev["type"][ev["type"] == ge.EV_ACTIVE] = ge.EV_ACCEPT
    run.batch(ev)
    run.flush(5)


def test_eviction_starts_a_recycled_slot_from_zero():
    """services idle for 20 s are evicted, new ones take their slots: every row stays the restatement's, which drops the evicted
    services' summaries"""
    rng = np.random.default_rng(11)
    keys = rng.integers(1, 1 << 62, 40, dtype=np.uint64)
    run = Run(max_svcs=64, idle_evict_secs=20)
    for i, t in enumerate(range(5, 305, 5)):
        ev = flow_events(rng, 2000, keys, nsvc=32)
        base = np.uint64(1 + (i // 8) * 32)
        ev["svc_id"] = (ev["svc_id"] // np.uint64(2654435761) - np.uint64(1) + base) * np.uint64(2654435761)
        run.batch(ev, ("evict", i))
        run.flush(t, ("evict", i, t))
        assert run.eng.stats()["events_dropped"] == 0
    assert run.eng.stats()["svcs_evicted"] >= 5 * 32


def test_growth_keeps_every_answer():
    """gysk_grow inside a window, and auto-grow at flushes: every row the restatement's"""
    rng = np.random.default_rng(12)
    keys = rng.integers(1, 1 << 62, 50, dtype=np.uint64)
    run = Run(max_svcs=32)
    run.eng.set_auto_grow(max_svcs_limit=512)
    for i, (t, nsvc) in enumerate(zip(range(5, 200, 15), [12, 12, 20, 40, 40, 80, 80, 150, 150, 150, 150, 150, 150])):
        ev = flow_events(rng, 3000, keys, nsvc=nsvc)
        half = len(ev) // 2
        run.batch(ev[:half], ("grow", i))
        if i == 2:
            run.eng.grow(max_svcs=run.eng.cfg.max_svcs * 2)
            run.check(WHICH, ("grown", i))
        run.batch(ev[half:], ("grow", i))
        run.flush(t, ("grow", i, t))
        assert run.eng.stats()["events_dropped"] == 0
    assert run.eng.capacity()["ngrows"] >= 3


def test_refusals():
    off = ge.Engine(**CFG)
    ids = np.array([1], dtype=np.uint64)
    for call in (lambda: off.query_svc_top_clients(ids), lambda: off.query_top_clients_window()):
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == NOTSUP
    on = ge.Engine(svc_top_clients=True, **CFG)
    for w in (-1, 3):
        for call in (lambda: on.query_svc_top_clients(ids, w), lambda: on.query_top_clients_window(w)):
            with pytest.raises(ge.GyskError) as ex:
                call()
            assert ex.value.code == INVAL
    r = on.query_svc_top_clients(np.array([0, 99], dtype=np.uint64), ge.TOPC_LAST)
    assert r["glob_id"].tolist() == [0, 99] and (r["found"] == 0).all() and not _body(r).strip(b"\0")


FLAG_SETS = [dict(), dict(client_levels=True, flow_level=True, flow_queries=True, flow_query_level=True, flow_resp_hist=True, flow_topk=True,
                          flow_topk_5min=True, flow_topk_slow=True, flow_errors=True, merge_levels=True, merge_states=True, merge_topn=True,
                          merge_traces=True, max_trace_svcs=64, idle_evict_secs=20)]


@pytest.mark.parametrize("flags", range(len(FLAG_SETS)))
def test_flag_off_and_on_answer_alike(flags):
    """the same stream through an engine without the flag and one with it: every existing answer and stat byte-equal (kernel launches
    aside), every merge array byte-equal"""
    import torch
    from tests.test_gpu_client_levels import _regions
    from tests.test_gpu_merge import _emulate_collectives
    rng = np.random.default_rng(40 + flags)
    keys = rng.integers(1, 1 << 62, 500, dtype=np.uint64)
    kw = {**CFG, **FLAG_SETS[flags]}
    off, on = ge.Engine(**kw), ge.Engine(svc_top_clients=True, **kw)
    sids = np.unique(flow_events(np.random.default_rng(0), 5000, keys)["svc_id"])
    for e in (off, on):
        e.set_logical_map(sids, sids % np.uint64(5) + np.uint64(70))
    for t in (5, 10, 10, 40, 345):
        ev = np.concatenate([flow_events(rng, 4000, keys), _noise(rng, sids, 1000)])
        for e in (off, on):
            e.ingest_events(ev); e.sync()
            e.flush(t)
        for lw in (False, True):
            assert off.export_cms(lw).tobytes() == on.export_cms(lw).tobytes()
        assert _rowbytes(off.query_svcs(sids)) == _rowbytes(on.query_svcs(sids))
        assert all(off.export_hll(s).tobytes() == on.export_hll(s).tobytes() for s in sids.tolist())
        (wa, na), (wb, nb) = off.query_window(), on.query_window()
        assert na == nb and sorted(bytes(r) for r in wa) == sorted(bytes(r) for r in wb)
        sa, sb = off.stats(), on.stats()
        assert {k: v for k, v in sa.items() if k != "kernel_launches"} == {k: v for k, v in sb.items() if k != "kernel_launches"}
        for e in (off, on):
            _emulate_collectives(torch, [e])
        lids = np.unique(sids % np.uint64(5) + np.uint64(70))
        assert _rowbytes(off.query_logical(lids)) == _rowbytes(on.query_logical(lids))
        ra, rb = _regions(off, torch), _regions(on, torch)
        assert sorted(ra) == sorted(rb)
        for region in ra:
            assert ra[region][0] == rb[region][0] and ra[region][1].tobytes() == rb[region][1].tobytes(), region
        assert (on.query_svc_top_clients(sids, ge.TOPC_LAST)["n"] > 0).any()
