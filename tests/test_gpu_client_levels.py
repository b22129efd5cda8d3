"""Distinct clients per window on the device (GYSK_FLAG_CLIENT_LEVELS). After every flush of the flow level's scripted sequences, each
service's exported last and 300-s registers must be byte-equal to the restatement of tests/client_levels.py, the by-id and window-read
estimates equal gysk_hll_estimate of those registers, and the window read's ids and order gysk_query_window_hosts'. Against the all-time
registers: last <= level <= fold(all-time), equal to the fold while every window is held and the open window is empty. Also every
ingest route (and the ones that never count), the hll_p edges, eviction, growth and auto-grow, a batch of more than 2^21 flows, the flag
off against on, the merge step at world 1 ... 8 (emulated) and once through NCCL, and the estimates against exact counts."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests.client_levels import BOUND, NREG, P, History, fold_registers
from tests.flow_level import SEQUENCES, flow_events
from tests.test_gpu_flow_level import _route_window, _rowbytes
from tests.test_gpu_merge import _emulate_collectives
from tests.trace_agg import api_tran

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
CFG = dict(max_svcs=1024, max_tasks=64, max_batch=1 << 14, cms_log2_width=12)


class Run:
    """one engine with the flag and the restated history of its closed windows"""

    def __init__(self, **kw):
        self.eng = ge.Engine(client_levels=True, **{**CFG, **kw})
        self.hist = History()
        self.pending = []

    def ingest(self, ev, batch=None):
        batch = batch or len(ev)
        for off in range(0, len(ev), batch):
            self.eng.ingest_events(ev[off: off + batch])
        self.eng.sync()
        self.pending.append(ev)

    def flush(self, t):
        self.eng.flush(t)
        self.hist.flush(t, np.concatenate(self.pending) if self.pending else np.zeros(0, dtype=ge.EVENT_DTYPE))
        self.pending = []

    def check(self, what=None):
        e = self.eng
        rows, hosts, n = e.query_window_hosts()
        crows, chosts, cn = e.query_clients_window()
        assert cn == n and [r.glob_id for r in crows] == [r.glob_id for r in rows] and chosts.tolist() == hosts.tolist(), what
        ids = np.array([r.glob_id for r in rows], dtype=np.uint64)
        byid = e.query_svc_clients(ids)
        assert [bytes(a) for a in byid] == [bytes(b) for b in crows], what
        for sid, r in zip(ids.tolist(), byid):
            last, lvl = e.export_hll_window(sid, ge.CLIENTS_LAST), e.export_hll_window(sid, ge.CLIENTS_5MIN)
            assert last.tobytes() == self.hist.last(sid).tobytes(), (what, sid)
            assert lvl.tobytes() == self.hist.level(sid).tobytes(), (what, sid)
            assert r.found == 1 and r.glob_id == sid
            assert r.last_5s == e.L.gysk_hll_estimate(_p(last), P) and r.last_5min == e.L.gysk_hll_estimate(_p(lvl), P), (what, sid)
            assert (last <= lvl).all()
            p = e.cfg.hll_p
            if p >= P:
                assert (lvl <= fold_registers(e.export_hll(sid), p)).all(), (what, sid)
        return ids


def _p(a):
    return a.ctypes.data_as(ge.C.c_void_p)


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_registers_after_every_flush(name):
    tsecs = SEQUENCES[name]
    rng = np.random.default_rng(200 + len(tsecs))
    keys = rng.integers(1, 1 << 62, 3000, dtype=np.uint64)
    run = Run()
    for i, t in enumerate(tsecs):
        run.ingest(flow_events(rng, int(rng.integers(500, 6000)), keys), batch=int(rng.integers(1000, 1 << 14)))
        run.flush(t)
        run.check((name, i, t))
    unknown = run.eng.query_svc_clients(np.array([0, 12345], dtype=np.uint64))
    assert [(r.found, r.last_5s, r.last_5min, r.glob_id) for r in unknown] == [(0, 0.0, 0.0, 0), (0, 0.0, 0.0, 12345)]
    assert run.eng.export_hll_window(12345) is None
    run.ingest(flow_events(rng, 3000, keys))                         # the open window is in neither answer
    run.check((name, "open"))


def test_fold_equals_the_level_while_every_window_is_held():
    """all windows inside 300 s, the open window empty: the level is the fold of the all-time registers, bit for bit"""
    rng = np.random.default_rng(3)
    keys = rng.integers(1, 1 << 62, 5000, dtype=np.uint64)
    for p in (8, 12, 16):
        run = Run(hll_p=p)
        for t in (5, 10, 40, 100, 200):
            run.ingest(flow_events(rng, 4000, keys))
            run.flush(t)
        for sid in run.check(("fold", p)).tolist():
            assert run.eng.export_hll_window(sid, ge.CLIENTS_5MIN).tobytes() == fold_registers(run.eng.export_hll(sid), p).tobytes(), (p, sid)


@pytest.mark.parametrize("hll_p", [4, 12, 16])
def test_hll_p_settings(hll_p):
    rng = np.random.default_rng(hll_p)
    keys = rng.integers(1, 1 << 62, 2000, dtype=np.uint64)
    run = Run(hll_p=hll_p)
    for t in SEQUENCES["gaps"]:
        run.ingest(flow_events(rng, 3000, keys))
        run.flush(t)
        run.check(("hll_p", hll_p, t))


@pytest.mark.parametrize("route", ["event32", "tcp24", "ipv4_raw", "ipv6_raw", "notify_tcp_conn", "notify_active_conn"])
def test_every_route_counts_and_the_others_never(route):
    """one window of the route: for every service, last = level = fold(all-time) (a record raises the window set exactly when it raises
    the all-time one). Then a window of response samples with error flags, trace events and API_TRAN records (with and without an error,
    new connections among them; the services hold trace rows, so each record is both a response sample and a trace event) only: every
    last set is empty and the all-time registers do not move"""
    rng = np.random.default_rng(sum(map(ord, route)))
    keys = rng.integers(1, 1 << 62, 500, dtype=np.uint64)
    eng = ge.Engine(client_levels=True, max_trace_svcs=64, **CFG)
    ingest, _ev, nkept, _units = _route_window(rng, route, keys, host=3)
    assert ingest(eng) in (None, 0)
    eng.sync()
    eng.flush(30)
    rows, _, n = eng.query_window_hosts()
    assert n > 0 and nkept > 0
    for r in rows:
        last, lvl = eng.export_hll_window(r.glob_id, ge.CLIENTS_LAST), eng.export_hll_window(r.glob_id, ge.CLIENTS_5MIN)
        assert last.tobytes() == lvl.tobytes() == fold_registers(eng.export_hll(r.glob_id), 12).tobytes(), (route, r.glob_id)
    ids = np.array([r.glob_id for r in rows], dtype=np.uint64)
    ev = np.zeros(4000, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = ids[rng.integers(0, len(ids), len(ev))]
    ev["flow_key"] = rng.integers(1, 1 << 62, len(ev), dtype=np.uint64)
    ev["type"] = rng.choice(np.array([ge.EV_RESP, ge.EV_TRACE], dtype=np.uint16), len(ev))
    ev["value"] = rng.integers(100, 1 << 20, len(ev))
    ev["flags"] = rng.integers(0, 4, len(ev))
    rec = api_tran(ids[rng.integers(0, len(ids), 3000)], rng.integers(100, 3_000_000, 3000).astype(np.uint64), reqlen=100, reslen=200,
                   reqnum=rng.integers(0, 3, 3000), errorcode=rng.integers(0, 2, 3000) * 500, cliport=rng.integers(40000, 40100, 3000))
    alltime = [eng.export_hll(s).tobytes() for s in ids.tolist()]
    tcp0 = eng.stats()["events_tcp"]
    eng.ingest_events(ev)
    assert eng.ingest_raw(ge.RAW_API_TRAN, rec, len(rec)) in (None, 0)
    eng.sync()
    assert eng.stats()["events_tcp"] == tcp0 and eng.trace_info()[0] > 0
    eng.flush(35)
    for s, a in zip(ids.tolist(), alltime):
        assert not eng.export_hll_window(s, ge.CLIENTS_LAST).any(), (route, s)
        assert eng.export_hll(s).tobytes() == a
    assert all(r.last_5s == 0.0 for r in eng.query_svc_clients(ids))


def test_eviction_starts_a_recycled_slot_from_zero():
    """services idle for 20 s are evicted; new services take their slots. Every answer stays the restatement's, by id: a recycled slot
    holding anything of its old service would differ. 32 new services every 8 windows, 64 slots: from the third set on every service
    takes a slot an evicted one left"""
    rng = np.random.default_rng(11)
    keys = rng.integers(1, 1 << 62, 3000, dtype=np.uint64)
    run = Run(max_svcs=64, idle_evict_secs=20)
    for i, t in enumerate(range(5, 305, 5)):
        ev = flow_events(rng, 2000, keys, nsvc=32)
        base = np.uint64(1 + (i // 8) * 32)
        ev["svc_id"] = (ev["svc_id"] // np.uint64(2654435761) - np.uint64(1) + base) * np.uint64(2654435761)
        run.ingest(ev)
        run.flush(t)
        assert run.eng.stats()["events_dropped"] == 0
        run.check(("evict", i, t))
    assert run.eng.stats()["svcs_evicted"] >= 5 * 32


def test_growth_keeps_every_answer():
    """gysk_grow inside windows, and auto-grow at flushes: every answer as the restatement's and as an engine that never grows"""
    rng = np.random.default_rng(12)
    keys = rng.integers(1, 1 << 62, 3000, dtype=np.uint64)
    run = Run(max_svcs=32)
    run.eng.set_auto_grow(max_svcs_limit=512)
    plain = ge.Engine(client_levels=True, **{**CFG, "max_svcs": 512})
    # the services in use stay below the capacity: the manual growth to 64 in window 2, then auto-grow to 128 and 256
    for i, (t, nsvc) in enumerate(zip(range(5, 200, 15), [12, 12, 20, 40, 40, 80, 80, 150, 150, 150, 150, 150, 150])):
        ev = flow_events(rng, 3000, keys, nsvc=nsvc)
        half = len(ev) // 2
        run.ingest(ev[:half])
        if i == 2:
            run.eng.grow(max_svcs=run.eng.cfg.max_svcs * 2)
        run.ingest(ev[half:])
        plain.ingest_events(ev); plain.sync()
        run.flush(t); plain.flush(t)
        assert run.eng.stats()["events_dropped"] == 0
        ids = run.check(("grow", i, t))
        assert [bytes(r) for r in run.eng.query_svc_clients(ids)] == [bytes(r) for r in plain.query_svc_clients(ids)]
    assert run.eng.capacity()["ngrows"] >= 3


def test_a_batch_of_more_than_2_21_flows():
    """3 M distinct flows in one batch over 8 services: past the batch flow table's 2^21 entries; the registers stay the restatement's"""
    rng = np.random.default_rng(13)
    n = 3_000_000
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = rng.integers(1, 9, n).astype(np.uint64)
    ev["flow_key"] = rng.permutation(n).astype(np.uint64) + np.uint64(1 << 40)
    ev["type"] = ge.EV_ACCEPT
    run = Run(max_batch=1 << 22)
    run.ingest(ev)
    run.flush(5)
    run.check("2^21")
    for r in run.eng.query_svc_clients(np.arange(1, 9, dtype=np.uint64)):
        exact = int((ev["svc_id"] == r.glob_id).sum())
        assert abs(r.last_5s - exact) <= BOUND * exact


@pytest.mark.parametrize("n", [10, 100, 1000, 10_000, 100_000])
def test_accuracy_against_exact_counts(n):
    rng = np.random.default_rng(n)
    eng = ge.Engine(client_levels=True, **{**CFG, "max_batch": 1 << 18})
    clients = rng.integers(1, 1 << 62, n, dtype=np.uint64)
    ev = np.zeros(3 * n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["type"] = 77, ge.EV_CONNECT
    ev["flow_key"] = clients[rng.integers(0, n, 3 * n)]
    ev["flow_key"][:n] = clients                           # every client at least once, most several times
    for off in range(0, len(ev), 1 << 18):
        eng.ingest_events(ev[off: off + (1 << 18)])
    eng.sync()
    eng.flush(10)
    r = eng.query_svc_clients(np.array([77], dtype=np.uint64))[0]
    assert abs(r.last_5s - n) <= BOUND * n and abs(r.last_5min - n) <= BOUND * n, (n, r.last_5s)
    assert eng.export_hll_window(77).tobytes() == po.hll_registers(clients, P).tobytes()


def _regions(eng, torch):
    from tests.test_gpu_merge_exact import _dev_bytes
    return {name.split(": ")[0]: (name, _dev_bytes(torch, ptr, nbytes)) for name, ptr, nbytes, _redop in eng.merge_buffers()}


FLAG_SETS = [dict(), dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, merge_traces=True, max_trace_svcs=64),
             dict(flow_level=True, flow_queries=True, flow_query_level=True, flow_resp_hist=True, flow_topk=True, flow_topk_5min=True,
                  flow_topk_slow=True)]


@pytest.mark.parametrize("flags", range(len(FLAG_SETS)))
def test_flag_off_and_on_answer_alike(flags):
    """the same stream through an engine without the flag and one with it: every existing answer and stat byte-equal, every merge array
    byte-equal (the client registers come after the rest of the u8 MAX region); the new calls GYSK_ERR_NOTSUP without it"""
    import torch
    rng = np.random.default_rng(40 + flags)
    keys = rng.integers(1, 1 << 62, 500, dtype=np.uint64)
    kw = {**CFG, **FLAG_SETS[flags]}
    off, on = ge.Engine(**kw), ge.Engine(client_levels=True, **kw)
    sids = np.unique(flow_events(np.random.default_rng(0), 5000, keys)["svc_id"])
    for e in (off, on):
        e.set_logical_map(sids, sids % np.uint64(5) + np.uint64(70))
    for t in (5, 10, 10, 40, 345):
        ev = flow_events(rng, 4000, keys)
        resp = np.zeros(1000, dtype=ge.EVENT_DTYPE)
        resp["svc_id"], resp["type"], resp["value"] = sids[rng.integers(0, len(sids), 1000)], ge.EV_RESP, rng.integers(100, 1 << 22, 1000)
        resp["flow_key"] = keys[rng.integers(0, len(keys), 1000)]
        ev = np.concatenate([ev, resp])
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
            (na_, a), (nb_, b) = ra[region], rb[region]
            if region == "max_u8":
                assert nb_ == na_ + "|client registers"
                b = b[: len(a)]
            else:
                assert na_ == nb_
            assert a.tobytes() == b.tobytes(), region
        assert on.query_logical_clients(lids)[0].found == 1
    calls = (lambda: off.query_svc_clients(sids), lambda: off.query_clients_window(), lambda: off.export_hll_window(int(sids[0])),
             lambda: off.query_logical_clients(sids), lambda: off.export_logical_hll_window(70))
    for call in calls:
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == NOTSUP
    fresh = ge.Engine(client_levels=True, **CFG)
    fresh.set_logical_map(sids, sids)
    for call in (lambda: fresh.query_logical_clients(sids), lambda: fresh.export_logical_hll_window(int(sids[0]))):
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == INVAL
    with pytest.raises(ge.GyskError) as ex:
        fresh.export_hll_window(int(sids[0]), 2)
    assert ex.value.code == INVAL


def _shard(ev, world):
    return [ev[ev["host_idx"] % world == r] for r in range(world)]


@pytest.mark.parametrize("spread", [True, False])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_merge_takes_the_registerwise_maximum(world, spread):
    """members spread over the ranks (events of every service on every host) or each on one rank (a service's events on one host):
    each logical service's merged registers are the registerwise maximum of every rank's member registers, and its row their estimates"""
    import torch
    rng = np.random.default_rng(world * 10 + spread)
    keys = rng.integers(1, 1 << 62, 2000, dtype=np.uint64)
    engines = [ge.Engine(client_levels=True, merge_levels=True, rank=r, world=world, **CFG) for r in range(world)]
    sids = np.arange(1, 41, dtype=np.uint64) * np.uint64(2654435761)
    lmap = sids % np.uint64(7) + np.uint64(500)
    for e in engines:
        e.set_logical_map(sids, lmap)
    lids = np.unique(lmap)
    for step, t in enumerate([30, 35, 60, 95, 300, 305]):
        ev = flow_events(rng, 6000, keys, nsvc=40)
        if not spread:
            ev["host_idx"] = (ev["svc_id"] // np.uint64(2654435761)).astype(np.uint32) % 16
        for e, sh in zip(engines, _shard(ev, world)):
            e.ingest_events(sh); e.sync()
            e.flush(t)
        _emulate_collectives(torch, engines)
        for which in (ge.CLIENTS_LAST, ge.CLIENTS_5MIN):
            for lid in lids.tolist():
                want = np.zeros(NREG, np.uint8)
                for e in engines:
                    for s in sids[lmap == np.uint64(lid)].tolist():
                        r = e.export_hll_window(s, which)
                        if r is not None:
                            np.maximum(want, r, out=want)
                for e in engines:
                    assert e.export_logical_hll_window(lid, which).tobytes() == want.tobytes(), (world, step, which, lid)
        for e in engines:
            rows = e.query_logical_clients(np.concatenate([lids, np.array([1], dtype=np.uint64)]))
            assert rows[-1].found == 0 and rows[-1].glob_id == 1 and rows[-1].last_5s == 0.0
            for lid, r in zip(lids.tolist(), rows):
                assert r.found == 1 and r.glob_id == lid
                assert r.last_5s == e.L.gysk_hll_estimate(_p(e.export_logical_hll_window(lid, ge.CLIENTS_LAST)), P)
                assert r.last_5min == e.L.gysk_hll_estimate(_p(e.export_logical_hll_window(lid, ge.CLIENTS_5MIN)), P)
            assert e.export_logical_hll_window(1) is None


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(5)
    keys = rng.integers(1, 1 << 62, 2000, dtype=np.uint64)
    eng = ge.Engine(client_levels=True, **CFG)
    sids = np.unique(flow_events(np.random.default_rng(0), 5000, keys)["svc_id"])
    eng.set_logical_map(sids, sids % np.uint64(3))
    for t in (30, 35, 65):
        eng.ingest_events(flow_events(rng, 5000, keys)); eng.sync()
        eng.flush(t)
    _emulate_collectives(torch, [eng])
    lids = np.arange(3, dtype=np.uint64)
    emulated = [bytes(r) for r in eng.query_logical_clients(lids)]
    regs = [eng.export_logical_hll_window(int(l), w).tobytes() for l in lids for w in (0, 1)]
    eng.nccl_comm_init(eng.nccl_unique_id(), 1, 0)
    eng.merge_global()
    eng.sync()
    assert [bytes(r) for r in eng.query_logical_clients(lids)] == emulated
    assert [eng.export_logical_hll_window(int(l), w).tobytes() for l in lids for w in (0, 1)] == regs
