"""GYSK_FLAG_FLOW_QUERIES on the device. After every batch and flush: gysk_export_cms_queries (open and last window) byte-equal to the
tables restated from the events (tests/flow_queries.py), each point query equal to the min-over-rows restatement and at least the exact
per-key counts, every row's query halves summing to the services' open-window request counts, and the batch flow tables empty. Covered:
event32 mixed batches with hot rows forced on and off, RESP16, raw IPv4 / IPv6, API_TRAN with and without trace rows, more distinct flows
in one batch than the flow table holds, the sketch-setting edges, samples beyond the validity rule, unknown ids and a full service table,
eviction with recycled slots and a gysk_grow inside a window, GYSK_FLAG_FLOW_LEVEL on; then flag off against on in every existing answer
and merge array, the accuracy bound, and the merge at 1, 2, 3, 5 and 8 emulated ranks and through the library's NCCL path."""
import math

import numpy as np
import pytest

from gyeeta_b200 import engine as ge, synth
from gyeeta_b200.wire import RESP4, RESP6
from tests import flow_queries as fq
from tests.test_gpu_flow_level import _arrays, _rowbytes
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_sketch_accuracy import fold_ip6, raw_svc_id
from tests.trace_agg import api_tran, resp_events

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
FLOW_ENT_MAX = 1 << 21
CFG = dict(max_svcs=1024, max_tasks=64, max_batch=1 << 17, cms_depth=4, cms_log2_width=14)


class Run:
    """one engine with the flag and the restated tables, fed the same samples"""

    def __init__(self, **kw):
        self.eng = ge.Engine(flow_queries=True, **kw)
        c = self.eng.cfg
        self.d, self.w = c.cms_depth, c.cms_log2_width
        self.cur = np.zeros(self.d << self.w, dtype=np.uint64)
        self.last = self.cur.copy()
        self.samples = []                       # the open window's counted samples
        self.ids = set()                        # services with counted samples in the open window

    def batch(self, ev, known=None, ingest=None, what=None):
        """ev: the batch as the library expands it; known: the ids that have a slot (None: every id)"""
        (ingest or (lambda e: e.ingest_events(ev)))(self.eng)
        self.eng.sync()
        s = fq.counted(ev, known)
        fq.add_samples(self.cur, s, self.d, self.w)
        self.samples.append(s)
        self.ids |= set(np.unique(s["svc_id"]).tolist())
        self.check(what, nqrys=True)

    def flush(self, t, what=None):
        self.eng.flush(t)
        self.last, self.cur = self.cur, np.zeros_like(self.cur)
        self.samples, self.ids = [], set()
        self.check(what)

    def check(self, what, nqrys=False):
        e = self.eng
        assert e.flow_table_used() == 0, what
        assert e.export_cms_queries().tobytes() == self.cur.tobytes(), what
        assert e.export_cms_queries(last_window=True).tobytes() == self.last.tobytes(), what
        s = np.concatenate(self.samples) if self.samples else np.zeros(0, dtype=ge.EVENT_DTYPE)
        keys = np.unique(s["flow_key"])[:3000]
        if len(keys):
            got = e.query_flow_queries(keys)
            q, m = fq.point_query(self.cur, keys, self.d, self.w)
            assert np.array_equal(got["flow_key"], keys) and np.array_equal(got["queries"], q) and np.array_equal(got["resp_ms"], m), what
            for (eq, em), a, b in zip(fq.exact(s, keys), q.tolist(), m.tolist()):
                assert a >= eq and b >= em, what
            lastq = e.query_flow_queries(keys, last_window=True)
            assert np.array_equal(lastq["queries"], fq.point_query(self.last, keys, self.d, self.w)[0]), what
        if nqrys:
            # the request count of every service's open window, from its histogram
            total = sum(int(e.export_hist(int(i), 0)[1]) for i in self.ids)
            assert total == len(s), what
            assert fq.row_sums(self.cur, self.d, self.w) == [total & fq.U32] * self.d, what


def _mixed(rng, n, nsvc=300, nclients=4000):
    ev = synth.gen_mixed(rng, n, nsvc, ntask=32, nhosts=16, nclients=nclients)
    r = np.flatnonzero(ev["type"] == ge.EV_RESP)
    ev["value"][r[::211]] = fq.VALID_USEC + 5            # beyond the validity rule: not counted
    return ev


@pytest.mark.parametrize("hot", ["on", "off"])
def test_event32_hot_rows_on_and_off(hot, monkeypatch):
    if hot == "on":
        monkeypatch.setenv("GYSK_HOT_MIN", "64")        # busy services turn hot after their first batch
    else:
        monkeypatch.setenv("GYSK_HOT_ROWS", "0")
    rng = np.random.default_rng(1 if hot == "on" else 2)
    run = Run(**CFG)
    for i, step in enumerate(["b", "b", "b", 5, "b", "b", 10, 15, "b"]):
        if step == "b":
            run.batch(_mixed(rng, int(rng.integers(30_000, 90_000))), what=(hot, i))
        else:
            run.flush(step, what=(hot, i))
    assert (run.eng.hot_rows_in_use() > 0) == (hot == "on")
    assert run.eng.last_batch_flow_query_direct() == 0
    st = run.eng.stats()
    assert st["events_resp"] > 0 and st["events_tcp"] > 0


def _raw_resp(rng, n, dtype, ipv6):
    rec = np.zeros(n, dtype=dtype)
    if ipv6:
        rec["saddr"] = [0x20010DB8, 0, 0, 1]
        rec["daddr"] = rng.integers(0, 1 << 32, (n, 4)) & np.array([0xFFFFFFFF, 0, 0, 0xFF], dtype=np.int64)
    else:
        rec["saddr"], rec["daddr"] = 0x0A000001, rng.integers(1, 200, n)
    rec["netns"] = 4026531840
    rec["sport"] = np.uint16(8080).byteswap()
    rec["dport"] = rng.integers(30000, 30050, n).astype(np.uint16).byteswap()
    rec["lrcvtime"] = rng.integers(0, 1 << 30, n)
    ms = rng.integers(0, 20000, n).astype(np.uint32)
    ms[::40] = 2_000_000                                  # dropped on the host
    rec["lsndtime"] = rec["lrcvtime"] + ms
    return rec


def _expanded(svc, keys, usec, ok):
    ev = np.zeros(int(ok.sum()), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"], ev["value"], ev["type"] = svc, keys[ok], usec[ok], ge.EV_RESP
    return ev


@pytest.mark.parametrize("route", ["ipv4", "ipv6", "resp16", "api_tran", "api_tran_traced"])
def test_every_response_route(route):
    rng = np.random.default_rng(sum(map(ord, route)))
    run = Run(max_trace_svcs=64 if route == "api_tran_traced" else 0, **CFG)
    for w, t in enumerate([5, 10, 15]):
        for b in range(2):
            n = 6000
            if route in ("ipv4", "ipv6"):
                rec = _raw_resp(rng, n, RESP6 if route == "ipv6" else RESP4, route == "ipv6")
                ms, ok = fq.resp_usec_raw(rec)
                keys = fq.route_key_ipv6(rec) if route == "ipv6" else fq.route_key_ipv4(rec)
                svc = raw_svc_id(fold_ip6([0x20010DB8, 0, 0, 1]) if route == "ipv6" else 0x0A000001, 8080)
                ev = _expanded(svc, keys, ms * np.uint32(1000), ok)
                kind = ge.RAW_TCP_IPV6_RESP if route == "ipv6" else ge.RAW_TCP_IPV4_RESP
            elif route == "resp16":
                rec = np.zeros(n, dtype=ge.RESP16_DTYPE)
                rec["svc_id"] = rng.integers(1, 40, n).astype(np.uint64) * np.uint64(1000003)
                rec["usec"], rec["cli_port"] = rng.integers(0, 3_000_000, n), rng.integers(0, 256, n)
                rec["usec"][::50] = fq.VALID_USEC + 1
                ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
                ev["svc_id"], ev["flow_key"], ev["value"], ev["type"] = rec["svc_id"], fq.route_key_resp16(rec), rec["usec"], ge.EV_RESP
                kind = ge.RAW_RESP16
            else:
                ids = rng.integers(1, 40, n).astype(np.uint64) * np.uint64(1000003)
                usec = rng.integers(0, 3_000_000, n).astype(np.uint64)
                usec[::50] = fq.VALID_USEC + 7
                rec = api_tran(ids, usec, reqlen=100, reslen=200, cliport=rng.integers(40000, 40100, n))
                ev = resp_events(rec)
                assert np.array_equal(ev["flow_key"], fq.route_key_api_tran(rec))
                kind = ge.RAW_API_TRAN
            run.batch(ev, ingest=lambda e, kind=kind, rec=rec: e.ingest_raw(kind, rec, len(rec)), what=(route, w, b))
        run.flush(t, what=(route, w))


def test_more_flows_than_the_table():
    """2.5 M response samples of distinct flows in one batch: the query flow table takes at most 2^21 of them, the rest update their
    cells directly; a small batch after it goes through the table again"""
    rng = np.random.default_rng(7)
    run = Run(max_svcs=1024, max_tasks=64, max_batch=1 << 22, stage_batch=1 << 22, cms_depth=4, cms_log2_width=20)
    n = 2_500_000
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = rng.integers(1, 200, n).astype(np.uint64) * np.uint64(7919)
    ev["flow_key"] = synth.splitmix64(np.arange(1, n + 1, dtype=np.uint64))
    ev["value"], ev["type"] = rng.integers(0, 1 << 22, n), ge.EV_RESP
    run.batch(ev, what="distinct")
    assert run.eng.last_batch_flow_query_direct() >= n - FLOW_ENT_MAX
    assert run.eng.last_batch_flow_direct() == 0
    run.batch(_mixed(rng, 50_000), what="after")
    assert run.eng.last_batch_flow_query_direct() == 0
    run.flush(5, what="flush")


@pytest.mark.parametrize("depth,log2w,flow_level", [(1, 4, False), (8, 4, True), (1, 22, False), (8, 22, True)])
def test_sketch_edges_and_flow_level(depth, log2w, flow_level):
    rng = np.random.default_rng(depth * 100 + log2w)
    run = Run(**dict(CFG, cms_depth=depth, cms_log2_width=log2w), flow_level=flow_level)
    for i, step in enumerate(["b", "b", 30, "b", 35]):
        if step == "b":
            run.batch(_mixed(rng, 60_000), what=(depth, log2w, i))
        else:
            run.flush(step, what=(depth, log2w, i))


def test_unknown_ids_and_a_full_table():
    """without auto-registration only registered ids count; with it, ids beyond a full table do not"""
    rng = np.random.default_rng(11)
    run = Run(**dict(CFG, auto_register=False))
    ev = _mixed(rng, 50_000, nsvc=200)
    ids = np.unique(ev["svc_id"][ev["type"] == ge.EV_RESP])
    reg = ids[::2]
    run.eng.register_ids(reg)
    run.batch(ev, known=set(reg.tolist()), what="registered")
    run.flush(5, what="flush")
    full = Run(**dict(CFG, max_svcs=64))
    first = np.zeros(20_000, dtype=ge.EVENT_DTYPE)
    svc = (np.arange(64, dtype=np.uint64) + np.uint64(1)) * np.uint64(104729)
    first["svc_id"], first["type"] = svc[rng.integers(0, 64, len(first))], ge.EV_RESP
    first["svc_id"][:64] = svc                          # every one of the 64 ids: the table is full after this batch
    first["flow_key"], first["value"] = rng.integers(1, 5000, len(first)), rng.integers(0, 1 << 22, len(first))
    full.batch(first, what="fill")
    more = first.copy()
    more["svc_id"][::3] = (np.arange(len(more[::3]), dtype=np.uint64) % np.uint64(30) + np.uint64(100)) * np.uint64(7)     # new ids: no slot
    full.batch(more, known=set(svc.tolist()), what="full")
    assert full.eng.stats()["events_dropped"] > 0


def test_eviction_recycled_slots_and_grow():
    rng = np.random.default_rng(13)
    run = Run(**dict(CFG, max_svcs=256, idle_evict_secs=10))
    def ev_of(lo, hi, n=20_000):
        ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = rng.integers(lo, hi, n).astype(np.uint64) * np.uint64(6151)
        ev["flow_key"], ev["value"], ev["type"] = rng.integers(1, 3000, n), rng.integers(0, 1 << 22, n), ge.EV_RESP
        return ev
    run.batch(ev_of(1, 150), what="a")
    for t in (5, 10, 20, 35, 60):
        run.flush(t, what=("idle", t))
    run.batch(ev_of(200, 380), what="recycled")            # the first services were evicted: their slots taken by new ids
    assert run.eng.stats()["svcs_evicted"] > 0
    run.eng.grow(max_svcs=1024)
    run.batch(ev_of(400, 900), what="after grow")
    run.flush(65, what="flush")
    assert run.eng.stats()["events_dropped"] == 0


def test_flag_off_and_on_answer_alike():
    import torch
    rng = np.random.default_rng(17)
    for flags in (dict(), dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, flow_level=True)):
        off, on = ge.Engine(**CFG, **flags), ge.Engine(flow_queries=True, **CFG, **flags)
        ev0 = _mixed(np.random.default_rng(0), 20_000)
        sids = np.unique(ev0["svc_id"][ev0["type"] != ge.EV_TASK])
        for e in (off, on):
            e.set_logical_map(sids, sids % np.uint64(7) + np.uint64(50))
        for t in (5, 10, 40):
            ev = _mixed(rng, 40_000)
            for e in (off, on):
                e.ingest_events(ev); e.sync()
            keys = np.unique(ev["flow_key"])[:2000]
            for lw in (False, True):
                assert off.export_cms(lw).tobytes() == on.export_cms(lw).tobytes()
                assert off.query_flows(keys, lw).tobytes() == on.query_flows(keys, lw).tobytes()
            assert _rowbytes(off.query_svcs(sids)) == _rowbytes(on.query_svcs(sids))
            for i in sids[:40].tolist():
                a, b = off.export_hist(i, 0), on.export_hist(i, 0)
                assert (a is None) == (b is None) and (a is None or (np.array_equal(a[0], b[0]) and a[1:] == b[1:]))
                assert np.array_equal(off.export_hll(i), on.export_hll(i))
            sa, sb = off.stats(), on.stats()
            assert sa == sb
            for e in (off, on):
                e.flush(t)
            for e in (off, on):
                _emulate_collectives(torch, [e])
            a, b = _arrays(off, torch), _arrays(on, torch)
            for k in [k for k in a if k[1] != "rest"]:
                buf, o, size = a[k]
                buf2, o2, _ = b[k]
                assert buf[o: o + size].tobytes() == buf2[o2: o2 + size].tobytes(), k
            for region in ("sum_u64", "max_i64", "max_u8"):
                assert a[region, "rest"].tobytes() == b[region, "rest"].tobytes(), (flags, region)
            assert ("sum_u64", "cms_qry_cur") in b and ("sum_u64", "cms_qry_cur") not in a
    for call in (lambda: off.query_flow_queries(keys), off.export_cms_queries, lambda: off.query_flow_queries_global(keys),
                 off.last_batch_flow_query_direct):
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == NOTSUP
    fresh = ge.Engine(flow_queries=True, **CFG)
    with pytest.raises(ge.GyskError) as ex:
        fresh.query_flow_queries_global(keys)
    assert ex.value.code == INVAL


@pytest.mark.parametrize("depth", [1, 4, 8])
@pytest.mark.parametrize("log2w", [10, 16, 20])
def test_accuracy_bound(depth, log2w):
    """the share of keys whose estimate exceeds the exact count by more than ceil(e / w * N) stays within e^-d + 0.01"""
    rng = np.random.default_rng(depth * 31 + log2w)
    w = 1 << log2w
    nkeys = min(4 * w, 1 << 20)
    keys = synth.splitmix64(np.arange(1, nkeys + 1, dtype=np.uint64) + np.uint64(log2w << 40))
    n = min(8 * nkeys, 1 << 22)
    zipf = np.minimum(rng.zipf(1.3, n) - 1, nkeys - 1)
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"], ev["value"], ev["type"] = 12345, keys[zipf], rng.integers(0, 1 << 20, n), ge.EV_RESP
    eng = ge.Engine(flow_queries=True, max_svcs=64, max_tasks=16, max_batch=1 << 22, stage_batch=1 << 22, cms_depth=depth, cms_log2_width=log2w)
    eng.ingest_events(ev); eng.sync()
    sample = keys[rng.choice(nkeys, min(nkeys, 200_000), replace=False)]
    got = eng.query_flow_queries(sample)["queries"].astype(np.int64)
    exact = np.array([e[0] for e in fq.exact(ev, sample)], dtype=np.int64)
    assert np.all(got >= exact)
    slack = math.ceil(math.e / w * n)
    share = float(np.mean(got - exact > slack))
    assert share <= math.exp(-depth) + 0.01, (depth, log2w, share)


def _shard(ev, world):
    return [ev[ev["host_idx"] % world == r] for r in range(world)]


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_merge_sums_the_ranks_tables(world):
    import torch
    rng = np.random.default_rng(world)
    engines = [ge.Engine(flow_queries=True, rank=r, world=world, **CFG) for r in range(world)]
    for e in engines:
        e.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    for t in (5, 10):
        ev = _mixed(rng, 40_000)
        for e in engines:
            e.ingest_events(ev); e.sync()          # each rank keeps its own hosts' events
        if t == 5:
            for e in engines:
                e.flush(t)
    _emulate_collectives(torch, engines)
    keys = np.unique(ev["flow_key"])[:500]
    for lw, name in ((False, "cms_qry_cur"), (True, "cms_qry_last")):
        want = sum((e.export_cms_queries(lw) for e in engines[1:]), engines[0].export_cms_queries(lw).copy())
        for e in engines:
            buf, off, size = _arrays(e, torch)["sum_u64", name]
            assert buf[off: off + size].view(np.uint64).tobytes() == want.tobytes(), (world, name)
            got = e.query_flow_queries_global(keys, lw)
            q, m = fq.point_query(want, keys, e.cfg.cms_depth, e.cfg.cms_log2_width)
            assert np.array_equal(got["queries"], q) and np.array_equal(got["resp_ms"], m), (world, lw)


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(5)
    eng = ge.Engine(flow_queries=True, **CFG)
    eng.set_logical_map(np.array([1], dtype=np.uint64), np.array([1], dtype=np.uint64))
    for t in (5, 10):
        eng.ingest_events(_mixed(rng, 30_000)); eng.sync()
        eng.flush(t)
    eng.ingest_events(_mixed(rng, 30_000)); eng.sync()
    keys = rng.integers(1, 5000, 300).astype(np.uint64)
    _emulate_collectives(torch, [eng])
    emulated = [eng.query_flow_queries_global(keys, lw).tobytes() for lw in (False, True)]
    eng.nccl_comm_init(eng.nccl_unique_id(), 1, 0)
    eng.merge_global()
    eng.sync()
    assert [eng.query_flow_queries_global(keys, lw).tobytes() for lw in (False, True)] == emulated
    assert emulated[0] == eng.query_flow_queries(keys).tobytes()
