"""The flow error tables and the server-error sets on the device (GYSK_FLAG_FLOW_ERRORS). Batches are driven one by one, and after every
batch and flush the open, last and 300-s exports must equal the restatement of tests/flow_errors.py byte for byte; every error half must be
at most the query half of the same flow query cell; after each flush each row's error halves of the last table must sum to the services'
last-window cli_errors / ser_errors; the point queries must equal the min-over-rows restatement and be at least the exact counts; and the
sets must equal their restatement, with the guarantee and B_L holding against exact counts.
Covered: event32 with hot rows on and off, API_TRAN with errorcode 0 / 1 / 499 / 500 / 503 (traced and not), raw IPv4 / IPv6 responses,
trace events and samples beyond the validity rule, the direct path, the sketch edges, eviction with growth, the level's flush sequences,
set sizes around K with ties, client-error-only flows, the flag off against on, and the merge at world 1 ... 8 emulated on one GPU and once
through NCCL."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import flow_errors as fe
from tests import flow_level as fl
from tests import flow_queries as fq
from tests.test_gpu_flow_level import _rowbytes
from tests.test_gpu_flow_query_level import _regions, _route_batch
from tests.test_gpu_flow_topk import CFG, _mixed, _shard
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import _dev_bytes
from tests.trace_agg import api_tran, resp_events

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
K = fe.K
LEVEL = dict(flow_topk_5min=True, flow_query_level=True)
SLAB_ENTRY = 4128                                                       # sizeof(SlabEntry)
U32 = np.uint64(0xFFFFFFFF)


def _slab_bytes(nsets):
    return -(-nsets * (K + 2) * 8 // SLAB_ENTRY) * SLAB_ENTRY


def _resp(keys, flags, msec=20, svc=1000003):
    ev = np.zeros(len(keys), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"], ev["type"] = svc, keys, ge.EV_RESP
    ev["value"] = np.uint32(msec * 1000 + 500)
    ev["flags"] = flags
    return ev


def _err_mixed(rng, n, share=0.05, **kw):
    """_mixed with a share of its responses carrying the client and / or server error bit, and a few low-volume clients that always get
    server errors"""
    ev = _mixed(rng, n, **kw)
    r = np.flatnonzero(ev["type"] == ge.EV_RESP)
    pick = r[rng.random(len(r)) < share]
    ev["flags"][pick] = rng.choice([1, 2, 3], len(pick), p=[0.5, 0.4, 0.1])
    few = r[:40]
    ev["flow_key"][few] = np.uint64(1 << 50) + (np.arange(len(few), dtype=np.uint64) % np.uint64(8))
    ev["flags"][few] = ge.EVF_SER_ERROR
    return ev


class Run:
    """one engine with the flag (topk: the server-error sets; level: the 300-s tables and sets), the restated tables and sets"""

    def __init__(self, topk=True, level=False, svc_check=True, **kw):
        flags = dict(flow_queries=True, flow_topk=topk, flow_query_level=level, flow_topk_5min=level and topk)
        self.eng = ge.Engine(flow_errors=True, **{**CFG, **flags, **kw})
        c = self.eng.cfg
        self.d, self.w = c.cms_depth, c.cms_log2_width
        self.topk, self.level, self.svc_check = topk, level, svc_check
        self.open, self.last = fe.empty(self.d, self.w), fe.empty(self.d, self.w)
        self.ring = fl.FlowLevelRing(self.d << self.w) if level else None
        self.sets = fe.Sets(self.d, self.w)
        self.lv = fe.LevelSets(self.d, self.w) if level and topk else None
        self.win, self.tsecs, self.history, self.ids = [], [], [], set()
        self.nb = 0

    def batch(self, ev, known=None, ingest=None, what=None):
        assert len(ev) <= (self.eng.cfg.stage_batch or min(self.eng.cfg.max_batch, 1 << 22))      # one device batch
        (ingest or (lambda e: e.ingest_events(ev)))(self.eng)
        self.eng.sync()
        self.nb += 1
        assert self.eng.stats()["batches"] == self.nb, what
        s = fq.counted(ev, known)
        fe.add_samples(self.open, s, self.d, self.w)
        self.sets.batch(fe.ser_keys(s), self.open)
        self.win.append(s)
        self.ids |= set(np.unique(ev["svc_id"][ev["type"] == ge.EV_RESP]).tolist())
        self.check(what)

    def flush(self, t, what=None):
        closing = self.open
        self.eng.flush(t)
        if self.ring is not None:
            self.ring.flush(t, closing)
            self.tsecs.append(t)
            self.history.append(np.concatenate(self.win) if self.win else fq.counted(np.zeros(0, dtype=ge.EVENT_DTYPE), None))
        if self.lv is not None:
            self.lv.flush(t, self.sets.open, closing)
        self.sets.flush()
        self.last, self.open = closing, fe.empty(self.d, self.w)
        self.last_win = np.concatenate(self.win) if self.win else fq.counted(np.zeros(0, dtype=ge.EVENT_DTYPE), None)
        self.win = []
        self.check(what, flushed=True)

    def check(self, what, flushed=False):
        e, d, w = self.eng, self.d, self.w
        for lw, want in ((False, self.open), (True, self.last)):
            got = e.export_cms_errors(lw).reshape(-1)
            assert got.tobytes() == want.tobytes(), (what, lw)
            q = e.export_cms_queries(lw).reshape(-1)
            assert np.all((got & U32) <= (q & U32)) and np.all((got >> np.uint64(32)) <= (q & U32)), (what, lw)
        if self.win:
            s = np.concatenate(self.win)
            keys = np.unique(np.concatenate([s["flow_key"][:3000], np.arange(7, 70, dtype=np.uint64) << np.uint64(40)]))
            rows = e.query_flow_errors(keys, False)
            assert rows.tobytes() == fe.point_query(self.open, e.export_cms_queries(False).reshape(-1), keys, d, w).tobytes(), what
            ex = fe.exact(s, keys)
            assert np.all(rows["cli_errors"] >= ex[:, 0]) and np.all(rows["ser_errors"] >= ex[:, 1]), what
            assert rows["queries"].tobytes() == e.query_flow_queries(keys, False)["queries"].tobytes(), what
        if flushed and self.svc_check and self.ids:
            sv = e.query_svcs(np.array(sorted(self.ids), dtype=np.uint64))
            cli = int(sum(int(r["cli_errors"]) for r in sv)) & 0xFFFFFFFF
            ser = int(sum(int(r["ser_errors"]) for r in sv)) & 0xFFFFFFFF
            assert all(rs == (cli, ser) for rs in fe.row_sums(self.last, d, w)), (what, cli, ser)
        if self.ring is not None:
            level = e.export_cms_errors_5min().reshape(-1)
            assert level.tobytes() == self.ring.level.tobytes(), what
            q5 = e.export_cms_queries_5min().reshape(-1)
            assert np.all((level & U32) <= (q5 & U32)) and np.all((level >> np.uint64(32)) <= (q5 & U32)), what
        if not self.topk:
            return
        for lw, keys, tab in ((False, self.sets.open, self.open), (True, self.sets.last, self.last)):
            got = e.topk_flow_errors(K, lw)
            want = fe.read(keys, tab, e.export_cms_queries(lw).reshape(-1), d, w)
            assert got.tobytes() == want.tobytes(), (what, lw, len(got), len(want))
            assert got.tobytes() == e.query_flow_errors(got["flow_key"], lw).tobytes(), (what, lw)
            assert np.all(got["ser_errors"] > 0) and np.all(got["ser_errors"][:-1] >= got["ser_errors"][1:]), (what, lw)
        if self.win:
            s = np.concatenate(self.win)
            allk = np.unique(s["flow_key"])
            ex = fe.exact(s, allk)[:, 1]
            members = set(self.sets.open.tolist())
            t = fe.fs.thr(self.sets.open, self.open, d, w, fe.ser_score) if len(self.sets.open) == K else 0
            assert all(k in members for k, x in zip(allk.tolist(), ex.tolist()) if x > t), what
        if self.lv is not None:
            rows, bound = e.topk_flow_errors_5min(K)
            level = e.export_cms_errors_5min().reshape(-1)
            assert rows.tobytes() == fe.read(self.lv.L, level, e.export_cms_queries_5min().reshape(-1), d, w).tobytes(), what
            assert bound == self.lv.B, (what, bound, self.lv.B)
            assert rows.tobytes() == e.query_flow_errors_5min(rows["flow_key"]).tobytes(), what
            if self.tsecs:
                held = [self.history[j] for j in fl.held_windows(self.tsecs)]
                held = np.concatenate(held)
                keys = np.unique(held["flow_key"])
                members = set(self.lv.L.tolist())
                assert all(x <= bound for k, x in zip(keys.tolist(), fe.exact(held, keys)[:, 1].tolist()) if k not in members), what


@pytest.mark.parametrize("hot", ["on", "off"])
def test_event32_hot_rows_on_and_off(hot, monkeypatch):
    if hot == "on":
        monkeypatch.setenv("GYSK_HOT_MIN", "64")
    else:
        monkeypatch.setenv("GYSK_HOT_ROWS", "0")
    rng = np.random.default_rng(1 if hot == "on" else 2)
    run = Run()
    for i, step in enumerate(["b", "b", "b", 5, "b", "b", 10, 15, "b"]):
        if step == "b":
            run.batch(_err_mixed(rng, int(rng.integers(30_000, 90_000))), what=(hot, i))
        else:
            run.flush(step, what=(hot, i))
    assert (run.eng.hot_rows_in_use() > 0) == (hot == "on")
    assert run.eng.last_batch_flow_err_direct() == 0


@pytest.mark.parametrize("traced", [False, True])
def test_api_tran_errorcodes(traced):
    """API_TRAN: errorcode 0 counts nowhere, 1 and 499 as client errors, 500 and 503 as server errors, all under the client port; the
    trace events beside them never count"""
    rng = np.random.default_rng(3 + traced)
    run = Run(max_trace_svcs=8 if traced else 0)
    for i in range(3):
        n = 6000
        ids = rng.integers(1, 20, n).astype(np.uint64) * np.uint64(1000003)
        usec = rng.integers(0, 3_000_000, n).astype(np.uint64)
        usec[::50] = fq.VALID_USEC + 7
        rec = api_tran(ids, usec, reqlen=100, reslen=200, errorcode=rng.choice([0, 1, 499, 500, 503], n), cliport=rng.integers(40000, 40100, n))
        run.batch(resp_events(rec), ingest=lambda e: e.ingest_raw(ge.RAW_API_TRAN, rec, len(rec)), what=(traced, i))
        if i == 1:
            run.flush(5, what=(traced, i))
    assert run.open.any()
    got = run.eng.topk_flow_errors(K)["flow_key"]
    assert np.all(got >= 40000) and np.all(got < 40100)


@pytest.mark.parametrize("route", ["ipv4", "ipv6"])
def test_raw_responses_never_count(route):
    rng = np.random.default_rng(5)
    run = Run()
    ev, ingest = _route_batch(rng, route)
    run.batch(ev, ingest=ingest, what=route)
    run.flush(5, what=route)
    assert not run.last.any() and len(run.eng.topk_flow_errors(K, True)) == 0


def test_trace_and_invalid_samples_never_count():
    rng = np.random.default_rng(6)
    run = Run(max_trace_svcs=8)
    ev = _err_mixed(rng, 20_000)
    tr = ev[:500].copy()
    tr["type"], tr["value"], tr["flags"] = ge.EV_TRACE, 5_000, 3
    tr["flow_key"] = np.arange(10**9, 10**9 + 500, dtype=np.uint64)
    bad = _resp(np.arange(2 * 10**9, 2 * 10**9 + 300, dtype=np.uint64), 3)
    bad["value"] = fq.VALID_USEC + 5
    unknown = _resp(np.arange(3 * 10**9, 3 * 10**9 + 300, dtype=np.uint64), 2, svc=0)
    known = set(np.unique(ev["svc_id"]).tolist()) | {1000003}
    run.batch(np.concatenate([ev, tr, bad, unknown]), known=known, what="trace")
    keys = np.concatenate([tr["flow_key"], bad["flow_key"], unknown["flow_key"]])
    assert not set(run.eng.topk_flow_errors(K)["flow_key"].tolist()) & set(keys.tolist())
    run.flush(5)


@pytest.mark.parametrize("nflows", [K - 1, K, K + 1, 3 * K])
def test_set_sizes_and_ties(nflows):
    rng = np.random.default_rng(nflows)
    run = Run(cms_log2_width=20)
    keys = rng.choice(1 << 40, nflows, replace=False).astype(np.uint64)
    nser = np.where(np.arange(nflows) % 3 == 0, 4, rng.integers(0, 3, nflows))      # a long run of score 4, many 0, 1 and 2
    ev = np.concatenate([_resp(np.repeat(keys, nser), ge.EVF_SER_ERROR), _resp(keys, 0), _resp(keys[::5], ge.EVF_CLI_ERROR)])
    run.batch(ev, what=nflows)
    assert len(run.eng.topk_flow_errors(K)) == min(K, int((nser > 0).sum()))
    run.batch(_resp(keys[: nflows // 2], 3), what=nflows)
    run.flush(5)


def test_client_error_only_flows_never_listed():
    rng = np.random.default_rng(7)
    run = Run(cms_log2_width=16)
    cli = rng.choice(1 << 40, 3000, replace=False).astype(np.uint64)
    ser = rng.choice(1 << 40, 20, replace=False).astype(np.uint64) | np.uint64(1 << 41)
    ev = np.concatenate([_resp(np.repeat(cli, 14), ge.EVF_CLI_ERROR), _resp(np.repeat(ser, 2), ge.EVF_SER_ERROR)])
    run.batch(ev, what="cli")
    assert set(run.eng.topk_flow_errors(K)["flow_key"].tolist()) == set(ser.tolist())


def test_direct_path():
    """more than 2^21 distinct error flows in one batch: most error samples take the direct path of the error flow table"""
    rng = np.random.default_rng(8)
    n = (1 << 21) + 300_000
    run = Run(max_batch=1 << 22, cms_log2_width=20, svc_check=False)
    keys = rng.integers(1, 1 << 62, n, dtype=np.uint64)
    run.batch(_resp(keys, rng.integers(1, 4, n)), what="direct")
    assert run.eng.last_batch_flow_err_direct() > 0
    run.flush(5, what="direct")
    run.batch(_resp(keys[:100_000], 2), what="direct2")
    assert run.eng.last_batch_flow_err_direct() < 100                  # a batch the table holds goes through it again


@pytest.mark.parametrize("depth,log2w", [(1, 4), (8, 4), (1, 22), (8, 22)])
def test_sketch_edges(depth, log2w):
    rng = np.random.default_rng(depth * 100 + log2w)
    run = Run(cms_depth=depth, cms_log2_width=log2w)
    for i, step in enumerate(["b", "b", 5, "b"]):
        if step == "b":
            run.batch(_err_mixed(rng, 40_000), what=(depth, log2w, i))
        else:
            run.flush(step)


def test_eviction_recycled_slots_and_growth():
    rng = np.random.default_rng(19)
    run = Run(max_svcs=256, idle_evict_secs=20, svc_check=False)
    for i, t in enumerate([5, 10, 100, 105, 140]):
        run.batch(_err_mixed(rng, 20_000, nsvc=200 if i < 2 else 60), what=("evict", i))
        if i == 2:
            run.eng.grow(512, 128)
            run.batch(_err_mixed(rng, 20_000, nsvc=60), what=("grown", i))
        run.flush(t, what=("evict", i))
    assert run.eng.stats()["svcs_evicted"] > 0


@pytest.mark.parametrize("seq", sorted(fl.SEQUENCES))
def test_level_flush_sequences(seq):
    rng = np.random.default_rng(len(seq) + 40)
    run = Run(level=True, flow_level=True)
    for i, t in enumerate(fl.SEQUENCES[seq]):
        run.batch(_err_mixed(rng, 20_000, nclients=3000), what=(seq, i))
        run.flush(t, what=(seq, i))


def test_without_topk_and_refusals():
    rng = np.random.default_rng(9)
    run = Run(topk=False, level=True)
    for i, t in enumerate((5, 30, 35)):
        run.batch(_err_mixed(rng, 20_000), what=i)
        run.flush(t, what=i)
    for call in (lambda e: e.topk_flow_errors(), lambda e: e.topk_flow_errors_global(), lambda e: e.topk_flow_errors_5min(),
                 lambda e: e.topk_flow_errors_global_5min()):
        with pytest.raises(ge.GyskError) as ex:
            call(run.eng)
        assert ex.value.code == NOTSUP
    without = ge.Engine(**CFG, flow_queries=True, flow_topk=True, **LEVEL)
    for call in (lambda e: e.query_flow_errors([1]), lambda e: e.query_flow_errors_5min([1]), lambda e: e.query_flow_errors_global([1]),
                 lambda e: e.query_flow_errors_global_5min([1]), lambda e: e.export_cms_errors(), lambda e: e.export_cms_errors_5min(),
                 lambda e: e.topk_flow_errors(), lambda e: e.topk_flow_errors_5min(), lambda e: e.topk_flow_errors_global(),
                 lambda e: e.topk_flow_errors_global_5min(), lambda e: e.last_batch_flow_err_direct()):
        with pytest.raises(ge.GyskError) as ex:
            call(without)
        assert ex.value.code == NOTSUP
    with pytest.raises(ge.GyskError) as ex:
        ge.Engine(flow_errors=True, **CFG)
    assert ex.value.code == INVAL
    nolevel = ge.Engine(flow_errors=True, flow_queries=True, flow_topk=True, **CFG)
    for call in (lambda e: e.query_flow_errors_5min([1]), lambda e: e.export_cms_errors_5min(), lambda e: e.topk_flow_errors_5min()):
        with pytest.raises(ge.GyskError) as ex:
            call(nolevel)
        assert ex.value.code == NOTSUP
    for call in (lambda e: e.topk_flow_errors_global(), lambda e: e.query_flow_errors_global([1])):
        with pytest.raises(ge.GyskError) as ex:
            call(nolevel)
        assert ex.value.code == INVAL                  # before the first merge


OTHER = {"alone": {}, "flow_level": dict(flow_level=True), "query_level": dict(flow_query_level=True),
         "resp_hist": dict(flow_resp_hist=True), "topk": dict(flow_topk=True),
         "topk_all": dict(flow_topk=True, flow_resp_hist=True, flow_topk_slow=True, flow_level=True, **LEVEL),
         "client_levels": dict(client_levels=True),
         "merge": dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True, merge_traces=True, max_trace_svcs=64,
                       flow_topk=True, flow_resp_hist=True, flow_topk_slow=True, flow_level=True, client_levels=True, **LEVEL)}


def _calls(flags):
    topk, level, rh = flags.get("flow_topk"), flags.get("flow_query_level"), flags.get("flow_resp_hist")
    out = [lambda e, k, lw: e.export_cms(lw), lambda e, k, lw: e.export_cms_queries(lw), lambda e, k, lw: e.query_flow_queries(k, lw),
           lambda e, k, lw: e.query_flows(k, lw)]
    if topk:
        out += [lambda e, k, lw: e.topk_flows(K, lw), lambda e, k, lw: e.topk_flow_queries(K, lw)]
    if rh:
        out += [lambda e, k, lw: e.export_cms_resp(lw)]
    if flags.get("flow_topk_slow"):
        out += [lambda e, k, lw: e.topk_flow_slow(K, lw)]
    if level:
        out += [lambda e, k, lw: e.export_cms_queries_5min()]
    if flags.get("flow_level"):
        out += [lambda e, k, lw: e.export_cms_5min()]
    return out


@pytest.mark.parametrize("other", sorted(OTHER))
def test_flag_off_and_on_answer_alike(other):
    import torch
    rng = np.random.default_rng(27)
    flags = {**CFG, "flow_queries": True, **OTHER[other]}
    off, on = ge.Engine(**flags), ge.Engine(flow_errors=True, **flags)
    topk, level = flags.get("flow_topk"), "flow_topk_5min" in flags
    ncms = (off.cfg.cms_depth << off.cfg.cms_log2_width) * 8
    ev0 = _mixed(np.random.default_rng(0), 20_000)
    sids = np.unique(ev0["svc_id"][ev0["type"] != ge.EV_TASK])
    for e in (off, on):
        e.set_logical_map(sids, sids % np.uint64(7) + np.uint64(50))
    lids = np.unique(sids % np.uint64(7) + np.uint64(50))
    for i, t in enumerate((5, 10, 40, 40, 300)):
        ev = _err_mixed(rng, 40_000)
        for e in (off, on):
            e.ingest_events(ev); e.sync()
        keys = np.unique(ev["flow_key"])[:2000]
        for lw in (False, True):
            for call in _calls(flags):
                assert call(off, keys, lw).tobytes() == call(on, keys, lw).tobytes(), (other, i)
        if level:
            for call in (lambda e: e.topk_flows_5min(K), lambda e: e.topk_flow_queries_5min(K)):
                a, b = call(off), call(on)
                assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1]
        assert _rowbytes(off.query_svcs(sids)) == _rowbytes(on.query_svcs(sids))
        sa, sb = off.stats(), on.stats()
        sa.pop("kernel_launches"); sb.pop("kernel_launches")
        assert sa == sb
        assert off.last_batch_flow_query_direct() == on.last_batch_flow_query_direct() and on.last_batch_flow_err_direct() == 0
        for e in (off, on):
            e.flush(t)
        for e in (off, on):
            _emulate_collectives(torch, [e])
        ra, rb = _regions(off, torch), _regions(on, torch)
        assert set(ra) == set(rb)
        for region in ra:
            na, ba = ra[region]
            nb, bb = rb[region]
            if region != "sum_u64":
                assert (na, ba.tobytes()) == (nb, bb.tobytes()), region
                continue
            # the error tables follow the other count-min tables; everything else is byte-equal
            errs = [n for n in nb if n.startswith("cms_err_")]
            assert [n for n in nb if n not in errs] == na and errs == (["cms_err_cur", "cms_err_last"] + (["cms_err_5min"] if level or
                                                                       flags.get("flow_query_level") else []))
            size = lambda n: (ncms * (8 if n.startswith("cms_resp_") else 1) + 255) & ~255
            step = size("cms_err_cur")
            lo = sum(size(n) for n in nb[: nb.index(errs[0])])
            hi = lo + len(errs) * step
            assert bb[:lo].tobytes() + bb[hi:].tobytes() == ba.tobytes(), region
            assert bb[lo: lo + ncms].tobytes() == on.export_cms_errors(False).tobytes()
            assert bb[lo + step: lo + step + ncms].tobytes() == on.export_cms_errors(True).tobytes()
        pa, na_ = off.merge_tdigest_slab()
        pb, nb_ = on.merge_tdigest_slab()
        sa_, sb_ = _dev_bytes(torch, pa, na_).tobytes(), _dev_bytes(torch, pb, nb_).tobytes()
        assert sa_[: len(lids) * SLAB_ENTRY] == sb_[: len(lids) * SLAB_ENTRY]
        if topk:
            # the heaviest-flow, level and slow sets, before the server-error ones
            tk = _slab_bytes(2) * (2 if level else 1) + (_slab_bytes(2 if level else 1) if flags.get("flow_topk_slow") else 0)
            assert sa_[na_ - tk:] == sb_[na_ - tk: na_]
            assert nb_ - na_ == _slab_bytes(2 if level else 1)
            new = np.frombuffer(sb_[na_:], dtype=np.uint64)
            rows = on.topk_flow_errors(K, True)
            assert new[0] >= len(rows) and new[2: 2 + len(rows)].tolist() == rows["flow_key"].tolist()
            assert off.topk_flows_global().tobytes() == on.topk_flows_global().tobytes()
            assert off.topk_flow_queries_global().tobytes() == on.topk_flow_queries_global().tobytes()
        else:
            assert nb_ == na_
        assert _rowbytes(off.query_logical(lids)) == _rowbytes(on.query_logical(lids))
        for lw in (False, True):
            assert off.query_flow_queries_global(keys, lw).tobytes() == on.query_flow_queries_global(keys, lw).tobytes()
        if level:
            for call in (lambda e: e.topk_flows_global_5min(K), lambda e: e.topk_flow_queries_global_5min(K)):
                a, b = call(off), call(on)
                assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1]
            assert off.merge_flush_range() == on.merge_flush_range()
    assert off.capacity()["device_bytes"] < on.capacity()["device_bytes"]


def _check_merge(ranks, what):
    engines = [r.eng for r in ranks]
    d, w, level = ranks[0].d, ranks[0].w, ranks[0].level
    total = lambda f: sum((f(e).reshape(-1) for e in engines[1:]), f(engines[0]).reshape(-1).copy())
    summed, summed_q = total(lambda e: e.export_cms_errors(True)), total(lambda e: e.export_cms_queries(True))
    keys = np.unique(np.concatenate([r.last_win["flow_key"][:3000] for r in ranks] + [np.arange(1, 50, dtype=np.uint64)]))
    g = fe.merged([r.sets.last for r in ranks], summed, d, w)
    want = fe.read(g, summed, summed_q, d, w)
    for e in engines:
        assert e.query_flow_errors_global(keys, True).tobytes() == fe.point_query(summed, summed_q, keys, d, w).tobytes(), what
        got = e.topk_flow_errors_global()
        assert got.tobytes() == want.tobytes(), what
        assert got.tobytes() == e.query_flow_errors_global(got["flow_key"], True).tobytes(), what
    if level:
        summed5, summed5_q = total(lambda e: e.export_cms_errors_5min()), total(lambda e: e.export_cms_queries_5min())
        g5, bg = fe.merged([r.lv.L for r in ranks], summed5, d, w, bounds=[r.lv.B for r in ranks])
        want5 = fe.read(g5, summed5, summed5_q, d, w)
        for e in engines:
            rows, bound = e.topk_flow_errors_global_5min()
            assert rows.tobytes() == want5.tobytes() and bound == bg, what
            assert rows.tobytes() == e.query_flow_errors_global_5min(rows["flow_key"]).tobytes(), what


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("others", ["alone", "merge"])
def test_merge_sums_and_ranks_the_union(world, others):
    import torch
    rng = np.random.default_rng(world * 10 + 7)
    extra = {k: v for k, v in OTHER["merge"].items() if k not in LEVEL and k != "flow_topk"} if others == "merge" else {}
    level = others == "merge"
    ranks = [Run(level=level, rank=r, world=world, svc_check=False, **extra) for r in range(world)]
    for step, t in enumerate([30, 35, 60]):
        ev = _err_mixed(rng, 60_000, nclients=3000)
        for run, sh in zip(ranks, _shard(ev, world)):
            run.batch(sh, what=(world, others, step))
            run.flush(t, what=(world, others, step))
        _emulate_collectives(torch, [r.eng for r in ranks])
        _check_merge(ranks, (world, others, step))


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(5)
    run = Run(level=True, flow_level=True)
    for t in (30, 35):
        run.batch(_err_mixed(rng, 30_000))
        run.flush(t)
    _emulate_collectives(torch, [run.eng])
    keys = np.arange(1, 3000, dtype=np.uint64)
    emulated = run.eng.topk_flow_errors_global().tobytes(), run.eng.topk_flow_errors_global_5min(), run.eng.query_flow_errors_global(keys, True)
    assert emulated[0] == run.eng.topk_flow_errors(K, True).tobytes()
    run.eng.nccl_comm_init(run.eng.nccl_unique_id(), 1, 0)
    run.eng.merge_global()
    run.eng.sync()
    got = run.eng.topk_flow_errors_global().tobytes(), run.eng.topk_flow_errors_global_5min(), run.eng.query_flow_errors_global(keys, True)
    assert got[0] == emulated[0] and got[1][0].tobytes() == emulated[1][0].tobytes() and got[1][1] == emulated[1][1]
    assert got[2].tobytes() == emulated[2].tobytes()
