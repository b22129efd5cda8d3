"""The rolling 300-s count-min level on the device (GYSK_FLAG_FLOW_LEVEL). After every flush of the scripted sequences of
tests/flow_level.py, gysk_export_cms_5min must be byte-equal to the host sum of the live windows' gysk_export_cms(last_window=1) tables
and to the oracle's level (the ring restatement fed the oracle's closed windows), and gysk_query_flows_5min must equal the min-over-rows
restatement of that table and be at least the exact counts and kbytes of the stream. Also: every ingest route, the sketch-setting
edges with a wrapping kbytes half, growth and eviction, the flag off against on over the same stream, and the merge step at world 1 ... 8
with the collectives emulated on one GPU, and once through the library's NCCL path."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200.wire import TCP_CONN, build_msg
from oracle import pyoracle as po
from tests.flow_level import M32, SEQUENCES, FlowLevelRing, exact_flows, flow_events, held_windows, level_of_history, point_query
from tests.test_gpu_boundary import ACTIVE, CONN6, fixed_msg
from tests.test_gpu_merge import _emulate_collectives

pytestmark = pytest.mark.gpu

NOTSUP = -95
CFG = dict(max_svcs=1024, max_tasks=64, max_batch=1 << 14, cms_log2_width=12)
CONN4 = np.dtype([("ts_ns", "<u8"), ("bytes_received", "<u8"), ("bytes_acked", "<u8"), ("pid", "<u4"), ("tid", "<u4"), ("comm", "S16"),
                  ("saddr", "<u4"), ("daddr", "<u4"), ("netns", "<u4"), ("sport", "<u2"), ("dport", "<u2"), ("ipver", "u1"), ("type", "u1")],
                 align=True)
assert CONN4.itemsize == 72


def _ocfg(kw):
    return {k: kw[k] for k in ("max_svcs", "max_tasks", "cms_depth", "cms_log2_width") if k in kw}


class Run:
    """one engine with the flag, the history of its closed windows (tsec, device table, events) and, fed the same events, the oracle
    and its ring"""

    def __init__(self, oracle=True, **kw):
        self.eng = ge.Engine(flow_level=True, **kw)
        c = self.eng.cfg
        self.depth, self.log2w = c.cms_depth, c.cms_log2_width
        self.orc = po.OracleEngine(**_ocfg(kw)) if oracle else None
        self.ring = FlowLevelRing(self.depth << self.log2w) if oracle else None
        self.tsecs, self.tables, self.streams, self.pending = [], [], [], []

    def ingest(self, ev, batch=None):
        batch = batch or len(ev)
        for off in range(0, len(ev), batch):
            self.eng.ingest_events(ev[off: off + batch])
            self.eng.sync()
            if self.orc:
                self.orc.ingest(ev[off: off + batch])
        self.pending.append(ev)

    def flush(self, t):
        self.eng.flush(t)
        self.tsecs.append(t)
        self.tables.append(self.eng.export_cms(last_window=True))
        self.streams.append(np.concatenate(self.pending) if self.pending else np.zeros(0, dtype=ge.EVENT_DTYPE))
        self.pending = []
        if self.orc:
            self.orc.flush(t)
            self.ring.flush(t, self.orc.cms(last_window=True))

    def check(self, keys, exact=True, what=None):
        got = self.eng.export_cms_5min()
        assert got.tobytes() == level_of_history(self.tsecs, self.tables).tobytes(), what
        if self.ring:
            assert got.tobytes() == self.ring.level.tobytes(), what
        q = self.eng.query_flows_5min(keys)
        assert q["flow_key"].tolist() == np.asarray(keys, dtype=np.uint64).tolist()
        assert [(int(r["count"]), int(r["kbytes"])) for r in q] == point_query(got, keys, self.depth, self.log2w), what
        if exact:
            ex = exact_flows(np.concatenate([self.streams[j] for j in held_windows(self.tsecs)]), keys)
            for k, r in zip(np.asarray(keys, dtype=np.uint64).tolist(), q):
                if ex[k][1] <= M32 and ex[k][0] <= M32:
                    assert r["count"] >= ex[k][0] and r["kbytes"] >= ex[k][1], (what, hex(k))
        return got


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_level_after_every_flush(name):
    tsecs = SEQUENCES[name]
    rng = np.random.default_rng(100 + len(tsecs))
    keys = rng.integers(1, 1 << 62, 400, dtype=np.uint64)
    run = Run(**CFG)
    assert not run.eng.export_cms_5min().any()                       # empty before the first flush
    for i, t in enumerate(tsecs):
        run.ingest(flow_events(rng, int(rng.integers(500, 6000)), keys), batch=int(rng.integers(1000, 1 << 14)))
        run.flush(t)
        run.check(keys[:64], what=(name, i, t))
    run.ingest(flow_events(rng, 3000, keys))                         # the open window stays out of the level
    run.eng.sync()
    run.check(keys[:64], what=(name, "open"))


def _route_window(rng, route, keys, host):
    """one window's records of one ingest route: (a callable that ingests them, the oracle's events or None, the connection events
    kept, the count units they add to each row: 1 an event, an ACTIVE_CONN_STATS record its active connections)"""
    n = int(rng.integers(300, 1500))
    if route in ("event32", "tcp24"):
        ev = flow_events(rng, n, keys)
        ev = ev[ev["type"] != ge.EV_ACTIVE] if route == "tcp24" else ev
        if route == "event32":
            return (lambda e: e.ingest_events(ev)), ev, len(ev), _units(ev)
        t24 = np.zeros(len(ev), dtype=ge.TCP24_DTYPE)
        t24["svc_id"], t24["flow_key"], t24["bytes"], t24["host_idx"], t24["type"] = ev["svc_id"], ev["flow_key"], ev["value"], ev["host_idx"], ev["type"]
        return (lambda e: e.ingest_raw(ge.RAW_TCP24, t24, len(t24))), ev, len(ev), _units(ev)
    if route == "notify_tcp_conn":
        recs, exp = [], []
        for _ in range(min(n, 1000)):
            r = np.zeros(1, dtype=TCP_CONN)
            r["ser_glob_id"], r["cli_task_aggr_id"] = 1000 + int(rng.integers(0, 20)), int(keys[int(rng.integers(0, len(keys)))])
            acc, closed = bool(rng.integers(0, 2)), bool(rng.integers(0, 2))
            r["is_accept"], r["is_connect"] = acc, not acc
            r["tusec_start"], r["tusec_close"] = 3_000_000, 7_000_000 if closed else 0
            r["bytes_sent"], r["bytes_rcvd"] = int(rng.integers(0, 1 << 20)), int(rng.integers(0, 1 << 26))
            recs.append((r, b""))
            e = np.zeros(1, dtype=ge.EVENT_DTYPE)
            e["svc_id"], e["flow_key"] = r["ser_glob_id"], r["cli_task_aggr_id"]
            e["value"] = int(r["bytes_sent"][0]) + int(r["bytes_rcvd"][0]) if closed else 0
            e["type"] = (4 if closed else 2) if acc else (3 if closed else 1)
            exp.append(e)
        msg = build_msg(ge.NOTIFY_TCP_CONN, recs)
        return (lambda e: e.ingest_msg(msg, host_idx=host)), np.concatenate(exp), len(exp), len(exp)
    if route == "notify_active_conn":
        recs = np.zeros(min(n, 1000), dtype=ACTIVE)
        recs["listener_glob_id"] = 9000 + rng.integers(0, 40, len(recs))
        recs["cli_aggr_task_id"] = keys[rng.integers(0, len(keys), len(recs))]
        recs["bytes_sent"], recs["bytes_received"] = rng.integers(0, 1 << 24, len(recs)), rng.integers(0, 1 << 24, len(recs))
        recs["active_conns"] = rng.integers(0, 50, len(recs))
        ev = np.zeros(len(recs), dtype=ge.EVENT_DTYPE)
        ev["svc_id"], ev["flow_key"] = recs["listener_glob_id"], recs["cli_aggr_task_id"]
        ev["value"] = (recs["bytes_sent"] + recs["bytes_received"]) >> np.uint64(10)
        ev["type"], ev["flags"], ev["host_idx"] = ge.EV_ACTIVE, recs["active_conns"], host
        msg = fixed_msg(ge.NOTIFY_ACTIVE_CONN_STATS, recs)
        return (lambda e: e.ingest_msg(msg, host_idx=host)), ev, len(ev), _units(ev)
    # raw eBPF connection events: the service and flow ids are derived from the addresses on the host, so the check is the device's own
    # history and the count halves: every kept event adds 1 to one cell of each row
    # a connect-side record keys its service by the remote end: few remote addresses and ports, so every service fits the table
    rec = np.zeros(n, dtype=CONN4 if route == "ipv4_raw" else CONN6)
    if route == "ipv4_raw":
        rec["saddr"], rec["daddr"] = 0x0A000001 + rng.integers(0, 8, n), 0x0B000001 + rng.integers(0, 16, n)
    else:
        rec["saddr"][:, 0], rec["saddr"][:, 3] = 0x20010DB8, rng.integers(1, 9, n)
        rec["daddr"][:, 0], rec["daddr"][:, 3] = 0x20010DB9, rng.integers(1, 17, n)
    rec["netns"] = 4026531840
    rec["sport"] = rng.choice(np.array([80, 443, 8080], dtype=np.uint16).byteswap(), n)
    rec["dport"] = rng.choice(np.arange(40000, 40016, dtype=np.uint16).byteswap(), n)
    rec["type"] = rng.choice(np.array([0, 1, 2, 3, 4], dtype=np.uint8), n, p=[0.1, 0.2, 0.3, 0.2, 0.2])      # 0: dropped
    rec["bytes_received"], rec["bytes_acked"] = rng.integers(0, 1 << 30, n), rng.integers(0, 1 << 20, n)
    kind = ge.RAW_TCP_IPV4_EVENT if route == "ipv4_raw" else ge.RAW_TCP_IPV6_EVENT
    kept = int(((rec["type"] >= 1) & (rec["type"] <= 4)).sum())
    return (lambda e: e.ingest_raw(kind, rec, n)), None, kept, kept


def _units(ev):
    return int(np.where(ev["type"] == ge.EV_ACTIVE, ev["flags"].astype(np.int64), 1).sum())


@pytest.mark.parametrize("route", ["event32", "tcp24", "ipv4_raw", "ipv6_raw", "notify_tcp_conn", "notify_active_conn"])
def test_every_ingest_route_feeds_the_level(route):
    rng = np.random.default_rng(sum(map(ord, route)))
    keys = rng.integers(1, 1 << 62, 200, dtype=np.uint64)
    oracle = route not in ("ipv4_raw", "ipv6_raw")
    run = Run(oracle=oracle, **CFG)
    kept, units = [], []
    for i, t in enumerate(SEQUENCES["gaps"]):
        ingest, ev, nkept, nunits = _route_window(rng, route, keys, host=3)
        rc = ingest(run.eng)
        assert rc in (None, 0)
        run.eng.sync()
        if oracle:
            run.orc.ingest(ev)
            run.pending.append(ev)
        kept.append(nkept); units.append(nunits)
        run.flush(t)
        got = run.check(keys[:32], exact=oracle, what=(route, i, t))
        assert int((got & np.uint64(M32)).sum()) == run.depth * sum(units[j] for j in held_windows(run.tsecs)), (route, i)
    assert sum(kept) > 0 and run.eng.stats()["events_tcp"] == sum(kept)


@pytest.mark.parametrize("depth,log2w", [(1, 4), (8, 4), (1, 22), (8, 22)])
def test_sketch_edges_and_a_wrapping_kbytes_half(depth, log2w):
    """1100 close events of 4 GB - 1 bytes a window on one key: 4 194 303 kbytes each, so its cells' kbytes half passes 2^32 within a
    window and again in the level"""
    rng = np.random.default_rng(depth * 100 + log2w)
    keys = rng.integers(1, 1 << 62, 100, dtype=np.uint64)
    kw = dict(CFG, cms_depth=depth, cms_log2_width=log2w)
    run = Run(oracle=log2w < 20, **kw)
    for i, t in enumerate([5, 35, 40] if log2w >= 20 else [5, 35, 40, 299, 400, 405]):
        run.ingest(flow_events(rng, 3000, keys, huge=1100), batch=1 << 13)
        run.flush(t)
        run.check(keys[:16], what=(depth, log2w, i))
        held = np.concatenate([run.streams[j] for j in held_windows(run.tsecs)])
        assert exact_flows(held, keys[:1])[int(keys[0])][1] > M32                      # keys[0]'s kbytes half has wrapped
    if log2w >= 20:
        assert run.eng.capacity()["device_bytes"] >= 13 * (depth << log2w) * 8


def test_growth_and_eviction_leave_the_level():
    """gysk_grow in the middle of windows and services evicted for idleness: the level depends on neither, so it stays equal to the
    oracle's (fed the same stream at the final capacity) and to an engine that neither grows nor evicts"""
    rng = np.random.default_rng(77)
    keys = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
    kw = dict(CFG, max_svcs=64)
    run = Run(idle_evict_secs=20, **kw)
    run.orc = po.OracleEngine(**_ocfg(dict(kw, max_svcs=256)))
    run.orc.set_idle_evict(20)
    plain = ge.Engine(flow_level=True, **dict(CFG, max_svcs=256))
    for i, t in enumerate(range(5, 205, 5)):
        ev = flow_events(rng, 2000, keys, nsvc=48 if i < 4 else 16)         # services 17 .. 48 go idle after four windows
        half = len(ev) // 2
        run.ingest(ev[:half])
        if i in (2, 11):
            run.eng.grow(max_svcs=run.eng.cfg.max_svcs * 2)
        run.ingest(ev[half:])
        plain.ingest_events(ev); plain.sync()
        run.flush(t); plain.flush(t)
        got = run.check(keys[:32], what=("grow/evict", i, t))
        assert got.tobytes() == plain.export_cms_5min().tobytes()
    assert run.eng.stats()["svcs_evicted"] >= 32 and run.eng.capacity()["ngrows"] == 2
    assert run.eng.stats()["events_dropped"] == 0


def _rowbytes(rows):
    return [tuple(np.float64(v).tobytes() if isinstance(v, float) else v for v in r.values()) for r in rows]


def _arrays(eng, torch):
    """{(region, count-min table): (region bytes, offset, size)} and {(region, "rest"): the region's bytes after its count-min tables},
    from the names gysk_merge_buffers gives (each array 256-byte aligned)"""
    from tests.test_gpu_merge_exact import _dev_bytes
    c = eng.cfg
    ncms = (c.cms_depth << c.cms_log2_width) * 8
    out = {}
    for name, ptr, nbytes, _redop in eng.merge_buffers():
        region, arrays = name.split(": ")
        buf = _dev_bytes(torch, ptr, nbytes)
        off = 0
        for a in arrays.split("|"):
            if not a.startswith("cms_"):
                break
            out[region, a] = (buf, off, ncms)
            off += (ncms + 255) & ~255
        out[region, "rest"] = buf[off:]
    return out


def test_flag_off_and_on_answer_alike():
    """the same stream through an engine without the flag and one with it: every existing answer byte-equal, the flow level's calls
    GYSK_ERR_NOTSUP without it"""
    import torch
    rng = np.random.default_rng(9)
    keys = rng.integers(1, 1 << 62, 500, dtype=np.uint64)
    kw = dict(CFG, merge_levels=True, merge_states=True, merge_topn=True)
    off, on = ge.Engine(**kw), ge.Engine(flow_level=True, **kw)
    sids = np.unique(flow_events(np.random.default_rng(0), 5000, keys)["svc_id"])
    for e in (off, on):
        e.set_logical_map(sids, sids % np.uint64(5) + np.uint64(70))
    for i, t in enumerate(SEQUENCES["same_tsec"] + [700, 905]):
        ev = flow_events(rng, 4000, keys)
        resp = np.zeros(1000, dtype=ge.EVENT_DTYPE)
        resp["svc_id"], resp["type"], resp["value"] = sids[rng.integers(0, len(sids), 1000)], ge.EV_RESP, rng.integers(100, 1 << 22, 1000)
        ev = np.concatenate([ev, resp])
        for e in (off, on):
            e.ingest_events(ev); e.sync()
            e.flush(t)
        for lw in (False, True):
            assert off.export_cms(lw).tobytes() == on.export_cms(lw).tobytes()
            assert off.query_flows(keys, lw).tobytes() == on.query_flows(keys, lw).tobytes()
        assert _rowbytes(off.query_svcs(sids)) == _rowbytes(on.query_svcs(sids))
        (wa, na), (wb, nb) = off.query_window(), on.query_window()      # rows as a set: a service's slot depends on the insert race
        assert na == nb and sorted(bytes(r) for r in wa) == sorted(bytes(r) for r in wb)
        for e in (off, on):
            _emulate_collectives(torch, [e])
        lids = np.unique(sids % np.uint64(5) + np.uint64(70))
        assert _rowbytes(off.query_logical(lids)) == _rowbytes(on.query_logical(lids))
        for lw in (False, True):
            assert off.query_flows_global(keys, lw).tobytes() == on.query_flows_global(keys, lw).tobytes()
        assert off.merge_flush_range() == on.merge_flush_range() == (t, t)
        a, b = _arrays(off, torch), _arrays(on, torch)
        for k in [k for k in a if k[1] != "rest"]:
            buf, o, size = a[k]
            buf2, o2, _ = b[k]
            assert buf[o: o + size].tobytes() == buf2[o2: o2 + size].tobytes(), k
        for region in ("sum_u64", "max_i64", "max_u8"):
            assert a[region, "rest"].tobytes() == b[region, "rest"].tobytes(), region
    for call in (lambda: off.query_flows_5min(keys), off.export_cms_5min, lambda: off.query_flows_global_5min(keys)):
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == NOTSUP
    alone = ge.Engine(**CFG)
    alone.set_logical_map(sids, sids)
    _emulate_collectives(torch, [alone])
    with pytest.raises(ge.GyskError) as ex:
        alone.merge_flush_range()
    assert ex.value.code == NOTSUP


def _shard_events(ev, world):
    return [ev[ev["host_idx"] % world == r] for r in range(world)]


@pytest.mark.parametrize("other_flags", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_merge_sums_the_ranks_levels(world, other_flags):
    import torch
    rng = np.random.default_rng(world * 10 + other_flags)
    keys = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
    flags = dict(merge_levels=True, merge_states=True, merge_clusters=True, merge_topn=True) if other_flags else {}
    engines = [ge.Engine(flow_level=True, rank=r, world=world, **flags, **CFG) for r in range(world)]
    sids = np.unique(flow_events(np.random.default_rng(0), 5000, keys)["svc_id"])
    for e in engines:
        e.set_logical_map(sids, sids % np.uint64(3) + np.uint64(10))
    ncell = engines[0].cfg.cms_depth << engines[0].cfg.cms_log2_width
    for step, t in enumerate([30, 35, 60, 95, 300, 305]):
        shards = _shard_events(flow_events(rng, 6000, keys), world)
        last = step == 5
        tsec = [t + (5 * (r % 3) if last else 0) for r in range(world)]       # at the last flush the ranks close different windows
        for e, ev, ts in zip(engines, shards, tsec):
            e.ingest_events(ev); e.sync()
            e.flush(ts)
        _emulate_collectives(torch, engines)
        levels = [e.export_cms_5min() for e in engines]
        want = sum(levels[1:], levels[0].copy())
        arrays = [_arrays(e, torch) for e in engines]
        for a in arrays:
            buf, off, size = a["sum_u64", "cms_5min"]
            assert buf[off: off + size].view(np.uint64).tobytes() == want.tobytes(), (world, step)
            cur = buf[0: size].view(np.uint64)
            assert cur.tobytes() == sum((e.export_cms(False) for e in engines[1:]), engines[0].export_cms(False)).tobytes()
        for e in engines:
            got = e.query_flows_global_5min(keys[:48])
            assert [(int(r["count"]), int(r["kbytes"])) for r in got] == point_query(want, keys[:48], e.cfg.cms_depth, e.cfg.cms_log2_width)
            assert e.merge_flush_range() == (min(tsec), max(tsec))
        assert want.shape == (ncell,)


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(5)
    keys = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
    eng = ge.Engine(flow_level=True, merge_levels=True, **CFG)
    sids = np.unique(flow_events(np.random.default_rng(0), 5000, keys)["svc_id"])
    eng.set_logical_map(sids, sids)
    for t in (30, 35, 65):
        eng.ingest_events(flow_events(rng, 5000, keys)); eng.sync()
        eng.flush(t)
    _emulate_collectives(torch, [eng])
    emulated = eng.query_flows_global_5min(keys)
    arrays = _arrays(eng, torch)
    eng.nccl_comm_init(eng.nccl_unique_id(), 1, 0)
    eng.merge_global()
    eng.sync()
    assert eng.query_flows_global_5min(keys).tobytes() == emulated.tobytes()
    after = _arrays(eng, torch)
    for k in arrays:
        if k[1] == "rest":
            assert arrays[k].tobytes() == after[k].tobytes(), k
            continue
        buf, off, size = arrays[k]
        buf2, off2, _ = after[k]
        assert buf[off: off + size].tobytes() == buf2[off2: off2 + size].tobytes(), k
    assert eng.merge_flush_range() == (65, 65)
