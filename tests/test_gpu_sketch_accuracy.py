"""The per-service HyperLogLog and the count-min on the device against exact answers computed in numpy, through every ingest route
that feeds them and on the key shapes of tests/test_sketch_accuracy_host.py: (client ip << 32) | port from raw IPv4 and IPv6 events,
a caller's 5-tuple fold, small sequential client-process ids of the wire records, and pre-mixed random keys.

HyperLogLog: each service's registers (gysk_export_hll) equal gyo_hll_registers over the service's distinct keys so far, and its
distinct_clients (gysk_query_svcs, gysk_query_window rows, gysk_hll_estimate of the exported registers) is within the bounds of the
host test of the exact distinct count. The registers live as long as the slot: keys arrive over many batches and windows with
duplicates, and an evicted service starts again from zero. Merged logical services (world 1 ... 8, collectives emulated on one GPU
by tests/test_gpu_merge._emulate_collectives) answer the exact union of their members' client sets, and gysk_export_logical_hll is the element-wise
maximum of the members' registers.

Count-min (gysk_query_flows on the open and the last window, gysk_query_flows_5min, gysk_query_flows_global after a merge): every
count is at least the exact count and every kbytes half at least the exact sum of bytes >> 10 (of the kbytes of ACTIVE_CONN_STATS
records); the share of keys whose count exceeds the exact one by more than ceil(e / w * N), N the table's total count, is at most
e^-d + 0.01."""
import math

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200.wire import TCP_CONN, build_msg_fixed
from oracle import pyoracle as po
from tests.test_gpu_boundary import ACTIVE, CONN6
from tests.test_gpu_flow_level import CONN4
from tests.test_gpu_merge import _emulate_collectives
from tests.test_sketch_accuracy_host import bound, distinct_keys, sigma

pytestmark = pytest.mark.gpu

GY_SEED = 0xCEEDFEAD
NETNS = 4026531840
M32 = 0xFFFFFFFF
WINDOWS = (5, 10, 15)                   # three closed windows, then an open one
REC_DTYPE = np.dtype([("key", "<u8"), ("cnt", "<u8"), ("kb", "<u8")])       # what one record adds to its flow
MAX_MSG = 2048                          # records per wire message (MAX_NUM_CONNS)


def jh(a, b, iv):
    return po.lib().gyo_jhash_2words(a & M32, b & M32, iv & M32)


def raw_svc_id(ip, port):
    """the listener id the library gives a raw event's {ip, netns, port} (raw_svc_id in gysk_engine.cu)"""
    id_ = (jh(ip, NETNS, GY_SEED) << 32) | jh(port, NETNS, GY_SEED ^ ip)
    return id_ or 1


def fold_ip6(w):
    return jh(int(w[2]), int(w[3]), jh(int(w[0]), int(w[1]), GY_SEED))


def bswap16(a):
    return a.astype(np.uint16).byteswap()


# ---- one service's records on one route: (ingest callables, the records' flow keys, count units and kbytes) -------------------------

def _conn_events(svc, keys, rng, t):
    ev = np.zeros(len(keys), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"], ev["tsec"] = svc, keys, t
    ev["type"] = rng.choice(np.array([ge.EV_CONNECT, ge.EV_ACCEPT, ge.EV_CLOSE_CLI, ge.EV_CLOSE_SER], dtype=np.uint16), len(keys))
    ev["value"] = rng.integers(0, 1 << 26, len(keys))
    return ev


def _recs(keys, cnt, kb):
    r = np.zeros(len(keys), dtype=REC_DTYPE)
    r["key"], r["cnt"], r["kb"] = keys, cnt, kb
    return r


class Route:
    """the service ids of a route and the records a slice of each service's client keys becomes"""

    def __init__(self, name, nsvc):
        self.name = name
        if name in ("ipv4_raw", "ipv6_raw"):
            self.srv = [(0x0A640001 + j, 8080 + j) for j in range(nsvc)]
            self.ids = [raw_svc_id(ip if name == "ipv4_raw" else fold_ip6([0x20010DB8, 0, 0, ip]), port) for ip, port in self.srv]
        else:
            self.ids = [int(x) for x in (np.arange(1, nsvc + 1, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))]

    def client_keys(self, keys):
        """the flow keys the engine derives from the client keys the test draws"""
        if self.name != "ipv6_raw":
            return keys
        ip = (keys >> np.uint64(32)).astype(np.uint32)
        fold = np.array([fold_ip6([0x20010DB8, 0, 0, int(a)]) for a in ip.tolist()], dtype=np.uint64)
        return (fold << np.uint64(32)) | (keys & np.uint64(0xFFFF))

    def records(self, j, keys, rng, t):
        """(list of callables ingesting the records into an engine, REC_DTYPE array of what they add)"""
        n, svc = len(keys), self.ids[j]
        if self.name in ("event32", "tcp24"):
            ev = _conn_events(svc, keys, rng, t)
            recs = _recs(keys, 1, ev["value"] >> np.uint32(10))
            if self.name == "event32":
                return [lambda e: e.ingest_events(ev)], recs
            t24 = np.zeros(n, dtype=ge.TCP24_DTYPE)
            t24["svc_id"], t24["flow_key"], t24["bytes"], t24["type"] = ev["svc_id"], ev["flow_key"], ev["value"], ev["type"]
            return [lambda e: e.ingest_raw(ge.RAW_TCP24, t24, n)], recs
        if self.name in ("ipv4_raw", "ipv6_raw"):
            v4 = self.name == "ipv4_raw"
            rec = np.zeros(n, dtype=CONN4 if v4 else CONN6)
            sip, sport = self.srv[j]
            cip, cport = (keys >> np.uint64(32)).astype(np.uint32), (keys & np.uint64(0xFFFF)).astype(np.uint16)
            ser = rng.integers(0, 2, n).astype(bool)                 # accept side: the listener is the source
            rec["type"] = np.where(ser, rng.choice([ge.EV_ACCEPT, ge.EV_CLOSE_SER], n), rng.choice([ge.EV_CONNECT, ge.EV_CLOSE_CLI], n))
            if v4:
                rec["saddr"], rec["daddr"] = np.where(ser, sip, cip), np.where(ser, cip, sip)
            else:
                for f, mine in (("saddr", ser), ("daddr", ~ser)):
                    rec[f][:, 0] = 0x20010DB8
                    rec[f][:, 3] = np.where(mine, sip, cip)
            rec["sport"], rec["dport"] = bswap16(np.where(ser, sport, cport)), bswap16(np.where(ser, cport, sport))
            rec["netns"], rec["ts_ns"] = NETNS, t * 1_000_000_000
            rec["bytes_received"], rec["bytes_acked"] = rng.integers(0, 1 << 30, n), rng.integers(0, 1 << 20, n)
            kind = ge.RAW_TCP_IPV4_EVENT if v4 else ge.RAW_TCP_IPV6_EVENT
            return [lambda e: e.ingest_raw(kind, rec, n)], _recs(self.client_keys(keys), 1, (rec["bytes_received"] + rec["bytes_acked"]) >> np.uint64(10))
        if self.name == "notify_tcp_conn":
            rec = np.zeros(n, dtype=TCP_CONN)
            rec["ser_glob_id"], rec["cli_task_aggr_id"] = svc, keys
            acc, closed = rng.integers(0, 2, n).astype(bool), rng.integers(0, 2, n).astype(bool)
            rec["is_accept"], rec["is_connect"] = acc, ~acc
            rec["tusec_start"], rec["tusec_close"] = t * 1_000_000 - 1, np.where(closed, t * 1_000_000, 0)
            rec["bytes_sent"], rec["bytes_rcvd"] = rng.integers(0, 1 << 20, n), rng.integers(0, 1 << 26, n)
            kb = np.where(closed, (rec["bytes_sent"] + rec["bytes_rcvd"]) >> np.uint64(10), 0)
            msgs = [build_msg_fixed(ge.NOTIFY_TCP_CONN, rec[o: o + MAX_MSG]) for o in range(0, n, MAX_MSG)]
            return [lambda e, m=m: _msg_ok(e, m) for m in msgs], _recs(keys, 1, kb)
        assert self.name == "active_conn"
        rec = np.zeros(n, dtype=ACTIVE)
        rec["listener_glob_id"], rec["cli_aggr_task_id"] = svc, keys
        rec["bytes_sent"], rec["bytes_received"] = rng.integers(0, 1 << 24, n), rng.integers(0, 1 << 24, n)
        rec["active_conns"] = rng.integers(1, 50, n)
        msgs = [build_msg_fixed(ge.NOTIFY_ACTIVE_CONN_STATS, rec[o: o + MAX_MSG]) for o in range(0, n, MAX_MSG)]
        kb = (rec["bytes_sent"] + rec["bytes_received"]) >> np.uint64(10)
        return [lambda e, m=m: _msg_ok(e, m) for m in msgs], _recs(keys, rec["active_conns"], kb)


def _msg_ok(e, m):
    assert e.ingest_msg(m) == 0


# ---- exact answers and the checks ------------------------------------------------------------------------------------------------------

def exact_flows(recs):
    """(distinct keys, exact count, exact kbytes) of the records"""
    keys, inv = np.unique(recs["key"], return_inverse=True)
    return keys, np.bincount(inv, weights=recs["cnt"]).astype(np.int64), np.bincount(inv, weights=recs["kb"]).astype(np.int64)


def check_cms(got, recs, depth, log2w, what):
    """got: gysk_flow_est rows of the distinct keys of recs, in np.unique order"""
    keys, cnt, kb = exact_flows(recs)
    assert got["flow_key"].tolist() == keys.tolist(), what
    assert cnt.max() <= M32 and kb.max() <= M32                      # neither half of a cell wraps at these sizes
    gc, gk = got["count"].astype(np.int64), got["kbytes"].astype(np.int64)
    assert np.all(gc >= cnt), (what, int(np.argmin(gc - cnt)))
    assert np.all(gk >= kb), (what, int(np.argmin(gk - kb)))
    over = math.ceil(math.e / (1 << log2w) * int(cnt.sum()))
    share = float(np.mean(gc - cnt > over))
    assert share <= math.exp(-depth) + 0.01, (what, share, over)
    return share


def check_hll(eng, ids, keysets, p, what):
    """every service's registers, and its three distinct_clients answers, against its exact distinct keys"""
    L = eng.L
    rows = {r.glob_id: r.distinct_clients for r in eng.query_window()[0]}
    for id_, s, keys in zip(ids, eng.query_svcs(ids), keysets):
        exact = len(keys)
        regs = eng.export_hll(id_)
        assert np.array_equal(regs, po.hll_registers(keys, p)), (what, hex(id_))
        est = L.gysk_hll_estimate(ge._p(regs), p)
        assert s["found"] and s["distinct_clients"] == est and rows[id_] == est, (what, hex(id_), s["distinct_clients"], rows.get(id_), est)
        assert abs(est - exact) <= bound(p, exact) * max(exact, 1), (what, hex(id_), exact, est, (est / max(exact, 1) - 1) / sigma(p))


def service_streams(rng, route, plan, nparts):
    """per service: the distinct client keys of its shape and cardinality, and its key stream (a third repeated, shuffled) cut in nparts"""
    out = []
    for shape, n in plan:
        if route.name == "notify_tcp_conn":
            shape = "seq"
        elif route.name in ("ipv4_raw", "ipv6_raw") and not shape.startswith("ip_port_"):
            shape = "ip_port_64"
        keys = distinct_keys(shape, n, rng)
        s = np.concatenate([keys, keys[rng.integers(0, n, n // 3)]])
        out.append(np.array_split(s[rng.permutation(len(s))], nparts))
    return out


def plan_for(p):
    return [("ip_port_64", 10), ("tuple5", 3000), ("ip_port_1024", 60_000)] if p < 16 else \
           [("seq", 10), ("ip_port_8", 30_000), ("ip_port_28232", 400_000)]


ROUTES = ["event32", "tcp24", "ipv4_raw", "ipv6_raw", "notify_tcp_conn", "active_conn"]


@pytest.mark.parametrize("route,p", [(r, 12) for r in ROUTES] + [("event32", 4), ("event32", 16), ("ipv4_raw", 4), ("ipv4_raw", 16)])
def test_every_route_against_exact_answers(route, p):
    """three services of each route, their keys over three closed windows and an open one, each window's part in four ingest calls
    split further by a small device batch"""
    rng = np.random.default_rng(sum(map(ord, route)) * 100 + p)
    plan = plan_for(p)
    r = Route(route, len(plan))
    depth, log2w = 4, 20
    eng = ge.Engine(max_svcs=64, max_tasks=16, max_batch=1 << 15, stage_batch=1 << 14, hll_p=p, cms_depth=depth, cms_log2_width=log2w,
                    flow_level=True)
    streams = service_streams(rng, r, plan, 4 * (len(WINDOWS) + 1))
    seen = [np.zeros(0, dtype=np.uint64) for _ in plan]
    closed = []
    for w in range(len(WINDOWS) + 1):
        t = WINDOWS[w] if w < len(WINDOWS) else WINDOWS[-1] + 2
        wrecs = []
        for part in range(4):
            calls = []
            for j in range(len(plan)):
                keys = streams[j][4 * w + part]
                c, recs = r.records(j, keys, rng, t)
                calls += c
                wrecs.append(recs)
                seen[j] = np.concatenate([seen[j], r.client_keys(keys)])
            for i in rng.permutation(len(calls)):
                calls[i](eng)
            eng.sync()
        wrecs = np.concatenate(wrecs)
        keys = np.unique(wrecs["key"])
        check_cms(eng.query_flows(keys), wrecs, depth, log2w, (route, p, w, "open"))
        if w < len(WINDOWS):
            eng.flush(t)
            closed.append(wrecs)
            check_cms(eng.query_flows(keys, last_window=True), wrecs, depth, log2w, (route, p, w, "last"))
            held = np.concatenate(closed)
            check_cms(eng.query_flows_5min(np.unique(held["key"])), held, depth, log2w, (route, p, w, "5min"))
        check_hll(eng, r.ids, [np.unique(s) for s in seen], p, (route, p, w))
    st = eng.stats()
    assert st["events_dropped"] == 0 and st["nsvcs"] == len(plan)


def test_evicted_service_starts_from_zero():
    """A's first life (20 000 keys) is evicted for idleness; in its second life the registers hold only the new keys"""
    rng = np.random.default_rng(31)
    p = 12
    eng = ge.Engine(max_svcs=16, max_tasks=4, max_batch=1 << 14, hll_p=p, idle_evict_secs=20)
    A, B = 0xA11CE, 0xB0B
    first, other = distinct_keys("ip_port_64", 20_000, rng), distinct_keys("random", 5000, rng)
    second = distinct_keys("ip_port_1024", 7000, rng)

    def feed(svc, keys, t):
        ev = _conn_events(svc, keys, rng, t)
        for off in range(0, len(ev), 6000):
            eng.ingest_events(ev[off: off + 6000])
        eng.sync()

    for i, t in enumerate((5, 10)):
        feed(A, first[i::2], t); feed(B, other[i::2], t)
        eng.flush(t)
    check_hll(eng, [A, B], [np.unique(first), np.unique(other)], p, "first life")
    evicted = set()
    for t in range(15, 200, 5):
        feed(B, other[:100], t)
        eng.flush(t)
        evicted |= set(int(x) for x in eng.evicted_ids())
        if A in evicted:
            break
    assert evicted == {A}
    assert eng.query_svcs([A])[0]["found"] == 0
    feed(A, second, t + 5)
    feed(A, second[:3000], t + 5)                   # duplicates in a later batch
    check_hll(eng, [A, B], [np.unique(second), np.unique(other)], p, "second life")
    eng.flush(t + 5)
    check_hll(eng, [A, B], [np.unique(second), np.unique(other)], p, "second life, flushed")


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_merged_logical_services_count_the_union(world):
    """logical 500: 2 * world members on hosts 0 .. 2 world - 1 (two on every rank), each with 20 000 client keys of one
    structured run, consecutive members overlapping by 12 000; logical 501: one member with pre-mixed keys. Every rank answers the
    exact union, and gysk_query_flows_global the exact flows of every rank"""
    import torch
    rng = np.random.default_rng(600 + world)
    p, depth, log2w = 12, 4, 16
    engines = [ge.Engine(rank=r, world=world, max_svcs=64, max_tasks=16, max_batch=1 << 15, hll_p=p, cms_depth=depth,
                         cms_log2_width=log2w) for r in range(world)]
    nm = 2 * world
    members = [int(x) for x in np.arange(1, nm + 2, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)]
    glob = np.array(members, dtype=np.uint64)
    logical = np.array([500] * nm + [501], dtype=np.uint64)
    for e in engines:
        e.set_logical_map(glob, logical)
    run = distinct_keys("ip_port_1024", 8000 * (nm - 1) + 20_000, rng)
    keysets = [run[8000 * j: 8000 * j + 20_000] for j in range(nm)] + [distinct_keys("random", 30_000, rng)]
    windows = []
    for t in (5, 7):                    # every key in the closed window, a third of them again in the open one
        evs = []
        for j, keys in enumerate(keysets):
            part = keys if t == 5 else keys[rng.permutation(len(keys))[: len(keys) // 3]]
            ev = _conn_events(members[j], part, rng, t)
            ev["host_idx"] = j if j < nm else 0
            evs.append(ev)
        ev = np.concatenate(evs)
        ev = ev[rng.permutation(len(ev))]
        for off in range(0, len(ev), 1 << 15):
            for e in engines:
                e.ingest_events(ev[off: off + (1 << 15)])
        for e in engines:
            e.sync()
        windows.append(ev)
        if t == 5:
            for e in engines:
                e.flush(t)
    _emulate_collectives(torch, engines)
    owner = lambda j: engines[(j if j < nm else 0) % world]
    union = np.unique(np.concatenate(keysets[:nm]))
    for lid, js, exact in ((500, range(nm), union), (501, [nm], np.unique(keysets[nm]))):
        want = np.maximum.reduce([owner(j).export_hll(members[j]) for j in js])
        assert np.array_equal(want, po.hll_registers(exact, p)), lid
        est = po.hll_estimate(want, p)
        assert abs(est / len(exact) - 1) <= bound(p, len(exact)), (world, lid, est, len(exact))
        for r, e in enumerate(engines):
            assert np.array_equal(e.export_logical_hll(lid), want), (world, r, lid)
            row = e.query_logical([lid])[0]
            assert row["found"] and row["distinct_clients"] == est, (world, r, lid, row["distinct_clients"], est)
    for lw, ev in ((True, windows[0]), (False, windows[1])):
        recs = _recs(ev["flow_key"], 1, ev["value"] >> np.uint32(10))
        keys = np.unique(recs["key"])
        for e in engines:
            check_cms(e.query_flows_global(keys, last_window=lw), recs, depth, log2w, (world, lw))


@pytest.mark.parametrize("log2w", [10, 16, 20])
@pytest.mark.parametrize("depth", [1, 4, 8])
def test_count_min_bounds_at_every_size(depth, log2w):
    """200 000 connection events over 40 000 structured and 20 000 pre-mixed flows, a few heavy: the open and the last window, the
    300-s level and the merged global table at world 1"""
    import torch
    rng = np.random.default_rng(depth * 100 + log2w)
    eng = ge.Engine(max_svcs=64, max_tasks=16, max_batch=1 << 16, cms_depth=depth, cms_log2_width=log2w, flow_level=True)
    eng.set_logical_map(np.array([7], dtype=np.uint64), np.array([7], dtype=np.uint64))
    flows = np.concatenate([distinct_keys("ip_port_64", 40_000, rng), distinct_keys("random", 20_000, rng)])
    weight = rng.pareto(1.2, len(flows)) + 1.0
    shares = []
    held = []
    for w, t in enumerate((5, 10, 12)):
        keys = flows[rng.choice(len(flows), 200_000, p=weight / weight.sum())]
        ev = _conn_events(7, keys, rng, t)
        ev["svc_id"] = rng.integers(1, 9, len(ev)).astype(np.uint64)
        ev["value"] = rng.integers(0, 1 << 20, len(ev))             # the heaviest flow's kbytes stay below 2^32
        for off in range(0, len(ev), 1 << 16):
            eng.ingest_events(ev[off: off + (1 << 16)])
        eng.sync()
        recs = _recs(ev["flow_key"], 1, ev["value"] >> np.uint32(10))
        uk = np.unique(keys)
        shares.append(check_cms(eng.query_flows(uk), recs, depth, log2w, (w, "open")))
        if t == 12:
            _emulate_collectives(torch, [eng])
            shares.append(check_cms(eng.query_flows_global(uk), recs, depth, log2w, (w, "global open")))
            prev = np.unique(held[-1]["key"])
            check_cms(eng.query_flows_global(prev, last_window=True), held[-1], depth, log2w, (w, "global last"))
            break
        eng.flush(t)
        held.append(recs)
        shares.append(check_cms(eng.query_flows(uk, last_window=True), recs, depth, log2w, (w, "last")))
        allr = np.concatenate(held)
        shares.append(check_cms(eng.query_flows_5min(np.unique(allr["key"])), allr, depth, log2w, (w, "5min")))
    if (depth, log2w) == (1, 10):
        assert max(shares) > 0                 # one row of 2^10 cells: some keys do pass the bound, so the check has teeth
