"""Host clusters across GPUs (GYSK_FLAG_MERGE_CLUSTERS): gysk_set_cluster_map, gysk_query_cluster_states and
gysk_query_cluster_states_all at world 1 ... 8, with and without the other two merge flags. Each cluster row is restated from what every
rank answers right after the merge: its gysk_query_host_listen rows, and LISTEN_SUMM_STATS (server/gy_msocket.h:853-864) over the
records gysk_encode_listener_state writes from its gysk_query_window_hosts(-1, 0) rows, folded by CLUSTER_STATE_ONE::update_from_state
(server/gy_mconnhdlr.cc:16032-16050) and summed over ranks modulo 2^32."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

from gyeeta_b200 import dist as gd
from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth, wire
from tests.test_gpu_logical_states import KW, TIMES, _ids, state_events, state_map
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import Shards, _align256, _dev_bytes

INVAL, NOTSUP = -22, -95
M32 = 0xFFFFFFFF
UNKNOWN = 987654321
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROW = struct.Struct("<QiI8I")
assert ROW.size == C.sizeof(ge.ClusterRow) == 48
# the fields of LISTENER_STATE_NOTIFY (88 bytes, common/gy_comm_proto.h:2183-2254) that LISTEN_SUMM_STATS::update reads
LSN = np.dtype({"names": ["nqrys_5s", "kb_in", "kb_out", "curr_state", "query_flags"], "formats": ["<u4", "<u4", "<u4", "u1", "u1"],
                "offsets": [8, 36, 40, 79, 84], "itemsize": 88})
LISTEN_FLAG_DELETE = 0xC0
# hosts 0 .. 15 carry the services of state_events; cluster 500 has one host on each rank at world 8, host 16 and 99 have no service,
# host 15 is in no cluster
CLUSTERS = {500: list(range(8)), 502: list(range(8, 15)) + [16], 503: [99]}
LATE_HOSTS = [2, 9, 15, 20]             # services whose first events arrive after the last flush


def _code(fn):
    with pytest.raises(ge.GyskError) as ei:
        fn()
    return ei.value.code


def _i32(v):
    v &= M32
    return v - (1 << 32) if v >> 31 else v


def _div1024(v):
    """int32 division by 1024 as C does it (toward zero), stored into a uint32"""
    v = _i32(v)
    return (-((-v) // 1024) if v < 0 else v // 1024) & M32


def cluster_map(rng, clusters=CLUSTERS):
    pairs = [(h, c) for c, hs in clusters.items() for h in hs]
    perm = rng.permutation(len(pairs))
    return np.array([pairs[i][0] for i in perm], dtype=np.uint32), np.array([pairs[i][1] for i in perm], dtype=np.uint64)


def host_summ(e):
    """{host: (tot_qps, tot_kb_inbound + tot_kb_outbound)} mod 2^32: LISTEN_SUMM_STATS over the encoded window rows of each host"""
    rows, hosts, _ = e.query_window_hosts()
    out = {}
    for h in sorted(set(hosts.tolist())):
        idx = np.nonzero(hosts == h)[0]
        qps = kb = 0
        for off in range(0, len(idx), 512):                     # one NOTIFY_LISTENER_STATE message holds 512 records
            part = idx[off: off + 512]
            sums = (ge.SvcSummary * len(part))(*[rows[i] for i in part])
            buf = C.create_string_buffer(88 * len(part))
            nrecs, nbytes = C.c_uint32(), C.c_uint32()
            e._chk(e.L.gysk_encode_listener_state(sums, len(part), buf, len(buf), C.byref(nrecs), C.byref(nbytes)))
            recs = np.frombuffer(buf.raw[: nbytes.value], dtype=LSN)
            recs = recs[(recs["query_flags"] != LISTEN_FLAG_DELETE) & (recs["curr_state"] <= ge.STATE_DOWN)]
            qps += sum(int(q) // 5 for q in recs["nqrys_5s"])       # nqrys_5s_ is uint32: unsigned division
            kb += sum(int(x) for x in recs["kb_in"]) + sum(int(x) for x in recs["kb_out"])
        out[h] = (qps & M32, kb & M32)
    return out


def restate(engines, hosts, cids):
    """{cluster id: the row's 48 bytes} from every rank's host listen rows and host summaries"""
    of = dict(zip(hosts.tolist(), cids.tolist()))
    words = {c: [0] * 6 for c in cids.tolist()}
    for e in engines:
        summ = host_summ(e)
        listen, _ = e.query_host_listen()
        assert sorted(summ) == [x.host_idx for x in listen]
        for x in listen:
            c = of.get(x.host_idx)
            if c is None:
                continue
            qps, kb = summ[x.host_idx]
            w = words[c]
            w[0] += 1; w[1] += x.nlisten_issue; w[2] += x.nlisten_issue != 0; w[3] += x.nlisten; w[4] += qps; w[5] += _div1024(kb)
    return {c: ROW.pack(c, 1, 0, *[v & M32 for v in w], 0, 0) for c, w in words.items()}


def check_clusters(torch, engines, hosts, cids):
    """merge with the collectives emulated, then every read on every rank against the restatement; returns the restated rows"""
    _emulate_collectives(torch, engines)
    want = restate(engines, hosts, cids)
    dense = list(dict.fromkeys(cids.tolist()))
    ordered = sorted(dense)
    active = [c for c in ordered if ROW.unpack(want[c])[6]]       # nsvc > 0
    missing = ROW.pack(UNKNOWN, 0, 0, *([0] * 8))
    for r, e in enumerate(engines):
        assert [bytes(x) for x in e.query_cluster_states(dense + [UNKNOWN])] == [want[c] for c in dense] + [missing], r
        rows, n = e.query_cluster_states_all()
        assert n == len(ordered) and [bytes(x) for x in rows] == [want[c] for c in ordered], r
        arows, an = e.query_cluster_states_all(active_only=True)
        assert an == len(active) and [bytes(x) for x in arows] == [want[c] for c in active], r
        assert e.query_cluster_states_all(cap=0) == ([], len(ordered))
        part, pn = e.query_cluster_states_all(cap=1)
        assert pn == len(ordered) and [bytes(x) for x in part] == [want[ordered[0]]], r
    return {c: ROW.unpack(b)[3:9] for c, b in want.items()}


def late_events(rng, t):
    ids = synth.splitmix64(np.arange(1, len(LATE_HOSTS) + 1, dtype=np.uint64) + np.uint64(t << 40))
    ev = np.zeros(50 * len(ids), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = np.repeat(ids, 50); ev["host_idx"] = np.repeat(np.array(LATE_HOSTS, dtype=np.uint32), 50)
    ev["type"] = ge.EV_RESP; ev["value"] = rng.integers(1000, 50_000, len(ev)); ev["tsec"] = t
    return ev


@pytest.mark.gpu
@pytest.mark.parametrize("others", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_clusters_equal_the_restatement(world, others):
    """a stream that turns slow, error-prone and busy, with services that arrive after the last flush: every rank's rows equal the
    restatement at early and late flushes. Without the other flags no logical map is set: gysk_set_cluster_map alone sets up the merge"""
    import torch
    rng = np.random.default_rng(3100 + 10 * world + others)
    ids, conn_ids, ghost_ids = _ids()
    sh = Shards(world, merge_clusters=True, merge_levels=others, merge_states=others, **KW)
    hosts, cids = cluster_map(rng)
    if others:
        sh.set_map(*state_map(rng, ids, conn_ids, ghost_ids))
    for e in sh.engines:
        e.set_cluster_map(hosts, cids)
    issue_seen = 0
    for w, t in enumerate(TIMES):
        sh.feed(state_events(rng, w, ids, conn_ids), 1 << 14)
        sh.flush(t)
        if w not in (0, 9, 16, len(TIMES) - 1):
            continue
        sh.feed(late_events(rng, t), 1 << 14)
        got = check_clusters(torch, sh.engines, hosts, cids)
        issue_seen += sum(g[1] for g in got.values())
        assert got[500][0] == 8 and got[503] == (0,) * 6           # nhosts; a cluster of hosts without services
    assert issue_seen > 0


@pytest.mark.gpu
def test_net_mb_is_divided_per_host():
    """two hosts of one cluster with 1000 KB each give svc_net_mb 0, not 1; a host whose int32 kbyte sum wraps gives what the
    reference's int arithmetic gives"""
    import torch
    e = ge.Engine(merge_clusters=True, **KW)
    a, b, w = (int(x) for x in synth.splitmix64(np.arange(1, 4, dtype=np.uint64) + np.uint64(1 << 54)))
    hosts, cids = np.array([3, 4, 5], dtype=np.uint32), np.array([600, 600, 601], dtype=np.uint64)
    e.set_cluster_map(hosts, cids)
    ev = np.zeros(602, dtype=ge.EVENT_DTYPE)
    ev["type"] = ge.EV_ACCEPT; ev["flow_key"] = np.arange(1, 603); ev["tsec"] = 5
    ev["svc_id"][:2] = [a, b]; ev["host_idx"][:2] = [3, 4]; ev["value"][:2] = 1000 << 10
    ev["svc_id"][2:] = w; ev["host_idx"][2:] = 5; ev["value"][2:] = 0xFFFFFFFF
    e.ingest_events(ev)
    e.flush(5)
    got = check_clusters(torch, [e], hosts, cids)
    kb = 600 * (0xFFFFFFFF >> 10)
    assert kb >= 1 << 31 and got[600][5] == 0 and got[600][0] == 2
    assert got[601][5] == _div1024(kb) == (1 << 32) - ((1 << 32) - kb) // 1024                  # a negative int32, divided toward zero


@pytest.mark.gpu
def test_clusters_across_eviction_and_recycled_slots():
    """A is evicted and its slot goes to U, then A returns into G's slot after G is evicted: a host counts while it holds a live
    service, so host 0 leaves nhosts with A and comes back with it"""
    import torch
    sh = Shards(2, max_svcs=3, max_tasks=8, max_batch=1 << 14, cms_log2_width=10, idle_evict_secs=300, merge_clusters=True)
    A, B, U, F, G = (int(x) for x in synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 53)))
    host = {A: 0, F: 2, G: 4, U: 6, B: 1}
    hosts, cids = np.array([0, 1, 2, 4, 6], dtype=np.uint32), np.array([700, 700, 701, 701, 702], dtype=np.uint64)
    for e in sh.engines:
        e.set_cluster_map(hosts, cids)
    rng = np.random.default_rng(58)

    def window(t, live, n=400):
        ev = np.zeros(n * len(live), dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = np.repeat(np.array(live, dtype=np.uint64), n)
        ev["host_idx"] = np.repeat(np.array([host[x] for x in live], dtype=np.uint32), n)
        ev["type"] = np.where(rng.random(len(ev)) < 0.8, ge.EV_RESP, ge.EV_ACCEPT)
        ev["value"] = np.minimum(np.exp(rng.normal(np.log(3000.0), 1.2, len(ev))), 9.0e8).astype(np.uint32)
        ev["flow_key"] = rng.integers(1, 1 << 62, len(ev), dtype=np.uint64)
        ev["tsec"] = t
        sh.feed(ev[rng.permutation(len(ev))], 1 << 14)
        sh.flush(t)
        return set().union(*[set(int(i) for i in e.evicted_ids()) for e in sh.engines])

    def nhosts():
        got = check_clusters(torch, sh.engines, hosts, cids)
        return [got[c][0] for c in (700, 701, 702)]

    for t in (5, 10, 200, 400):
        window(t, [A, B, F, G] if t < 100 else [B, F, G])
    assert window(606, [B, F]) == {A}
    assert nhosts() == [1, 2, 0]
    window(620, [B, F, U])                                      # U takes A's slot
    assert nhosts() == [1, 2, 1]
    assert window(720, [B, F, U]) == {G}
    assert nhosts() == [1, 1, 1]
    window(730, [A, B, F, U])                                   # A returns into G's slot
    assert nhosts() == [2, 1, 1]


@pytest.mark.gpu
def test_cross_check_with_the_host_summary_path():
    """world 1: the shim's round trip (window rows -> LISTENER_STATE_NOTIFY -> gysk_ingest -> gysk_query_cluster_state over the cluster's
    hosts) gives the new row's nhosts, nsvc, total_qps and svc_net_mb"""
    import torch
    rng = np.random.default_rng(77)
    ids, conn_ids, _ = _ids()
    e = ge.Engine(merge_clusters=True, **KW)
    hosts, cids = cluster_map(rng)
    e.set_cluster_map(hosts, cids)
    for w, t in enumerate(TIMES[:12]):
        _feed_one(e, state_events(rng, w, ids, conn_ids), t)
    got = check_clusters(torch, [e], hosts, cids)
    rows, rhosts, _ = e.query_window_hosts()
    for h in sorted(set(rhosts.tolist())):
        part = [rows[i] for i in np.nonzero(rhosts == h)[0]]
        sums = (ge.SvcSummary * len(part))(*part)
        buf = C.create_string_buffer(88 * len(part))
        nrecs, nbytes = C.c_uint32(), C.c_uint32()
        e._chk(e.L.gysk_encode_listener_state(sums, len(part), buf, len(buf), C.byref(nrecs), C.byref(nbytes)))
        msg = wire.build_msg_fixed(ge.NOTIFY_LISTENER_STATE, np.frombuffer(buf.raw[: nbytes.value], dtype=np.dtype((np.void, 88))))
        assert e.ingest_msg(msg, host_idx=h) == 0
    for c, hs in CLUSTERS.items():
        old = e.cluster_state(hs)
        assert (old["nhosts"], old["nsvc"], old["total_qps"], old["svc_net_mb"]) == (got[c][0], got[c][3], got[c][4], got[c][5]), c
    assert got[500][3] > 0


def _feed_one(e, ev, t):
    for off in range(0, len(ev), KW["max_batch"]):
        e.ingest_events(ev[off: off + KW["max_batch"]])
        e.sync()
    e.flush(t)


@pytest.mark.gpu
def test_flag_off_is_unchanged_and_reads_are_read_only():
    """without the flag the arena's regions (names, sizes, bytes), the merge's launches and the rows are today's, and the new calls are
    GYSK_ERR_NOTSUP; with it the SUM region grows by the cluster words, the merge by two launches, and every read before a finished
    merge is GYSK_ERR_INVAL. The reads change nothing the merge left. Map errors, and either order of the two maps, give the same rows"""
    import torch
    rng = np.random.default_rng(29)
    ids, conn_ids, ghost_ids = _ids()
    glob, logical = state_map(rng, ids, conn_ids, ghost_ids)
    hosts, cids = cluster_map(rng)
    off, cl, late = ge.Engine(merge_states=True, **KW), ge.Engine(merge_states=True, merge_clusters=True, **KW), \
        ge.Engine(merge_states=True, merge_clusters=True, **KW)
    calls = [lambda: cl.query_cluster_states([500]), lambda: cl.query_cluster_states_all(), lambda: cl.query_cluster_states_all(True, cap=0)]
    assert [_code(c) for c in calls] == [INVAL] * 3                  # no map, no merge
    off.set_logical_map(glob, logical)
    cl.set_logical_map(glob, logical)
    cl.set_cluster_map(hosts, cids)
    late.set_cluster_map(hosts, cids)                                  # the cluster map first, the logical map after it
    late.set_logical_map(glob, logical)
    assert [_code(c) for c in calls] == [INVAL] * 3
    assert _code(lambda: off.set_cluster_map(hosts, cids)) == NOTSUP
    assert _code(lambda: cl.set_cluster_map(np.array([1, 2, 1], dtype=np.uint32), np.array([5, 6, 7], dtype=np.uint64))) == INVAL
    assert _code(lambda: cl.set_cluster_map(np.array([1 << 24], dtype=np.uint32), np.array([5], dtype=np.uint64))) == INVAL
    for w, t in enumerate(TIMES[:12]):
        for e in (off, cl, late):
            _feed_one(e, state_events(np.random.default_rng(w), w, ids, conn_ids), t)

    def launches(e, fn):
        k0 = e.stats()["kernel_launches"]
        fn()
        return e.stats()["kernel_launches"] - k0

    cl.merge_prepare()
    cl.sync()
    assert [_code(c) for c in calls] == [INVAL] * 3                  # prepared, not finished
    assert [launches(e, lambda: _emulate_collectives(torch, [e])) for e in (off, cl, late)] == [6, 8, 8]
    nl, c = len(set(logical.tolist())), off.cfg
    ncms = c.cms_depth << c.cms_log2_width
    sum0 = 2 * _align256(ncms * 8) + 2 * _align256(nl * 16 * 16) + _align256(nl * 32) + _align256(nl * 15 * 8)
    assert [(n, b, r) for n, _, b, r in off.merge_buffers()] == [
        ("sum_u64: cms_cur|cms_last|hist_last|hist_all|conn|states", sum0, gd.RED_SUM_U64),
        ("max_i64: hist max_val_seen", _align256(nl * 16), gd.RED_MAX_I64), ("max_u8: hll registers", _align256(nl << c.hll_p), gd.RED_MAX_U8)]
    nc = len(CLUSTERS)
    for e in (cl, late):
        bufs = e.merge_buffers()
        assert [(n, b) for n, _, b, _ in bufs] == [("sum_u64: cms_cur|cms_last|hist_last|hist_all|conn|states|clusters", sum0 + _align256(nc * 48)),
                                                   ("max_i64: hist max_val_seen", _align256(nl * 16)), ("max_u8: hll registers", _align256(nl << c.hll_p))]
        for (_, pa, na, _), (_, pb, nb, _) in zip(bufs, off.merge_buffers()):
            assert _dev_bytes(torch, pa, na).tobytes()[:nb] == _dev_bytes(torch, pb, nb).tobytes()
    lids = list(dict.fromkeys(logical.tolist()))
    assert repr(cl.query_logical(lids)) == repr(off.query_logical(lids))
    assert [bytes(x) for x in cl.query_logical_states(lids)] == [bytes(x) for x in off.query_logical_states(lids)]
    assert _code(lambda: off.query_cluster_states([500])) == NOTSUP
    assert _code(lambda: off.query_cluster_states_all()) == NOTSUP
    dense = list(dict.fromkeys(cids.tolist()))
    rows = [bytes(x) for x in cl.query_cluster_states(dense)]
    assert [bytes(x) for x in late.query_cluster_states(dense)] == rows
    regions = [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in cl.merge_buffers()]
    assert launches(cl, lambda: cl.query_cluster_states(dense)) == 1
    assert launches(cl, lambda: cl.query_cluster_states_all(cap=nc)) == 1
    assert launches(cl, lambda: cl.query_cluster_states_all(cap=0)) == 0
    assert launches(cl, lambda: cl.query_cluster_states_all(active_only=True, cap=nc)) == 2
    assert [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in cl.merge_buffers()] == regions
    assert [bytes(x) for x in cl.query_cluster_states(dense)] == rows
    assert launches(cl, lambda: _emulate_collectives(torch, [cl])) == 8          # the host words were cleared: the same rows again
    assert [bytes(x) for x in cl.query_cluster_states(dense)] == rows


def _nccl_uid():
    try:
        return ge.Engine(max_svcs=64, max_tasks=8, max_batch=4096, cms_log2_width=8).nccl_unique_id()
    except ge.GyskError as ex:
        pytest.skip(f"NCCL not loadable: {ex}")


def _run(engines, ids, conn_ids):
    for w, t in enumerate(TIMES[:12]):
        for e in engines:
            _feed_one(e, state_events(np.random.default_rng(w), w, ids, conn_ids), t)


@pytest.mark.gpu
def test_library_nccl_merge_equals_the_emulation():
    """gysk_merge_global (NCCL inside the library) at world 1 leaves the same region bytes and cluster rows as the emulated collectives"""
    import torch
    uid = _nccl_uid()
    ids, conn_ids, _ = _ids()
    hosts, cids = cluster_map(np.random.default_rng(92))
    dense = list(dict.fromkeys(cids.tolist()))
    e = ge.Engine(merge_clusters=True, **KW)
    e.set_cluster_map(hosts, cids)
    _run([e], ids, conn_ids)
    _emulate_collectives(torch, [e])
    region = lambda x: [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in x.merge_buffers()]     # noqa: E731
    emu_bytes, emu_rows = region(e), [bytes(x) for x in e.query_cluster_states(dense)]
    e.nccl_comm_init(uid, 1, 0)
    e.merge_global()
    e.sync()
    assert region(e) == emu_bytes and [bytes(x) for x in e.query_cluster_states(dense)] == emu_rows


@pytest.mark.gpu
def test_two_device_nccl_merge_equals_the_emulation():
    """two engines on two devices merged by gysk_merge_global equal two emulated shards on one device"""
    import threading

    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("the two-device NCCL merge needs two GPUs")
    _nccl_uid()
    ids, conn_ids, _ = _ids()
    hosts, cids = cluster_map(np.random.default_rng(93))
    dense = list(dict.fromkeys(cids.tolist()))
    emu = [ge.Engine(rank=r, world=2, merge_clusters=True, **KW) for r in range(2)]
    lib = [ge.Engine(device=r, rank=r, world=2, merge_clusters=True, **KW) for r in range(2)]
    for x in emu + lib:
        x.set_cluster_map(hosts, cids)
    _run(emu + lib, ids, conn_ids)
    _emulate_collectives(torch, emu)
    uid2 = lib[0].nccl_unique_id()
    errs = []

    def merge(r):
        try:
            lib[r].nccl_comm_init(uid2, 2, r)
            lib[r].merge_global()
            lib[r].sync()
        except Exception as ex:      # noqa: BLE001
            errs.append(ex)
    th = [threading.Thread(target=merge, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errs, errs
    want = [bytes(x) for x in emu[0].query_cluster_states(dense)]
    assert [bytes(x) for x in lib[0].query_cluster_states(dense)] == want and [bytes(x) for x in lib[1].query_cluster_states(dense)] == want


def test_symbols_and_layout_match_the_header():
    """no device needed: the new entry points are exported and answer GYSK_ERR_INVAL without an engine; the flag and the row layout are
    the header's"""
    L = ge.load_library()
    n = C.c_uint32()
    ids = np.array([1], dtype=np.uint64)
    hosts = np.array([1], dtype=np.uint32)
    out = (ge.ClusterRow * 1)()
    assert L.gysk_set_cluster_map(None, ge._p(hosts), ge._p(ids), 1) == INVAL
    assert L.gysk_query_cluster_states(None, ge._p(ids), 1, out) == INVAL
    assert L.gysk_query_cluster_states_all(None, 0, out, 1, C.byref(n)) == INVAL
    hdr = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert int(re.search(r"#define GYSK_FLAG_MERGE_CLUSTERS\s+(0x[0-9a-fA-F]+)u", hdr).group(1), 16) == ge.FLAG_MERGE_CLUSTERS == 8
    body = re.search(r"typedef struct gysk_cluster_row\s*\{(.*?)\}\s*gysk_cluster_row;", hdr, re.S).group(1)
    fields = re.findall(r"^\s*(\w+)\s+(\w+);", body, re.M)
    assert fields == [("uint64_t", "cluster_id"), ("int32_t", "found"), ("uint32_t", "pad"), ("gysk_cluster_state", "st")]
    assert [(f, getattr(ge.ClusterRow, f).offset) for f, _ in ge.ClusterRow._fields_] == [("cluster_id", 0), ("found", 8), ("pad", 12), ("st", 16)]
    assert [(f, getattr(ge.ClusterState, f).offset) for f, _ in ge.ClusterState._fields_] == [
        ("nhosts", 0), ("nsvc_issue", 4), ("nsvcissue_hosts", 8), ("nsvc", 12), ("total_qps", 16), ("svc_net_mb", 20), ("pad", 24)]
    assert C.sizeof(ge.ClusterState) == 32 and C.sizeof(ge.ClusterRow) == 48
