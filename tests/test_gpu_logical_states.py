"""The listener states of logical services (GYSK_FLAG_MERGE_STATES): gysk_query_logical_states, gysk_query_logical_states_all and the
GYSK_TOPN_ISSUE ranking of gysk_topn_logical, at world 1 ... 8 with and without GYSK_FLAG_MERGE_LEVELS, over late members, ghost ids,
connection-only members, eviction and recycled slots. Each logical row is restated from the member rows every rank gives with
gysk_query_svcs right after the merge: LISTEN_SUMM_STATS::update (server/gy_msocket.h:853-864) of each member's LISTENER_STATE_NOTIFY,
int32 wrap-around, summed over ranks. The members' states themselves are pinned to the CPU oracle's."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

from gyeeta_b200 import dist as gd
from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import Shards, _align256, _dev_bytes

INVAL, NOENT, NOTSUP = -22, -2, -95
M32 = 0xFFFFFFFF
UNKNOWN = 123456789
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(max_svcs=256, max_tasks=16, max_batch=1 << 14, cms_log2_width=10)
NSVC, NHOSTS = 64, 16
LATE = range(56, 64)                    # services whose first events arrive at window 10, after the map was set
TIMES = [5 + 40 * w for w in range(24)]
ROW = struct.Struct("<QiI16i")
assert ROW.size == C.sizeof(ge.LogicalState) == 80


def _code(fn):
    with pytest.raises(ge.GyskError) as ei:
        fn()
    return ei.value.code


def _i32(v):
    v &= M32
    return v - (1 << 32) if v >> 31 else v


def _ids():
    ids = synth.service_ids(NSVC)
    conn_ids = synth.splitmix64(np.arange(1, 3, dtype=np.uint64) + np.uint64(1 << 51))
    ghost_ids = synth.splitmix64(np.arange(1, 4, dtype=np.uint64) + np.uint64(1 << 52))
    return ids, conn_ids, ghost_ids


def state_map(rng, ids, conn_ids, ghost_ids):
    """(glob ids, logical ids) in a shuffled map order:
      8000: services 0..15, one per host => members on every rank
      8100 + i: singletons (services 16..31)
      8001: services 32..55
      8002: ids that never register
      8003: services that register at window 10
      8004: two members with connection events only
    Every id maps to one logical service."""
    pairs = [(ids[i], 8000) for i in range(16)] + [(ids[i], 8100 + i) for i in range(16, 32)]
    pairs += [(ids[i], 8001) for i in range(32, 56)] + [(g, 8002) for g in ghost_ids]
    pairs += [(ids[i], 8003) for i in LATE] + [(c, 8004) for c in conn_ids]
    perm = rng.permutation(len(pairs))
    return (np.array([int(pairs[i][0]) for i in perm], dtype=np.uint64), np.array([pairs[i][1] for i in perm], dtype=np.uint64))


def state_events(rng, w, ids, conn_ids, n=6000):
    """the stream of test_gpu_day_stats that drives device-evaluated states to BAD and SEVERE (slow responses, server errors, more
    queries and many active connections), spread over NHOSTS hosts, plus connection events of the connection-only members"""
    k = rng.integers(0, NSVC, n)
    k = k[(k < LATE.start) | (w >= 10)]
    ev = np.zeros(len(k), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = ids[k]; ev["host_idx"] = k % NHOSTS; ev["type"] = ge.EV_RESP
    slow = (w >= 6) & (k % 4 == 0)
    ev["value"] = np.minimum(np.exp(rng.normal(np.log(20_000.0), 1.0, len(k))) * np.where(slow, 8.0, 1.0), 9e8).astype(np.uint32)
    ev["flow_key"] = rng.integers(0, 1 << 16, len(k))
    err = (w >= 4) & (k % 5 == 1) & (rng.random(len(k)) < (0.7 if w % 2 else 0.15))
    ev["flags"] = np.where(err, ge.EVF_SER_ERROR, 0)
    ev["tsec"] = TIMES[w]
    if w >= 8:
        ev = np.concatenate([ev] + [ev[(k % 4 == 2)]] * 5)
    parts = [ev]
    if w % 3 == 0:
        act = np.zeros(48, dtype=ge.EVENT_DTYPE)
        act["svc_id"] = ids[:48]; act["host_idx"] = np.arange(48) % NHOSTS; act["type"] = ge.EV_ACTIVE; act["flow_key"] = 77
        act["flags"] = np.where((np.arange(48) % 8 == 3) & (w >= 9), 400, 3 + (np.arange(48) % 5))
        parts.append(act)
    cn = np.zeros(60 * len(conn_ids), dtype=ge.EVENT_DTYPE)
    cn["svc_id"] = np.repeat(conn_ids, 60); cn["host_idx"] = np.repeat(np.arange(1, len(conn_ids) + 1, dtype=np.uint32), 60)
    cn["type"] = rng.choice([ge.EV_ACCEPT, ge.EV_CLOSE_SER, ge.EV_CONNECT], len(cn))
    cn["value"] = rng.integers(0, 1 << 22, len(cn)); cn["flow_key"] = rng.integers(1, 1 << 62, len(cn), dtype=np.uint64)
    parts.append(cn)
    ev = np.concatenate(parts)
    return ev[rng.permutation(len(ev))]


def restate(sh):
    """{logical id: the row's 80 bytes} from every rank's gysk_query_svcs rows of the members; each found member's curr_state is
    checked against its rank's oracle. Returns (rows, nsvc_issue by logical id, members in BAD or worse, members found)"""
    members = {}
    for g, l in zip(sh.glob.tolist(), sh.logical.tolist()):
        members.setdefault(l, []).append(g)
    rows, issue, bad, found = {}, {}, 0, 0
    for lid, gs in members.items():
        w = [0] * 15
        for r, e in enumerate(sh.engines):
            for g, s in zip(gs, e.query_svcs(gs)):
                if not s["found"]:
                    continue
                assert s["curr_state"] == sh.oracles[r].export_state(g)[0], (r, g)
                st = s["curr_state"]
                if st > ge.STATE_DOWN:
                    continue
                found += 1
                bad += st >= ge.STATE_BAD
                w[st] += 1
                w[8] += s["nqrys_5s"] // 5                           # LISTENER_STATE_NOTIFY::nqrys_5s_ is uint32: unsigned division
                w[9] += s["nconns_active"]
                w[10] += s["kbytes_5s"]                              # curr_kbytes_inbound_; curr_kbytes_outbound_ stays 0
                w[12] += s["ser_errors"]
                w[13] += 1
                w[14] += s["nqrys_5s"] != 0
        issue[lid] = (w[3] + w[4] + w[5]) & M32
        rows[lid] = ROW.pack(lid, 1, issue[lid], *[_i32(x) for x in w], 0)
    return rows, issue, bad, found


def _feed(engines, ev, t):
    for e in engines:
        for off in range(0, len(ev), KW["max_batch"]):
            e.ingest_events(ev[off: off + KW["max_batch"]])
            e.sync()
        e.flush(t)


def _raw_states(e, ids):
    return [bytes(x) for x in e.query_logical_states(ids)]


def _raw_topn(e, metric, n):
    out = (ge.TopnEntry * n)()
    k = C.c_uint32()
    e._chk(e.L.gysk_topn_logical(e.h, metric, n, out, C.byref(k)))
    return b"".join(bytes(o) for o in out[: k.value])


def check_states(torch, sh):
    """merge with the collectives emulated, restate, then every new read on every rank; returns the restated nsvc_issue by logical id
    and the members in BAD or worse"""
    _emulate_collectives(torch, sh.engines)
    want, issue, bad, found = restate(sh)
    dense = list(dict.fromkeys(sh.logical.tolist()))          # dense logical index = order of first appearance
    lids = sorted(dense)
    missing = ROW.pack(UNKNOWN, 0, 0, *([0] * 16))
    order = sorted(((s, dense.index(l), l) for l, s in issue.items() if s > 0), reverse=True)
    tops = {}
    for r, e in enumerate(sh.engines):
        assert _raw_states(e, dense + [UNKNOWN]) == [want[l] for l in dense] + [missing], r
        rows, n = e.query_logical_states_all()
        assert n == len(lids) and [bytes(x) for x in rows] == [want[l] for l in lids], r
        active = [x.glob_id for x in e.query_logical_all(active_only=True)[0]]
        arows, an = e.query_logical_states_all(active_only=True)
        assert an == len(active) and [bytes(x) for x in arows] == [want[l] for l in active], r
        assert e.query_logical_states_all(cap=0) == ([], len(lids))
        for cap in (1, max(1, len(lids) // 3)):
            part, pn = e.query_logical_states_all(cap=cap)
            assert pn == len(lids) and [bytes(x) for x in part] == [want[l] for l in lids[:cap]], (r, cap)
        for k in (1, 7, 64):
            assert e.topn_logical(ge.TOPN_ISSUE, k) == [(l, s, 0) for s, _, l in order[:k]], (r, k)
            tops.setdefault(k, set()).add(_raw_topn(e, ge.TOPN_ISSUE, k))
        assert all(x["curr_state"] == 0 and x["curr_issue"] == 0 for x in e.query_logical(lids))     # logical services stay unclassified
    assert all(len(v) == 1 for v in tops.values())                 # identical bytes on every rank
    return issue, bad, found


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_states_equal_the_restatement(world, levels):
    """a stream that turns slow, error-prone and busy: every rank's rows, the all-rows read and the issue ranking equal the restatement
    at early and late flushes; by the end some logical services have members in issue and others none"""
    import torch
    rng = np.random.default_rng(2100 + 10 * world + levels)
    ids, conn_ids, ghost_ids = _ids()
    sh = Shards(world, merge_levels=levels, merge_states=True, **KW)
    sh.set_map(*state_map(rng, ids, conn_ids, ghost_ids))
    bad_seen = 0
    for w, t in enumerate(TIMES):
        sh.feed(state_events(rng, w, ids, conn_ids), 1 << 14)
        sh.flush(t)
        if w not in (0, 9, 16, len(TIMES) - 1):
            continue
        issue, bad, found = check_states(torch, sh)
        bad_seen += bad
        assert found > 0
    assert bad_seen > 0
    assert any(s > 0 for s in issue.values()) and any(s == 0 for l, s in issue.items() if l != 8002)
    assert issue[8002] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [False, True])
def test_states_across_eviction_and_recycled_slots(levels):
    """test_gpu_logical_reads' eviction scenario: A (logical 7000 with B) is evicted, its slot goes to U outside the map, then A returns
    into another slot; the members counted are the ones holding a slot at each merge"""
    import torch
    sh = Shards(2, max_svcs=3, max_tasks=8, max_batch=1 << 14, cms_log2_width=10, idle_evict_secs=300, merge_levels=levels, merge_states=True)
    A, B, U, F, G = (int(x) for x in synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 53)))
    host = {A: 0, F: 2, G: 4, U: 6, B: 1}
    sh.set_map(np.array([B, A], dtype=np.uint64), np.array([7000, 7000], dtype=np.uint64))
    rng = np.random.default_rng(48 + levels)

    def window(t, live, n=400):
        ev = np.zeros(n * len(live), dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = np.repeat(np.array(live, dtype=np.uint64), n)
        ev["host_idx"] = np.repeat(np.array([host[a] for a in live], dtype=np.uint32), n)
        ev["type"] = np.where(rng.random(len(ev)) < 0.8, ge.EV_RESP, ge.EV_ACCEPT)
        ev["value"] = np.minimum(np.exp(rng.normal(np.log(3000.0), 1.2, len(ev))), 9.0e8).astype(np.uint32)
        ev["flags"] = np.where((ev["type"] == ge.EV_RESP) & (rng.random(len(ev)) < 0.3), ge.EVF_SER_ERROR, 0)
        ev["flow_key"] = rng.integers(1, 1 << 62, len(ev), dtype=np.uint64)
        ev["tsec"] = t
        sh.feed(ev[rng.permutation(len(ev))], 1 << 14)
        sh.flush(t)
        return set().union(*[set(int(i) for i in e.evicted_ids()) for e in sh.engines])

    for t in (5, 10, 200, 400):
        window(t, [A, B, F, G] if t < 100 else [B, F, G])
    assert window(606, [B, F]) == {A}
    assert check_states(torch, sh)[2] == 1                      # B alone
    window(620, [B, F, U])                                      # U takes A's slot
    assert check_states(torch, sh)[2] == 1
    assert window(720, [B, F, U]) == {G}
    window(730, [A, B, F, U])                                   # A returns into G's slot
    assert check_states(torch, sh)[2] == 2


@pytest.mark.gpu
def test_every_read_needs_a_finished_merge():
    """GYSK_ERR_INVAL without a map, with a map before a merge, and after gysk_merge_prepare before gysk_merge_finish"""
    rng = np.random.default_rng(9)
    ids, conn_ids, ghost_ids = _ids()
    e = ge.Engine(merge_states=True, **KW)
    calls = [lambda: e.query_logical_states([8000]), lambda: e.query_logical_states_all(), lambda: e.query_logical_states_all(True, cap=0),
             lambda: e.topn_logical(ge.TOPN_ISSUE)]
    assert [_code(c) for c in calls] == [INVAL] * len(calls)
    e.set_logical_map(*state_map(rng, ids, conn_ids, ghost_ids))
    assert [_code(c) for c in calls] == [INVAL] * len(calls)
    _feed([e], state_events(rng, 0, ids, conn_ids), 5)
    e.merge_prepare()
    e.sync()
    assert [_code(c) for c in calls] == [INVAL] * len(calls)
    e.merge_finish()
    rows, n = e.query_logical_states_all()
    assert n == len(rows) > 0 and e.query_logical_states([8000])[0].found == 1
    e.close()


@pytest.mark.gpu
def test_flag_off_is_unchanged_and_reads_are_read_only():
    """engines without the flag, with it alone and with both flags, fed the same stream: without it the arena's regions (names, sizes),
    the merge's five launches and the rows are today's, the new reads are GYSK_ERR_NOTSUP and the issue ranking GYSK_ERR_INVAL; the flag
    adds one launch and its words behind the old part of the SUM region, and leaves every gysk_query_logical row as it was. The reads
    change nothing the merge left"""
    import torch
    rng = np.random.default_rng(23)
    ids, conn_ids, ghost_ids = _ids()
    off, st, both = ge.Engine(**KW), ge.Engine(merge_states=True, **KW), ge.Engine(merge_levels=True, merge_states=True, **KW)
    glob, logical = state_map(rng, ids, conn_ids, ghost_ids)
    lids = list(dict.fromkeys(logical.tolist()))
    for e in (off, st, both):
        e.set_logical_map(glob, logical)
    for w, t in enumerate(TIMES[:12]):
        _feed((off, st, both), state_events(rng, w, ids, conn_ids), t)

    def launches(e, fn):
        k0 = e.stats()["kernel_launches"]
        fn()
        return e.stats()["kernel_launches"] - k0

    assert [launches(e, lambda: _emulate_collectives(torch, [e])) for e in (off, st, both)] == [5, 6, 7]
    nl, c = len(lids), off.cfg
    ncms = c.cms_depth << c.cms_log2_width
    sizes = [2 * _align256(ncms * 8) + 2 * _align256(nl * 16 * 16) + _align256(nl * 32), _align256(nl * 16), _align256(nl << c.hll_p)]
    assert [(n, b, r) for n, _, b, r in off.merge_buffers()] == [
        ("sum_u64: cms_cur|cms_last|hist_last|hist_all|conn", sizes[0], gd.RED_SUM_U64),
        ("max_i64: hist max_val_seen", sizes[1], gd.RED_MAX_I64), ("max_u8: hll registers", sizes[2], gd.RED_MAX_U8)]
    states_bytes = _align256(nl * 15 * 8)
    assert [(n, b) for n, _, b, _ in st.merge_buffers()] == [("sum_u64: cms_cur|cms_last|hist_last|hist_all|conn|states", sizes[0] + states_bytes),
                                                            ("max_i64: hist max_val_seen", sizes[1]), ("max_u8: hll registers", sizes[2])]
    lvl_sum = _align256(2 * nl * 16 * 16) + _align256(nl * 32)
    assert [(n, b) for n, _, b, _ in both.merge_buffers()][0] == ("sum_u64: cms_cur|cms_last|hist_last|hist_all|conn|levels|aux|states",
                                                                 sizes[0] + lvl_sum + states_bytes)
    for (_, pa, _, _), (_, pb, nb, _) in zip(st.merge_buffers(), off.merge_buffers()):
        assert _dev_bytes(torch, pa, nb).tobytes() == _dev_bytes(torch, pb, nb).tobytes()
    assert repr(st.query_logical(lids)) == repr(off.query_logical(lids))
    # without the flag
    assert _code(lambda: off.query_logical_states(lids)) == NOTSUP
    assert _code(lambda: off.query_logical_states_all()) == NOTSUP
    assert _code(lambda: off.topn_logical(ge.TOPN_ISSUE, 5)) == INVAL
    assert off.topn_logical(ge.TOPN_QPS, 5)
    # read-only reads, and their launches: one per by-id chunk, one per all-rows pass, one select more under ACTIVE_ONLY, a top-N as
    # many as gysk_topn_svcs
    for e, merge_launches in ((st, 6), (both, 7)):
        regions = [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in e.merge_buffers()]
        rows, srows = repr(e.query_logical(lids)), _raw_states(e, lids)
        assert launches(e, lambda: e.query_logical_states(lids)) == 1
        assert launches(e, lambda: e.query_logical_states_all(cap=nl)) == 1
        assert launches(e, lambda: e.query_logical_states_all(cap=0)) == 0
        assert launches(e, lambda: e.query_logical_states_all(active_only=True, cap=nl)) == 2
        assert launches(e, lambda: e.topn_logical(ge.TOPN_ISSUE, 64)) == launches(e, lambda: e.topn(ge.TOPN_ISSUE, 64))
        assert [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in e.merge_buffers()] == regions
        assert repr(e.query_logical(lids)) == rows and _raw_states(e, lids) == srows
        assert launches(e, lambda: _emulate_collectives(torch, [e])) == merge_launches
        assert repr(e.query_logical(lids)) == rows and _raw_states(e, lids) == srows
    assert _raw_states(st, lids) == _raw_states(both, lids)          # the levels flag changes no state word


def _nccl_uid():
    try:
        return ge.Engine(max_svcs=64, max_tasks=8, max_batch=4096, cms_log2_width=8).nccl_unique_id()
    except ge.GyskError as ex:
        pytest.skip(f"NCCL not loadable: {ex}")


def _nccl_setup():
    ids, conn_ids, ghost_ids = _ids()
    glob, logical = state_map(np.random.default_rng(91), ids, conn_ids, ghost_ids)

    def run(engines, times=TIMES[:12]):
        for w, t in enumerate(times):
            _feed(engines, state_events(np.random.default_rng(w), w, ids, conn_ids), t)
    return glob, logical, list(dict.fromkeys(logical.tolist())), run


@pytest.mark.gpu
def test_library_nccl_merge_equals_the_emulation():
    """gysk_merge_global (NCCL inside the library) at world 1 leaves the same region bytes and state rows as the emulated collectives"""
    import torch
    uid = _nccl_uid()
    glob, logical, lids, run = _nccl_setup()
    e = ge.Engine(merge_states=True, **KW)
    e.set_logical_map(glob, logical)
    run([e])
    _emulate_collectives(torch, [e])
    region = lambda x: [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in x.merge_buffers()]     # noqa: E731
    emu_bytes, emu_rows = region(e), _raw_states(e, lids)
    e.nccl_comm_init(uid, 1, 0)
    e.merge_global()
    e.sync()
    assert region(e) == emu_bytes and _raw_states(e, lids) == emu_rows


@pytest.mark.gpu
def test_two_device_nccl_merge_equals_the_emulation():
    """two engines on two devices merged by gysk_merge_global equal two emulated shards on one device"""
    import threading

    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("the two-device NCCL merge needs two GPUs")
    _nccl_uid()
    glob, logical, lids, run = _nccl_setup()
    emu = [ge.Engine(rank=r, world=2, merge_states=True, **KW) for r in range(2)]
    lib = [ge.Engine(device=r, rank=r, world=2, merge_states=True, **KW) for r in range(2)]
    for x in emu + lib:
        x.set_logical_map(glob, logical)
    run(emu + lib)
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
    want = _raw_states(emu[0], lids)
    assert _raw_states(lib[0], lids) == want and _raw_states(lib[1], lids) == want


def test_symbols_and_layout_match_the_header():
    """no device needed: the new entry points are exported and answer GYSK_ERR_INVAL without an engine; the flag and the struct layout
    are the header's"""
    L = ge.load_library()
    n = C.c_uint32()
    ids = np.array([1], dtype=np.uint64)
    out = (ge.LogicalState * 1)()
    assert L.gysk_query_logical_states(None, ge._p(ids), 1, out) == INVAL
    assert L.gysk_query_logical_states_all(None, 0, out, 1, C.byref(n)) == INVAL
    hdr = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert int(re.search(r"#define GYSK_FLAG_MERGE_STATES\s+(0x[0-9a-fA-F]+)u", hdr).group(1), 16) == ge.FLAG_MERGE_STATES == 4
    body = re.search(r"typedef struct gysk_logical_state\s*\{(.*?)\}\s*gysk_logical_state;", hdr, re.S).group(1)
    fields = re.findall(r"^\s*(\w+)\s+(\w+);", body, re.M)
    assert fields == [("uint64_t", "logical_id"), ("int32_t", "found"), ("uint32_t", "nsvc_issue"), ("gysk_host_summary", "summ")]
    assert [(f, getattr(ge.LogicalState, f).offset) for f, _ in ge.LogicalState._fields_] == [("logical_id", 0), ("found", 8), ("nsvc_issue", 12),
                                                                                            ("summ", 16)]
    assert C.sizeof(ge.HostSummary) == 64 and C.sizeof(ge.LogicalState) == 80
