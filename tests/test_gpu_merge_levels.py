"""The merge step with GYSK_FLAG_MERGE_LEVELS: the 300-s / 5-day levels, active connections, errors and max rtt of the member
services folded into each logical service. Every one of them is an integer sum or maximum, so the logical rows are pinned bit for
bit: against a restatement from one oracle engine per rank (the level cells of export_hist(g, 6 / 7), the aux words of export_aux,
both as each member's own row shows them), against a single unsharded engine, and against the compiled reference's
update_from_serialized + get_percentiles. Without the flag the merge must be exactly what it was."""
import numpy as np
import pytest

from gyeeta_b200 import dist as gd
from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import DOUBLE_FIELDS, INT_FIELDS, NSVC, Shards, _align256, _dev_bytes, assert_summary, logical_map, window_events
from tests.util import M32, MergeRestatement, same_double

pytestmark = pytest.mark.gpu

# the flush schedule of test_gpu_parity.test_rolling_levels_300s_and_5days: its time jumps expire slots of both rings
TIMES = [5, 10, 15, 35, 65, 300, 305, 310, 3905, 3910, 50_000, 50_005, 500_000, 500_005]
CHECK_AT = {15, 310, 3910, 50_005, 500_005}
LEVEL_FIELDS = ["p95_5min_resp_ms", "p99_5min_resp_ms", "nqrys_5min", "p95_5day_resp_ms", "nqrys_5day", "nconns_active", "active_kbytes",
                "max_rtt_msec", "cli_errors", "ser_errors"]
STATE_FIELDS = ["curr_state", "curr_issue", "issue_bit_hist", "high_resp_bit_hist"]
KW = dict(max_svcs=1024, max_tasks=128, max_batch=1 << 16, cms_log2_width=12)
INT64_MIN = -(1 << 63)


def _f32_bits(x):
    return int(np.array([x], dtype=np.float32).view(np.uint32)[0])


def _pct(lib, cells, pcts):
    ser = np.zeros(15, dtype=po.SERIAL_DTYPE)
    ser[:] = cells
    p = np.array(pcts, dtype=np.float32)
    out = np.zeros(len(p), dtype=np.int64)
    assert lib.gysk_hist_percentiles(0, 0, po._p(ser), int(cells["count"].sum()), po._p(p), len(p), po._p(out)) == 0
    return out.tolist()


class LevelRestatement(MergeRestatement):
    """MergeRestatement plus what the flag adds: each member's level cells (its own export_hist(g, 6 / 7)) summed over members and
    ranks, the level maxima, the aux halves summed, the largest rtt bit pattern"""

    def levels(self, lid):
        lvl = [np.zeros(15, dtype=po.SERIAL_DTYPE) for _ in range(2)]
        mx, aux, rtt = [INT64_MIN, INT64_MIN], [0, 0, 0, 0], 0
        for orc in self.oracles:
            for g in self.members.get(int(lid), []):
                if orc.export_hist(g, 1) is None:
                    continue
                for k, which in enumerate((ge.HIST_RESP_5MIN, ge.HIST_RESP_5DAY)):
                    h = orc.export_hist(g, which)
                    lvl[k]["count"] += h[0]["count"]; lvl[k]["sum"] += h[0]["sum"]
                    mx[k] = max(mx[k], h[2])
                a = orc.export_aux(g)
                aux[0] += a["act_last"] & M32; aux[1] += a["act_last"] >> 32
                aux[2] += a["err_last"] & M32; aux[3] += a["err_last"] >> 32
                rtt = max(rtt, _f32_bits(a["rtt_last"]))
        return dict(lvl=lvl, max=mx, aux=aux, rtt=rtt)

    def summary(self, lid, eng_lib):
        d = super().summary(lid, eng_lib)
        c = self.levels(lid)
        p5m, p5d = _pct(eng_lib, c["lvl"][0], [95.0, 99.0]), _pct(eng_lib, c["lvl"][1], [95.0])
        d.update(p95_5min_resp_ms=p5m[0], p99_5min_resp_ms=p5m[1], nqrys_5min=int(c["lvl"][0]["count"].sum()), p95_5day_resp_ms=p5d[0],
                 nqrys_5day=int(c["lvl"][1]["count"].sum()), nconns_active=c["aux"][0] & M32, active_kbytes=c["aux"][1] & M32,
                 cli_errors=c["aux"][2] & M32, ser_errors=c["aux"][3] & M32,
                 max_rtt_msec=float(np.array([c["rtt"]], dtype=np.uint32).view(np.float32)[0]))
        return d


def _events(rng, w, n, ids, conn_ids):
    """test_gpu_merge_exact's window stream, with 3 % of its response samples marked as API client or server errors"""
    ev = window_events(rng, w, n, ids, conn_ids)
    err = (ev["type"] == ge.EV_RESP) & (rng.random(len(ev)) < 0.03)
    ev["flags"][err] = rng.choice([ge.EVF_CLI_ERROR, ge.EVF_SER_ERROR, ge.EVF_CLI_ERROR | ge.EVF_SER_ERROR], int(err.sum()))
    return ev


def _stream_ids():
    ids = synth.service_ids(NSVC)
    conn_ids = synth.splitmix64(np.arange(1, 4, dtype=np.uint64) + np.uint64(1 << 51))
    ghost_ids = synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 52))
    return ids, conn_ids, ghost_ids


def _feed(engines, ev, batch=1 << 16):
    for off in range(0, len(ev), batch):
        for e in engines:
            e.ingest_events(ev[off: off + batch])
            e.sync()


def _check_levels(torch, sh):
    """merge with the collectives emulated, then every field of every logical row on every rank against LevelRestatement, and
    gysk_export_logical_hist against the restated cells; returns the restated rows"""
    _emulate_collectives(torch, sh.engines)
    rs = LevelRestatement(sh.oracles, sh.glob, sh.logical, sh.delta, sh.hll_p)
    lids = list(dict.fromkeys(sh.logical.tolist()))
    lib = ge.load_library()
    want = {lid: rs.summary(lid, lib) for lid in lids}
    for r, e in enumerate(sh.engines):
        for lid, got in zip(lids, e.query_logical(lids)):
            assert_summary(got, want[lid], (r, lid))
    e = sh.engines[-1]
    for lid in lids:
        c, cl = rs.levels(lid), rs.cells(lid)
        for which, cells, mx in ((ge.HIST_RESP_LAST, cl["last"], cl["max_last"]), (ge.HIST_RESP_ALL, cl["all"], cl["max_all"]),
                                 (ge.HIST_RESP_5MIN, c["lvl"][0], c["max"][0]), (ge.HIST_RESP_5DAY, c["lvl"][1], c["max"][1])):
            ser, total, gmx = e.export_logical_hist(lid, which)
            assert np.array_equal(ser["count"], cells["count"]) and np.array_equal(ser["sum"], cells["sum"]), (lid, which)
            assert total == int(cells["count"].sum()), (lid, which, total)
            if which in (ge.HIST_RESP_5MIN, ge.HIST_RESP_5DAY) and total == 0:
                mx = INT64_MIN
            assert gmx == mx, (lid, which, gmx, mx)
    assert e.export_logical_hist(123456789, ge.HIST_RESP_5MIN) is None
    return want


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_levels_equal_the_restatement(world):
    """the map of test_gpu_merge_exact (late members, ghost ids, members with connection events only) over the flush schedule whose
    jumps expire slots of both rings: every field of every logical row equals the restatement at every checked flush"""
    import torch
    rng = np.random.default_rng(900 + world)
    ids, conn_ids, ghost_ids = _stream_ids()
    sh = Shards(world, merge_levels=True, **KW)
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    sh.set_map(glob, logical)
    seen = dict(lvl5m=0, lvl5d=0, act=0, err=0, rtt=0, expired5m=0, expired5d=0)
    for w, t in enumerate(TIMES):
        sh.feed(_events(rng, w, 20_000, ids, conn_ids), 1 << 16)
        sh.flush(t)
        if t not in CHECK_AT:
            continue
        want = _check_levels(torch, sh)
        assert all(e.merge_flush_range() == (t, t) for e in sh.engines)
        for row in want.values():
            seen["lvl5m"] += row["nqrys_5min"] > 0; seen["lvl5d"] += row["nqrys_5day"] > 0
            seen["act"] += row["nconns_active"] > 0; seen["err"] += row["cli_errors"] + row["ser_errors"] > 0
            seen["rtt"] += row["max_rtt_msec"] > 0
            seen["expired5m"] += row["nqrys_5min"] < row["nqrys_5day"]; seen["expired5d"] += row["nqrys_5day"] < row["nqrys_all"]
        assert want[9002]["nqrys_5day"] == 0 and want[9002]["p95_5day_resp_ms"] == -1       # ghosts only
        assert want[9003]["nqrys_5min"] == 0 and want[9003]["found"] == 1                     # connection events only
    # the stream exercised what the flag merges: levels, active connections, errors, rtt, and expiry of ring slots
    for k, v in seen.items():
        assert v > 0, (k, seen)


def test_eviction_with_recycled_slots():
    """test_gpu_merge_exact's eviction scenario with the flag: A (logical 7000 with B) is evicted, its slot goes to U outside the map,
    then A returns into another slot. The levels of A's first life and U's never count"""
    import torch
    sh = Shards(2, max_svcs=3, max_tasks=8, max_batch=1 << 14, cms_log2_width=10, idle_evict_secs=300, merge_levels=True)
    A, B, U, F, G = (int(x) for x in synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 53)))
    host = {A: 0, F: 2, G: 4, U: 6, B: 1}
    sh.set_map(np.array([B, A], dtype=np.uint64), np.array([7000, 7000], dtype=np.uint64))
    rng = np.random.default_rng(45)

    def window(t, active, n=400):
        ev = np.zeros(n * len(active), dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = np.repeat(np.array(active, dtype=np.uint64), n)
        ev["host_idx"] = np.repeat(np.array([host[a] for a in active], dtype=np.uint32), n)
        ev["type"] = np.where(rng.random(len(ev)) < 0.8, ge.EV_RESP, ge.EV_ACCEPT)
        act = ev["type"] == ge.EV_ACCEPT
        act &= rng.random(len(ev)) < 0.1
        ev["type"][act] = ge.EV_ACTIVE
        ev["flags"][act] = rng.integers(1, 50, int(act.sum()))
        ev["value"] = np.minimum(np.exp(rng.normal(np.log(3000.0), 1.2, len(ev))), 9.0e8).astype(np.uint32)
        ev["flow_key"] = rng.integers(1, 1 << 62, len(ev), dtype=np.uint64)
        ev["tsec"] = t
        ev["tsec"][act] = (rng.random(int(act.sum())) * 300).astype(np.float32).view(np.uint32)
        sh.feed(ev[rng.permutation(len(ev))], 1 << 14)
        sh.flush(t)
        return set().union(*[set(int(i) for i in e.evicted_ids()) for e in sh.engines])

    for t in (5, 10, 200, 400):
        window(t, [A, B, F, G] if t < 100 else [B, F, G])
    assert window(606, [B, F]) == {A}
    _check_levels(torch, sh)
    window(620, [B, F, U])
    w = _check_levels(torch, sh)
    assert w[7000]["nqrys_5day"] == sh.oracles[1].export_hist(B, ge.HIST_RESP_5DAY)[1]
    assert window(720, [B, F, U]) == {G}
    window(730, [A, B, F, U])
    w = _check_levels(torch, sh)
    assert w[7000]["nqrys_5min"] > sh.oracles[1].export_hist(B, ge.HIST_RESP_5MIN)[1]


def _run_engines(engines, rng, ids, conn_ids, times=TIMES[:8], n=20_000):
    for w, t in enumerate(times):
        _feed(engines, _events(rng, w, n, ids, conn_ids))
        for e in engines:
            e.flush(t)


def test_singleton_answers_like_its_service():
    """world 1: the row of a one-member logical service equals its member's gysk_query_svcs row in every field but glob_id and the
    four listener-state fields (0 in a logical row); the t-digest goes through one more merge-compress, so its quantiles equal the
    fold of the member's digest"""
    import torch
    rng = np.random.default_rng(31)
    ids, conn_ids, ghost_ids = _stream_ids()
    e = ge.Engine(merge_levels=True, **KW)
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    e.set_logical_map(glob, logical)
    _run_engines([e], rng, ids, conn_ids)
    _emulate_collectives(torch, [e])
    single = [i for i in range(16, 48)]
    svc = e.query_svcs(ids[single])
    got = e.query_logical([9100 + i for i in single])
    from tests.util import Digest, td_fold
    states = found = 0
    for i, s, g in zip(single, svc, got):
        assert g["found"] == s["found"], i
        if not s["found"]:
            continue
        found += 1
        for f in s:
            if f == "glob_id" or f in DOUBLE_FIELDS[1:]:
                continue
            if f in STATE_FIELDS:
                assert g[f] == 0
                states += s[f] != 0
                continue
            assert g[f] == s[f] or same_double(g[f], s[f]), (i, f, g[f], s[f])
        means, weights, mn, mx = e.export_tdigest(int(ids[i]))
        cent = np.zeros(len(means), dtype=po.CENTROID_DTYPE)
        cent["mean"], cent["weight"] = means, weights
        d = td_fold([Digest(cent, int(weights.sum()), mn, mx)], e.cfg.td_compression)
        for f, q in (("td_p50_us", 0.50), ("td_p95_us", 0.95), ("td_p99_us", 0.99)):
            assert same_double(g[f], d.quantile(q)), (i, f, g[f], d.quantile(q))
    assert found >= 24 and states > 0 and any(s["nconns_active"] for s in svc) and any(s["cli_errors"] for s in svc)
    assert sum(s["nqrys_5day"] for s in svc) > sum(s["nqrys_5min"] for s in svc) > 0


@pytest.mark.parametrize("world", [2, 4])
def test_shards_equal_one_engine(world):
    """every integer field of the logical rows of `world` host shards equals the same fold by one engine over the whole stream"""
    import torch
    rng = np.random.default_rng(70 + world)
    ids, conn_ids, ghost_ids = _stream_ids()
    shards = [ge.Engine(rank=r, world=world, merge_levels=True, **KW) for r in range(world)]
    one = ge.Engine(merge_levels=True, **KW)
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    for e in shards + [one]:
        e.set_logical_map(glob, logical)
    _run_engines(shards + [one], rng, ids, conn_ids, times=TIMES[:10])
    _emulate_collectives(torch, shards)
    _emulate_collectives(torch, [one])
    lids = list(dict.fromkeys(logical.tolist()))
    want = one.query_logical(lids)
    for e in shards:
        for lid, g, w in zip(lids, e.query_logical(lids), want):
            for f in INT_FIELDS + ["distinct_clients"]:
                assert g[f] == w[f], (lid, f, g[f], w[f])
    assert sum(w["nqrys_5min"] > 0 for w in want) > 10 and sum(w["nconns_active"] > 0 for w in want) > 2


def test_export_round_trips_through_the_reference():
    """gysk_export_logical_hist fed to the reference's update_from_serialized + get_percentiles gives the row's percentiles back for
    all four histograms; without the flag the two levels are GYSK_ERR_NOTSUP"""
    import torch
    R = po.ref()
    if R is None:
        pytest.skip("the compiled reference (oracle/_ref) is not available")
    rng = np.random.default_rng(53)
    ids, conn_ids, ghost_ids = _stream_ids()
    on, off = ge.Engine(merge_levels=True, **KW), ge.Engine(**KW)
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    for e in (on, off):
        e.set_logical_map(glob, logical)
        with pytest.raises(ge.GyskError) as ei:
            e.export_logical_hist(9000, ge.HIST_RESP_LAST)                 # before a finished merge
        assert ei.value.code == -22
    _run_engines([on, off], rng, ids, conn_ids, times=TIMES[:10])
    _emulate_collectives(torch, [on])
    _emulate_collectives(torch, [off])
    lids = list(dict.fromkeys(logical.tolist()))
    checks = {ge.HIST_RESP_LAST: ("p95_5s_resp_ms", "p99_5s_resp_ms", "p25_5s_resp_ms"), ge.HIST_RESP_ALL: ("p95_all_resp_ms", "p99_all_resp_ms"),
              ge.HIST_RESP_5MIN: ("p95_5min_resp_ms", "p99_5min_resp_ms"), ge.HIST_RESP_5DAY: ("p95_5day_resp_ms",)}
    pmap = {"p95": 95.0, "p99": 99.0, "p25": 25.0}
    nonempty = 0
    for lid, row in zip(lids, on.query_logical(lids)):
        for which, fields in checks.items():
            ser, total, mx = on.export_logical_hist(lid, which)
            pcts = np.array([pmap[f[:3]] for f in fields], dtype=np.float32)
            out = np.zeros(len(pcts), dtype=np.int64)
            R.gyref_hist_pct_from_serial(0, 0, po._p(ser), total, mx, po._p(pcts), len(pcts), po._p(out), None)
            assert out.tolist() == [row[f] for f in fields], (lid, which, out.tolist(), [row[f] for f in fields])
            nonempty += total > 0
        for which in (ge.HIST_RESP_5MIN, ge.HIST_RESP_5DAY):
            with pytest.raises(ge.GyskError) as ei:
                off.export_logical_hist(lid, which)
            assert ei.value.code == -95
        a, b = on.export_logical_hist(lid, ge.HIST_RESP_ALL), off.export_logical_hist(lid, ge.HIST_RESP_ALL)
        assert a[0].tobytes() == b[0].tobytes() and a[1:] == b[1:]
    assert nonempty > 2 * len(lids)
    with pytest.raises(ge.GyskError):
        on.export_logical_hist(lids[0], ge.HIST_RESP_CUR)


def test_flag_off_is_unchanged():
    """two engines fed the same stream, one with the flag: the one without keeps today's arena (the three regions' sizes and names),
    five kernel launches per merge, and rows whose untouched fields equal the flag's rows and whose level / aux fields are 0 / -1"""
    import torch
    rng = np.random.default_rng(61)
    ids, conn_ids, ghost_ids = _stream_ids()
    on, off = ge.Engine(merge_levels=True, **KW), ge.Engine(**KW)
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    for e in (on, off):
        e.set_logical_map(glob, logical)
    _run_engines([on, off], rng, ids, conn_ids)
    launches = []
    for e in (on, off):
        k0 = e.stats()["kernel_launches"]
        _emulate_collectives(torch, [e])
        launches.append(e.stats()["kernel_launches"] - k0)
    assert launches == [6, 5]
    nl, c = len(set(logical.tolist())), off.cfg
    ncms = c.cms_depth << c.cms_log2_width
    sizes = [2 * _align256(ncms * 8) + 2 * _align256(nl * 16 * 16) + _align256(nl * 32), _align256(nl * 16), _align256(nl << c.hll_p)]
    assert [(n, b, r) for n, _, b, r in off.merge_buffers()] == [
        ("sum_u64: cms_cur|cms_last|hist_last|hist_all|conn", sizes[0], gd.RED_SUM_U64),
        ("max_i64: hist max_val_seen", sizes[1], gd.RED_MAX_I64), ("max_u8: hll registers", sizes[2], gd.RED_MAX_U8)]
    grown = [b for _, _, b, _ in on.merge_buffers()]
    assert grown == [sizes[0] + _align256(2 * nl * 16 * 16) + _align256(nl * 32),
                     sizes[1] + _align256(nl * 16) + _align256(nl * 8) + _align256(16), sizes[2]]
    # the flag's arrays sit behind the old ones: the old part of every region is byte for byte the flag-off engine's
    for (_, pa, _, _), (_, pb, nb, _) in zip(on.merge_buffers(), off.merge_buffers()):
        assert _dev_bytes(torch, pa, nb).tobytes() == _dev_bytes(torch, pb, nb).tobytes()
    lids = list(dict.fromkeys(logical.tolist()))
    for lid, a, b in zip(lids, on.query_logical(lids), off.query_logical(lids)):
        for f in a:
            if f in LEVEL_FIELDS:
                assert b[f] == (-1 if f.startswith("p9") else 0), (lid, f, b[f])
            else:
                assert a[f] == b[f] or same_double(a[f], b[f]), (lid, f, a[f], b[f])
    with pytest.raises(ge.GyskError) as ei:
        off.merge_flush_range()
    assert ei.value.code == -95


def test_flush_range():
    """(t, t) after a common flush; the true earliest and latest tsec after the ranks flushed at different times"""
    import torch
    rng = np.random.default_rng(67)
    ids, conn_ids, ghost_ids = _stream_ids()
    engs = [ge.Engine(rank=r, world=3, merge_levels=True, **KW) for r in range(3)]
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    for e in engs:
        e.set_logical_map(glob, logical)
    _feed(engs, _events(rng, 0, 20_000, ids, conn_ids))
    for e in engs:
        e.flush(305)
    _emulate_collectives(torch, engs)
    assert [e.merge_flush_range() for e in engs] == [(305, 305)] * 3
    _feed(engs, _events(rng, 1, 20_000, ids, conn_ids))
    for e, t in zip(engs, (320, 43_210, 315)):
        e.flush(t)
    _emulate_collectives(torch, engs)
    assert [e.merge_flush_range() for e in engs] == [(315, 43_210)] * 3


def _region_bytes(torch, e):
    return [_dev_bytes(torch, p, nb).tobytes() for _, p, nb, _ in e.merge_buffers()]


def test_library_nccl_merge_equals_the_emulation():
    """gysk_merge_global (NCCL inside the library) at world 1 leaves the same region bytes and rows as the emulated collectives; on a
    box with two GPUs, two engines on two devices merged by the library equal two emulated shards on one device"""
    import torch
    try:
        uid = ge.Engine(max_svcs=64, max_tasks=8, max_batch=4096, cms_log2_width=8).nccl_unique_id()
    except ge.GyskError as ex:
        pytest.skip(f"NCCL not loadable: {ex}")
    rng = np.random.default_rng(88)
    ids, conn_ids, ghost_ids = _stream_ids()
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    lids = list(dict.fromkeys(logical.tolist()))
    e = ge.Engine(merge_levels=True, **KW)
    e.set_logical_map(glob, logical)
    _run_engines([e], rng, ids, conn_ids, times=TIMES[:6])
    _emulate_collectives(torch, [e])
    emu_bytes, emu_rows = _region_bytes(torch, e), repr(e.query_logical(lids))
    e.nccl_comm_init(uid, 1, 0)
    e.merge_global()
    e.sync()
    assert _region_bytes(torch, e) == emu_bytes and repr(e.query_logical(lids)) == emu_rows
    assert e.merge_flush_range() == (TIMES[5], TIMES[5])
    if torch.cuda.device_count() < 2:
        return
    import threading
    emu = [ge.Engine(rank=r, world=2, merge_levels=True, **KW) for r in range(2)]
    lib = [ge.Engine(device=r, rank=r, world=2, merge_levels=True, **KW) for r in range(2)]
    for x in emu + lib:
        x.set_logical_map(glob, logical)
    _run_engines(emu + lib, np.random.default_rng(89), ids, conn_ids, times=TIMES[:6])
    _emulate_collectives(torch, emu)
    uid2 = lib[0].nccl_unique_id()
    errs = []

    def run(r):
        try:
            lib[r].nccl_comm_init(uid2, 2, r)
            lib[r].merge_global()
            lib[r].sync()
        except Exception as ex:      # noqa: BLE001
            errs.append(ex)
    th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errs, errs
    want = repr(emu[0].query_logical(lids))
    assert repr(lib[0].query_logical(lids)) == want and repr(lib[1].query_logical(lids)) == want
