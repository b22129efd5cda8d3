"""Each logical service's heaviest clients merged across GPUs (GYSK_FLAG_SVC_TOP_CLIENTS with a logical map). After every merge of the
flow level's scripted flush sequences, at world 1, 2, 3, 5 and 8 with the collectives emulated, both reads must be byte-equal to the
restatement of tests/logical_top_clients.py for GYSK_TOPC_LAST and GYSK_TOPC_5MIN, the all-rows read must follow gysk_query_logical_all
row for row, and the last-window guarantees must hold against exact per-client sums whose total is query_logical's kbytes_5s. Also a
one-member logical service, K - 1 / K / K + 1 / 3K clients, a fold of about 2 000 members, ghost ids, eviction with recycled slots, a
map change between merges, gysk_grow between prepare and finish, the refusals, the flag off against on, and the library's NCCL path."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import logical_top_clients as lt
from tests import svc_top_clients as tc
from tests.flow_level import SEQUENCES
from tests.test_gpu_merge import _emulate_collectives

pytestmark = pytest.mark.gpu

NOTSUP, INVAL = -95, -22
K = tc.K
CFG = dict(max_svcs=256, max_tasks=64, max_batch=1 << 14, cms_log2_width=12)
WHICH = (ge.TOPC_LAST, ge.TOPC_5MIN)
GOLD = np.uint64(2654435761)


def _body(r):
    """the bytes of a row after its id and found word"""
    return np.asarray(r["n"]).tobytes() + np.asarray(r["delta"]).tobytes() + np.asarray(r["entries"]).tobytes()


def _expect(summary):
    out = np.zeros(1, dtype=ge.SVC_TOP_CLIENTS_DTYPE)[0]
    n, delta, a = tc.row(summary)
    out["n"], out["delta"] = n, delta
    out["entries"]["flow_key"], out["entries"]["kbytes"], out["entries"]["conns"] = a[:, 0], a[:, 1], a[:, 2]
    return out


class Fleet:
    """world engines with the flag, one restatement per rank, and each rank's exact per-(service, client) sums of its open and last
    windows"""

    def __init__(self, world, **kw):
        import torch
        self.torch = torch
        self.world = world
        self.engines = [ge.Engine(svc_top_clients=True, rank=r, world=world, **{**CFG, **kw}) for r in range(world)]
        self.models = [tc.TopClients() for _ in range(world)]
        self.open_exact = [{} for _ in range(world)]
        self.last_exact = [{} for _ in range(world)]
        self.members = {}

    def set_map(self, glob_ids, logical_ids):
        for e in self.engines:
            e.set_logical_map(glob_ids, logical_ids)
        self.members = lt.members_of(np.asarray(glob_ids, dtype=np.uint64), np.asarray(logical_ids, dtype=np.uint64))

    def batch(self, ev):
        """one device batch per rank: the events of the hosts the rank owns (host_idx % world)"""
        for r, e in enumerate(self.engines):
            sh = ev[ev["host_idx"] % self.world == r]
            e.ingest_events(sh)
            e.sync()
            self.models[r].batch(sh)
            for s, d in tc.batch_sums(sh).items():
                o = self.open_exact[r].setdefault(s, {})
                for k, (kb, c) in d.items():
                    a = o.setdefault(k, [0, 0])
                    a[0] += kb
                    a[1] += c

    def flush(self, t):
        for r, e in enumerate(self.engines):
            e.flush(t)
            gone = e.evicted_ids()
            self.models[r].evict(gone)
            for s in gone.tolist():
                self.open_exact[r].pop(int(s), None)
            self.models[r].flush(t)
            self.last_exact[r], self.open_exact[r] = self.open_exact[r], {}

    def merge(self, what=None):
        _emulate_collectives(self.torch, self.engines)
        self.check(what)

    def want(self, which, lid):
        return lt.logical_summary(self.models, which, self.members.get(lid, []))

    def check(self, what=None):
        lids = sorted(self.members)
        ids = np.array(lids + [0, 12345], dtype=np.uint64)
        for which in WHICH:
            want = {lid: _expect(self.want(which, lid)) for lid in lids}
            for e in self.engines:
                rows = e.query_logical_top_clients(ids, which)
                assert rows["glob_id"].tolist() == ids.tolist(), what
                for lid, r in zip(lids, rows):
                    assert r["found"] == 1 and _body(r) == _body(want[lid]), (what, which, lid, r, want[lid])
                assert (rows["found"][-2:] == 0).all() and not _body(rows[-2:]).strip(b"\0"), what
                for active in (False, True):
                    arows, n = e.query_logical_top_clients_all(which, active_only=active)
                    vrows, vn = e.query_logical_all(active_only=active)
                    assert n == vn and arows["glob_id"].tolist() == [v.glob_id for v in vrows], (what, which, active)
                    assert arows.tobytes() == e.query_logical_top_clients(arows["glob_id"], which).tobytes(), (what, which, active)
                if len(lids) > 2:
                    part, n = e.query_logical_top_clients_all(which, cap=2)
                    assert n == len(lids) and len(part) == 2
        # the last-window guarantees against the exact sums over every member on every rank; N_L = the logical kbytes_5s
        summ = {r["glob_id"]: r for r in self.engines[0].query_logical(np.array(lids, dtype=np.uint64))}
        for lid in lids:
            exact = {}
            for r in range(self.world):
                for m in self.members[lid]:
                    for k, (kb, c) in self.last_exact[r].get(m, {}).items():
                        a = exact.setdefault(k, [0, 0])
                        a[0] += kb
                        a[1] += c
            n_l = sum(v[0] for v in exact.values())
            assert n_l & 0xFFFFFFFF == summ[lid]["kbytes_5s"], (what, lid)
            tc.check_guarantees(self.want(ge.TOPC_LAST, lid), exact, n_s=n_l)


# 48 services: service 0 alone in logical 900; services 1 .. 23 in logical 500 .. 505, each logical's members on one host (so on one
# rank); services 24 .. 47 in logical 600 .. 603 on every host (spread over the ranks). Each logical service draws its clients from its
# own pool of K - 1, K, K + 1, 3K or 300 keys. Ghost ids join 500 and 600, and logical 950 has ghosts only.
NSVC = 48
SIDS = np.arange(1, NSVC + 1, dtype=np.uint64) * GOLD
LMAP = np.array([900] + [500 + j % 6 for j in range(1, 24)] + [600 + j % 4 for j in range(24, NSVC)], dtype=np.uint64)
GHOSTS = np.array([777, 778, 779], dtype=np.uint64) * GOLD
MAP_IDS = np.concatenate([SIDS, GHOSTS])
MAP_LIDS = np.concatenate([LMAP, np.array([500, 600, 950], dtype=np.uint64)])
POOL = {lid: size for lid, size in zip(sorted(set(LMAP.tolist())), [K - 1, K, K + 1, 3 * K, 300] * 3)}


def _events(rng, n, keys, sids=SIDS, lmap=LMAP):
    """n connection events of the services, each client from its logical service's pool, and response samples that never count"""
    i = rng.integers(0, len(sids), n)
    lid = lmap[i]
    lids = sorted(set(lmap.tolist()))
    off = np.array([lids.index(int(l)) * 1000 for l in lid.tolist()])
    size = np.array([POOL.get(int(l), 300) for l in lid.tolist()])
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = sids[i]
    ev["flow_key"] = keys[off + (rng.random(n) * size).astype(np.int64)]
    ev["type"] = rng.choice(np.array(tc.COUNTED + (ge.EV_RESP,), dtype=np.uint16), n)
    ev["value"] = rng.integers(0, 1 << 22, n)
    pinned = (lid >= 500) & (lid < 600)
    ev["host_idx"] = np.where(pinned, lid.astype(np.int64) % 16, rng.integers(0, 16, n))
    return ev


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_rows_after_every_merge(name, world):
    rng = np.random.default_rng(700 + world + len(SEQUENCES[name]))
    keys = rng.integers(1, 1 << 62, 20_000, dtype=np.uint64)
    fleet = Fleet(world)
    fleet.set_map(MAP_IDS, MAP_LIDS)
    for i, t in enumerate(SEQUENCES[name]):
        for _ in range(int(rng.integers(1, 3))):
            fleet.batch(_events(rng, int(rng.integers(500, 4000)), keys))
        fleet.flush(t)
        fleet.merge((name, world, i, t))
    # the one-member logical service 900: its member's own row on the rank that holds it (one host, so one rank), apart from glob_id
    fleet2 = Fleet(world)
    fleet2.set_map(MAP_IDS, MAP_LIDS)
    ev = _events(rng, 3000, keys)
    ev["host_idx"][ev["svc_id"] == SIDS[0]] = 5
    fleet2.batch(ev)
    fleet2.flush(30)
    fleet2.merge((name, world, "one member"))
    for which in WHICH:
        own = fleet2.engines[5 % world].query_svc_top_clients(SIDS[:1], which)[0]
        for e in fleet2.engines:
            r = e.query_logical_top_clients(np.array([900], dtype=np.uint64), which)[0]
            assert r["glob_id"] == 900 and r["found"] == 1 and _body(r) == _body(own) and r["n"] > 0


def test_a_long_fold_of_2000_members():
    """one logical service of 2 000 members (and a few small ones) at world 2: the fold runs through every member in map order"""
    n = 2000
    rng = np.random.default_rng(31)
    keys = rng.integers(1, 1 << 62, 4000, dtype=np.uint64)
    sids = np.arange(1, n + 9, dtype=np.uint64) * GOLD
    lmap = np.where(np.arange(n + 8) < n, 4242, 10 + np.arange(n + 8) % 4).astype(np.uint64)
    order = rng.permutation(n + 8)
    fleet = Fleet(2, max_svcs=4096, max_batch=1 << 16)
    fleet.set_map(sids[order], lmap[order])
    for step, t in enumerate((5, 10, 40, 300)):
        ev = np.zeros(40_000, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = sids[rng.integers(0, len(sids), len(ev))]
        ev["flow_key"] = keys[np.minimum(rng.zipf(1.2, len(ev)), len(keys)) - 1]
        ev["type"], ev["value"], ev["host_idx"] = ge.EV_CLOSE_SER, rng.integers(0, 1 << 22, len(ev)), rng.integers(0, 16, len(ev))
        fleet.batch(ev)
        fleet.flush(t)
        fleet.merge(("long", step))
    r = fleet.engines[0].query_logical_top_clients(np.array([4242], dtype=np.uint64), ge.TOPC_5MIN)[0]
    assert r["n"] == K and r["delta"] > 0


def test_eviction_recycled_slots_and_a_map_change():
    """services idle for 20 s are evicted and new ids take their slots; the map names old and new ids, and changes between merges"""
    rng = np.random.default_rng(41)
    keys = rng.integers(1, 1 << 62, 20_000, dtype=np.uint64)
    fleet = Fleet(3, max_svcs=64, idle_evict_secs=20)
    allsids = np.arange(1, 200, dtype=np.uint64) * GOLD
    for i, t in enumerate(range(5, 205, 5)):
        if i % 7 == 0:                                          # a new map: every id, logical ids reshuffled
            fleet.set_map(allsids, (allsids // GOLD + np.uint64(i)) % np.uint64(9) + np.uint64(300))
        base = (i // 8) * 32
        sids = allsids[base: base + 32]
        lmap = np.full(len(sids), 600, dtype=np.uint64)         # pools by _events' rule
        fleet.batch(_events(rng, 3000, keys, sids, lmap))
        fleet.flush(t)
        fleet.merge(("evict", i, t))
        assert all(e.stats()["events_dropped"] == 0 for e in fleet.engines)
    assert sum(e.stats()["svcs_evicted"] for e in fleet.engines) >= 64


def test_grow_between_prepare_and_finish():
    """gysk_grow after gysk_merge_prepare moves every slot; finish reads only the slab, so every row is the restatement's"""
    rng = np.random.default_rng(51)
    keys = rng.integers(1, 1 << 62, 20_000, dtype=np.uint64)
    fleet = Fleet(2, max_svcs=64)
    fleet.set_map(MAP_IDS, MAP_LIDS)
    for e in fleet.engines:
        prepare = e.merge_prepare

        def prepare_then_grow(e=e, prepare=prepare):
            prepare()
            e.grow(max_svcs=e.cfg.max_svcs * 2)
        e.merge_prepare = prepare_then_grow
    for i, t in enumerate((5, 10, 35)):
        fleet.batch(_events(rng, 3000, keys))
        fleet.flush(t)
        fleet.merge(("grow", i))
    assert all(e.cfg.max_svcs == 64 * 8 for e in fleet.engines)


def test_refusals():
    ids = np.array([500], dtype=np.uint64)
    off = ge.Engine(**CFG)
    off.set_logical_map(SIDS, LMAP)
    for call in (lambda: off.query_logical_top_clients(ids), lambda: off.query_logical_top_clients_all()):
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == NOTSUP
    on = ge.Engine(svc_top_clients=True, **CFG)
    on.set_logical_map(SIDS, LMAP)
    for call in (lambda: on.query_logical_top_clients(ids), lambda: on.query_logical_top_clients_all()):    # no finished merge
        with pytest.raises(ge.GyskError) as ex:
            call()
        assert ex.value.code == INVAL
    on.merge_prepare()
    on.merge_finish()
    assert on.query_logical_top_clients(ids)[0]["found"] == 1
    for w in (ge.TOPC_OPEN, -1, 3):
        for call in (lambda: on.query_logical_top_clients(ids, w), lambda: on.query_logical_top_clients_all(w)):
            with pytest.raises(ge.GyskError) as ex:
                call()
            assert ex.value.code == INVAL
    on.set_logical_map(SIDS, LMAP)                              # a new map drops the last merge's results
    with pytest.raises(ge.GyskError) as ex:
        on.query_logical_top_clients(ids)
    assert ex.value.code == INVAL


FLAG_SETS = [dict(), dict(client_levels=True, flow_level=True, flow_queries=True, flow_query_level=True, flow_resp_hist=True, flow_topk=True,
                          flow_topk_5min=True, flow_topk_slow=True, flow_errors=True, merge_levels=True, merge_states=True, merge_topn=True,
                          merge_traces=True, max_trace_svcs=64, idle_evict_secs=20)]


@pytest.mark.parametrize("flags", range(len(FLAG_SETS)))
def test_flag_off_and_on_answer_alike(flags):
    """the same stream through engines without and with the flag, merged at world 2: every existing answer and merge region byte-equal,
    each off engine's slab a byte-equal prefix of the on engine's, which is longer by exactly ceil(nl x 528 / 4128) entries"""
    import torch
    from tests.test_gpu_client_levels import _regions
    from tests.test_gpu_flow_level import _rowbytes
    from tests.test_gpu_merge_exact import _dev_bytes
    rng = np.random.default_rng(60 + flags)
    keys = rng.integers(1, 1 << 62, 20_000, dtype=np.uint64)
    kw = {**CFG, **FLAG_SETS[flags]}
    off = [ge.Engine(rank=r, world=2, **kw) for r in range(2)]
    on = [ge.Engine(svc_top_clients=True, rank=r, world=2, **kw) for r in range(2)]
    for e in off + on:
        e.set_logical_map(MAP_IDS, MAP_LIDS)
        for s in SIDS.tolist():             # one id per call: each id takes the same slot in every engine, so top-N ties break alike
            e.register_ids([s])
    nl = len(set(MAP_LIDS.tolist()))
    entry = 4128
    for t in (5, 10, 10, 40, 345):
        ev = _events(rng, 4000, keys)
        for fleet in (off, on):
            for r, e in enumerate(fleet):
                e.ingest_events(ev[ev["host_idx"] % 2 == r]); e.sync()
                e.flush(t)
            _emulate_collectives(torch, fleet)
        lids = np.array(sorted(set(MAP_LIDS.tolist())), dtype=np.uint64)
        for a, b in zip(off, on):
            assert _rowbytes(a.query_logical(lids)) == _rowbytes(b.query_logical(lids))
            assert _rowbytes(a.query_svcs(SIDS)) == _rowbytes(b.query_svcs(SIDS))
            ra, rb = _regions(a, torch), _regions(b, torch)
            assert sorted(ra) == sorted(rb)
            for region in ra:
                assert ra[region][0] == rb[region][0] and ra[region][1].tobytes() == rb[region][1].tobytes(), region
            (pa, na), (pb, nb) = a.merge_tdigest_slab(), b.merge_tdigest_slab()
            assert nb - na == -(-nl * 528 // entry) * entry
            assert _dev_bytes(torch, pa, na).tobytes() == _dev_bytes(torch, pb, nb)[:na].tobytes()
            sa, sb = a.stats(), b.stats()
            assert {k: v for k, v in sa.items() if k != "kernel_launches"} == {k: v for k, v in sb.items() if k != "kernel_launches"}
        assert (on[0].query_logical_top_clients(lids, ge.TOPC_LAST)["n"] > 0).any()


def test_library_nccl_path_equals_the_emulation():
    import torch
    rng = np.random.default_rng(71)
    keys = rng.integers(1, 1 << 62, 20_000, dtype=np.uint64)
    eng = ge.Engine(svc_top_clients=True, **CFG)
    eng.set_logical_map(MAP_IDS, MAP_LIDS)
    for t in (30, 35, 65):
        eng.ingest_events(_events(rng, 5000, keys)); eng.sync()
        eng.flush(t)
    _emulate_collectives(torch, [eng])
    lids = np.array(sorted(set(MAP_LIDS.tolist())), dtype=np.uint64)
    emulated = [eng.query_logical_top_clients(lids, w).tobytes() for w in WHICH]
    assert any(np.frombuffer(b, dtype=ge.SVC_TOP_CLIENTS_DTYPE)["n"].any() for b in emulated)
    eng.nccl_comm_init(eng.nccl_unique_id(), 1, 0)
    eng.merge_global()
    eng.sync()
    assert [eng.query_logical_top_clients(lids, w).tobytes() for w in WHICH] == emulated
