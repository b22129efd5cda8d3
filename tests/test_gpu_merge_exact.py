"""The merge step (gysk_merge.cu) pinned bit for bit. Shard engines on one GPU at world 1 ... 8, the collectives emulated element-wise
(test_gpu_merge._emulate_collectives), one oracle engine per rank. The merge is deterministic: members fold in map order, ranks in
ascending order, each step a stable merge by mean (accumulator first on equal means) plus one K_1 compress. tests.util.MergeRestatement
states the same steps on the CPU with the oracle's primitives, so every answer of gysk_query_logical — the t-digest quantiles
included — must equal the restatement exactly, as must each rank's folded slab and the all-reduced count-min tables."""
import numpy as np
import pytest

from gyeeta_b200 import dist as gd
from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po
from tests.test_gpu_merge import _emulate_collectives
from tests.util import M32, Digest, MergeRestatement, k1_cell_weights, same_double, td_fold, td_merge_compress

pytestmark = pytest.mark.gpu

TD_HEAD_DTYPE = np.dtype([("total", "<u8"), ("minv", "<f8"), ("maxv", "<f8"), ("n", "<u4"), ("pad", "<u4")])
SLAB_DTYPE = np.dtype([("head", TD_HEAD_DTYPE), ("cent", po.CENTROID_DTYPE, (po.TD_CAP,))])
assert TD_HEAD_DTYPE.itemsize == 32 and SLAB_DTYPE.itemsize == 4128          # SlabEntry: TdHead + TD_CAP centroids

DOUBLE_FIELDS = ["distinct_clients", "td_p50_us", "td_p95_us", "td_p99_us"]
INT_FIELDS = [f for f, _ in ge.SvcSummary._fields_ if f not in DOUBLE_FIELDS]      # every other field, glob_id included

NSVC, NHOSTS = 400, 40
LATE = range(300, 340)                  # services whose first events arrive in the second window, after the map was set


def _dev_bytes(torch, ptr, nbytes):
    return torch.as_tensor(gd._DevBuf(ptr, nbytes, "|u1", 1), device="cuda:0").cpu().numpy()


def _align256(v):
    return (v + 255) & ~255


def logical_map(rng, ids, conn_ids, ghost_ids):
    """(glob ids, logical ids) in a shuffled map order:
      9000: services 0..15, on hosts 0..15 => members on every rank at world <= 8
      9100 + i: singletons (services 16..47)
      9001: 84 members (services 48..131) and one with connection events only
      9002: ids that never register
      9003: two members with connection events only: found, but an empty digest
      9004: services that register in the second window, and eight that were there from the start"""
    pairs = [(ids[i], 9000) for i in range(16)]
    pairs += [(ids[i], 9100 + i) for i in range(16, 48)]
    pairs += [(ids[i], 9001) for i in range(48, 132)] + [(conn_ids[0], 9001)]
    pairs += [(g, 9002) for g in ghost_ids]
    pairs += [(conn_ids[1], 9003), (conn_ids[2], 9003)]
    pairs += [(ids[i], 9004) for i in list(LATE) + list(range(132, 140))]
    perm = rng.permutation(len(pairs))
    return (np.array([int(pairs[i][0]) for i in perm], dtype=np.uint64), np.array([pairs[i][1] for i in perm], dtype=np.uint64))


def conn_only_events(rng, conn_ids, n, tsec):
    """connection events of services that never see a response sample; each on its own host"""
    ev = np.zeros(n * len(conn_ids), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = np.repeat(conn_ids, n)
    ev["host_idx"] = np.repeat(np.arange(1, len(conn_ids) + 1, dtype=np.uint32), n)
    ev["type"] = rng.choice([ge.EV_ACCEPT, ge.EV_CLOSE_SER, ge.EV_CONNECT], len(ev))
    ev["value"] = rng.integers(0, 1 << 22, len(ev))
    ev["flow_key"] = rng.integers(1, 1 << 62, len(ev), dtype=np.uint64)
    ev["tsec"] = tsec
    return ev


def window_events(rng, w, n, ids, conn_ids):
    """the mixed stream; 2 % of its connection events are ACTIVE_CONN_STATS records, so the services' own rows carry active
    connections and a max rtt"""
    ev = synth.gen_mixed(rng, n, NSVC, ntask=32, nhosts=NHOSTS, nclients=5000)
    if w == 0:
        late = ids[list(LATE)]
        ev = ev[(ev["type"] == ge.EV_TASK) | ~np.isin(ev["svc_id"], late)]
    act = (ev["type"] >= ge.EV_CONNECT) & (ev["type"] <= ge.EV_CLOSE_SER) & (rng.random(len(ev)) < 0.02)
    k = int(act.sum())
    ev["type"][act] = ge.EV_ACTIVE
    ev["flags"][act] = rng.integers(1, 200, k)                                       # active connections
    ev["tsec"][act] = (rng.random(k) * 500).astype(np.float32).view(np.uint32)       # max rtt, msec
    return np.concatenate([ev, conn_only_events(rng, conn_ids, 200, 1)])


class Shards:
    """world engines of one configuration, rank r = shard r, and the oracle engine of every rank"""

    def __init__(self, world, **kw):
        self.world = world
        okw = {k: kw[k] for k in ("max_svcs", "max_tasks", "cms_depth", "cms_log2_width", "hll_p", "td_compression") if k in kw}
        self.engines = [ge.Engine(rank=r, world=world, **kw) for r in range(world)]
        self.oracles = [po.OracleEngine(rank=r, world=world, **okw) for r in range(world)]
        if kw.get("idle_evict_secs"):
            for o in self.oracles:
                o.set_idle_evict(kw["idle_evict_secs"])
        c = self.engines[0].cfg
        self.depth, self.log2w, self.hll_p, self.delta = c.cms_depth, c.cms_log2_width, c.hll_p, c.td_compression

    def set_map(self, glob, logical):
        self.glob, self.logical = glob, logical
        for e in self.engines:
            e.set_logical_map(glob, logical)

    def feed(self, ev, batch):
        for off in range(0, len(ev), batch):
            chunk = ev[off: off + batch]
            for e in self.engines:
                e.ingest_events(chunk)
                e.sync()
            for o in self.oracles:
                o.ingest(chunk)

    def flush(self, tsec):
        for e in self.engines:
            e.flush(tsec)
        for o in self.oracles:
            o.flush(tsec)

    def check_merge(self, torch, flow_keys=()):
        """merge, then compare every rank's folded slab, the all-reduced count-min tables, the global point queries and every
        logical service's answers with the restatement; returns the restated answers by logical id"""
        _emulate_collectives(torch, self.engines)
        rs = MergeRestatement(self.oracles, self.glob, self.logical, self.delta, self.hll_p)
        lids = list(dict.fromkeys(self.logical.tolist()))           # dense logical index = order of first appearance
        # per-rank fold, whole digests: the slab is not touched by the gather or the finish
        for r, e in enumerate(self.engines):
            p, nb = e.merge_tdigest_slab()
            assert nb == len(lids) * SLAB_DTYPE.itemsize
            slab = _dev_bytes(torch, p, nb).view(SLAB_DTYPE)
            for l, lid in enumerate(lids):
                assert_slab_entry(slab[l], rs.rank_digest(r, lid), (r, lid))
        # global count-min, whole tables: cms_cur | cms_last at the start of the sum_u64 region, each padded to 256 B
        ncms = self.depth << self.log2w
        want_cur, want_last = rs.cms(False), rs.cms(True)
        for e in self.engines:
            name, ptr, nbytes, redop = e.merge_buffers()[0]
            assert redop == gd.RED_SUM_U64 and name.startswith("sum_u64") and nbytes >= 2 * _align256(ncms * 8)
            buf = _dev_bytes(torch, ptr, 2 * _align256(ncms * 8)).view(np.uint64)
            assert np.array_equal(buf[:ncms], want_cur)
            assert np.array_equal(buf[_align256(ncms * 8) // 8:][:ncms], want_last)
        if len(flow_keys):
            L = po.lib()
            tbl = want_last.reshape(self.depth, -1)
            got = self.engines[-1].query_flows_global(flow_keys, last_window=True)
            for k, g in zip(np.asarray(flow_keys).tolist(), got):
                cells = [int(tbl[r, L.gyo_cms_index(k, r, self.log2w)]) for r in range(self.depth)]
                assert (g["count"], g["kbytes"]) == (min(c & M32 for c in cells), min(c >> 32 for c in cells)), hex(k)
        # every logical service's answers, on every rank, each engine having just read its own services by id: a logical row
        # carries none of their values
        self.svc_rows = [s for e in self.engines for s in e.query_svcs([r.glob_id for r in e.query_window()[0]])]
        lib = ge.load_library()
        want = {lid: rs.summary(lid, lib) for lid in lids}
        for r, e in enumerate(self.engines):
            for lid, got in zip(lids, e.query_logical(lids)):
                assert_summary(got, want[lid], (r, lid))
            assert e.query_logical([123456789])[0]["found"] == 0
        return want


def assert_slab_entry(entry, want, ctx):
    h = entry["head"]
    n = len(want.cent)
    assert (int(h["n"]), int(h["total"]), int(h["pad"])) == (n, want.total, 0), (ctx, int(h["n"]), n, int(h["total"]), want.total)
    assert same_double(h["minv"], want.minv) and same_double(h["maxv"], want.maxv), (ctx, h["minv"], want.minv, h["maxv"], want.maxv)
    c = entry["cent"]
    assert np.array_equal(c["weight"][:n], want.cent["weight"]), ctx
    assert c["mean"][:n].tobytes() == want.cent["mean"].tobytes(), ctx
    assert not c["weight"][n:].any() and not c["mean"][n:].any(), ctx


def assert_summary(got, want, ctx):
    for f in INT_FIELDS:
        assert got[f] == want[f], (ctx, f, got[f], want[f])
    for f in DOUBLE_FIELDS:
        assert same_double(got[f], want[f]), (ctx, f, got[f], want[f])


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_merged_answers_equal_the_restatement(world):
    import torch
    rng = np.random.default_rng(500 + world)
    ids = synth.service_ids(NSVC)
    conn_ids = synth.splitmix64(np.arange(1, 4, dtype=np.uint64) + np.uint64(1 << 51))
    ghost_ids = synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 52))
    sh = Shards(world, max_svcs=1024, max_tasks=128, max_batch=1 << 16, cms_log2_width=12)
    glob, logical = logical_map(rng, ids, conn_ids, ghost_ids)
    sh.set_map(glob, logical)                                       # before any service registered
    for w in range(2):
        ev = window_events(rng, w, 120_000, ids, conn_ids)
        sh.feed(ev, 1 << 16)
        sh.flush(5 * (w + 1))
        keys = np.unique(ev["flow_key"][(ev["type"] >= ge.EV_CONNECT) & (ev["type"] <= ge.EV_CLOSE_SER)])[:300]
        want = sh.check_merge(torch, keys)
        # the by-id reads before the logical ones returned active connections and listener states
        assert any(s["nconns_active"] for s in sh.svc_rows) and any(s["curr_state"] for s in sh.svc_rows)
        # the map covers what it should: every rank holds members of 9000 and 9001, the late services count from window 2 on
        assert want[9000]["td_count"] > 10_000 and want[9001]["td_count"] > 1000
        assert want[9003]["found"] == 1 and want[9003]["td_count"] == 0 and want[9003]["nconns_all"] > 0
        assert want[9002]["found"] == 1 and want[9002]["nqrys_all"] == 0
        late_resp = int(np.isin(ev["svc_id"][ev["type"] == ge.EV_RESP], ids[list(LATE)]).sum())
        assert (late_resp == 0) == (w == 0)
        assert (want[9004]["td_count"] > 0) and (w == 0 or want[9004]["td_count"] > late_resp)
    for o in sh.oracles:                                            # 9000 has a non-empty digest on every rank
        assert any(o.export_tdigest(int(g)) is not None and o.export_tdigest(int(g)).n for g in ids[:16])


def _digest(rng, n, lo=1.0, hi=1.0e6, wmax=1000):
    means = np.sort(np.exp(rng.uniform(np.log(lo), np.log(hi), n)))
    w = rng.integers(1, wmax + 1, n).astype(np.uint64)
    return means, w


def test_finish_on_crafted_gathered_slabs():
    """gysk_merge_finish on hand-built gathered slabs of 8 ranks at delta = 256: equal means across ranks, empty ranks between
    non-empty ones (their head fields must not count), all ranks empty, a single centroid, 256 centroids on every rank (the
    512-entry work area filled exactly at every step) and a total weight above 2^53, where (double) W rounds"""
    import torch
    world, delta = 8, 256
    rng = np.random.default_rng(8)
    cases = ["equal_means", "empty_between", "all_empty", "single", "full", "beyond_2_53"]
    nl = len(cases)
    eng = ge.Engine(max_svcs=64, max_tasks=16, max_batch=4096, cms_log2_width=8, td_compression=delta)
    lids = np.arange(7000, 7000 + nl, dtype=np.uint64)
    eng.set_logical_map(synth.splitmix64(lids), lids)               # never registered: the own fold is empty
    eng.merge_prepare()
    eng.sync()
    g = crafted_slabs(rng, world, nl)
    # the inputs decide what they are meant to: on equal means the accumulator goes first (a fold that lets the later rank go
    # first gives other centroids), and no partial sum of the heavy case is a double
    swapped = Digest()
    for d in slab_digests(g, world, nl, 0):
        swapped = Digest(td_merge_compress(d.cent, swapped.cent, delta), swapped.total + d.total)
    assert swapped.cent.tobytes() != td_fold(slab_digests(g, world, nl, 0), delta).cent.tobytes()
    heavy = np.cumsum([d.total for d in slab_digests(g, world, nl, 5)], dtype=object)
    assert all(int(float(w)) != w for w in heavy) and (1 << 53) < heavy[-1] < (1 << 64)
    dev =torch.from_numpy(g.view(np.uint8).copy()).to("cuda:0")
    torch.cuda.synchronize()
    eng.merge_finish(dev.data_ptr(), world)
    got = eng.query_logical(lids)
    for l, case in enumerate(cases):
        want = td_fold(slab_digests(g, world, nl, l), delta)
        assert got[l]["found"] == 1 and got[l]["td_count"] == want.total, (case, got[l]["td_count"], want.total)
        for f, q in (("td_p50_us", 0.50), ("td_p95_us", 0.95), ("td_p99_us", 0.99)):
            assert same_double(got[l][f], want.quantile(q)), (case, f, got[l][f], want.quantile(q))
        if case == "all_empty":
            assert want.total == 0 and np.isnan(got[l]["td_p50_us"])
        elif case == "single":
            assert len(want.cent) == 1 and got[l]["td_count"] == 1
        elif case == "full":
            assert all(len(td_fold(slab_digests(g, r + 1, nl, l), delta).cent) == 256 for r in range(world))


def slab_digests(g, world, nl, l):
    """the digests of logical index l on every rank of a gathered [world][nl] slab array"""
    out = []
    for r in range(world):
        h, c = g["head"][r * nl + l], g["cent"][r * nl + l]
        out.append(Digest(c[: int(h["n"])], int(h["total"]), float(h["minv"]), float(h["maxv"])))
    return out


def crafted_slabs(rng, world, nl):
    """[world][nl] SlabEntry: 0 identical means on every rank with rank-dependent weights; 1 non-empty on ranks 0, 3, 7 only, the
    empty ranks' heads carrying a count, min and max that must not count; 2 empty everywhere; 3 one centroid on rank 5; 4 256
    centroids on every rank, one in each K_1 cell, so that the accumulator keeps 256 and every merge fills the 512-entry work
    area; 5 256 centroids of weight about 2^51 on every rank (total about 2^62)"""
    g = np.zeros(world * nl, dtype=SLAB_DTYPE)
    H, Cm, Cw = g["head"], g["cent"]["mean"], g["cent"]["weight"]

    def put(r, l, means, w, total=None, minv=None, maxv=None):
        i, n = r * nl + l, len(means)
        H["n"][i] = n
        H["total"][i] = sum(int(x) for x in w) if total is None else total
        H["minv"][i] = (means[0] * 0.5 if n else np.inf) if minv is None else minv
        H["maxv"][i] = (means[-1] * 2.0 if n else -np.inf) if maxv is None else maxv
        Cm[i, :n] = means
        Cw[i, :n] = w

    shared = np.sort(rng.uniform(10.0, 5000.0, 120)).round(1)
    for r in range(world):
        put(r, 0, shared, rng.integers(1, 50, len(shared)).astype(np.uint64))
        if r in (0, 3, 7):
            put(r, 1, *_digest(rng, 60 + 20 * r))
        else:
            put(r, 1, [], [], total=99, minv=-5.0, maxv=1.0e12)
        put(r, 2, [], [], total=7 * r, minv=float(r), maxv=float(r))
        if r == 5:
            put(r, 3, [1234.5], [1])
        put(r, 4, np.geomspace(1.0, 1.0e6, 256) * (1.0 + 1.0e-3 * r), k1_cell_weights(256, (1 << 20) + r))
        m, _ = _digest(rng, 256)
        put(r, 5, m, (rng.integers(1, 1 << 8, 256).astype(np.uint64) << np.uint64(44)) | rng.integers(0, 1 << 20, 256).astype(np.uint64))
    return g


def test_eviction_only_the_new_life_counts():
    """A (logical 7000 with B) goes idle and is evicted; its slot goes to U, an id outside the map, the one free slot of rank 0; a
    second eviction frees a slot and A returns. At every merge the answers equal the restatement: A's first life is gone, U never
    counts."""
    import torch
    world = 2
    sh = Shards(world, max_svcs=3, max_tasks=8, max_batch=1 << 14, cms_log2_width=10, idle_evict_secs=300)
    A, B, U, F, G = (int(x) for x in synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 53)))
    host = {A: 0, F: 2, G: 4, U: 6, B: 1}                           # A, F, G, U on rank 0; B on rank 1
    sh.set_map(np.array([B, A], dtype=np.uint64), np.array([7000, 7000], dtype=np.uint64))
    rng = np.random.default_rng(44)

    def window(t, active, n=400):
        ev = np.zeros(n * len(active), dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = np.repeat(np.array(active, dtype=np.uint64), n)
        ev["host_idx"] = np.repeat(np.array([host[a] for a in active], dtype=np.uint32), n)
        ev["type"] = np.where(rng.random(len(ev)) < 0.8, ge.EV_RESP, ge.EV_ACCEPT)
        ev["value"] = np.minimum(np.exp(rng.normal(np.log(3000.0), 1.2, len(ev))), 9.0e8).astype(np.uint32)
        ev["flow_key"] = rng.integers(1, 1 << 62, len(ev), dtype=np.uint64)
        ev["tsec"] = t
        sh.feed(ev[rng.permutation(len(ev))], 1 << 14)
        sh.flush(t)
        got = [set(int(i) for i in e.evicted_ids()) for e in sh.engines]
        want = [set(int(i) for i in o.evicted_ids()[0]) for o in sh.oracles]
        assert got == want, (t, got, want)
        return set().union(*got), int((ev["type"][ev["svc_id"] == A] == ge.EV_RESP).sum())

    for t in (5, 10):
        window(t, [A, B, F, G])
    for t in (200, 400):
        window(t, [B, F, G])
    ev_ids, _ = window(606, [B, F])
    assert ev_ids == {A}
    sh.check_merge(torch)
    window(620, [B, F, U])                                          # U takes A's slot: the only free one on rank 0
    w = sh.check_merge(torch)
    b_all = sh.oracles[1].export_hist(B, 2)[1]
    assert w[7000]["nqrys_all"] == b_all                           # neither A's first life nor U
    ev_ids, _ = window(720, [B, F, U])
    assert ev_ids == {G}
    _, a_new = window(730, [A, B, F, U])                            # A returns into G's slot
    w = sh.check_merge(torch)
    assert a_new > 0 and w[7000]["nqrys_all"] == sh.oracles[1].export_hist(B, 2)[1] + a_new
    assert sh.engines[0].stats()["nsvcs"] == 3
