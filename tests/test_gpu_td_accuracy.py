"""The all-time t-digest against the TRUTH, in the regime it runs in: a service's samples arrive over many device batches (one batch
down to one sample per batch, with and without flushes, beside other services' events, on the sort-key and on the hot-row route),
and a logical service's digest is folded again across members and ranks by the merge step.

The other t-digest tests pin the device's centroids to oracle/gysk_oracle.c, which restates the same algorithm, so a flaw of the
algorithm is on both sides; here the bit-identity is kept, and on top of it the answers are checked against numpy float64 over the
raw samples:

- the exact quantile is the ceil(q n) - 1 order statistic (tests.util.exact_quantile);
- the rank error of an estimate g at q is the distance of q from the rank interval [#{v < g} / n, #{v <= g} / n]. Where g is
  not a sample value that is |midrank(g) / n - q|; where it is one, the interval covers its ties, so a constant stream answered
  with its value has rank error 0. It does not depend on the distribution, so it is asserted for every stream;
- the value error |g - exact| / exact is asserted on the sigma <= 1.5 log-normal streams only.

Rank bound. The K_1 grid's cell at q is dq(q) = (pi / delta) sqrt(q (1 - q)) wide in rank. A cluster is its cell plus at most half
of its first and half of its last item, and an item is a sample, a value bin of one batch or an old centroid of about one cell, so a
cluster spans at most ~2 cells; the quantile interpolates between cluster centres, so it is off by at most about one cluster
width. RANK_FACTOR = 2 cells, plus 1 / n for the rank granularity of n samples, for every stream and schedule. One exception, which
no compress rule can change: a batch's samples of one value bin become ONE item, and the quantile interpolates linearly between
centroid centres. Where one value repeats within one batch more often than pi / delta of the stream (the weight of the two widest
cells), that item is a centroid wider than the bound assumes, and an estimate beside it lands off the point mass. Such a stream
(a point mass fed in a few big batches) keeps every other assertion, and its many-batch schedules keep the rank bound too."""
import math
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po
from tests.util import exact_quantile, same_double, td_p99_tolerance

pytestmark = pytest.mark.gpu

QS = (0.01, 0.1, 0.5, 0.9, 0.95, 0.99, 0.999)
QGRID = np.linspace(0.0, 1.0, 2001)
VMAX = 1_000_000_999                        # the largest response time the engine accepts (usec < 1 000 001 000)
RANK_FACTOR = 2.0                           # cells of the K_1 grid (module docstring)
# An i.i.d. stream fed evenly through many batches keeps at least this share of delta centroids once n >> delta. With the centre
# rule an old centroid whose centre lies in a cell stays a cluster of that cell, so nearly every cell stays occupied: 197..200 of
# 200 measured on the oracle for 20 K .. 400 K log-normal samples at 4 096 down to 1 sample per batch. 0.9 leaves room for the
# tail cells narrower than a sample or a heavy bin; the start rule, whose clusters widen by their last item at every merge, kept
# 70..150 there.
MIN_CENT_SHARE = 0.9
SMOOTH = ("lognormal-1.0", "lognormal-1.5", "ascending", "descending")
IID = ("lognormal-1.0", "lognormal-1.5")


# ---------------------------------------------------------------------------------------------------------------------------
# the truth
# ---------------------------------------------------------------------------------------------------------------------------
def rank_error(sorted_v, g, q):
    n = len(sorted_v)
    lo, hi = np.searchsorted(sorted_v, g, side="left") / n, np.searchsorted(sorted_v, g, side="right") / n
    return max(0.0, lo - q, q - hi)


def rank_bound(q, n, delta):
    return RANK_FACTOR * (math.pi / delta) * math.sqrt(q * (1.0 - q)) + 1.0 / n


def point_mass_in_a_batch(vals, k, delta):
    """one value repeats within one batch of k samples more often than pi / delta of the stream (module docstring)"""
    vals = np.asarray(vals)
    top = max(int(np.unique(vals[o:o + k], return_counts=True)[1].max()) for o in range(0, len(vals), k)) if k > 1 else 1
    return top > 1 and top > math.pi / delta * len(vals)


def check_against_truth(est, vals, delta, ctx, value_check=False, rank_check=True):
    """est: the digest's answers at QS; vals: every raw sample"""
    sv = np.sort(np.asarray(vals, dtype=np.float64))
    n = len(sv)
    for q, g in zip(QS, est):
        re_ = rank_error(sv, g, q)
        assert not rank_check or re_ <= rank_bound(q, n, delta), (ctx, "rank", q, g, re_, rank_bound(q, n, delta))
        if value_check and q in (0.5, 0.95, 0.99):
            x = exact_quantile(sv, q)
            tol = td_p99_tolerance(n) if q == 0.99 else 0.01
            assert abs(g - x) / x <= tol, (ctx, "value", q, g, x, abs(g - x) / x, tol)


# ---------------------------------------------------------------------------------------------------------------------------
# streams and schedules
# ---------------------------------------------------------------------------------------------------------------------------
def _u32(x):
    return np.minimum(np.maximum(np.asarray(x, dtype=np.float64), 0.0), VMAX).astype(np.uint32)


def streams(rng, n):
    """every stream of n samples (the tiny ones excepted), in arrival order"""
    ln = lambda s, m: rng.lognormal(math.log(20_000.0), s, m)
    base = ln(1.0, n)
    t = np.arange(n) / n
    tail = rng.random(n) < 0.01
    bimodal = np.where(rng.random(n) < 0.95, 100, 10_000_000)
    return {
        "lognormal-1.0": _u32(base),
        "lognormal-1.5": _u32(ln(1.5, n)),
        "ascending": np.sort(_u32(ln(1.0, n))),
        "descending": np.sort(_u32(ln(1.0, n)))[::-1].copy(),
        "step-10x": _u32(base * np.where(t >= 0.9, 10.0, 1.0)),
        "drift-25x": _u32(ln(1.0, n) * np.exp(math.log(25.0) * t)),
        "bimodal": _u32(bimodal),
        "constant": np.full(n, 20_000, dtype=np.uint32),
        "one-value-99": np.where(tail, _u32(rng.lognormal(math.log(2.0e5), 1.0, n)), 5_000).astype(np.uint32),
        "edges": rng.choice(np.array([0, 1, 31, 32, 33, 1000, VMAX], dtype=np.uint32), n),
        "n1": _u32(ln(1.0, 1)), "n2": _u32(ln(1.0, 2)), "n3": _u32(ln(1.0, 3)), "n5": _u32(ln(1.0, 5)),
    }


def stream_ids(names):
    return dict(zip(names, (int(x) for x in synth.splitmix64(np.arange(1, len(names) + 1, dtype=np.uint64) + np.uint64(1 << 53)))))


def _resp(ids, vals, host_idx=0):
    ev = np.zeros(len(vals), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = ids
    ev["type"] = ge.EV_RESP
    ev["value"] = vals
    ev["host_idx"] = host_idx
    ev["flow_key"] = np.arange(1, len(vals) + 1, dtype=np.uint64)
    ev["tsec"] = 1
    return ev


def batches(rng, data, ids, k, background=True):
    """the device batches: batch b holds samples [b k, (b + 1) k) of every stream, and (background) other services' response and
    connection events, a quarter as many as the streams bring, all shuffled together"""
    n = max(len(v) for v in data.values())
    nb = -(-n // k)
    bg = synth.gen_mixed(rng, max(64, (k * len(data)) // 4) * nb, 64, ntask=8, nhosts=8, nclients=500) if background else None
    per_bg = 0 if bg is None else len(bg) // nb
    out = []
    for b in range(nb):
        parts = [_resp(ids[s], v[b * k:(b + 1) * k]) for s, v in data.items() if b * k < len(v)]
        if per_bg:
            parts.append(bg[b * per_bg:(b + 1) * per_bg])
        ev = np.concatenate(parts)
        out.append(ev[rng.permutation(len(ev))])
    return out


def feed(eng, orc, evs, flush):
    for b, ev in enumerate(evs):
        eng.ingest_events(ev)
        eng.sync()
        orc.ingest(ev)
        if flush:
            eng.flush(5 * (b + 1))
            orc.flush(5 * (b + 1))


# ---------------------------------------------------------------------------------------------------------------------------
# one service's digest: bit-identity, invariants, truth
# ---------------------------------------------------------------------------------------------------------------------------
def check_digest(eng, orc, id_, vals, delta, ctx, many_batches, k):
    vals = np.asarray(vals)
    n = len(vals)
    means, weights, mn, mx = eng.export_tdigest(id_)
    td = orc.export_tdigest(id_)
    om, ow = td.centroids()
    # bit-identity with the oracle fed the same device batches
    assert np.array_equal(weights, ow) and means.tobytes() == om.tobytes(), ctx
    assert same_double(mn, td.minv) and same_double(mx, td.maxv) and td.total == n, ctx
    row = eng.query_svcs([id_])[0]
    assert row["td_count"] == n, (ctx, row["td_count"], n)
    # invariants
    assert int(weights.sum()) == n and (weights > 0).all(), ctx
    assert np.all(np.diff(means) >= 0), ctx
    assert mn == float(vals.min()) and mx == float(vals.max()), (ctx, mn, mx)
    assert np.all((means >= mn) & (means <= mx)), ctx
    assert 1 <= len(means) <= delta, (ctx, len(means))
    grid = eng.quantiles(id_, QGRID)
    assert np.all(np.diff(grid) >= 0) and grid.min() >= mn and grid.max() <= mx, ctx
    if mn == mx:                                         # n = 1 and constant streams: the value itself at every q
        assert np.all(grid == mn) and np.all(means == mn), ctx
    est = eng.quantiles(id_, QS)
    three = eng.quantiles(id_, [0.5, 0.95, 0.99])
    for f, v in zip(("td_p50_us", "td_p95_us", "td_p99_us"), three):
        assert same_double(row[f], v), (ctx, f, row[f], v)
    if many_batches and n >= 50 * delta:
        assert len(means) >= MIN_CENT_SHARE * delta, (ctx, "centroids", len(means))
    # the value tolerances are those of delta = 200 (tests.util.td_p99_tolerance); other deltas are held to the rank bound only
    check_against_truth(est, vals, delta, ctx, value_check=ctx[0] in SMOOTH and delta == 200,
                        rank_check=not point_mass_in_a_batch(vals, k, delta))
    return len(means)


# samples per batch -> samples per stream: the many-batch schedules keep their batch count (and so the test's time) bounded
SCHEDULES = [
    pytest.param(None, 400_000, "keys", False, id="one-batch-keys"),
    pytest.param(65_536, 400_000, "keys", False, id="65536-keys"),
    pytest.param(65_536, 400_000, "hot", True, id="65536-hot-flush"),
    pytest.param(4_096, 400_000, "keys", True, id="4096-keys-flush"),
    pytest.param(4_096, 400_000, "hot", False, id="4096-hot"),
    pytest.param(512, 400_000, "keys", False, id="512"),
    pytest.param(512, 200_000, "keys", True, id="512-flush"),
    pytest.param(64, 100_000, "keys", False, id="64"),
    pytest.param(8, 40_000, "keys", False, id="8"),
    pytest.param(1, 20_000, "keys", False, id="1"),
]


@pytest.mark.parametrize("k,n,route,flush", SCHEDULES)
def test_digest_against_truth_over_batches(monkeypatch, k, n, route, flush):
    """every stream as its own service, k samples of each per device batch beside other services' events; the digest equals the
    oracle's bit for bit, keeps its invariants and answers within the rank bound (and the value tolerance on the smooth streams)"""
    if route == "hot":                                  # a service with 8 samples in a batch owns a row of dense bins from then on
        monkeypatch.setenv("GYSK_HOT_ROWS", "2048")
        monkeypatch.setenv("GYSK_HOT_MIN", "8")
    else:
        monkeypatch.setenv("GYSK_HOT_ROWS", "0")
    rng = np.random.default_rng(1000 + (k or 0) + n // 1000 + 7 * flush)
    data = streams(rng, n)
    ids = stream_ids(list(data))
    kk = k or n
    evs = batches(rng, data, ids, kk, background=k is not None and k >= 8)
    max_batch = max(1024, max(len(e) for e in evs))
    eng = ge.Engine(max_svcs=256, max_tasks=64, max_batch=max_batch, cms_log2_width=10)
    orc = po.OracleEngine(max_svcs=256, max_tasks=64, cms_log2_width=10)
    feed(eng, orc, evs, flush)
    if route == "hot":
        assert eng.hot_rows_in_use() > 0
    for name, v in data.items():
        check_digest(eng, orc, ids[name], v, 200, (name, k, route, flush), k is not None and k <= 4096 and name in IID, kk)
    eng.close(); orc.close()


@pytest.mark.parametrize("delta", [10, 100, 256])
def test_digest_edges_of_delta(delta):
    """delta = 10, 100 and 256 at 256 samples per batch: invariants, centroid count and the rank bound scaled by 1 / delta"""
    rng = np.random.default_rng(delta)
    data = {k: v for k, v in streams(rng, 100_000).items() if k in ("lognormal-1.0", "lognormal-1.5", "drift-25x", "edges", "n3")}
    ids = stream_ids(list(data))
    evs = batches(rng, data, ids, 256)
    eng = ge.Engine(max_svcs=256, max_tasks=64, max_batch=1 << 12, cms_log2_width=10, td_compression=delta)
    orc = po.OracleEngine(max_svcs=256, max_tasks=64, cms_log2_width=10, td_compression=delta)
    feed(eng, orc, evs, False)
    for name, v in data.items():
        m = check_digest(eng, orc, ids[name], v, delta, (name, delta), name in IID, 256)
        if name in IID:
            assert m >= MIN_CENT_SHARE * delta, (name, delta, m)
    eng.close(); orc.close()


# ---------------------------------------------------------------------------------------------------------------------------
# the merge step: logical services of 1, 8 and 64 members folded across 1 .. 8 ranks
# ---------------------------------------------------------------------------------------------------------------------------
def parse_pgtext(text):
    """'flags 1 count N compression 100 centroids n (mean, weight) ...' -> (N, compression, CENTROID_DTYPE array)"""
    head = re.match(r"flags 1 count (\d+) compression (\d+) centroids (\d+)", text)
    pairs = re.findall(r"\(([^,()]+), (\d+)\)", text)
    c = np.zeros(len(pairs), dtype=po.CENTROID_DTYPE)
    c["mean"] = [float(m) for m, _ in pairs]
    c["weight"] = [int(w) for _, w in pairs]
    assert int(head.group(3)) == len(pairs)
    return int(head.group(1)), int(head.group(2)), c


LOGICAL = {7001: 1, 7008: 8, 7064: 64}                  # logical id -> members


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_merged_digest_against_truth(world):
    """73 member services, each a log-normal stream with its own median, 16 samples per device batch spread over 16 hosts (so
    every rank holds a share of every member and builds it over ~16 / world samples per batch). After the merge, every rank's
    logical quantiles, the td_p*_us of its logical row and the delta = 100 Postgres export answer within the rank bound of the
    union of all members' samples."""
    import torch
    from tests.test_gpu_merge import _emulate_collectives
    rng = np.random.default_rng(90 + world)
    nmem, per_batch, nbatch = sum(LOGICAL.values()), 16, 200
    mids = synth.splitmix64(np.arange(1, nmem + 1, dtype=np.uint64) + np.uint64(3 << 52))
    lids = np.repeat(np.array(list(LOGICAL), dtype=np.uint64), list(LOGICAL.values()))
    medians = 20_000.0 * np.exp(0.5 * rng.standard_normal(nmem))
    vals = _u32(rng.lognormal(np.log(medians)[:, None], 1.0, (nmem, per_batch * nbatch)))
    engines = [ge.Engine(rank=r, world=world, max_svcs=256, max_tasks=16, max_batch=1 << 12, cms_log2_width=10) for r in range(world)]
    for e in engines:
        e.set_logical_map(mids, lids)
    for b in range(nbatch):
        v = vals[:, b * per_batch:(b + 1) * per_batch]
        ev = _resp(np.repeat(mids, per_batch), v.reshape(-1), rng.integers(0, 16, v.size).astype(np.uint32))
        ev = ev[rng.permutation(len(ev))]
        for e in engines:
            e.ingest_events(ev)
            e.sync()
    _emulate_collectives(torch, engines)
    for lid in LOGICAL:
        union = vals[lids == lid].reshape(-1)
        n = len(union)
        for r, e in enumerate(engines):
            ctx = (world, lid, r)
            means, weights, mn, mx = e.export_logical_tdigest(lid)
            assert int(weights.sum()) == n and np.all(np.diff(means) >= 0) and len(means) <= 200, ctx
            assert mn == float(union.min()) and mx == float(union.max()), ctx
            est = e.logical_quantiles(lid, QS)
            check_against_truth(est, union, 200, ctx)
            row = e.query_logical([lid])[0]
            assert row["td_count"] == n, ctx
            row_q = [row["td_p50_us"], row["td_p95_us"], row["td_p99_us"]]
            assert all(same_double(a, b) for a, b in zip(row_q, e.logical_quantiles(lid, [0.5, 0.95, 0.99]))), ctx
            sv = np.sort(union.astype(np.float64))
            for q, g in zip((0.5, 0.95, 0.99), row_q):
                assert rank_error(sv, g, q) <= rank_bound(q, n, 200), (ctx, "row", q)
            total, comp, cent = parse_pgtext(e.export_logical_tdigest_pgtext(lid))
            assert (total, comp) == (n, 100) and int(cent["weight"].sum()) == n and len(cent) <= 100, ctx
            pg = [po.lib().gyo_td_quantile(po._p(cent), len(cent), mn, mx, q) for q in QS]
            check_against_truth(pg, union, 100, ctx + ("pgtext",))
    for e in engines:
        e.close()
