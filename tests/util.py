"""shared helpers for the GPU parity tests: run the same seeded event stream through the CUDA engine (via the C ABI)
and through the CPU oracle, and compare."""
import numpy as np

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po

assert ge.EVENT_DTYPE == po.EVENT_DTYPE


def make_pair(**kw):
    """(Engine, OracleEngine) with identical configuration"""
    eng = ge.Engine(**kw)
    idle = kw.get("idle_evict_secs", 0)
    ocfg = dict(max_svcs=kw.get("max_svcs", 1 << 14), max_tasks=kw.get("max_tasks", 1 << 12), cms_depth=kw.get("cms_depth", 4),
                cms_log2_width=kw.get("cms_log2_width", 20), hll_p=kw.get("hll_p", 12), td_compression=kw.get("td_compression", 200),
                flags=1 if kw.get("auto_register", True) else 0, rank=kw.get("rank", 0), world=kw.get("world", 1))
    orc = po.OracleEngine(**ocfg)
    if idle:
        orc.set_idle_evict(idle)
    return eng, orc


def feed_both(eng, orc, ev, batch):
    """identical device batches on both sides (the t-digest update is per batch)"""
    for off in range(0, len(ev), batch):
        chunk = ev[off: off + batch]
        eng.ingest_events(chunk)
        eng.sync()
        orc.ingest(chunk)


def assert_hist_equal(eng, orc, id_, which):
    a = eng.export_hist(id_, which)
    b = orc.export_hist(id_, which)
    assert (a is None) == (b is None), (hex(id_), which)
    if a is None:
        return 0
    assert np.array_equal(a[0]["count"], b[0]["count"]), (hex(id_), which, a[0]["count"], b[0]["count"])
    assert np.array_equal(a[0]["sum"], b[0]["sum"]), (hex(id_), which)
    assert a[1] == b[1] and a[2] == b[2], (hex(id_), which, a[1:], b[1:])
    return a[1]


def exact_quantile(vals, q):
    v = np.sort(np.asarray(vals, dtype=np.float64))
    return float(v[min(len(v) - 1, max(0, int(np.ceil(q * len(v))) - 1))])


def threaded_oracle(ev, nthreads, **ocfg):
    """The CPU oracle over a large stream: events pre-sharded by host_idx % nthreads (every per-service / per-task sketch lives
    wholly in one shard, SURVEY.md §8e), one oracle engine per thread, each shard ingested as ONE device batch. Returns
    (engines, owner) with owner(id, host_idx) -> engine; the count-min table of the whole stream is the sum of the shard tables."""
    import ctypes as C
    L = po.lib()
    owner = (ev["host_idx"] % nthreads).astype(np.int32)
    order = np.argsort(owner, kind="stable")
    cuts = np.searchsorted(owner[order], np.arange(1, nthreads))
    shards = [np.ascontiguousarray(a) for a in np.split(ev[order], cuts)]
    engines = [po.OracleEngine(**ocfg) for _ in range(nthreads)]
    eh = (C.c_void_p * nthreads)(*[e.h for e in engines])
    sp = (C.c_void_p * nthreads)(*[s_.ctypes.data for s_ in shards])
    cn = (C.c_uint64 * nthreads)(*[len(s_) for s_ in shards])
    L.gyo_bench_ingest(eh, sp, cn, nthreads, 0)               # batch 0 = the whole shard in one gyo_ingest call
    return engines, shards


M32 = 0xFFFFFFFF


def td_bins(usec):
    """the value bin of every response sample, the oracle's td_bin_index: gyo_td_code(usec) + the RESP_TIME bucket of usec / 1000"""
    L = po.lib()
    usec = np.asarray(usec, dtype=np.uint32)
    u, inv = np.unique(usec, return_inverse=True)
    b = np.array([L.gyo_td_code(int(v)) + L.gyo_bucket(0, int(v) // 1000) for v in u.tolist()], dtype=np.int64)
    return b[inv.reshape(-1)]


def td_bin_usec():
    """(bins, usec): every value bin a response time below the 10^6 msec cut-off can fall in, ascending, and one response time in
    each. td_bins is monotone in usec and changes only where the td_code changes ((32 + m) << sh) or the RESP_TIME bucket of the
    msec does, so those points reach every bin."""
    L = po.lib()
    ms = np.arange(0, 1_000_001)
    bk = np.array([L.gyo_bucket(0, m) for m in ms.tolist()])
    cand = list(range(32)) + [(32 + m) << sh for sh in range(26) for m in range(32)] + (ms[1:][np.diff(bk) != 0] * 1000).tolist()
    cand = np.unique(np.array(cand, dtype=np.int64))
    cand = cand[cand < 1_000_000_000].astype(np.uint32)
    bins, first = np.unique(td_bins(cand), return_index=True)
    return bins, cand[first]


def td_batch_items(usec):
    """one batch of one service as gyo_td_add_batch sees it: every non-empty value bin, in bin order, becomes the item
    {(double) usec sum / (double) samples, samples}"""
    usec = np.asarray(usec, dtype=np.uint32)
    bins = td_bins(usec)
    order = np.argsort(bins, kind="stable")
    ub, starts, cnt = np.unique(bins[order], return_index=True, return_counts=True)
    sums = np.add.reduceat(usec[order].astype(np.uint64), starts) if len(usec) else np.zeros(0, dtype=np.uint64)
    items = np.zeros(len(ub), dtype=po.CENTROID_DTYPE)
    items["mean"] = sums.astype(np.float64) / cnt.astype(np.float64)
    items["weight"] = cnt
    return items


def td_merge_compress(a, b, delta):
    """the CPU statement of warp_merge_compress: a stable merge by mean of two mean-sorted CENTROID_DTYPE lists, `a` first on equal
    means (the oracle's merge_sorted), then one gyo_td_compress pass with room for TD_CAP centroids"""
    a = np.asarray(a, dtype=po.CENTROID_DTYPE)
    b = np.asarray(b, dtype=po.CENTROID_DTYPE)
    am, bm = a["mean"].tolist(), b["mean"].tolist()
    na, nb = len(am), len(bm)
    order, i, j = [], 0, 0
    while i < na and j < nb:
        if bm[j] < am[i]:
            order.append(na + j); j += 1
        else:
            order.append(i); i += 1
    order += list(range(i, na)) + [na + k for k in range(j, nb)]
    merged = np.concatenate([a, b])[np.asarray(order, dtype=np.int64)]
    return po.td_compress(merged, delta) if len(merged) else merged


def k1_cell_weights(delta, W):
    """delta weights summing to W whose exclusive prefixes sit one in each cell of the K_1 grid (item 0 at 0, item j > 0 at the
    middle of cell j): compressed on its own, such a list keeps all delta items apart — a digest of exactly delta centroids"""
    import math
    q = [0.5 * (math.sin(math.pi * (j / delta - 0.5)) + 1.0) for j in range(delta + 1)]
    q[0], q[delta] = 0.0, 1.0
    T = [int(x * float(W)) for x in q]
    assert min(b - a for a, b in zip(T, T[1:])) >= 4, "W too small for the narrowest cell"
    starts = [0] + [(T[j] + T[j + 1]) // 2 for j in range(1, delta)] + [W]
    return np.diff(np.array(starts, dtype=np.int64)).astype(np.uint64)


class Digest:
    """a t-digest as the merge step carries it: centroids, sample count, min and max (an empty one has min +inf, max -inf)"""

    def __init__(self, cent=None, total=0, minv=np.inf, maxv=-np.inf):
        self.cent = np.zeros(0, dtype=po.CENTROID_DTYPE) if cent is None else np.asarray(cent, dtype=po.CENTROID_DTYPE)
        self.total, self.minv, self.maxv = int(total), float(minv), float(maxv)

    @classmethod
    def of_oracle(cls, td):
        c = np.frombuffer(bytes(td.c), dtype=po.CENTROID_DTYPE)[: td.n].copy()
        return cls(c, td.total, td.minv, td.maxv)

    def quantile(self, q):
        c = np.ascontiguousarray(self.cent)
        return po.lib().gyo_td_quantile(po._p(c), len(c), self.minv, self.maxv, q) if len(c) else float("nan")


def td_fold(digests, delta):
    """fold_td_kernel / finish_td_kernel: merge the non-empty digests one after the other into an accumulator that starts empty
    (so even a lone digest is compressed once more); count, min and max over the non-empty ones only"""
    acc = Digest()
    for d in digests:
        if d is None or not len(d.cent):
            continue
        acc = Digest(td_merge_compress(acc.cent, d.cent, delta), acc.total + d.total, min(acc.minv, d.minv), max(acc.maxv, d.maxv))
    return acc


class MergeRestatement:
    """What the merge step computes for every logical service, restated from one oracle engine per rank (OracleEngine(rank=r,
    world=W), fed the whole stream). Members are taken in map order, ranks in ascending order; a member without a service on a rank
    is skipped there, the way resolve_members_kernel maps it to the null slot."""

    def __init__(self, oracles, glob_ids, logical_ids, delta, hll_p):
        self.oracles, self.delta, self.hll_p = oracles, delta, hll_p
        self.members = {}
        for g, l in zip(np.asarray(glob_ids, dtype=np.uint64).tolist(), np.asarray(logical_ids, dtype=np.uint64).tolist()):
            self.members.setdefault(l, []).append(g)

    def rank_digest(self, r, lid):
        orc = self.oracles[r]
        tds = [orc.export_tdigest(g) for g in self.members.get(int(lid), [])]
        return td_fold([Digest.of_oracle(t) for t in tds if t is not None], self.delta)

    def digest(self, lid):
        return td_fold([self.rank_digest(r, lid) for r in range(len(self.oracles))], self.delta)

    def cells(self, lid):
        """summed {count, sum} cells of the last and all-time histograms, their max_val_seen, the connection sums and the
        per-byte max of the HLL registers"""
        last, all_ = np.zeros(15, dtype=po.SERIAL_DTYPE), np.zeros(15, dtype=po.SERIAL_DTYPE)
        mx_last = mx_all = -(1 << 63)
        conn = [0, 0, 0, 0]
        regs = np.zeros(1 << self.hll_p, dtype=np.uint8)
        for orc in self.oracles:
            for g in self.members.get(int(lid), []):
                hl, ha = orc.export_hist(g, 1), orc.export_hist(g, 2)
                if hl is None:
                    continue
                for h, acc in ((hl[0], last), (ha[0], all_)):
                    acc["count"] += h["count"]; acc["sum"] += h["sum"]
                mx_last, mx_all = max(mx_last, hl[2]), max(mx_all, ha[2])
                _cur, cl, ac, ak = orc.export_conn(g)
                conn[0] += cl & M32; conn[1] += cl >> 32; conn[2] += ac; conn[3] += ak
                regs = np.maximum(regs, orc.export_hll(g))
        return dict(last=last, all=all_, max_last=mx_last, max_all=mx_all, conn=conn, regs=regs)

    def summary(self, lid, eng_lib):
        """every field of the gysk_query_logical row of one logical service; the percentiles of the summed cells go through the
        library's gysk_hist_percentiles. The merge folds no rolling levels, active connections, errors or listener state: those
        fields are 0, and the percentiles of the empty 5-min / 5-day histograms -1."""
        import ctypes as C
        c = self.cells(lid)
        pcts = np.array([95.0, 99.0, 25.0], dtype=np.float32)

        def pct(cells, k):
            ser = np.zeros(15, dtype=po.SERIAL_DTYPE)
            ser[:] = cells
            out = np.zeros(3, dtype=np.int64)
            assert eng_lib.gysk_hist_percentiles(0, 0, po._p(ser), int(cells["count"].sum()), po._p(pcts), k, po._p(out)) == 0
            return out.tolist()

        p5, pa = pct(c["last"], 3), pct(c["all"], 2)
        d = self.digest(lid)
        return dict(glob_id=int(lid), found=1, p95_5min_resp_ms=-1, p99_5min_resp_ms=-1, nqrys_5min=0, p95_5day_resp_ms=-1, nqrys_5day=0,
                    nconns_active=0, active_kbytes=0, max_rtt_msec=0.0, cli_errors=0, ser_errors=0, curr_state=0, curr_issue=0,
                    issue_bit_hist=0, high_resp_bit_hist=0, nqrys_5s=int(c["last"]["count"].sum()) & M32, total_resp_5sec=int(c["last"]["sum"].sum()),
                    p95_5s_resp_ms=p5[0], p99_5s_resp_ms=p5[1], p25_5s_resp_ms=p5[2], p95_all_resp_ms=pa[0], p99_all_resp_ms=pa[1],
                    nqrys_all=int(c["all"]["count"].sum()), max_resp_ms=c["max_all"], nconns_5s=c["conn"][0] & M32,
                    kbytes_5s=c["conn"][1] & M32, nconns_all=c["conn"][2], kbytes_all=c["conn"][3],
                    distinct_clients=po.lib().gyo_hll_estimate(po._p(c["regs"]), self.hll_p), td_count=d.total,
                    td_p50_us=d.quantile(0.50), td_p95_us=d.quantile(0.95), td_p99_us=d.quantile(0.99))

    def cms(self, last_window):
        """the global count-min table: the sum of the per-rank tables"""
        return sum(o.cms(last_window) for o in self.oracles)


def same_double(a, b):
    """bit-identical doubles (NaN included)"""
    return np.float64(a).tobytes() == np.float64(b).tobytes()


def td_p99_tolerance(n, eps=0.01):
    """value tolerance of the digest's p99 against the EXACT sample quantile on the sigma <= 1.5 log-normal streams.
    Two parts: the systematic interpolation error of a delta = 200 K_1 digest (~0.3 %) — and the order-statistic noise of the
    sample itself: the p99 cluster holds n pi sqrt(.0099) / 200 samples whose individual positions the digest does not keep; the
    exact quantile, one of them, deviates from the cluster's straight line by ~ sqrt(cluster / 4) sample spacings of
    sigma / (phi(z_99) n) each (1 sigma = 0.5 % at n = 47 K, falling as 1 / sqrt(n)). 1 % holds from n = 150 K on; below that
    no sketch of a few hundred centroids can promise it, and the bound is 3.5 sigma of that noise."""
    return max(eps, 3.5 * 0.005 * float(np.sqrt(47_000.0 / n)))
