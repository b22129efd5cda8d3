"""CPU-only probe of the all-time t-digest's accuracy when a service's samples arrive over many device batches (DESIGN.md §2).

Every device batch turns one service's samples into value-bin items, merges them with the service's old centroids and compresses
the list on the K_1 grid (gyo_td_add_batch). Which K_1 cell an item joins is the compress rule:

  start   the cell that holds the item's exclusive weight prefix P_i (the rule before the centre rule);
  centre  the cell that holds its weight centre P_i + w_i / 2 (the rule the engine and the oracle implement).

Both are restated here in numpy; the centre column is checked bit for bit against the oracle's gyo_td_add_batch on every run, so
the table shows what the device computes. For each stream and batch size it prints, over the seeds, the p99 relative value
error against the exact order statistic (mean / max), the largest rank error |midrank(estimate) / n - q| over
q in {0.01, 0.1, 0.5, 0.9, 0.95, 0.99, 0.999}, and the number of centroids left (mean).

    python scripts/td_accuracy_probe.py [--seeds 4] [--n 400000]
"""
import argparse
import ctypes as C
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import pyoracle as po  # noqa: E402

QS = (0.01, 0.1, 0.5, 0.9, 0.95, 0.99, 0.999)
_bucket_of_ms = {}


def items_of(vals):
    """one batch as gyo_td_add_batch sees it: bin = gyo_td_code(usec) + RESP_TIME bucket of usec / 1000; every non-empty bin is
    the item {usec sum / samples, samples}, in bin order"""
    v = vals.astype(np.int64)
    e = np.frexp(np.maximum(v, 1).astype(np.float64))[1].astype(np.int64)       # bit length, exact below 2^53
    sh = np.maximum(e - 6, 0)
    code = np.where(v < 32, v, ((sh + 1) << 5) | ((v >> sh) & 31))
    ms = v // 1000
    L = po.lib()
    for m in np.unique(ms).tolist():
        if m not in _bucket_of_ms:
            _bucket_of_ms[m] = L.gyo_bucket(0, m)
    b = code + np.array([_bucket_of_ms[m] for m in ms.tolist()], dtype=np.int64)
    ub, inv = np.unique(b, return_inverse=True)
    cnt = np.bincount(inv)
    sums = np.zeros(len(ub), dtype=np.uint64)
    np.add.at(sums, inv, vals.astype(np.uint64))
    return sums.astype(np.float64) / cnt.astype(np.float64), cnt.astype(np.int64)


def k1_starts(delta, W):
    j = np.arange(delta + 1)
    q = 0.5 * (np.sin(math.pi * (j / float(delta) - 0.5)) + 1.0)
    q[0], q[delta] = 0.0, 1.0
    T = (q * float(W)).astype(np.uint64).astype(np.int64)
    T[delta] = W
    return T


def compress(m, w, delta, rule):
    W = int(w.sum())
    pref = np.cumsum(w) - w
    T = k1_starts(delta, W)[1:delta]
    if rule == "start":
        cell = np.searchsorted(T, pref, side="right")                            # T_c <= P_i < T_c+1
    else:
        cell = np.searchsorted(2 * T, 2 * pref + w, side="right")                # T_c <= P_i + w_i / 2 < T_c+1
    cw = np.bincount(cell, weights=w.astype(np.float64), minlength=delta)
    cs = np.bincount(cell, weights=m * w.astype(np.float64), minlength=delta)    # sequential sums, input order, as the oracle
    nz = cw > 0
    return cs[nz] / cw[nz], cw[nz].astype(np.int64)


def add_batch(td, vals, delta, rule):
    m, w = items_of(vals)
    if td is not None:
        om, ow = td
        mm, ww = np.concatenate([om, m]), np.concatenate([ow, w])
        o = np.argsort(mm, kind="stable")                                        # old centroids first on equal means
        m, w = mm[o], ww[o]
    return compress(m, w, delta, rule)


def quantile(td, vmin, vmax, q):
    c = np.zeros(len(td[0]), dtype=po.CENTROID_DTYPE)
    c["mean"], c["weight"] = td
    return po.lib().gyo_td_quantile(po._p(c), len(c), float(vmin), float(vmax), q)


def exact(sorted_v, q):
    return float(sorted_v[min(len(sorted_v) - 1, max(0, int(math.ceil(q * len(sorted_v))) - 1))])


def rank_err(sorted_v, g, q):
    lo, hi = np.searchsorted(sorted_v, g, side="left"), np.searchsorted(sorted_v, g, side="right")
    return abs((lo + hi) / 2.0 / len(sorted_v) - q)


def streams(n, seed):
    rng = np.random.default_rng(seed)
    clip = lambda x: np.minimum(np.maximum(x, 1.0), 1.0e9).astype(np.uint32)
    yield "lognormal s=1.0", clip(rng.lognormal(math.log(20000), 1.0, n))
    yield "lognormal s=1.5", clip(rng.lognormal(math.log(20000), 1.5, n))
    base = rng.lognormal(math.log(20000), 1.0, n)
    yield "10x step at 90 %", clip(base * np.where(np.arange(n) >= 0.9 * n, 10.0, 1.0))
    yield "x25 drift", clip(base * np.exp(np.log(25.0) * np.arange(n) / n))


def run(n, seeds, batches, delta=200):
    print(f"n = {n}, delta = {delta}, {seeds} seeds; p99 value error mean / max, worst rank error, centroids")
    print(f"{'stream':<18} {'per batch':>9} | {'start rule':^34} | {'centre rule':^34}")
    rows = {}
    for seed in range(seeds):
        for name, v in streams(n, 1000 + seed):
            sv = np.sort(v.astype(np.float64))
            for k in batches:
                for rule in ("start", "centre"):
                    td = None
                    orc = po.td_new() if rule == "centre" else None
                    for off in range(0, n, k):
                        part = v[off: off + k]
                        td = add_batch(td, part, delta, rule)
                        if orc is not None:
                            po.td_add(orc, part, float(delta))
                    if orc is not None:                                         # the restatement is the oracle, bit for bit
                        om, ow = orc.centroids()
                        assert np.array_equal(ow.astype(np.int64), td[1]) and om.tobytes() == td[0].tobytes(), (name, k)
                    est = {q: quantile(td, sv[0], sv[-1], q) for q in QS}
                    p99 = abs(est[0.99] - exact(sv, 0.99)) / exact(sv, 0.99)
                    rk = max(rank_err(sv, est[q], q) for q in QS)
                    rows.setdefault((name, k, rule), []).append((p99, rk, len(td[0])))
    for name in dict.fromkeys(r[0] for r in rows):
        for k in batches:
            line = f"{name:<18} {k:>9} |"
            for rule in ("start", "centre"):
                a = np.array(rows[(name, k, rule)])
                line += f" {100 * a[:, 0].mean():5.2f} % / {100 * a[:, 0].max():5.2f} %  rk {a[:, 1].max():.4f}  {a[:, 2].mean():5.0f} |"
            print(line)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=400_000)
    ap.add_argument("--seeds", type=int, default=4)
    ap.add_argument("--batches", type=str, default="400000,65536,4096,512")
    a = ap.parse_args()
    run(a.n, a.seeds, [int(x) for x in a.batches.split(",")])
