"""The slow-response sets of GYSK_FLAG_FLOW_TOPK_SLOW restated on the CPU (tests only), on the response tables of tests/flow_resp_hist.py
and the selection of tests/flow_topk.py with the score passed in. A counted sample is slow when its RESP_TIME_HASH bucket is b_slow or above
(b_slow = 2 + the index of the threshold T). A flow's score S on a response table is the sum of its per-bucket row minima (point_counts)
from b_slow on, saturated at 2^32 - 1. After each device batch the open set becomes the K best of C u B_slow (B_slow: the distinct flow keys
with a slow counted sample in the batch), by (score descending, key ascending) on the table after the batch; gysk_flush moves it to the
last set. The 300-s level sets follow tests/flow_topk_5min.py's rule on the response ring, scored by S."""
import numpy as np

from tests import flow_level as fl
from tests import flow_resp_hist as frh
from tests import flow_topk as ft

K = ft.K
THR = frh.THR
NSLOTS, WIDTH = fl.NSLOTS, fl.WIDTH
SAT = (1 << 32) - 1


def b_slow(above_ms):
    """the first slow bucket of threshold above_ms: msec > T <=> bucket >= 2 + index of T"""
    return 2 + int(np.flatnonzero(THR == above_ms)[0])


def score_of_counts(counts, bs):
    """S of [n, 15] bucket counts: their sum from bucket bs on, saturated at 2^32 - 1"""
    c = np.asarray(counts, dtype=np.uint64).reshape(-1, frh.NB)
    return np.minimum(c[:, bs:].sum(axis=1, dtype=np.uint64), np.uint64(SAT)).astype(np.int64)


def scorer(bs):
    """score(table, keys, depth, log2w) -> S per key"""
    def score(table, keys, depth, log2w):
        keys = np.asarray(keys, dtype=np.uint64)
        if not len(keys):
            return np.zeros(0, dtype=np.int64)
        return score_of_counts(frh.point_counts(table, keys, depth, log2w), bs)
    return score


def select(keys, table, depth, log2w, score, k=K):
    """the k best of the distinct keys by (score descending, key ascending)"""
    u = np.unique(np.asarray(keys, dtype=np.uint64))
    if not len(u):
        return u
    s = score(table, u, depth, log2w)
    return u[np.lexsort((u, -s))][:k]


def thr(keys, table, depth, log2w, score, k=K):
    """the smallest score of a full set (its last key), else 0"""
    return int(score(table, np.asarray(keys, dtype=np.uint64)[-1:], depth, log2w)[0]) if len(keys) == k else 0


def slow_keys(samples, bs):
    """B_slow: the distinct flow keys with at least one counted sample in bucket bs or above"""
    if not len(samples):
        return np.zeros(0, dtype=np.uint64)
    return np.unique(samples["flow_key"][frh.buckets(samples["value"]) >= bs])


def read(keys, table, depth, log2w, bs, n=K):
    """a read of a set: its first n keys as gysk_query_flow_resp rows, the zero scores left out"""
    rows = frh.point_query(table, np.asarray(keys, dtype=np.uint64)[:n], depth, log2w)
    return rows[score_of_counts(rows["counts"], bs) != 0] if len(rows) else rows


def exact_slow(samples, keys, bs):
    """each key's exact slow count (keys: ascending, unique)"""
    return frh.exact(samples, keys)[:, bs:].sum(axis=1)


def guarantee_holds(set_keys, table, depth, log2w, score, all_keys, exact, k=K):
    """with a full set every flow whose exact count exceeds the set's smallest score is in it; with fewer, every slow flow is"""
    members = set(np.asarray(set_keys, dtype=np.uint64).tolist())
    if len(set_keys) < k:
        return all(int(key) in members for key, x in zip(all_keys.tolist(), np.asarray(exact).tolist()) if x > 0)
    t = thr(set_keys, table, depth, log2w, score, k)
    return all(int(key) in members for key, x in zip(all_keys.tolist(), np.asarray(exact).tolist()) if x > t)


class Sets:
    """the open and last slow set, fed B_slow and the table after each batch"""

    def __init__(self, bs, depth, log2w, k=K):
        self.score, self.d, self.w, self.k = scorer(bs), depth, log2w, k
        self.open = np.zeros(0, dtype=np.uint64)
        self.last = np.zeros(0, dtype=np.uint64)

    def batch(self, b, table):
        self.open = select(np.concatenate([self.open, np.asarray(b, dtype=np.uint64)]), table, self.d, self.w, self.score, self.k)
        return self.open

    def flush(self):
        self.last, self.open = self.open, np.zeros(0, dtype=np.uint64)


class LevelSets:
    """the slot sets, L and their bounds on the response level ring, the rule of tests/flow_topk_5min.py scored by S"""

    def __init__(self, bs, depth, log2w, k=K):
        self.score, self.d, self.w, self.k = scorer(bs), depth, log2w, k
        self.ring = fl.FlowLevelRing((depth << log2w) * frh.WORDS)
        self.slots = [np.zeros(0, dtype=np.uint64) for _ in range(NSLOTS)]
        self.bounds = [0] * NSLOTS
        self.L = np.zeros(0, dtype=np.uint64)
        self.B = 0

    def _thr(self, keys, table):
        return thr(keys, table, self.d, self.w, self.score, self.k)

    def flush(self, tsec, win, closed):
        """the flush at tsec of the window whose slow set is win and whose response table is closed; returns (L, B_L)"""
        ep, s = tsec // WIDTH, (tsec // WIDTH) % NSLOTS
        fresh = self.ring.epoch[s] != ep
        level = self.ring.flush(tsec, closed)
        if fresh:
            self.slots[s], self.bounds[s] = np.zeros(0, dtype=np.uint64), 0
        win = np.asarray(win, dtype=np.uint64)
        acc = self.bounds[s] + self._thr(win, closed)
        self.slots[s] = select(np.concatenate([self.slots[s], win]), self.ring.ring[s], self.d, self.w, self.score, self.k)
        self.bounds[s] = max(self._thr(self.slots[s], self.ring.ring[s]), acc)
        live = [j for j in range(NSLOTS) if self.ring.epoch[j] is not None and ep - NSLOTS < self.ring.epoch[j] <= ep]
        self.L = select(np.concatenate([self.slots[j] for j in live] + [np.zeros(0, np.uint64)]), level, self.d, self.w, self.score,
                        self.k)
        self.B = max(self._thr(self.L, level), sum(self.bounds[j] for j in live))
        return self.L, self.B

    @property
    def level(self):
        return self.ring.level


def merged(sets, summed, depth, log2w, bs, bounds=None, k=K):
    """the merge: the k best of the union of the ranks' sets on the summed table; with bounds also B_G = max(thr(G), sum of bounds)"""
    score = scorer(bs)
    g = select(np.concatenate([np.asarray(s, dtype=np.uint64) for s in sets] + [np.zeros(0, np.uint64)]), summed, depth, log2w, score, k)
    return g if bounds is None else (g, max(thr(g, summed, depth, log2w, score, k), sum(bounds)))
