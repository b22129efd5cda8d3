"""The heaviest-flow sets of the rolling 300-s levels (GYSK_FLAG_FLOW_TOPK_5MIN) restated on the CPU (tests only), on top of the window
sets of tests/flow_topk.py and the level ring of tests/flow_level.py. At every flush, once the closing window's table is in ring slot
s = (tsec / 30) % 10: if the flush took the slot for a new epoch, its set S_s and bound B_s start empty; S_s becomes the K best of S_s u W
(W the closing window's set) scored on the slot, and B_s = max(thr(S_s), B_s + thr(W)). Then the level set L becomes the K best of the
live slots' sets scored on the level, and B_L = max(thr(L), sum of the live B_s). thr(X) is the smallest score of X when it holds K
flows, else 0. The merge keeps the K best of every rank's L on the summed levels, with B_G = max(thr(G), sum of the ranks' B_L)."""
import numpy as np

from tests import flow_level as fl
from tests import flow_queries as fq
from tests import flow_topk as ft

K = ft.K
NSLOTS, WIDTH = fl.NSLOTS, fl.WIDTH


def thr(keys, table, depth, log2w, half, k=K):
    """the smallest score of a full set (its last key: the sets are best first), else 0"""
    return int(ft.scores(table, keys[-1:], depth, log2w, half)[0]) if len(keys) == k else 0


def table_of(keys, inc, depth, log2w):
    """a count-min table of one u64 per cell holding the increments inc of the flow keys"""
    t = np.zeros((depth, 1 << log2w), dtype=np.uint64)
    cols = fq.columns(np.asarray(keys, dtype=np.uint64), depth, log2w)
    for r in range(depth):
        np.add.at(t[r], cols[r], np.asarray(inc, dtype=np.uint64))
    return t.reshape(-1)


class LevelSets:
    """the slot sets, the level set and their bounds of one level, fed each flush's tsec, closing window set and closing table. The
    ring is tests/flow_level.py's, so the slot decision is the level's own."""

    def __init__(self, half, depth, log2w, k=K):
        self.half, self.d, self.w, self.k = half, depth, log2w, k
        self.ring = fl.FlowLevelRing(depth << log2w)
        self.slots = [np.zeros(0, dtype=np.uint64) for _ in range(NSLOTS)]
        self.bounds = [0] * NSLOTS
        self.L = np.zeros(0, dtype=np.uint64)
        self.B = 0
        self.slot_thr = []              # (slot, epoch, thr(S_s)) after each fold

    def _thr(self, keys, table):
        return thr(keys, table, self.d, self.w, self.half, self.k)

    def flush(self, tsec, win, closed):
        """the flush at tsec of the window whose set is win and whose table is closed; returns (L, B_L)"""
        ep, s = tsec // WIDTH, (tsec // WIDTH) % NSLOTS
        fresh = self.ring.epoch[s] != ep
        level = self.ring.flush(tsec, closed)
        if fresh:
            self.slots[s], self.bounds[s] = np.zeros(0, dtype=np.uint64), 0
        acc = self.bounds[s] + self._thr(np.asarray(win, dtype=np.uint64), closed)
        self.slots[s] = ft.select(np.concatenate([self.slots[s], np.asarray(win, dtype=np.uint64)]), self.ring.ring[s], self.d, self.w,
                                  self.half, self.k)
        t = self._thr(self.slots[s], self.ring.ring[s])
        self.bounds[s] = max(t, acc)
        self.slot_thr.append((s, ep, t))
        live = self.live(ep)
        self.L = ft.select(np.concatenate([self.slots[j] for j in live] + [np.zeros(0, np.uint64)]), level, self.d, self.w, self.half,
                           self.k)
        self.B = max(self._thr(self.L, level), sum(self.bounds[j] for j in live))
        return self.L, self.B

    def live(self, ep):
        return [j for j in range(NSLOTS) if self.ring.epoch[j] is not None and ep - NSLOTS < self.ring.epoch[j] <= ep]

    @property
    def level(self):
        return self.ring.level


def merged(sets, bounds, summed, depth, log2w, half, k=K):
    """the merge of the ranks' level sets: (G, B_G) on the summed level"""
    g = ft.merged(sets, summed, depth, log2w, half, k)
    return g, max(thr(g, summed, depth, log2w, half, k), sum(bounds))


def exact_level(tsecs, windows):
    """each flow's exact score over the windows the level holds after the last of tsecs: {flow key: score}. windows[i]: {key: score}
    of the window flush i closed"""
    out = {}
    for i in fl.held_windows(tsecs):
        for key, x in windows[i].items():
            out[key] = out.get(key, 0) + x
    return out


def guarantee_holds(set_keys, bound, exact):
    """every flow outside the set has an exact score of at most the bound"""
    members = set(np.asarray(set_keys, dtype=np.uint64).tolist())
    return all(x <= bound for key, x in exact.items() if key not in members)
