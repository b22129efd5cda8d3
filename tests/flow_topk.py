"""The heaviest-flow sets of GYSK_FLAG_FLOW_TOPK restated on the CPU (tests only), on top of the table restatements of
tests/flow_queries.py. After each device batch the open set C becomes the K best of C u B by (score descending, flow key ascending), B the
distinct flow keys whose records reached the table in the batch, every key scored on the table as it is after the batch: the minimum over
rows of one half of its cells (the kbytes half of the connection table, the queries half of the flow query table). gysk_flush moves the
open set to the last one and starts an empty one. The merge keeps the K best of the union of every rank's last sets, scored on the summed
table. A read returns the set's first n entries with their estimates, the zero scores left out."""
import numpy as np

from gyeeta_b200 import engine as ge
from tests import flow_queries as fq

K = ge.FLOW_TOPK_CAP
CONN, QRY = 0, 1                  # the two sets; HALF: which half of a cell scores
HALF = {CONN: 1, QRY: 0}
TCP_TYPES = (ge.EV_CONNECT, ge.EV_ACCEPT, ge.EV_CLOSE_CLI, ge.EV_CLOSE_SER, ge.EV_ACTIVE)


def scores(table, keys, depth, log2w, half):
    """the point estimate of one half per key (uint32), the rule of gysk_query_flows"""
    lo, hi = fq.point_query(table, np.asarray(keys, dtype=np.uint64), depth, log2w)
    return hi if half else lo


def select(keys, table, depth, log2w, half, k=K):
    """the k best of the distinct keys by (score descending, key ascending)"""
    u = np.unique(np.asarray(keys, dtype=np.uint64))
    if not len(u):
        return u
    s = scores(table, u, depth, log2w, half).astype(np.int64)
    return u[np.lexsort((u, -s))][:k]


def batch_keys(ev, which, known=None):
    """B: the flow keys of the batch's records that reach the table (connection records of services holding a slot, ACTIVE ones
    included; counted response samples). known: the ids holding a slot (None: every id but 0 and ~0)"""
    if which == QRY:
        return np.unique(fq.counted(ev, known)["flow_key"])
    m = np.isin(ev["type"], TCP_TYPES) & (ev["svc_id"] != 0) & (ev["svc_id"] != np.uint64(0xFFFFFFFFFFFFFFFF))
    if known is not None:
        m &= np.isin(ev["svc_id"], np.fromiter(known, dtype=np.uint64, count=len(known)))
    return np.unique(ev["flow_key"][m])


def read(keys, table, depth, log2w, half, n=K):
    """a read of a set: its first n keys with their estimates as gysk_flow_est rows, the zero scores left out"""
    keys = np.asarray(keys, dtype=np.uint64)[:n]
    lo, hi = fq.point_query(table, keys, depth, log2w) if len(keys) else (np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    rows = np.zeros(len(keys), dtype=ge.FLOW_EST_DTYPE)
    rows["flow_key"], rows["count"], rows["kbytes"] = keys, lo, hi
    return rows[(hi if half else lo) != 0]


def conn_increments(ev):
    """{count | kbytes << 32} of each connection record: cms_increment(bytes) of a TCP event, {flags | value << 32} of ACTIVE"""
    inc = np.uint64(1) | ((ev["value"] >> np.uint32(10)).astype(np.uint64) << np.uint64(32))
    act = ev["type"] == ge.EV_ACTIVE
    inc[act] = ev["flags"][act].astype(np.uint64) | (ev["value"][act].astype(np.uint64) << np.uint64(32))
    return inc


def exact_scores(keys, flow_keys, inc, half):
    """each key's exact score: the half of the sum of its increments, mod 2^32"""
    keys = np.asarray(keys, dtype=np.uint64)
    part = (inc >> np.uint64(32)) if half else (inc & np.uint64(fq.U32))
    u, inv = np.unique(flow_keys, return_inverse=True)
    if not len(u):
        return np.zeros(len(keys), dtype=np.int64)
    tot = np.zeros(len(u), dtype=np.uint64)
    np.add.at(tot, inv.reshape(-1), part)
    pos = np.minimum(np.searchsorted(u, keys), len(u) - 1)
    out = np.where(u[pos] == keys, tot[pos], np.uint64(0))
    return (out & np.uint64(fq.U32)).astype(np.int64)


def guarantee_holds(set_keys, table, depth, log2w, half, all_keys, exact):
    """the guarantee: with a full set, every flow whose exact score exceeds the set's smallest score is in it; with fewer than K
    members, every flow of the window is (all_keys: every flow of the window, exact: their exact scores)"""
    members = set(np.asarray(set_keys, dtype=np.uint64).tolist())
    if len(set_keys) < K:
        return all(int(k) in members for k in all_keys)
    thr = int(scores(table, set_keys, depth, log2w, half).min())
    return all(int(k) in members for k, x in zip(all_keys.tolist(), exact.tolist()) if x > thr)


class Sets:
    """the open and last set of one table, fed the table after each batch"""

    def __init__(self, half, depth, log2w, k=K):
        self.half, self.d, self.w, self.k = half, depth, log2w, k
        self.open = np.zeros(0, dtype=np.uint64)
        self.last = np.zeros(0, dtype=np.uint64)
        self.floor = []                 # the K-th score after each batch of the window (full sets only)

    def batch(self, b, table):
        self.open = select(np.concatenate([self.open, np.asarray(b, dtype=np.uint64)]), table, self.d, self.w, self.half, self.k)
        if len(self.open) == self.k:
            self.floor.append(int(scores(table, self.open[-1:], self.d, self.w, self.half)[0]))
        return self.open

    def flush(self):
        self.last, self.open, self.floor = self.open, np.zeros(0, dtype=np.uint64), []


def merged(sets, table, depth, log2w, half, k=K):
    """the merge: the k best of the union of every rank's last set, scored on the summed table"""
    return select(np.concatenate([np.asarray(s, dtype=np.uint64) for s in sets] + [np.zeros(0, np.uint64)]), table, depth, log2w, half, k)
