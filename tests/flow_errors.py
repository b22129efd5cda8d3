"""The flow error tables of GYSK_FLAG_FLOW_ERRORS and their server-error sets restated on the CPU (tests only). A response sample counts
iff it counts in the flow query tables (tests/flow_queries.py: counted) and its event carries GYSK_EVF_CLI_ERROR and/or
GYSK_EVF_SER_ERROR; it adds {cli | ser << 32} (one per bit set) to its flow key's cell in every row, at the columns the numpy hashes of
tests/flow_queries.py give. A flow's server-error score is the minimum over rows of the high half. After each device batch the open set
becomes the K best of C u B_ser (B_ser: the distinct flow keys with a counted server-error sample in the batch) by (score descending, key
ascending) on the table after the batch; gysk_flush moves it to the last set. The 300-s sets follow tests/flow_topk_5min.py's rule on the
error ring, scored alike."""
import numpy as np

from gyeeta_b200 import engine as ge
from tests import flow_level as fl
from tests import flow_queries as fq
from tests import flow_topk_slow as fs

K = fs.K
U32 = fq.U32
NSLOTS, WIDTH = fl.NSLOTS, fl.WIDTH


def empty(depth, log2w):
    return np.zeros(depth << log2w, dtype=np.uint64)


def increments(samples):
    """{cli | ser << 32} of each sample (zero for a sample without an error bit)"""
    f = samples["flags"].astype(np.uint64)
    return (f & np.uint64(1)) | (((f >> np.uint64(1)) & np.uint64(1)) << np.uint64(32))


def add_samples(table, samples, depth, log2w):
    """table += the error increments of counted samples (fq.counted), mod 2^64 per cell"""
    inc = increments(samples)
    m = inc != 0
    if not m.any():
        return table
    t = table.reshape(depth, 1 << log2w)
    cols = fq.columns(samples["flow_key"][m], depth, log2w)
    for r in range(depth):
        np.add.at(t[r], cols[r], inc[m])
    return table


def point_query(err, qry, keys, depth, log2w):
    """gysk_query_flow_errors restated: queries from the query table qry, each error half's minimum over rows of err"""
    keys = np.asarray(keys, dtype=np.uint64)
    out = np.zeros(len(keys), dtype=ge.FLOW_ERR_EST_DTYPE)
    if not len(keys):
        return out
    out["flow_key"] = keys
    out["queries"] = fq.point_query(qry, keys, depth, log2w)[0]
    out["cli_errors"], out["ser_errors"] = fq.point_query(err, keys, depth, log2w)
    return out


def ser_score(table, keys, depth, log2w):
    keys = np.asarray(keys, dtype=np.uint64)
    if not len(keys):
        return np.zeros(0, dtype=np.int64)
    return fq.point_query(table, keys, depth, log2w)[1].astype(np.int64)


def ser_keys(samples):
    """B_ser: the distinct flow keys with a counted server-error sample"""
    return np.unique(samples["flow_key"][(samples["flags"] & ge.EVF_SER_ERROR) != 0])


def exact(samples, keys):
    """[n, 2] exact (cli, ser) errors of each key (keys: ascending, unique)"""
    keys = np.asarray(keys, dtype=np.uint64)
    out = np.zeros((len(keys), 2), dtype=np.int64)
    if not len(samples) or not len(keys):
        return out
    pos = np.searchsorted(keys, samples["flow_key"])
    hit = (pos < len(keys)) & (keys[np.minimum(pos, len(keys) - 1)] == samples["flow_key"])
    f = samples["flags"]
    np.add.at(out[:, 0], pos[hit], (f[hit] & 1).astype(np.int64))
    np.add.at(out[:, 1], pos[hit], ((f[hit] >> 1) & 1).astype(np.int64))
    return out


def row_sums(table, depth, log2w):
    """per row (sum of the low halves, sum of the high halves), each mod 2^32"""
    t = table.reshape(depth, 1 << log2w)
    return [(int((t[r] & np.uint64(U32)).sum(dtype=np.uint64)) & U32, int((t[r] >> np.uint64(32)).sum(dtype=np.uint64)) & U32)
            for r in range(depth)]


def read(keys, err, qry, depth, log2w, n=K):
    """a read of a set: its first n keys as gysk_query_flow_errors rows, the zero scores left out"""
    rows = point_query(err, qry, np.asarray(keys, dtype=np.uint64)[:n], depth, log2w)
    return rows[rows["ser_errors"] != 0]


class Sets:
    """the open and last server-error set, fed B_ser and the table after each batch"""

    def __init__(self, depth, log2w, k=K):
        self.d, self.w, self.k = depth, log2w, k
        self.open = np.zeros(0, dtype=np.uint64)
        self.last = np.zeros(0, dtype=np.uint64)

    def batch(self, b, table):
        self.open = fs.select(np.concatenate([self.open, np.asarray(b, dtype=np.uint64)]), table, self.d, self.w, ser_score, self.k)
        return self.open

    def flush(self):
        self.last, self.open = self.open, np.zeros(0, dtype=np.uint64)


class LevelSets(fs.LevelSets):
    """the slot sets, L and their bounds on the error level ring (one word a cell), scored by the server-error half"""

    def __init__(self, depth, log2w, k=K):
        super().__init__(2, depth, log2w, k)
        self.score = ser_score
        self.ring = fl.FlowLevelRing(depth << log2w)


def merged(sets, summed, depth, log2w, bounds=None, k=K):
    """the merge: the k best of the union on the summed table; with bounds also B_G = max(thr(G), sum of bounds)"""
    g = fs.select(np.concatenate([np.asarray(s, dtype=np.uint64) for s in sets] + [np.zeros(0, np.uint64)]), summed, depth, log2w,
                  ser_score, k)
    return g if bounds is None else (g, max(fs.thr(g, summed, depth, log2w, ser_score, k), sum(bounds)))
