"""The flow response histograms of GYSK_FLAG_FLOW_RESP_HIST restated on the CPU (tests only). They count the samples the flow query tables
count (tests/flow_queries.py: counted, the route keys) at the same columns (flow_queries.columns). A cell is 8 u64 words: the count of
RESP_TIME_HASH bucket b of the sample's msec sits in half b & 1 of word b >> 1, every word summed mod 2^64. Tables here are flat uint64
arrays of (depth << log2w) x 8 words, the layout of gysk_export_cms_resp. Also restated: the packed key the device sums a batch under
(packed_keys / apply_packed), the point query and the percentile rule of gysk_flow_resp_est."""
import numpy as np

from tests import flow_queries as fq

WORDS, NB = 8, 15
U32, M64 = fq.U32, (1 << 64) - 1
THR = np.array([1, 10, 30, 60, 100, 150, 200, 300, 450, 700, 1000, 3000, 15000], dtype=np.int64)    # RESP_TIME_HASH thresholds


def buckets(usec):
    """RESP_TIME_HASH bucket of each sample's msec = usec / 1000 (bucket_resp_time: 1 .. 14 for unsigned values)"""
    ms = (np.asarray(usec, dtype=np.uint32) // np.uint32(1000)).astype(np.int64)
    return np.where(ms >= 15001, 14, 1 + (ms[:, None] > THR[None, :]).sum(axis=1)).astype(np.int64)


def empty(depth, log2w):
    return np.zeros((depth << log2w) * WORDS, dtype=np.uint64)


def _add(table, cols, b, counts, depth, log2w):
    inc = np.asarray(counts, dtype=np.uint64) << (np.uint64(32) * (b & 1).astype(np.uint64))      # uint64: the high bits drop, mod 2^64
    for r in range(depth):
        np.add.at(table, ((np.int64(r) << log2w) + cols[r]) * WORDS + (b >> 1), inc)
    return table


def add_samples(table, samples, depth, log2w):
    """table += one count per sample in its bucket, in every row, as one RED.ADD.64 per sample and row would"""
    if len(samples):
        _add(table, fq.columns(samples["flow_key"], depth, log2w), buckets(samples["value"]), np.ones(len(samples), dtype=np.uint64), depth, log2w)
    return table


def packed_keys(keys, b, log2w):
    """the batch flow table key of each sample, one per cell word: ((b >> 1) + 1) << 56 | (h2 & wmask) << 28 | (h1 & wmask)"""
    h1, h2 = fq.flow_hashes(keys)
    wm = np.uint64((1 << log2w) - 1)
    w = np.asarray(b, dtype=np.uint64) >> np.uint64(1)
    return ((w + np.uint64(1)) << np.uint64(56)) | ((h2.astype(np.uint64) & wm) << np.uint64(28)) | (h1.astype(np.uint64) & wm)


def packed_incs(b):
    """the word increment of each sample: 1 << 32 * (b & 1)"""
    return np.uint64(1) << (np.uint64(32) * (np.asarray(b, dtype=np.uint64) & np.uint64(1)))


def decode_packed(pkeys, depth, log2w):
    """(cell word, [depth, n] columns) of each packed key, as the TASK pass decodes it"""
    pkeys = np.asarray(pkeys, dtype=np.uint64)
    w = (pkeys >> np.uint64(56)).astype(np.int64) - 1
    h1, h2 = (pkeys & np.uint64(0xFFFFFFF)).astype(np.uint32), ((pkeys >> np.uint64(28)) & np.uint64(0xFFFFFFF)).astype(np.uint32)
    with np.errstate(over="ignore"):
        cols = np.stack([(h1 + np.uint32(r) * (h2 | np.uint32(1))) & np.uint32((1 << log2w) - 1) for r in range(depth)]).astype(np.int64)
    return w, cols


def apply_packed(table, pkeys, incs, depth, log2w):
    """the TASK pass restated: each packed key's summed increment into its word of its cell in every row, mod 2^64"""
    w, cols = decode_packed(pkeys, depth, log2w)
    incs = np.asarray(incs, dtype=np.uint64)
    for r in range(depth):
        np.add.at(table, ((np.int64(r) << log2w) + cols[r]) * WORDS + w, incs)
    return table


def halves(table):
    """[cells, 16] the 32-bit halves of every cell, bucket order (the 16th is word 7's high half)"""
    t = np.asarray(table, dtype=np.uint64).reshape(-1, WORDS)
    return np.stack([t & np.uint64(U32), t >> np.uint64(32)], axis=2).reshape(-1, 2 * WORDS)


def point_counts(table, keys, depth, log2w):
    """[n, 15] per key and bucket the minimum over rows (gysk_query_flow_resp's counts)"""
    t = np.asarray(table, dtype=np.uint64).reshape(depth, 1 << log2w, WORDS)
    cols = fq.columns(keys, depth, log2w)
    return np.stack([halves(t[r][cols[r]]) for r in range(depth)]).min(axis=0)[:, :NB].astype(np.uint32)


def pct_bucket(counts, total, pct):
    """hist_pct_bucket (GY_HISTOGRAM::get_percentiles): the first bucket whose cumulative count reaches (uint64)((float)total * (float)(pct / 100.0))"""
    cut = int(np.float32(total) * np.float32(np.float64(np.float32(pct)) / 100.0))
    c = 0
    for i, x in enumerate(counts):
        c += int(x)
        if c >= cut:
            return i
    return len(counts)


def bucket_value(b, total):
    """get_bucket_max_threshold<RESP_TIME_HASH, int64_t>: the bucket's upper threshold, min_value - 1 = -1 for bucket 0 (and an empty
    histogram), INT16_MAX for the last bucket (max_value 15001 <= INT16_MAX / 2)"""
    if b >= NB:
        b = NB - 1 if total > 0 else 0
    return -1 if b == 0 else (32767 if b >= 14 else int(THR[b - 1]))


def percentiles(counts):
    """(p25, p95, p99) msec of 15 bucket counts, the total their full sum"""
    total = sum(int(x) for x in counts)
    return tuple(bucket_value(pct_bucket(counts, total, p), total) for p in (25, 95, 99))


def point_query(table, keys, depth, log2w):
    """gysk_query_flow_resp restated: a FLOW_RESP_EST_DTYPE row per key"""
    from gyeeta_b200 import engine as ge
    keys = np.asarray(keys, dtype=np.uint64)
    out = np.zeros(len(keys), dtype=ge.FLOW_RESP_EST_DTYPE)
    out["flow_key"] = keys
    if len(keys):
        c = point_counts(table, keys, depth, log2w)
        out["counts"] = c
        out["total"] = (c.astype(np.uint64).sum(axis=1) & np.uint64(U32)).astype(np.uint32)
        p = np.array([percentiles(row) for row in c], dtype=np.int64).reshape(-1, 3)
        out["p25_ms"], out["p95_ms"], out["p99_ms"] = p[:, 0], p[:, 1], p[:, 2]
    return out


def exact(samples, keys):
    """[n, 15] the exact bucket counts of each key (keys: ascending, unique)"""
    keys = np.asarray(keys, dtype=np.uint64)
    assert np.all(keys[:-1] < keys[1:]), "keys: ascending, unique"
    out = np.zeros((len(keys), NB), dtype=np.int64)
    if not len(samples) or not len(keys):
        return out
    u, inv = np.unique(samples["flow_key"], return_inverse=True)
    pos = np.searchsorted(keys, u)
    hit = (pos < len(keys)) & (keys[np.minimum(pos, len(keys) - 1)] == u)
    m = hit[inv.reshape(-1)]
    np.add.at(out, (pos[inv.reshape(-1)][m], buckets(samples["value"])[m]), 1)
    return out


def bucket_sums(table, depth, log2w):
    """[depth, 16] per row and bucket the column sum of that half, mod 2^32"""
    t = np.asarray(table, dtype=np.uint64).reshape(depth, 1 << log2w, WORDS)
    out = np.zeros((depth, 2 * WORDS), dtype=np.int64)
    for r in range(depth):
        out[r, 0::2] = ((t[r] & np.uint64(U32)).sum(axis=0, dtype=np.uint64) & np.uint64(U32)).astype(np.int64)
        out[r, 1::2] = ((t[r] >> np.uint64(32)).sum(axis=0, dtype=np.uint64) & np.uint64(U32)).astype(np.int64)
    return out


def cell_totals(table):
    """per cell the sum of its 16 halves mod 2^32: the query half of the same flow query cell (while no bucket count carries)"""
    t = np.asarray(table, dtype=np.uint64).reshape(-1, WORDS)
    lo = (t & np.uint64(U32)).sum(axis=1, dtype=np.uint64)
    return (lo + (t >> np.uint64(32)).sum(axis=1, dtype=np.uint64)) & np.uint64(U32)
