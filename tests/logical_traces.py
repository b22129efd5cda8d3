"""The merged trace rows of logical services restated (tests only): what GYSK_FLAG_MERGE_TRACES computes for every logical service, from
one TraceOracle per rank (tests/trace_agg.py), each fed the events its rank owns. Members are taken in map order on each rank and the
ranks in ascending order; a member without a trace row on a rank adds nothing there. Counters are summed, maxima taken, and the window
digests folded with td_fold at compression 100, as fold_td_kernel and finish_td_kernel fold them."""
import ctypes as C

import numpy as np

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests import trace_agg as ta
from tests.util import Digest, td_fold

DELTA = 100
SUMS = ("nreq", "nerr", "nconns", "sum_resp_us", "bytes_in", "bytes_out")
MAXES = ("max_resp_us", "max_bytes_in", "max_bytes_out")


def members_of(glob, logical):
    """{logical id: [glob ids in map order]}, logical ids in order of first appearance"""
    m = {}
    for g, l in zip(np.asarray(glob, dtype=np.uint64).tolist(), np.asarray(logical, dtype=np.uint64).tolist()):
        m.setdefault(l, []).append(g)
    return m


def window_digest(to, g):
    """the last closed window's digest of member g on one rank's TraceOracle, as a Digest (None without a row)"""
    d = to.digest(g, True)
    if d is None:
        return None
    means, weights, mn, mx = d
    cent = np.zeros(len(means), dtype=po.CENTROID_DTYPE)
    cent["mean"], cent["weight"] = means, weights
    return Digest(cent, int(np.asarray(weights).sum()), mn, mx)


def fold_counters(oracles, gs):
    """(window dict of the summed counters and maxima, ntraced) of members gs over the ranks' TraceOracles"""
    w = dict(ta.empty_window(), td_count=0)
    ntraced = 0
    for to in oracles:
        for g in gs:
            if g not in to.in_use:
                continue
            ntraced += 1
            x = to.last[g]
            for f in SUMS:
                w[f] += x[f]
            for f in MAXES:
                w[f] = max(w[f], x[f])
            w["resp_buckets"] = [a + b for a, b in zip(w["resp_buckets"], x["resp_buckets"])]
            d = window_digest(to, g)
            w["td_count"] += d.total
    return w, ntraced


def merged_digest(oracles, gs):
    """the members' window digests folded in map order on each rank, then the ranks' in ascending order"""
    return td_fold([td_fold([window_digest(to, g) for g in gs], DELTA) for to in oracles], DELTA)


def quantile(d, q):
    """gysk_tdigest_quantile of a Digest, NaN while it is empty"""
    if not len(d.cent):
        return float("nan")
    m, w = np.ascontiguousarray(d.cent["mean"]), np.ascontiguousarray(d.cent["weight"], dtype=np.uint64)
    return ge.load_library().gysk_tdigest_quantile(ge._p(m), ge._p(w), len(m), d.minv, d.maxv, q)


def row(oracles, lid, gs):
    """(the gysk_logical_trace of one mapped logical service as a LogicalTrace, its merged Digest)"""
    w, ntraced = fold_counters(oracles, gs)
    d = merged_digest(oracles, gs)
    r = ge.LogicalTrace()
    r.logical_id, r.found, r.ntraced = lid, 1, ntraced
    for f in SUMS + MAXES + ("td_count",):
        setattr(r.last, f, w[f])
    r.last.resp_buckets[:] = w["resp_buckets"]
    r.last.p99_resp_us = quantile(d, 0.99)
    return r, d


def missing(lid):
    """the row of an id the map does not have: all zero but the queried id"""
    r = ge.LogicalTrace()
    r.logical_id = lid
    return r


def pgtext(d):
    L = ge.load_library()
    buf = C.create_string_buffer(8192)
    m, w = np.ascontiguousarray(d.cent["mean"]), np.ascontiguousarray(d.cent["weight"], dtype=np.uint64)
    rc = L.gysk_tdigest_to_pgtext(ge._p(m), ge._p(w), len(m), DELTA, buf, len(buf))
    assert rc >= 0
    return buf.value.decode()


def row_bytes(r):
    return bytes(C.string_at(C.addressof(r), C.sizeof(r)))
