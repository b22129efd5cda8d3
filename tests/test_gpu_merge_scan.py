"""bins_merge_kernel reads a short key segment (at most LONG_SEG keys) in blocks of 256 keys, 8 consecutive keys per lane: each lane
sums its own runs of equal bin, one segmented scan per block joins the runs that cross lanes and blocks, and a bin's totals are
emitted at its last key. When the digest's old centroids and the batch's items fit the warp's shared-memory work area together
(head.n + items <= 540, TD_SMEM_N) the items are staged there and merged by warp_merge_compress_staged; otherwise they go to the
warp's L2 scratch. Here segments are laid out against those edges — a new bin at every key, runs across a lane (8-key) and a block
(256-key) boundary, a bin over a whole block, segments of 1, 7, 8, 9, 255, 256, 257 and LONG_SEG keys, at both parities of the
segment's first key — and services bring exactly 539, 540 and 541 - head.n items. After every batch each service's window histogram
and t-digest equal the oracle's bit for bit."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from tests.util import assert_hist_equal, feed_both, make_pair, td_bin_usec

pytestmark = pytest.mark.gpu

LONG_SEG = 8192                 # gysk_kernels.cuh
SMEM_N = 540                    # TD_SMEM_N, gysk_kernels.cu


def _resp(id_, usec, rng):
    ev = np.zeros(len(usec), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = id_
    ev["flow_key"] = rng.integers(1, 1 << 62, len(usec), dtype=np.uint64)
    ev["value"] = np.asarray(usec, dtype=np.uint32)
    ev["type"] = ge.EV_RESP
    ev["tsec"] = 1
    return ev


def _runs(usec, lengths, first):
    """one run of lengths[k] samples in the k-th bin from `first` on (ascending bins: the sorted segment is these runs in order)"""
    return np.repeat(usec[first: first + len(lengths)], lengths)


def _lognormal(rng, n):
    return np.minimum(np.exp(rng.normal(np.log(2000.0), 1.5, n)), 9.0e8).astype(np.uint32)


def _td_equal(eng, orc, id_, ctx):
    (means, weights, mn, mx), td = eng.export_tdigest(id_), orc.export_tdigest(id_)
    om, ow = td.centroids()
    assert np.array_equal(weights, ow) and means.tobytes() == om.tobytes(), ctx
    if len(ow):
        assert (mn, mx) == (td.minv, td.maxv) and int(weights.sum()) == td.total, ctx
    return len(ow)


def test_short_segment_scan_edges_are_bit_exact(monkeypatch):
    monkeypatch.setenv("GYSK_HOT_ROWS", "0")          # every sample travels as a sort key
    bins, usec = td_bin_usec()
    assert len(bins) >= 840
    rng = np.random.default_rng(256)
    # a new bin at every key (300 keys: one block and a bit); runs over key 5..12 (a lane boundary) and 250..262 (a block
    # boundary); one bin over keys 100..611 (the whole second block); then random segments of every edge length
    every_key = usec[200:500]
    across = _runs(usec, [5, 8] + [1] * 237 + [13] + [2] * 20, 100)
    whole_block = _runs(usec, [100, 512, 7], 300)
    fixed = [every_key, across, whole_block]
    lengths = [1, 7, 8, 9, 255, 256, 257, LONG_SEG]
    nedge = 3                                           # services at head.n + items = 539, 540, 541
    ids = synth.service_ids(1 + len(fixed) + len(lengths) + nedge + 5)[5:]
    pad_id, ids = int(ids[0]), [int(x) for x in ids[1:]]
    edge_ids = ids[len(fixed) + len(lengths):]

    eng, orc = make_pair(max_svcs=64, max_tasks=8, max_batch=1 << 16, cms_log2_width=8)
    for id_ in [pad_id] + ids:                          # one call per id: slot order = segment order in the sorted keys
        eng.register_ids(np.array([id_], dtype=np.uint64))
        orc.register_ids(np.array([id_], dtype=np.uint64))
    paths = set()
    for b in range(6):
        # the pad service's 1 or 2 keys flip the parity of every later segment's first key
        parts = [_resp(pad_id, usec[400: 401 + (b & 1)], rng)]
        parts += [_resp(id_, v, rng) for id_, v in zip(ids, fixed)]
        parts += [_resp(id_, _lognormal(rng, n), rng) for id_, n in zip(ids[len(fixed):], lengths)]
        for k, id_ in enumerate(edge_ids):
            if b == 0:
                parts.append(_resp(id_, _lognormal(rng, 3000), rng))       # a digest of old centroids first
            else:
                n_old = len(eng.export_tdigest(id_)[1])
                want = SMEM_N - 1 + k - n_old                               # items: head.n + items = 539, 540, 541
                pick = np.sort(rng.choice(len(bins), want, replace=False))
                parts.append(_resp(id_, np.repeat(usec[pick], rng.integers(1, 4, want)), rng))
                paths.add(n_old + want <= SMEM_N)
        ev = np.concatenate(parts)
        feed_both(eng, orc, ev[rng.permutation(len(ev))], 1 << 16)
        assert eng.last_batch_keys() == len(ev)
        for id_ in [pad_id] + ids:
            assert_hist_equal(eng, orc, id_, ge.HIST_RESP_CUR)
            _td_equal(eng, orc, id_, (b, hex(id_)))
        if b == 3:
            eng.flush(5); orc.flush(5)
    assert paths == {True, False}                       # both the staged and the L2 path ran
    eng.close(); orc.close()
