"""The batch's response keys are sorted by service only: inside a service's segment the bins arrive in any order, and
bins_merge_kernel sums a short segment (at most LONG_SEG keys) per bin in shared memory before it walks the bins in order. That
must not change a number: after every batch each service's window histogram and t-digest equal the oracle's bit for bit, and each
trace row's digest equals the restated trace view's. The services are registered one by one, so their segments lie in the sorted
keys in a known order. Segments: 1 key; every key in one bin; 31, 32, 33 and every reachable distinct bin; bins in ascending,
descending and shuffled order; the extremes 0 usec and the largest response time in one segment; LONG_SEG - 1, LONG_SEG and
LONG_SEG + 1 keys; and trace pseudo-slots beside the services that bring the same response times."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po
from tests import trace_agg as ta
from tests.util import assert_hist_equal, feed_both, make_pair, td_bin_usec

pytestmark = pytest.mark.gpu

LONG_SEG = 8192                 # gysk_kernels.cuh


@pytest.fixture(scope="module")
def bin_usec():
    """one response time in every reachable value bin, ascending by bin"""
    bins, usec = td_bin_usec()
    assert len(bins) > 800 and np.all(np.diff(bins) > 0)
    return usec.astype(np.uint32)


def _lognormal(rng, n):
    return np.minimum(np.exp(rng.normal(np.log(3000.0), 1.7, n)), 9.0e8).astype(np.uint32)


def _segments(rng, bu):
    """the usec of each service's samples of one batch, in the order they are fed"""
    shuffled = np.repeat(bu[:300], 3)
    return [
        np.array([4321], dtype=np.uint32),                        # 1 key
        np.full(700, 1500, dtype=np.uint32),                      # every key in one bin
        np.repeat(bu[100:131], 2),                                # 31 distinct bins
        np.repeat(bu[200:232], 3),                                # 32
        bu[400:433].copy(),                                       # 33
        bu.copy(),                                                # every reachable bin, ascending
        np.repeat(bu[::-1], 2),                                   # every reachable bin, descending
        np.repeat(bu[50:250][::-1], 5),                           # 200 bins, descending
        shuffled[rng.permutation(len(shuffled))],                 # 300 bins, shuffled
        np.array([0, 999_999_999, 0, 5, 999_999_999], dtype=np.uint32),   # both ends of the bin range
        _lognormal(rng, LONG_SEG - 1),
        _lognormal(rng, LONG_SEG),                                # the longest short segment
        _lognormal(rng, LONG_SEG + 1),                            # the shortest long segment
        np.full(LONG_SEG, 77, dtype=np.uint32),                   # LONG_SEG keys in one bin
        bu[rng.integers(0, len(bu), LONG_SEG)],                   # LONG_SEG keys over every bin, shuffled
    ]


def _events(ids, segs, rng):
    parts = []
    for id_, usec in zip(ids, segs):
        ev = np.zeros(len(usec), dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = id_
        ev["flow_key"] = rng.integers(1, 1 << 62, len(usec), dtype=np.uint64)
        ev["value"] = usec
        ev["type"] = ge.EV_RESP
        ev["tsec"] = 1
        parts.append(ev)
    return np.concatenate(parts)       # each service's samples together and in the order given


@pytest.mark.parametrize("rows", [0, 2048], ids=["hot-off", "hot-on"])
def test_short_segments_in_any_bin_order_are_bit_exact(monkeypatch, bin_usec, rows):
    monkeypatch.setenv("GYSK_HOT_ROWS", str(rows))
    rng = np.random.default_rng(90)
    segs = _segments(rng, bin_usec)
    ids = synth.service_ids(len(segs) + 3)[3:]
    eng, orc = make_pair(max_svcs=256, max_tasks=16, max_batch=1 << 20, cms_log2_width=12)
    for i in range(len(ids)):                         # one call per id: slot order = list order
        eng.register_ids(ids[i:i + 1])
        orc.register_ids(ids[i:i + 1])
    for b in range(3):
        ev = _events(ids, segs if b != 1 else [s[::-1] for s in segs], rng)
        feed_both(eng, orc, ev, 1 << 20)
        if b == 0:
            assert eng.last_batch_keys() == len(ev)
        for id_ in ids.tolist():
            assert_hist_equal(eng, orc, id_, ge.HIST_RESP_CUR)
            (means, weights, mn, mx), td = eng.export_tdigest(id_), orc.export_tdigest(id_)
            om, ow = td.centroids()
            assert means.tobytes() == om.tobytes() and np.array_equal(weights, ow), (b, hex(id_))
            assert mn == td.minv and mx == td.maxv and int(weights.sum()) == td.total, (b, hex(id_))
        if b == 1:
            eng.flush(5); orc.flush(5)
            for id_ in ids.tolist():
                assert_hist_equal(eng, orc, id_, ge.HIST_RESP_LAST)


def test_trace_pseudo_slots_beside_services(bin_usec):
    """trace rows' segments (the pseudo-slots after every service) hold the same bin layouts as their services' segments"""
    rng = np.random.default_rng(91)
    segs = [s for s in _segments(rng, bin_usec) if len(s) <= LONG_SEG]
    ids = (np.arange(1, len(segs) + 1, dtype=np.uint64) * np.uint64(0x9E3779B1)) | np.uint64(1 << 40)
    eng = ge.Engine(max_svcs=256, max_tasks=16, max_batch=1 << 20, max_trace_svcs=64)
    orc = po.OracleEngine(max_svcs=256, max_tasks=16)
    to = ta.TraceOracle(64)
    for b in range(2):
        gid = np.concatenate([np.full(len(s), i, dtype=np.uint64) for i, s in zip(ids, segs)])
        usec = np.concatenate([s if b == 0 else s[::-1] for s in segs]).astype(np.uint64)
        rec = ta.api_tran(gid, usec)
        tr = ta.trace_events(rec)
        rs = ta.resp_events(rec)
        ev = np.concatenate([rs, tr])
        eng.ingest_events(ev)
        eng.sync()
        orc.ingest(ev)
        to.ingest(ev)
        for id_ in ids.tolist():
            a, o = eng.export_hist(id_, ge.HIST_RESP_CUR), orc.export_hist(id_, ge.HIST_RESP_CUR)
            assert np.array_equal(a[0], o[0]) and a[1:] == o[1:], (b, hex(id_))
            m, w, mn, mx = eng.export_tdigest(id_)
            om, ow = orc.export_tdigest(id_).centroids()
            assert m.tobytes() == om.tobytes() and np.array_equal(w, ow), (b, hex(id_))
            tm, tw, tmn, tmx = eng.export_trace_tdigest(id_, False)
            rm, rw, rmn, rmx = to.digest(id_, False)
            assert tm.tobytes() == np.asarray(rm, dtype=np.float64).tobytes() and np.array_equal(tw, rw), (b, hex(id_))
            assert (tmn, tmx) == (rmn, rmx), (b, hex(id_))
        rows = eng.query_traces(ids.tolist())
        for id_, r in zip(ids.tolist(), rows):
            assert ta.row_bytes(r) == ta.row_bytes(to.row(id_, 0)), hex(id_)
