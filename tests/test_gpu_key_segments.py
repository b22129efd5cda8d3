"""The samples of a service that travel as sort keys reach bins_merge_kernel in one of two ways: a segment of at most LONG_SEG
keys is read by one warp straight from the sorted keys (bins found by a segmented scan over 32-key windows), a longer one is
summed into a dense batch row by long_sum_kernel first. That is routing only: after every batch each service's window histogram
and t-digest must equal the oracle's bit for bit. The services are registered one by one, so their slots, and with them the order
of their segments in the sorted keys, are known: segments start and end on 128-key chunk and 4096-key sort-tile boundaries, and
have 1, 31, 32, 33, LONG_SEG - 1, LONG_SEG and LONG_SEG + 1 keys; one service brings millions of keys over many bins, others
bring all their keys in one bin (the whole-chunk path of a long segment, and a short one)."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from tests.util import assert_hist_equal, feed_both, make_pair

pytestmark = pytest.mark.gpu

LONG_SEG = 8192                 # gysk_kernels.cuh
CHUNK, TILE = 128, 4096

# (keys per batch, one-bin value or None): the running sum of the keys marks where each segment ends
LAYOUT = [
    (CHUNK, None),                        # ends on a chunk boundary
    (TILE - CHUNK, None),                 # ends on a tile boundary
    (1, None), (31, None), (32, None), (33, None),
    (2 * TILE - (TILE + 97), None),       # pads to the next tile: 8192
    (LONG_SEG, None),                     # the longest short segment, from tile boundary to tile boundary
    (LONG_SEG + 1, None),                 # the shortest long segment, from a tile boundary
    (CHUNK - 1, None),                    # back onto a chunk boundary
    (LONG_SEG - 1, None),
    (3 * CHUNK + 1, None),
    (TILE, 1500),                         # short, every key in one bin
    (300_000, 1500),                      # long, every key in one bin: whole 128-key chunks of one bin
    (2_500_000, None),                    # millions of keys over hundreds of bins
    (LONG_SEG + 1, 777),
    (1, 3), (2, None), (40_000, None),
]


def _batch(rng, ids):
    parts = []
    for (n, one), id_ in zip(LAYOUT, ids):
        ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = id_
        ev["flow_key"] = rng.integers(1, 1 << 62, n, dtype=np.uint64)
        ev["value"] = one if one is not None else np.minimum(np.exp(rng.normal(np.log(2000.0), 1.5, n)), 9.0e8).astype(np.uint32)
        ev["type"] = ge.EV_RESP
        ev["tsec"] = 1
        parts.append(ev)
    ev = np.concatenate(parts)
    return ev[rng.permutation(len(ev))]


@pytest.mark.parametrize("rows,bin_max", [(0, None), (2048, None), (2048, 1)], ids=["hot-off", "hot-on", "hot-on-all-refused"])
def test_every_segment_length_is_bit_exact(monkeypatch, rows, bin_max):
    monkeypatch.setenv("GYSK_HOT_ROWS", str(rows))
    if bin_max is not None:
        monkeypatch.setenv("GYSK_HOT_BIN_MAX", str(bin_max))
    ends = np.cumsum([n for n, _ in LAYOUT])
    assert ends[0] == CHUNK and ends[1] == TILE and ends[6] == 2 * TILE and ends[7] == 4 * TILE and ends[9] % CHUNK == 0
    rng = np.random.default_rng(2024)
    ids = synth.service_ids(len(LAYOUT) + 7)[7:]
    eng, orc = make_pair(max_svcs=256, max_tasks=16, max_batch=1 << 22, cms_log2_width=12)
    for i in range(len(ids)):                         # one call per id: slot order = layout order
        eng.register_ids(ids[i:i + 1])
        orc.register_ids(ids[i:i + 1])
    total = int(ends[-1])
    for b in range(3):
        ev = _batch(rng, ids)
        feed_both(eng, orc, ev, 1 << 22)
        if b == 0:
            assert eng.last_batch_keys() == total     # no hot row yet: every sample is a key, the segments lie as laid out
        for id_ in ids.tolist():
            assert_hist_equal(eng, orc, id_, ge.HIST_RESP_CUR)
            (means, weights, mn, mx), td = eng.export_tdigest(id_), orc.export_tdigest(id_)
            om, ow = td.centroids()
            assert np.array_equal(weights, ow) and np.array_equal(means, om), (b, hex(id_))
            assert mn == td.minv and mx == td.maxv and int(weights.sum()) == td.total, (b, hex(id_))
        if b == 1:
            eng.flush(5); orc.flush(5)
    if rows and bin_max is None:
        assert eng.hot_rows_in_use() > 0
    s, o = eng.stats(), orc.counters()
    assert s["events_resp"] == o["resp"] and s["events_dropped"] == o["dropped"]
