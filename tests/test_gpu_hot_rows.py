"""Hot services take their response samples as direct updates of a dense, L2-resident row of value bins instead of sort keys
(DESIGN.md §4). That is routing only: every number must be the one the oracle (and the key path) produces. The parity tests are
re-run with the switch-over forced early (8 samples in a batch), with almost no rows (the overflow stays on the key path), and
with the path off; and with the fullest-bin limit (GYSK_HOT_BIN_MAX) low enough that the head services are refused a row."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po
from tests import test_gpu_parity as tp
from tests.util import assert_hist_equal, feed_both, make_pair

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows,hmin", [(2048, 8), (5, 8), (0, 4096)])
def test_hot_rows_do_not_change_any_number(monkeypatch, rows, hmin):
    monkeypatch.setenv("GYSK_HOT_ROWS", str(rows))
    monkeypatch.setenv("GYSK_HOT_MIN", str(hmin))
    tp.test_mixed_stream_bit_exact(3000, 300_000, 1 << 15)
    tp.test_tdigest_many_services_skewed()
    tp.test_idle_service_eviction_and_slot_reuse()
    tp.test_window_membership_is_by_arrival()
    tp.test_full_value_range_keys()


def _bin_counts(resp):
    """(service ids, response samples, samples in the fullest value bin) of one batch; a bin is td_code(usec) plus the RESP_TIME
    bucket of usec / 1000, the oracle's td_bin_index"""
    L = po.lib()
    code = np.fromiter((L.gyo_td_code(int(v)) for v in resp["value"]), dtype=np.int64, count=len(resp))
    ms, inv = np.unique(resp["value"] // 1000, return_inverse=True)
    bins = code + np.array([L.gyo_bucket(0, int(m)) for m in ms], dtype=np.int64)[inv.reshape(-1)]
    ids, svc = np.unique(resp["svc_id"], return_inverse=True)
    svc = svc.reshape(-1).astype(np.int64)
    keys, cnt = np.unique(svc * 4096 + bins, return_counts=True)          # < 4096 bins
    binmax = np.zeros(len(ids), dtype=np.int64)
    np.maximum.at(binmax, keys // 4096, cnt)
    return ids, np.bincount(svc, minlength=len(ids)), binmax


def _promoted(resp, hmin, bin_max):
    """the services a batch hands a hot row to (bins_merge_kernel): hmin or more samples, none of its bins with more than bin_max"""
    if not len(resp):
        return set()
    ids, n, binmax = _bin_counts(resp)
    return set(ids[(n >= hmin) & (binmax <= bin_max)].tolist())


HOT_BIN_MAX_DEFAULT = 131072


@pytest.mark.parametrize("rows,hmin,want,bin_max", [
    pytest.param(2048, 8, None, None, id="2048-8-None"), pytest.param(5, 8, 5, None, id="5-8-5"), pytest.param(0, 8, 0, None, id="0-8-0"),
    pytest.param(2048, 1 << 26, 0, None, id="2048-67108864-0"),
    # the fullest bins of the three busiest services hold 22 to 78 samples per batch: with 16 they stay on the key path
    pytest.param(2048, 8, "exact", 16, id="2048-8-exact-binmax16"),
    # the limit set to a head service's fullest bin, with another head service one sample above it
    pytest.param(2048, 256, "exact", "edge", id="2048-256-exact-binmax-edge"),
])
def test_hot_rows_are_taken_and_every_batch_is_bit_exact(monkeypatch, rows, hmin, want, bin_max):
    """eight batches; after each one histograms and centroids of hot and cold services equal the oracle's. With GYSK_HOT_BIN_MAX
    set ("exact"), the rows in use after every batch are the number of services the fullest-bin rule promoted so far."""
    monkeypatch.setenv("GYSK_HOT_ROWS", str(rows))
    monkeypatch.setenv("GYSK_HOT_MIN", str(hmin))
    rng = np.random.default_rng(77)
    nsvc = 400
    batches = []
    for b in range(8):
        ev = synth.gen_mixed(rng, 60_000, nsvc, ntask=8, nhosts=8, nclients=2000, zipf_s=1.05)
        if b == 5:
            ev = ev[ev["type"] != ge.EV_RESP]                 # a batch without a single response sample: hot rows stay empty
        batches.append(ev)
    if bin_max == "edge":
        ids, n, binmax = _bin_counts(batches[0][batches[0]["type"] == ge.EV_RESP])
        head = set(binmax[n >= hmin].tolist())
        edges = [v for v in head if v + 1 in head]
        assert edges, sorted(head)
        bin_max = max(edges)                                  # promoted at bin_max, not at bin_max + 1
    if bin_max is not None:
        monkeypatch.setenv("GYSK_HOT_BIN_MAX", str(bin_max))
    eng, orc = make_pair(max_svcs=512, max_tasks=64, max_batch=1 << 16, cms_log2_width=12)
    ids_seen = set()
    hot, hot_default = set(), set()
    for b, ev in enumerate(batches):
        feed_both(eng, orc, ev, 1 << 16)
        if want == "exact":
            resp = ev[ev["type"] == ge.EV_RESP]
            hot |= _promoted(resp, hmin, bin_max)
            hot_default |= _promoted(resp, hmin, HOT_BIN_MAX_DEFAULT)
            assert eng.hot_rows_in_use() == min(len(hot), rows), (b, len(hot))
        resp = ev[ev["type"] == ge.EV_RESP]
        ids, counts = np.unique(resp["svc_id"], return_counts=True)
        ids_seen |= set(int(i) for i in ids)
        order = np.argsort(-counts) if len(ids) else []
        pick = [int(ids[j]) for j in list(order[:12]) + list(order[-12:])] + sorted(ids_seen)[:6]
        for id_ in pick:
            assert_hist_equal(eng, orc, id_, ge.HIST_RESP_CUR)
            (means, weights, mn, mx), td = eng.export_tdigest(id_), orc.export_tdigest(id_)
            om, ow = td.centroids()
            assert np.array_equal(weights, ow) and np.array_equal(means, om) and mn == td.minv and mx == td.maxv, (b, hex(id_))
        if b == 3:
            eng.flush(5); orc.flush(5)
    got = eng.hot_rows_in_use()
    if want is None:
        assert 20 <= got <= nsvc, got                        # the head of the Zipf distribution turned hot
    elif want == "exact":
        assert got < min(len(hot_default), rows), (got, len(hot_default))     # the rule kept services on the key path
    else:
        assert got == want, got
    s, o = eng.stats(), orc.counters()
    assert s["events_resp"] == o["resp"] and s["events_dropped"] == o["dropped"]
