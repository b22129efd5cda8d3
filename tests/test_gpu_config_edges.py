"""The engine at the edges of every sketch setting. The kernels take the count-min depth and width, the HLL precision p and the
t-digest delta as runtime values (the row loops of both drain passes and of query_flows_kernel, hll_idx_rank2 with ranks up to 61 at
p = 4, fold_hll_kernel's 1 << (p - 2) words per logical service, the merge arena, the HLL alpha of p = 4, 5, 6, the delta + 1 entry
qtab); every other GPU test runs depth 4, p 12 and delta 200. Here each setting is compared with the oracle bit for bit and then
merged at world 3; gysk_create's bounds are pinned, and bins_merge_kernel is driven across its shared-memory / L2 switch."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po
from tests.test_gpu_merge_exact import NSVC as MERGE_NSVC
from tests.test_gpu_merge_exact import Shards, logical_map, window_events
from tests.util import M32, assert_hist_equal, feed_both, k1_cell_weights, make_pair, td_bin_usec

pytestmark = pytest.mark.gpu

SETTINGS = [
    pytest.param(dict(cms_depth=1, cms_log2_width=4, hll_p=4, td_compression=10), id="d1-w4-p4-td10"),
    pytest.param(dict(cms_depth=3, cms_log2_width=13, hll_p=5, td_compression=100), id="d3-w13-p5-td100"),
    pytest.param(dict(cms_depth=4, cms_log2_width=12, hll_p=6, td_compression=200), id="d4-w12-p6-td200"),
    pytest.param(dict(cms_depth=8, cms_log2_width=22, hll_p=16, td_compression=256), id="d8-w22-p16-td256"),
]
COUNTERS = (("events_in", "in"), ("events_dropped", "dropped"), ("events_resp", "resp"), ("events_tcp", "tcp"),
            ("events_task", "task"), ("nsvcs", "nsvcs"), ("ntasks", "ntasks"))
TASK_HISTS = (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY)
GRID_BATCH = 300_000                    # more events than one ingest grid (~200 K) takes in one pass


def _check(eng, orc, svcs, tasks, keys, p, flushed):
    """counters, both count-min tables whole, every service's and task's state, and the point queries"""
    s, o = eng.stats(), orc.counters()
    for k, ko in COUNTERS:
        assert s[k] == o[ko], (k, s[k], o[ko])
    assert np.array_equal(eng.export_cms(), orc.cms())
    assert np.array_equal(eng.export_cms(last_window=True), orc.cms(True))
    L = po.lib()
    summ = eng.query_svcs(svcs)
    for id_, q in zip(svcs.tolist(), summ):
        for which in ((ge.HIST_RESP_CUR, ge.HIST_RESP_LAST, ge.HIST_RESP_ALL) if flushed else (ge.HIST_RESP_CUR,)):
            assert_hist_equal(eng, orc, id_, which)
        regs, oregs = eng.export_hll(id_), orc.export_hll(id_)
        assert len(regs) == 1 << p and np.array_equal(regs, oregs), hex(id_)
        assert q["distinct_clients"] == L.gyo_hll_estimate(po._p(oregs), p), hex(id_)
        for lw in (False, True):
            g, w = eng.export_conn_bitmap(id_, lw), orc.export_conn_bitmap(id_, lw)
            assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]), (hex(id_), lw)
        (means, weights, mn, mx), td = eng.export_tdigest(id_), orc.export_tdigest(id_)
        om, ow = td.centroids()
        assert np.array_equal(weights, ow) and means.tobytes() == om.tobytes(), hex(id_)
        if len(ow):
            assert (mn, mx) == (td.minv, td.maxv), hex(id_)
    for id_ in tasks.tolist():
        for which in TASK_HISTS:
            assert_hist_equal(eng, orc, id_, which)
    depth, log2w = eng.cfg.cms_depth, eng.cfg.cms_log2_width
    for lw in (False, True):
        tbl = orc.cms(lw).reshape(depth, -1)
        for k, e_ in zip(keys.tolist(), eng.query_flows(keys, last_window=lw)):
            cells = [int(tbl[r, L.gyo_cms_index(k, r, log2w)]) for r in range(depth)]
            assert (e_["count"], e_["kbytes"]) == (min(c & M32 for c in cells), min(c >> 32 for c in cells)), (hex(k), lw)


@pytest.mark.parametrize("setting", SETTINGS)
def test_setting_equals_the_oracle_and_merges(setting):
    import torch
    rng = np.random.default_rng(setting["hll_p"] * 1000 + setting["td_compression"])
    nsvc = 300
    eng, orc = make_pair(max_svcs=1024, max_tasks=256, max_batch=1 << 19, **setting)
    svcs, tasks = set(), set()
    for w, (n, batch) in enumerate(((GRID_BATCH, GRID_BATCH), (100_000, 50_000))):
        ev = synth.gen_mixed(rng, n, nsvc, ntask=64, nhosts=64, nclients=50_000)
        feed_both(eng, orc, ev, batch)
        svcs |= set(np.unique(ev["svc_id"][ev["type"] != ge.EV_TASK]).tolist())
        tasks |= set(np.unique(ev["svc_id"][ev["type"] == ge.EV_TASK]).tolist())
        sv, tk = np.array(sorted(svcs), dtype=np.uint64), np.array(sorted(tasks), dtype=np.uint64)
        keys = np.unique(ev["flow_key"][(ev["type"] >= ge.EV_CONNECT) & (ev["type"] <= ge.EV_CLOSE_SER)])[:200]
        _check(eng, orc, sv, tk, keys, setting["hll_p"], flushed=w > 0)
        eng.flush(5 * (w + 1)); orc.flush(5 * (w + 1))
        _check(eng, orc, sv, tk, keys, setting["hll_p"], flushed=True)
    assert eng.stats()["events_in"] == GRID_BATCH + 100_000
    eng.close(); orc.close()

    # the merge step of test_gpu_merge_exact at world 3 with the same setting
    sh = Shards(3, max_svcs=1024, max_tasks=128, max_batch=1 << 16, **setting)
    ids = synth.service_ids(MERGE_NSVC)
    conn_ids = synth.splitmix64(np.arange(1, 4, dtype=np.uint64) + np.uint64(1 << 51))
    ghost_ids = synth.splitmix64(np.arange(1, 6, dtype=np.uint64) + np.uint64(1 << 52))
    sh.set_map(*logical_map(rng, ids, conn_ids, ghost_ids))
    for w in range(2):
        ev = window_events(rng, w, 120_000, ids, conn_ids)
        sh.feed(ev, 1 << 16)
        sh.flush(5 * (w + 1))
        keys = np.unique(ev["flow_key"][(ev["type"] >= ge.EV_CONNECT) & (ev["type"] <= ge.EV_CLOSE_SER)])[:200]
        want = sh.check_merge(torch, keys)
        assert want[9000]["td_count"] > 10_000 and want[9000]["distinct_clients"] > 0


BOUNDS = (("cms_depth", 1, 8), ("cms_log2_width", 4, 28), ("hll_p", 4, 16), ("td_compression", 10, 256))


def test_configuration_bounds():
    """gysk_create takes every bound and refuses each neighbour with GYSK_ERR_INVAL (the engines stay small: width 2^28 is tried
    at depth 1, already 2 x 2 GB of count-min; the max_svcs bound is left alone, 2^24 services need 64 GB of HLL registers)"""
    small = dict(max_svcs=16, max_tasks=16, max_batch=1024, cms_depth=1, cms_log2_width=4, hll_p=4, td_compression=10)
    for field, lo, hi in BOUNDS:
        for v, ok in ((lo - 1, False), (lo, True), (hi, True), (hi + 1, False)):
            kw = dict(small, **{field: v})
            if ok:
                e = ge.Engine(**kw)
                assert getattr(e.cfg, field) == v
                e.close()
            else:
                with pytest.raises(ge.GyskError) as ei:
                    ge.Engine(**kw)
                assert ei.value.code == -22, (field, v, ei.value.code)


@pytest.mark.parametrize("max_svcs", [1, 3, 8])
def test_batch_that_fills_the_service_table_keeps_every_event(max_svcs):
    """max_svcs new services in one batch, their events interleaved: the table ends exactly full and no event is dropped — an
    event that found its service's entry still empty must not be refused once the other events of that service have taken the last
    slot. Then every service goes idle and is evicted but one, and as many new ids arrive: they fill the recycled slots, again
    without a drop. Counters and every service's state equal the oracle's."""
    rng = np.random.default_rng(max_svcs)
    eng, orc = make_pair(max_svcs=max_svcs, max_tasks=8, max_batch=1 << 14, cms_log2_width=10, idle_evict_secs=300)
    first = [int(x) for x in synth.splitmix64(np.arange(1, max_svcs + 1, dtype=np.uint64) + np.uint64(1 << 54))]
    second = [int(x) for x in synth.splitmix64(np.arange(1, max_svcs + 1, dtype=np.uint64) + np.uint64(1 << 55))]

    def window(t, ids, n=1200):
        ev = np.zeros(n * len(ids), dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = np.repeat(np.array(ids, dtype=np.uint64), n)
        ev["type"] = np.where(rng.random(len(ev)) < 0.8, ge.EV_RESP, ge.EV_ACCEPT)
        ev["value"] = np.minimum(np.exp(rng.normal(np.log(3000.0), 1.2, len(ev))), 9.0e8).astype(np.uint32)
        ev["flow_key"] = rng.integers(1, 1 << 62, len(ev), dtype=np.uint64)
        ev["tsec"] = t
        feed_both(eng, orc, ev[rng.permutation(len(ev))], 1 << 14)
        s, o = eng.stats(), orc.counters()
        for k, ko in COUNTERS:
            assert s[k] == o[ko], (t, k, s[k], o[ko])
        assert s["events_dropped"] == 0 and s["nsvcs"] == max_svcs, (t, s)
        assert np.array_equal(eng.export_cms(), orc.cms()), t
        for id_ in ids:
            assert_hist_equal(eng, orc, id_, ge.HIST_RESP_CUR)
        eng.flush(t); orc.flush(t)
        return set(int(i) for i in eng.evicted_ids())

    window(5, first)
    window(10, first)
    keep = first[:1]
    for t in (400, 606):
        gone = window(t, keep)
    assert gone == set(first[1:])
    window(620, keep + second[: max_svcs - 1])                      # the recycled slots fill up in one batch
    assert eng.stats()["svcs_evicted"] == max_svcs - 1


def _resp(svc, usec, rng):
    ev = np.zeros(len(usec), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = svc
    ev["type"] = ge.EV_RESP
    ev["value"] = usec
    ev["flow_key"] = rng.integers(1, 1 << 62, len(ev), dtype=np.uint64)
    ev["tsec"] = 1
    return ev


def _td_equal(eng, orc, id_, ctx):
    (means, weights, mn, mx), td = eng.export_tdigest(id_), orc.export_tdigest(id_)
    om, ow = td.centroids()
    assert np.array_equal(weights, ow) and means.tobytes() == om.tobytes() and (mn, mx) == (td.minv, td.maxv), ctx
    return len(ow)


def test_td_lists_across_the_shared_memory_limit():
    """bins_merge_kernel merges a service's old centroids with its batch items in shared memory while head.n + nitems <= 384
    (TD_SMEM_N) and in the L2 scratch (TdWorkBig, 1120 entries) above that. One service brings exactly 384 - head.n distinct value
    bins, another 385 - head.n; at delta = 256 a third brings every bin a response time can reach (841 of the NBINS = 848) on top of
    exactly 256 old centroids, the longest list a batch can form. Centroids equal the oracle's after every batch."""
    rng = np.random.default_rng(384)
    bins, usec = td_bin_usec()
    assert len(bins) >= 840 and len(bins) + 256 <= 1120
    ids = [int(x) for x in synth.service_ids(3)]

    eng, orc = make_pair(max_svcs=16, max_tasks=8, max_batch=1 << 18, cms_log2_width=8, td_compression=200)
    first = [np.minimum(np.exp(rng.normal(np.log(2000.0), 1.5, n)), 9.0e8).astype(np.uint32) for n in (3000, 2500)]
    feed_both(eng, orc, np.concatenate([_resp(ids[0], first[0], rng), _resp(ids[1], first[1], rng)]), 1 << 18)
    n0, n1 = (_td_equal(eng, orc, ids[k], ("first", k)) for k in range(2))
    assert 0 < n0 <= 200 and 0 < n1 <= 200
    pick = [np.sort(rng.choice(len(bins), 384 - n0, replace=False)), np.sort(rng.choice(len(bins), 385 - n1, replace=False))]
    ev = np.concatenate([_resp(ids[0], usec[pick[0]], rng), _resp(ids[1], usec[pick[1]], rng)])
    feed_both(eng, orc, ev[rng.permutation(len(ev))], 1 << 18)
    for k in range(2):
        _td_equal(eng, orc, ids[k], ("boundary", k))
    eng.close(); orc.close()

    eng, orc = make_pair(max_svcs=16, max_tasks=8, max_batch=1 << 18, cms_log2_width=8, td_compression=256)
    w = k1_cell_weights(256, 200_000)                   # one K_1 cell per bin: a first batch that leaves exactly 256 centroids
    sel = np.linspace(0, len(bins) - 1, 256).round().astype(np.int64)
    assert len(np.unique(sel)) == 256
    feed_both(eng, orc, _resp(ids[2], np.repeat(usec[sel], w.astype(np.int64)), rng), 1 << 18)
    assert _td_equal(eng, orc, ids[2], "256 old") == 256
    for b in range(2):                                  # every reachable bin on top of 256 (then of whatever is left) centroids
        feed_both(eng, orc, _resp(ids[2], np.repeat(usec, 1 + b), rng), 1 << 18)
        _td_equal(eng, orc, ids[2], ("all bins", b))
