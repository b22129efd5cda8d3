"""merge step (SURVEY.md §8e) on one GPU: two engines configured as rank 0 / rank 1 of a 2-way host shard; the collectives are
emulated with torch ops on the wrapped device buffers (sum / max / concat), which is exactly what NCCL does element-wise. The
merged logical-service answers must equal (integers: bit-exact) a single engine that ingested the whole stream and the oracle."""
import numpy as np
import pytest

from tests.test_gpu_td_accuracy import rank_bound, rank_error
from tests.util import td_p99_tolerance

from gyeeta_b200 import dist as gd
from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu


def _emulate_collectives(torch, engines):
    dev = torch.device("cuda", 0)
    for e in engines:
        e.merge_prepare()
        e.sync()                     # merge_prepare is stream-ordered; the emulation below runs on torch's stream
    bufs = [e.merge_buffers() for e in engines]
    for k in range(len(bufs[0])):
        ts = [gd.wrap(torch, b[k][1], b[k][2], b[k][3], dev) for b in bufs]
        red = ts[0].clone()
        for t in ts[1:]:
            red = red + t if bufs[0][k][3] == gd.RED_SUM_U64 else torch.maximum(red, t)
        for t in ts:
            t.copy_(red)
    slabs = []
    for e in engines:
        p, nb = e.merge_tdigest_slab()
        slabs.append(torch.as_tensor(gd._DevBuf(p, nb, "|u1", 1), device=dev))
    gathered = torch.cat(slabs).contiguous()
    torch.cuda.synchronize()
    for e in engines:
        e.merge_finish(gathered.data_ptr(), len(engines))


def test_two_shards_merge_to_global_answers_and_exact_quantiles():
    import torch
    rng = np.random.default_rng(17)
    nsvc, nhosts = 320, 64
    ev = synth.gen_mixed(rng, 150_000, nsvc, ntask=16, nhosts=nhosts, nclients=4000)
    resp = ev[(ev["type"] == ge.EV_RESP) & (ev["value"] < 1_000_001_000)]
    resp_ids, resp_vals = resp["svc_id"], resp["value"].astype(np.float64)
    kw = dict(max_svcs=1024, max_tasks=64, max_batch=1 << 16, cms_log2_width=14)
    shards = [ge.Engine(rank=r, world=2, **kw) for r in range(2)]
    one = ge.Engine(**kw)
    orc = po.OracleEngine(max_svcs=1024, max_tasks=64, cms_log2_width=14)
    for off in range(0, len(ev), 1 << 16):
        chunk = ev[off: off + (1 << 16)]
        for e in shards + [one]:
            e.ingest_events(chunk); e.sync()
        orc.ingest(chunk)
    for e in shards + [one]:
        e.flush(5)
    orc.flush(5)

    ids = synth.service_ids(nsvc)
    logical = ids >> np.uint64(4) << np.uint64(4) | np.uint64(1)      # 16 hosts' instances -> one logical service key
    logical = (np.arange(nsvc, dtype=np.uint64) // np.uint64(16)) + np.uint64(1000)
    for e in shards + [one]:
        e.set_logical_map(ids, logical)
    _emulate_collectives(torch, shards)
    _emulate_collectives(torch, [one])

    lids = np.unique(logical)
    a = shards[0].query_logical(lids)
    b = shards[1].query_logical(lids)
    c = one.query_logical(lids)
    int_fields = ["found", "nqrys_5s", "total_resp_5sec", "p95_5s_resp_ms", "p99_5s_resp_ms", "p25_5s_resp_ms", "p95_all_resp_ms",
                  "p99_all_resp_ms", "nqrys_all", "max_resp_ms", "nconns_5s", "kbytes_5s", "nconns_all", "kbytes_all", "td_count"]
    nonzero = 0
    for x, y, z, lid in zip(a, b, c, lids):
        for f in int_fields:
            assert x[f] == y[f] == z[f], (int(lid), f, x[f], y[f], z[f])
        assert x["distinct_clients"] == y["distinct_clients"] == z["distinct_clients"]       # same registers -> same double
        # oracle: sum the member services' last-window histograms
        members = ids[logical == lid]
        tot = sum(orc.export_hist(int(m), 1)[1] for m in members if orc.export_hist(int(m), 1) is not None)
        assert x["nqrys_5s"] == tot
        regs = np.zeros(4096, dtype=np.uint8)
        for m in members:
            r = orc.export_hll(int(m))
            if r is not None:
                regs = np.maximum(regs, r)
        assert x["distinct_clients"] == po.lib().gyo_hll_estimate(po._p(regs), 12)
        # t-digests: rank-ascending merge of two shard digests vs one engine folding 16 members: same samples, different
        # clustering => epsilon parity on the quantiles, exact parity on the counts. Both answers are held to the rank bound of the
        # members' exact samples; the 1 % value parity from 5 000 samples on (at ~2 300 samples neighbouring samples near p95 lie
        # ~1 % apart in value, so two clusterings one sample apart differ by that much)
        if x["td_count"] >= 2000:
            sv = np.sort(resp_vals[np.isin(resp_ids, members)])
            assert len(sv) == x["td_count"]
            for f, q in (("td_p50_us", 0.5), ("td_p95_us", 0.95), ("td_p99_us", 0.99)):
                for g in (x[f], z[f]):
                    assert rank_error(sv, g, q) <= rank_bound(q, len(sv), 200), (int(lid), f, g)
                if f != "td_p99_us" and x["td_count"] >= 5000:
                    assert abs(x[f] - z[f]) / z[f] < 0.01, (f, x[f], z[f])
            assert abs(x["td_p99_us"] - z["td_p99_us"]) / z["td_p99_us"] < max(0.03, 2 * td_p99_tolerance(x["td_count"]))   # two clusterings of a few thousand samples
            assert x["td_p50_us"] == y["td_p50_us"]                                          # both ranks computed the same merge
            nonzero += 1
    assert nonzero >= 3
    # global count-min = sum of the shard tables = the single engine's table
    keys = np.unique(ev["flow_key"][(ev["type"] >= 1) & (ev["type"] <= 4)])[:1000]
    ga = shards[0].query_flows_global(keys, last_window=True)
    gc = one.query_flows(keys, last_window=True)
    assert np.array_equal(ga["count"], gc["count"]) and np.array_equal(ga["kbytes"], gc["kbytes"])
    assert shards[0].query_logical([999999])[0]["found"] == 0


def test_logical_map_set_before_the_services_register():
    """gysk_set_logical_map keeps every {glob_id, logical} pair and looks the slots up at every merge: a map handed over before any
    event arrived (or naming services that register later) gives the same merged answers as one set afterwards"""
    import torch
    rng = np.random.default_rng(23)
    nsvc = 200
    ids = synth.service_ids(nsvc)
    logical = (np.arange(nsvc, dtype=np.uint64) // np.uint64(8)) + np.uint64(500)
    kw = dict(max_svcs=512, max_tasks=32, max_batch=1 << 15, cms_log2_width=12)
    early, late = ge.Engine(**kw), ge.Engine(**kw)
    early.set_logical_map(ids, logical)                              # nothing is registered yet
    for w in range(2):
        ev = synth.gen_mixed(rng, 40_000, nsvc // 2 if w == 0 else nsvc, ntask=8, nhosts=16, nclients=2000)   # half of the services appear in window 2
        for e in (early, late):
            e.ingest_events(ev); e.sync(); e.flush(5 * (w + 1))
        if w == 0:
            late.set_logical_map(ids, logical)                      # after the first half registered, before the second
        _emulate_collectives(torch, [early]); _emulate_collectives(torch, [late])
        lids = np.unique(logical)
        a, b = early.query_logical(lids), late.query_logical(lids)
        assert repr(a) == repr(b)                                   # (NaN quantiles of empty logical services compare by text)
        assert sum(x["nqrys_5s"] for x in a) == int((ev["type"] == ge.EV_RESP).sum())
