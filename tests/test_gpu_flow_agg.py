"""The batch flow table: the TCP drain pass sums each flow's count-min increments in an entry keyed by its two hashes, and the TASK
drain pass adds every entry to the flow's cells once and empties the table. After every batch and every flush the whole count-min
table (the open window and the last closed one) must be byte-equal to the oracle's, and the flow table must be empty again: with about
20 records per flow, with more distinct flows in one batch than the table holds (so that records take the direct path), with several
batches in a window and flushes between them, at the sketch-setting edges, with the 300-s level on, with ACTIVE_CONN_STATS records in
the same batches, and through the event32, TCP24 and NOTIFY_TCP_CONN inputs."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge, synth
from oracle import pyoracle as po
from tests.flow_level import flow_events
from tests.test_gpu_flow_level import _route_window

pytestmark = pytest.mark.gpu

FLOW_ENT_MAX = 1 << 21


class Run:
    """one engine and the oracle, fed the same events; check() after every batch and flush"""

    def __init__(self, flow_level=False, **kw):
        self.eng = ge.Engine(flow_level=flow_level, **kw)
        self.orc = po.OracleEngine(**{k: kw[k] for k in ("max_svcs", "max_tasks", "cms_depth", "cms_log2_width") if k in kw})

    def batch(self, ev, ingest=None, what=None):
        (ingest or (lambda e: e.ingest_events(ev)))(self.eng)
        self.eng.sync()
        self.orc.ingest(ev)
        self.check(what)

    def flush(self, t, what=None):
        self.eng.flush(t)
        self.orc.flush(t)
        self.check(what)

    def check(self, what):
        assert self.eng.flow_table_used() == 0, what
        assert self.eng.export_cms().tobytes() == self.orc.cms().tobytes(), what
        assert self.eng.export_cms(last_window=True).tobytes() == self.orc.cms(last_window=True).tobytes(), what


@pytest.mark.parametrize("depth,log2w,flow_level", [(4, 20, False), (4, 20, True), (1, 4, False), (8, 4, False), (1, 22, False),
                                                    (8, 22, True)])
def test_about_20_records_per_flow(depth, log2w, flow_level):
    """mixed batches (RESP, TCP, TASK, ACTIVE_CONN_STATS) whose connection records come about 20 to a flow: three batches in one window,
    a flush, two more batches, a flush with nothing after it, one more batch"""
    rng = np.random.default_rng(depth * 1000 + log2w + flow_level)
    run = Run(flow_level=flow_level, max_svcs=1024, max_tasks=256, max_batch=1 << 17, cms_depth=depth, cms_log2_width=log2w)
    keys = rng.integers(1, 1 << 63, 600, dtype=np.uint64)
    steps = ["b", "b", "b", 5, "b", "b", 10, 15, "b"]
    for i, s in enumerate(steps):
        if s == "b":
            n = int(rng.integers(40_000, 120_000))
            ev = synth.gen_mixed(rng, n, 300, ntask=64, nhosts=16, nclients=n // 100)      # 20 % TCP: about 20 records per client
            act = flow_events(rng, 2000, keys)
            ev = np.concatenate([ev, act])[rng.permutation(n + len(act))]
            run.batch(ev, what=(depth, log2w, i))
        else:
            run.flush(s, what=(depth, log2w, i))
    assert run.eng.stats()["events_tcp"] > 0
    assert run.eng.last_batch_flow_direct() == 0


def test_more_flows_than_the_table():
    """2.5 M connection records of distinct flows in one batch: the table takes at most 2^21 of them, the rest update their cells
    directly; then a batch of a few flows, which the table takes again"""
    rng = np.random.default_rng(7)
    run = Run(max_svcs=1024, max_tasks=64, max_batch=1 << 22, stage_batch=1 << 22, cms_depth=4, cms_log2_width=20)
    n = 2_500_000
    ev = flow_events(rng, n, np.zeros(1, dtype=np.uint64))
    ev["flow_key"] = synth.splitmix64(np.arange(1, n + 1, dtype=np.uint64))                    # a bijection: n distinct flows
    ev["type"][ev["type"] == ge.EV_ACTIVE] = ge.EV_ACCEPT
    nflows = len(np.unique(ev["flow_key"]))
    assert nflows > FLOW_ENT_MAX
    run.batch(ev, what="distinct")
    assert run.eng.last_batch_flow_direct() >= nflows - FLOW_ENT_MAX
    run.batch(flow_events(rng, 50_000, rng.integers(1, 1 << 63, 2500, dtype=np.uint64)), what="after")
    assert run.eng.last_batch_flow_direct() == 0
    run.flush(5, what="flush")


@pytest.mark.parametrize("route", ["event32", "tcp24", "notify_tcp_conn"])
def test_every_connection_input(route):
    """each input of connection records, about 20 records per flow, two batches per window and a flush between windows"""
    rng = np.random.default_rng(sum(map(ord, route)) + 1)
    keys = rng.integers(1, 1 << 62, 40, dtype=np.uint64)
    run = Run(max_svcs=1024, max_tasks=64, max_batch=1 << 14, cms_depth=4, cms_log2_width=12)
    for w, t in enumerate([5, 10, 15, 20]):
        for b in range(2):
            ingest, ev, nkept, _ = _route_window(rng, route, keys, host=3)
            assert nkept > 0
            run.batch(ev, ingest=ingest, what=(route, w, b))
        run.flush(t, what=(route, w))
    assert run.eng.stats()["events_tcp"] > 0
