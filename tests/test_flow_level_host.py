"""The rolling 300-s count-min level (GYSK_FLAG_FLOW_LEVEL) on the CPU: the ring restatement of tests/flow_level.py fed the oracle's
closed-window tables equals the sum of those tables under the epoch rule after every flush of every scripted sequence, and the flushes
it holds are the ones the oracle's own 300-s response level holds."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests.flow_level import SEQUENCES, FlowLevelRing, exact_flows, flow_events, held_windows, level_of_history, point_query

DEPTH, LOG2W = 4, 10
TRACER = 0xF10E


def _tracer_samples(n):
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["type"], ev["value"], ev["host_idx"] = TRACER, ge.EV_RESP, 2000, 1
    return ev


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_ring_equals_the_epoch_rule_and_the_oracles_response_level(name):
    tsecs = SEQUENCES[name]
    rng = np.random.default_rng(len(tsecs))
    keys = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
    orc = po.OracleEngine(max_svcs=256, max_tasks=16, cms_depth=DEPTH, cms_log2_width=LOG2W)
    ring = FlowLevelRing(DEPTH << LOG2W)
    tables, streams, nresp = [], [], []
    for i, t in enumerate(tsecs):
        ev = flow_events(rng, int(rng.integers(200, 2000)), keys)
        n = int(rng.integers(1, 500))                  # the window's response samples of one service: a tag the 300-s level sums
        orc.ingest(np.concatenate([ev, _tracer_samples(n)]))
        orc.flush(t)
        tables.append(orc.cms(last_window=True))
        streams.append(ev); nresp.append(n)
        level = ring.flush(t, tables[-1])
        assert np.array_equal(level, level_of_history(tsecs[: i + 1], tables)), (name, i, t)
        held = held_windows(tsecs[: i + 1])
        assert orc.export_hist(TRACER, ge.HIST_RESP_5MIN)[1] == sum(nresp[j] for j in held), (name, i, t)
        exact = exact_flows(np.concatenate([streams[j] for j in held]), keys[:40])
        for k, est in zip(keys[:40].tolist(), point_query(level, keys[:40], DEPTH, LOG2W)):
            assert est[0] >= exact[k][0] and est[1] >= exact[k][1], (name, i, hex(k))
    assert np.array_equal(orc.cms(last_window=False), np.zeros(DEPTH << LOG2W, dtype=np.uint64))     # the open window is empty


def test_held_windows_by_hand():
    assert held_windows([0]) == [0]
    assert held_windows([5, 10, 305]) == [2]                       # epochs 0, 0, 10: 0 is ten epochs back
    assert held_windows([5, 10, 299]) == [0, 1, 2]                 # epoch 9: 0 .. 9 are live
    assert held_windows([600, 605, 605]) == [0, 1, 2]              # the same tsec twice adds twice
    assert held_windows([900, 930, 620]) == [2]                    # back to epoch 20: slot 0 leaves epoch 30, epoch 31 is ahead
    assert held_windows([900, 930, 960, 620, 930]) == [1, 4]       # epoch 31's slot kept its epoch through the step back
