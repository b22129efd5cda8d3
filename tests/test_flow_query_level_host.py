"""The rolling 300-s flow query level (GYSK_FLAG_FLOW_QUERY_LEVEL) on the CPU: the per-window flow query tables restated from the samples
(tests/flow_queries.py) and rolled by the ring of tests/flow_level.py equal the sum of those tables under the epoch rule after every
flush of every scripted sequence, and the level's cells are the table one window fed all the held samples would hold, a wrapping msec
half included. The header and the Python binding are pinned."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import flow_queries as fq
from tests.flow_level import SEQUENCES, FlowLevelRing, held_windows, level_of_history

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEPTH, LOG2W = 4, 10


def _samples(rng, n, keys, ms_hi=20_000):
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["type"], ev["host_idx"] = 1 + rng.integers(0, 40, n).astype(np.uint64), ge.EV_RESP, rng.integers(0, 8, n)
    ev["flow_key"] = keys[rng.integers(0, len(keys), n)]
    ev["value"] = rng.integers(0, ms_hi, n).astype(np.uint32) * np.uint32(1000) + rng.integers(0, 1000, n).astype(np.uint32)
    return ev


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_ring_of_query_tables_equals_the_epoch_rule(name):
    tsecs = SEQUENCES[name]
    rng = np.random.default_rng(200 + len(tsecs))
    keys = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
    ring = FlowLevelRing(DEPTH << LOG2W)
    tables, windows = [], []
    for i, t in enumerate(tsecs):
        s = _samples(rng, int(rng.integers(100, 3000)), keys)
        tables.append(fq.add_samples(np.zeros(DEPTH << LOG2W, dtype=np.uint64), s, DEPTH, LOG2W))
        windows.append(s)
        level = ring.flush(t, tables[-1])
        assert np.array_equal(level, level_of_history(tsecs[: i + 1], tables)), (name, i, t)
        held = np.concatenate([windows[j] for j in held_windows(tsecs[: i + 1])])
        # linear: the level is the table of one window fed every held sample
        assert level.tobytes() == fq.add_samples(np.zeros_like(level), held, DEPTH, LOG2W).tobytes(), (name, i, t)
        q, m = fq.point_query(level, keys[:40], DEPTH, LOG2W)
        for (eq, em), a, b in zip(fq.exact(held, keys[:40]), q.tolist(), m.tolist()):
            assert a >= eq and b >= em, (name, i)
        assert fq.row_sums(level, DEPTH, LOG2W) == [len(held) & fq.U32] * DEPTH


def test_msec_half_wraps_like_the_table():
    """4 400 samples of 1 000 000 ms on one key over three held windows: the msec half passes 2^32 and carries into nothing (the key's
    cell is {4400 | (4.4e9 mod 2^32) << 32} mod 2^64)"""
    key = np.array([0xABCDEF], dtype=np.uint64)
    ring = FlowLevelRing(DEPTH << LOG2W)
    tables = []
    for t in (5, 10, 15):
        s = np.zeros(1467, dtype=ge.EVENT_DTYPE)
        s["flow_key"], s["type"], s["value"], s["svc_id"] = key[0], ge.EV_RESP, 1_000_000_000, 7
        tables.append(fq.add_samples(np.zeros(DEPTH << LOG2W, dtype=np.uint64), s, DEPTH, LOG2W))
        ring.flush(t, tables[-1])
    n = 3 * 1467
    assert n * 1_000_000 > fq.U32
    q, m = fq.point_query(ring.level, key, DEPTH, LOG2W)
    assert int(q[0]) == n and int(m[0]) == (n * 1_000_000) & fq.U32
    want = (n + ((n * 1_000_000) << 32)) & ((1 << 64) - 1)
    cols = fq.columns(key, DEPTH, LOG2W)[:, 0]
    assert [int(ring.level.reshape(DEPTH, -1)[r, c]) for r, c in enumerate(cols)] == [want] * DEPTH


def test_header_and_binding():
    h = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert re.search(r"#define GYSK_FLAG_FLOW_QUERY_LEVEL\s+0x100u", h)
    assert ge.FLAG_FLOW_QUERY_LEVEL == 0x100
    for decl in ("int		gysk_query_flow_queries_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_qry_est *out);",
                 "int		gysk_export_cms_queries_5min(gysk_engine *e, uint64_t *cells",
                 "int		gysk_query_flow_queries_global_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_qry_est *out);"):
        assert decl in h, decl
    section = h.split("the rolling 300-s flow query level (GYSK_FLAG_FLOW_QUERY_LEVEL)")[1].split("int		gysk_query_flow_queries_5min")[0]
    assert "All three are GYSK_ERR_NOTSUP without the flag." in section
    flag = h.split("#define GYSK_FLAG_FLOW_QUERY_LEVEL")[1].split("*/")[0]
    assert "Needs" in flag and "GYSK_FLAG_FLOW_QUERIES" in flag and "gysk_create refuses it" in flag


def test_library_exports_the_calls():
    lib = os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    L = C.CDLL(lib)
    for name in ("gysk_query_flow_queries_5min", "gysk_export_cms_queries_5min", "gysk_query_flow_queries_global_5min"):
        assert hasattr(L, name), name
    assert L.gysk_export_cms_queries_5min(None, None) == -22
    # the configuration check comes before any device is looked for
    with pytest.raises(ge.GyskError) as ex:
        ge.Engine(flow_query_level=True)
    assert ex.value.code == -22 and "needs GYSK_FLAG_FLOW_QUERIES" in str(ex.value)
