"""The heaviest-flow rule of GYSK_FLAG_FLOW_TOPK on the CPU: the restatement of tests/flow_topk.py on scripted streams keeps its stated
properties (the K-th score never falls within a window, the guarantee, every flow when there are at most K, ties by key, a wrapping half
followed as the estimates wrap, the merge's union bound), and the header, the Python constants and the bindings pin the ABI."""
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import flow_queries as fq
from tests import flow_topk as ft

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, W = 4, 10


def _table(keys, inc, d=D, w=W):
    t = np.zeros(d << w, dtype=np.uint64).reshape(d, 1 << w)
    cols = fq.columns(keys, d, w)
    for r in range(d):
        np.add.at(t[r], cols[r], inc)
    return t.reshape(-1)


def _stream(rng, nbatches, nflows, per_batch, k):
    """scripted batches of (keys, kbytes increments): a Zipf-like weight per flow"""
    flows = rng.choice(1 << 40, nflows, replace=False).astype(np.uint64)
    w = 1.0 / np.arange(1, nflows + 1) ** 1.1
    for _ in range(nbatches):
        pick = flows[rng.choice(nflows, per_batch, p=w / w.sum())]
        yield pick, rng.integers(0, 64, per_batch).astype(np.uint64) << np.uint64(32)


@pytest.mark.parametrize("k,nflows,w", [(16, 200, 10), (64, 5000, 12), (64, 40, 10), (8, 3000, 4)])
def test_floor_never_falls_and_the_guarantee_holds(k, nflows, w):
    rng = np.random.default_rng(k + nflows + w)
    s = ft.Sets(1, D, w, k)
    table = np.zeros(D << w, dtype=np.uint64)
    seen_k, seen_inc = [], []
    for keys, inc in _stream(rng, 12, nflows, 400, k):
        tab = _table(keys, inc, D, w).reshape(D, -1)
        table = (table.reshape(D, -1) + tab).reshape(-1)
        s.batch(np.unique(keys), table)
        seen_k.append(keys); seen_inc.append(inc)
        assert s.floor == sorted(s.floor)
        fk, ic = np.concatenate(seen_k), np.concatenate(seen_inc)
        allk = np.unique(fk)
        ex = ft.exact_scores(allk, fk, ic, 1)
        members = set(s.open.tolist())
        if len(s.open) < k:
            assert members == set(allk.tolist())
        else:
            thr = int(ft.scores(table, s.open, D, w, 1).min())
            assert all(int(x) in members for x, e in zip(allk.tolist(), ex.tolist()) if e > thr)
    s.flush()
    assert len(s.open) == 0 and len(s.last) > 0


def test_ties_break_by_key_and_zero_scores_are_read_out():
    keys = np.array([50, 7, 30, 9, 11, 3], dtype=np.uint64)
    inc = np.array([5, 5, 5, 0, 9, 0], dtype=np.uint64) << np.uint64(32)
    table = _table(keys, inc, D, 16)
    sel = ft.select(keys, table, D, 16, 1, k=4)
    assert sel.tolist() == [11, 7, 30, 50]
    full = ft.select(keys, table, D, 16, 1, k=6)
    assert full.tolist() == [11, 7, 30, 50, 3, 9]
    rows = ft.read(full, table, D, 16, 1)
    assert rows["flow_key"].tolist() == [11, 7, 30, 50] and rows["kbytes"].tolist() == [9, 5, 5, 5]


def test_a_wrapping_half_is_followed():
    keys = np.array([1, 2, 3], dtype=np.uint64)
    table = _table(keys, np.array([0xFFFFFFF0, 0x10, 0x20], dtype=np.uint64) << np.uint64(32), D, 16)
    assert ft.select(keys, table, D, 16, 1, k=1).tolist() == [1]
    table = (table + _table(keys[:1], np.array([0x20], dtype=np.uint64) << np.uint64(32), D, 16))
    assert ft.select(keys, table, D, 16, 1, k=1).tolist() == [3]          # key 1's kbytes half wrapped to 0x10: a tie with 2 at 0x10 < 0x20


def test_merge_union_bound():
    """a flow whose exact global score exceeds the sum of the ranks' thresholds is in the union"""
    rng = np.random.default_rng(3)
    k, world = 16, 3
    sets, tables, fks, incs = [], [], [], []
    for r in range(world):
        s = ft.Sets(1, D, 12, k)
        table = np.zeros(D << 12, dtype=np.uint64)
        for keys, inc in _stream(np.random.default_rng(r), 4, 300, 500, k):
            table = table + _table(keys, inc, D, 12)
            s.batch(np.unique(keys), table)
            fks.append(keys); incs.append(inc)
        s.flush()
        sets.append(s.last); tables.append(table)
    summed = sum(tables[1:], tables[0].copy())
    thr = sum(int(ft.scores(t, s, D, 12, 1).min()) if len(s) == k else 0 for s, t in zip(sets, tables))
    union = set(np.concatenate(sets).tolist())
    fk, ic = np.concatenate(fks), np.concatenate(incs)
    allk = np.unique(fk)
    ex = ft.exact_scores(allk, fk, ic, 1)
    assert all(int(x) in union for x, e in zip(allk.tolist(), ex.tolist()) if e > thr)
    m = ft.merged(sets, summed, D, 12, 1, k)
    assert len(m) == k and set(m.tolist()) <= union


def test_header_constants_and_bindings():
    with open(os.path.join(ROOT, "include", "gysketch.h")) as f:
        h = f.read()
    assert re.search(r"#define GYSK_FLAG_FLOW_TOPK\s+0x400u", h)
    assert re.search(r"#define GYSK_FLOW_TOPK_CAP\s+4096u", h)
    assert re.search(r"#define GYSK_ABI_VERSION\s+2\b", h)
    for call in ("gysk_topk_flows(gysk_engine *e, int last_window, uint32_t n, gysk_flow_est *out, uint32_t *nout)",
                 "gysk_topk_flow_queries(gysk_engine *e, int last_window, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout)",
                 "gysk_topk_flows_global(gysk_engine *e, uint32_t n, gysk_flow_est *out, uint32_t *nout)",
                 "gysk_topk_flow_queries_global(gysk_engine *e, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout)"):
        assert call in h
    assert ge.FLAG_FLOW_TOPK == 0x400 and ge.FLOW_TOPK_CAP == 4096 == ft.K
    assert ge.FLOW_EST_DTYPE.itemsize == ge.FLOW_QRY_EST_DTYPE.itemsize == 16
    for name in ("topk_flows", "topk_flow_queries", "topk_flows_global", "topk_flow_queries_global"):
        assert callable(getattr(ge.Engine, name))
    with open(os.path.join(ROOT, "gyeeta_b200", "engine.py")) as f:
        src = f.read()
    for sym in ("gysk_topk_flows", "gysk_topk_flow_queries", "gysk_topk_flows_global", "gysk_topk_flow_queries_global"):
        assert f'"{sym}"' in src
