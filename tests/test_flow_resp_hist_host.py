"""The flow response histograms (GYSK_FLAG_FLOW_RESP_HIST) on the CPU: summing a batch's samples per packed key and applying the sums
equals one update per sample, over random keys and keys crafted to share the low hash bits; the cells tie to the flow query tables; the
packed key decodes to the flow's own cells at every width up to 2^28; the percentile rule of gysk_flow_resp_est equals
gysk_hist_percentiles and the compiled reference's get_percentiles on the same counts; the 300-s level rolled by the ring of tests/flow_level.py is the table one window fed every held sample would hold. The header, the Python
binding and the refusal without GYSK_FLAG_FLOW_QUERIES are pinned."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests import flow_queries as fq
from tests import flow_resp_hist as fr
from tests.flow_level import SEQUENCES, FlowLevelRing, held_windows, level_of_history

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEPTH, LOG2W = 4, 10


def _samples(rng, n, keys, ms_hi=20_000):
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["type"] = 1 + rng.integers(0, 40, n).astype(np.uint64), ge.EV_RESP
    ev["flow_key"] = keys[rng.integers(0, len(keys), n)]
    ev["value"] = rng.integers(0, ms_hi, n).astype(np.uint32) * np.uint32(1000) + rng.integers(0, 1000, n).astype(np.uint32)
    return ev


def _sharing_keys(rng, log2w, n):
    """n keys in groups whose (h1, h2) agree on the low log2w bits: distinct flows that share every cell"""
    cand = rng.integers(1, 1 << 62, 200_000, dtype=np.uint64)
    h1, h2 = fq.flow_hashes(cand)
    wm = np.uint32((1 << log2w) - 1)
    grp = (h2 & wm).astype(np.uint64) << np.uint64(32) | (h1 & wm).astype(np.uint64)
    u, inv, cnt = np.unique(grp, return_inverse=True, return_counts=True)
    shared = np.isin(inv.reshape(-1), np.flatnonzero(cnt >= 2))
    return cand[shared][:n]


def _sum_per_key(pk, inc):
    """the batch flow table restated: per packed key the sum of its samples' word increments, mod 2^64"""
    u, inv = np.unique(pk, return_inverse=True)
    tot = np.zeros(len(u), dtype=np.uint64)
    np.add.at(tot, inv.reshape(-1), inc)
    return u, tot


@pytest.mark.parametrize("depth,log2w,kind", [(4, 10, "random"), (1, 4, "random"), (8, 4, "shared"), (4, 6, "shared"), (3, 22, "random")])
def test_packed_key_sums_equal_per_sample_updates(depth, log2w, kind):
    rng = np.random.default_rng(depth * 31 + log2w)
    keys = _sharing_keys(rng, log2w, 400) if kind == "shared" else rng.integers(1, 1 << 62, 500, dtype=np.uint64)
    assert len(keys) >= 100
    s = _samples(rng, 40_000, keys)
    s["value"][::97] = rng.integers(15_000_000, 15_002_000, len(s["value"][::97]))      # both sides of the last bucket edge
    want = fr.add_samples(fr.empty(depth, log2w), s, depth, log2w)
    b = fr.buckets(s["value"])
    pk = fr.packed_keys(s["flow_key"], b, log2w)
    assert pk.min() > 0
    u, tot = _sum_per_key(pk, fr.packed_incs(b))
    pairs = np.unique(np.stack([s["flow_key"], b.astype(np.uint64)]), axis=1)
    assert len(u) < pairs.shape[1]                                      # a word's two buckets (and with kind "shared", flows) in one entry
    got = fr.apply_packed(fr.empty(depth, log2w), u, tot, depth, log2w)
    assert got.tobytes() == want.tobytes()
    # every cell's 15 counts sum to the query half of the same flow query cell (mod 2^32); word 7's high half stays 0
    q = fq.add_samples(np.zeros(depth << log2w, dtype=np.uint64), s, depth, log2w)
    h = fr.halves(got)
    assert not h[:, 15].any()
    assert np.array_equal(h[:, :15].sum(axis=1, dtype=np.uint64) & np.uint64(fq.U32), q & np.uint64(fq.U32))


@pytest.mark.parametrize("log2w", list(range(4, 29)))
def test_packed_key_decodes_at_every_width(log2w):
    """at every width gysk_create accepts (up to 2^28) a packed key decodes to the sample's word and to the columns of its flow in every
    row, so the cells a key names are the flow's own (the tables themselves are too large to restate beyond 2^22)"""
    rng = np.random.default_rng(log2w)
    depth = 8
    keys = rng.integers(1, 1 << 63, 100_000, dtype=np.uint64)
    b = rng.integers(0, 15, len(keys))
    w, cols = fr.decode_packed(fr.packed_keys(keys, b, log2w), depth, log2w)
    assert np.array_equal(w, b >> 1)
    assert np.array_equal(cols, fq.columns(keys, depth, log2w))
    assert (w >= 0).all() and (w < fr.WORDS).all()


def test_bucket_edges():
    ms = np.array([0, 1, 2, 10, 11, 1000, 1001, 3000, 3001, 15000, 15001, 1_000_000], dtype=np.uint32)
    assert fr.buckets(ms * np.uint32(1000) + np.uint32(999)).tolist() == [1, 1, 2, 2, 3, 11, 12, 12, 13, 13, 14, 14]
    lib = ge.load_library()
    for v in ms.tolist():
        assert lib.gysk_hist_bucket(0, int(v)) == int(fr.buckets(np.array([v * 1000]))[0])


def test_carry_into_the_next_bucket():
    """a bucket count past 2^32 in one cell carries into its neighbour, the known edge of a summed u64 word"""
    t = fr.apply_packed(fr.empty(1, 4), fr.packed_keys(np.array([7], dtype=np.uint64), [2], 4), np.array([(1 << 32) + 5], dtype=np.uint64), 1, 4)
    c = fr.point_counts(t, np.array([7], dtype=np.uint64), 1, 4)[0]
    assert c[2] == 5 and c[3] == 1


def test_percentile_rule_equals_the_library_and_the_reference():
    L, R = ge.load_library(), po.ref()
    rng = np.random.default_rng(9)
    pcts = np.array([25, 95, 99], dtype=np.float32)
    # empty, one sample (every cut-off is 0, met by bucket 0: -1 ms), four samples (cut-offs 1, 3, 3), the last bucket alone
    cases = [np.zeros(15, dtype=np.uint64), np.eye(15, dtype=np.uint64)[5], np.eye(15, dtype=np.uint64)[3] * 3 + np.eye(15, dtype=np.uint64)[9],
             np.eye(15, dtype=np.uint64)[14]]
    assert [fr.percentiles(c) for c in cases] == [(-1, -1, -1), (-1, -1, -1), (30, 30, 30), (-1, -1, -1)]
    for _ in range(3000):
        c = np.zeros(15, dtype=np.uint64)
        k = int(rng.integers(1, 16))
        c[rng.integers(0, 15, k)] = rng.integers(0, 1 << int(rng.integers(1, 32)), k)
        cases.append(c)
    for c in cases:
        ser = np.zeros(15, dtype=ge.SERIAL_DTYPE)
        ser["count"] = c
        total = int(c.sum())
        got = np.zeros(3, dtype=np.int64)
        assert L.gysk_hist_percentiles(0, 0, ge._p(ser), total, ge._p(pcts), 3, ge._p(got)) == 0
        assert fr.percentiles(c) == tuple(got.tolist()), c
        if R is not None:
            ref = np.zeros(3, dtype=np.int64)
            R.gyref_hist_pct_from_serial(0, 0, po._p(ser), total, 0, po._p(pcts), 3, po._p(ref), None)
            assert tuple(ref.tolist()) == fr.percentiles(c), c


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_ring_of_histogram_tables_equals_the_epoch_rule(name):
    tsecs = SEQUENCES[name]
    rng = np.random.default_rng(400 + len(tsecs))
    keys = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
    ring = FlowLevelRing((DEPTH << LOG2W) * fr.WORDS)
    tables, windows = [], []
    for i, t in enumerate(tsecs):
        s = _samples(rng, int(rng.integers(100, 2000)), keys)
        tables.append(fr.add_samples(fr.empty(DEPTH, LOG2W), s, DEPTH, LOG2W))
        windows.append(s)
        level = ring.flush(t, tables[-1])
        assert np.array_equal(level, level_of_history(tsecs[: i + 1], tables)), (name, i)
        held = np.concatenate([windows[j] for j in held_windows(tsecs[: i + 1])])
        assert level.tobytes() == fr.add_samples(fr.empty(DEPTH, LOG2W), held, DEPTH, LOG2W).tobytes(), (name, i)
        k = np.unique(keys[:40])
        assert (fr.point_counts(level, k, DEPTH, LOG2W) >= fr.exact(held, k)).all()
        assert (fr.bucket_sums(level, DEPTH, LOG2W)[:, :15] == np.bincount(fr.buckets(held["value"]), minlength=15)[None, :]).all()


def test_header_and_binding():
    h = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert re.search(r"#define GYSK_FLAG_FLOW_RESP_HIST\s+0x200u", h)
    assert ge.FLAG_FLOW_RESP_HIST == 0x200
    for decl in ("int		gysk_query_flow_resp(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_resp_est *out);",
                 "int		gysk_export_cms_resp(gysk_engine *e, int last_window, uint64_t *words",
                 "int		gysk_query_flow_resp_global(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_resp_est *out);",
                 "int		gysk_query_flow_resp_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_resp_est *out);",
                 "int		gysk_export_cms_resp_5min(gysk_engine *e, uint64_t *words",
                 "int		gysk_query_flow_resp_global_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_resp_est *out);",
                 "int64_t		gysk_last_batch_flow_resp_direct(gysk_engine *e);"):
        assert decl in h, decl
    st = h.split("typedef struct gysk_flow_resp_est")[1].split("} gysk_flow_resp_est;")[0]
    fields = re.findall(r"^\s*(u?int\d+_t)\s+([^;]+);", st, re.M)
    assert fields == [("uint64_t", "flow_key"), ("uint32_t", "counts[15]"), ("uint32_t", "total"), ("int64_t", "p25_ms, p95_ms, p99_ms")]
    d = ge.FLOW_RESP_EST_DTYPE
    assert d.itemsize == 96 and [d.fields[f][1] for f in d.names] == [0, 8, 68, 72, 80, 88]
    flag = h.split("#define GYSK_FLAG_FLOW_RESP_HIST")[1].split("*/")[0]
    assert "Needs GYSK_FLAG_FLOW_QUERIES" in flag and "gysk_create refuses it" in flag and "8x the words" in flag


def test_library_exports_the_calls():
    lib = os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    L = C.CDLL(lib)
    for name in ("gysk_query_flow_resp", "gysk_export_cms_resp", "gysk_query_flow_resp_global", "gysk_query_flow_resp_5min",
                 "gysk_export_cms_resp_5min", "gysk_query_flow_resp_global_5min", "gysk_last_batch_flow_resp_direct"):
        assert hasattr(L, name), name
    assert L.gysk_export_cms_resp(None, 0, None) == -22
    # the configuration check comes before any device is looked for
    for kw in (dict(flow_resp_hist=True), dict(flow_resp_hist=True, flow_query_level=True)):
        with pytest.raises(ge.GyskError) as ex:
            ge.Engine(**kw)
        assert ex.value.code == -22 and "needs GYSK_FLAG_FLOW_QUERIES" in str(ex.value)
