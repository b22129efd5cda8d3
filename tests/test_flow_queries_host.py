"""GYSK_FLAG_FLOW_QUERIES without a GPU: the numpy restatement of the flow query tables (tests/flow_queries.py) against the oracle's hash
and column definitions, the count-min properties of the restated tables (min over rows >= exact, every row's query halves summing to the
counted samples), the key each response route gives a sample, and the C header's flag, struct and calls."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests import flow_queries as fq
from tests.trace_agg import api_tran, resp_events

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M32 = 0xFFFFFFFF


def _resp(rng, n, keys, nsvc=50):
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = rng.integers(1, nsvc + 1, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15 & ((1 << 63) - 1))
    ev["flow_key"] = keys[rng.integers(0, len(keys), n)]
    ev["value"] = rng.integers(0, 3_000_000, n)
    ev["value"][::97] = fq.VALID_USEC + rng.integers(0, 1000, len(ev[::97]))      # beyond the validity rule
    ev["type"] = np.where(rng.random(n) < 0.8, ge.EV_RESP, ge.EV_ACCEPT)
    return ev


def test_hashes_and_columns_are_the_oracles():
    L = po.lib()
    rng = np.random.default_rng(1)
    keys = np.concatenate([np.array([0, 1, (1 << 64) - 1, 1 << 32, (10 << 56) | 443], dtype=np.uint64),
                           rng.integers(0, 1 << 64, 300, dtype=np.uint64, endpoint=False)])
    h1, h2 = fq.flow_hashes(keys)
    for i, k in enumerate(keys.tolist()):
        a, b = C.c_uint32(), C.c_uint32()
        L.gyo_flow_hashes(k, C.byref(a), C.byref(b))
        assert (int(h1[i]), int(h2[i])) == (a.value, b.value), hex(k)
    for depth, log2w in ((1, 4), (4, 20), (8, 22), (8, 4)):
        cols = fq.columns(keys, depth, log2w)
        for r in range(depth):
            assert cols[r].tolist() == [L.gyo_cms_index(k, r, log2w) for k in keys.tolist()], (depth, log2w, r)


@pytest.mark.parametrize("depth,log2w", [(1, 4), (4, 10), (8, 4), (8, 16)])
def test_min_over_rows_bounds_the_exact_counts_and_rows_sum_to_the_samples(depth, log2w):
    rng = np.random.default_rng(depth * 100 + log2w)
    keys = rng.integers(1, 1 << 63, 2000, dtype=np.uint64)
    ev = _resp(rng, 60_000, keys)
    known = set(np.unique(ev["svc_id"]).tolist()[:40])          # the other services have no slot: not counted
    s = fq.counted(ev, known)
    assert 0 < len(s) < int((ev["type"] == ge.EV_RESP).sum())
    table = fq.add_samples(np.zeros(depth << log2w, dtype=np.uint64), s, depth, log2w)
    assert fq.row_sums(table, depth, log2w) == [len(s) & M32] * depth
    qs, ms = fq.point_query(table, keys, depth, log2w)
    for (eq, em), q, m in zip(fq.exact(s, keys), qs.tolist(), ms.tolist()):
        assert q >= eq and m >= em
    if depth == 8 and log2w == 16:                               # wide enough: almost every key exact
        assert sum(e == (q, m) for e, q, m in zip(fq.exact(s, keys), qs.tolist(), ms.tolist())) > 0.99 * len(keys)


def test_cells_wrap_mod_2_64():
    """a query half that wraps carries into the msec half, as RED.ADD.64 does on the device"""
    t = np.zeros(1 << 4, dtype=np.uint64)
    s = np.zeros(3, dtype=ge.EVENT_DTYPE)
    s["flow_key"], s["value"], s["type"] = 7, 999, ge.EV_RESP
    col = int(fq.columns(np.array([7], dtype=np.uint64), 1, 4)[0, 0])
    t[col] = np.uint64(M32)
    fq.add_samples(t, s, 1, 4)
    assert int(t[col]) == (M32 + 3) & ((1 << 64) - 1)


def test_route_keys():
    """the key of each response route: the raw IPv4 / IPv6 events key (client ip << 32) | client port like the connection events of the
    same client (the address of IPv6 folded as the library folds it); RESP16 and API_TRAN only the client port"""
    L = po.lib()
    rng = np.random.default_rng(3)
    r4 = np.zeros(100, dtype=np.dtype([("daddr", "<u4"), ("dport", "<u2")]))
    r4["daddr"], r4["dport"] = rng.integers(1, 1 << 32, 100), rng.integers(0, 1 << 16, 100)
    k4 = fq.route_key_ipv4(r4)
    assert [int(k) for k in k4] == [(int(a) << 32) | int.from_bytes(int(p).to_bytes(2, "little"), "big") for a, p in zip(r4["daddr"], r4["dport"])]
    r6 = np.zeros(50, dtype=np.dtype([("daddr", "<u4", 4), ("dport", "<u2")]))
    r6["daddr"], r6["dport"] = rng.integers(0, 1 << 32, (50, 4)), rng.integers(0, 1 << 16, 50)
    k6 = fq.route_key_ipv6(r6)
    for w, p, k in zip(r6["daddr"].tolist(), r6["dport"].tolist(), k6.tolist()):
        fold = L.gyo_jhash_2words(w[2], w[3], L.gyo_jhash_2words(w[0], w[1], fq.GY_SEED))
        assert k == (fold << 32) | int.from_bytes(int(p).to_bytes(2, "little"), "big")
    rec = api_tran(np.arange(1, 11, dtype=np.uint64), 1000, cliport=np.arange(40000, 40010))
    assert fq.route_key_api_tran(rec).tolist() == resp_events(rec)["flow_key"].tolist()
    r16 = np.zeros(5, dtype=ge.RESP16_DTYPE)
    r16["cli_port"] = [0, 1, 31, 200, 255]
    assert fq.route_key_resp16(r16).tolist() == [0, 1, 31, 200, 255]


def test_header_declares_the_flag_struct_and_calls():
    h = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert re.search(r"#define GYSK_FLAG_FLOW_QUERIES\s+0x80u", h)
    assert ge.FLAG_FLOW_QUERIES == 0x80
    body = re.search(r"typedef struct gysk_flow_qry_est\s*\{(.*?)\}\s*gysk_flow_qry_est;", h, re.S).group(1)
    fields = re.findall(r"(uint\d+_t)\s+(\w+);", body)
    assert fields == [("uint64_t", "flow_key"), ("uint32_t", "queries"), ("uint32_t", "resp_ms")]
    assert ge.FLOW_QRY_EST_DTYPE.itemsize == 16 and ge.FLOW_QRY_EST_DTYPE.names == ("flow_key", "queries", "resp_ms")
    for decl in ("int		gysk_query_flow_queries(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_qry_est *out);",
                 "int		gysk_export_cms_queries(gysk_engine *e, int last_window, uint64_t *cells",
                 "int		gysk_query_flow_queries_global(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_qry_est *out);",
                 "int64_t		gysk_last_batch_flow_query_direct(gysk_engine *e);"):
        assert decl in h, decl


def test_library_exports_the_calls():
    lib = os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    L = C.CDLL(lib)
    for name in ("gysk_query_flow_queries", "gysk_export_cms_queries", "gysk_query_flow_queries_global", "gysk_last_batch_flow_query_direct"):
        assert hasattr(L, name), name
