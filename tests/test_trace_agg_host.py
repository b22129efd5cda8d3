"""Trace rows without a GPU: the restatement of tests/trace_agg.py against the SQL of the trace view column by column, the
GYSK_EV_TRACE layout, and the ABI (the config word, the entry points and their answers without an engine)."""
import ctypes as C
import os
import re

import numpy as np

from gyeeta_b200 import engine as ge
from tests import trace_agg as ta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EDGES = [0, 1, 299, 300, 999, 1000, 9999, 10000, 29999, 30000, 99999, 100000, 299999, 300000, 999999, 1000000, 1000000999, 1000001000,
         (1 << 32) + 5]


def records(rng, n, ids):
    pick = lambda opts: opts[int(rng.integers(len(opts)))]          # exact Python ints (rng.choice would go through float64)
    recs = []
    for i in range(n):
        recs.append(dict(glob_id=pick(ids), response=int(EDGES[i]) if i < len(EDGES) else int(np.exp(rng.normal(8, 2))),
                         reqlen=pick([0, 17, 1 << 31, (1 << 32) - 1, 1 << 32, 1 << 50]),
                         reslen=pick([0, 5, (1 << 32) + 1, (1 << 64) - 1]),
                         reqnum=pick([0, 0, 1, 7]), errorcode=pick([0, 0, 1, 499, 500])))
    return recs


def as_api_tran(recs):
    col = lambda k: np.array([r[k] for r in recs], dtype=np.uint64)
    return ta.api_tran(col("glob_id"), col("response"), col("reqlen"), col("reslen"), col("reqnum"),
                       np.array([r["errorcode"] for r in recs], dtype=np.int32))


def test_restatement_equals_the_sql_aggregate_over_windows_and_batches():
    rng = np.random.default_rng(0)
    ids = [3, 5, 8, 13]
    to = ta.TraceOracle(16)
    for _ in range(3):                                      # windows
        window = []
        for nb in (1, 40, 300):                             # batches of the window, one of a single sample
            recs = records(rng, nb, ids)
            window += recs
            to.ingest(ta.trace_events(as_api_tran(recs)))
        want = ta.sql_aggregate(window)
        for id_ in ids:
            got = to.cur.get(id_, ta.empty_window()) if id_ in to.in_use else None
            if id_ in want:
                assert got == want[id_], id_
                w = to.window(id_, False)
                valid = [min(r["response"], ta.U32) for r in window if r["glob_id"] == id_ and min(r["response"], ta.U32) < ta.VALID_USEC]
                assert w["td_count"] == len(valid)
                assert (w["p99_resp_us"] != w["p99_resp_us"]) == (not valid)
        to.flush()
        for id_ in ids:
            if id_ in want:
                assert to.last[id_] == want[id_]
    assert to.dropped == 0


def test_bucket_edges_and_saturation():
    recs = [dict(glob_id=1, response=v, reqlen=(1 << 40), reslen=3, reqnum=1, errorcode=0) for v in EDGES]
    agg = ta.sql_aggregate(recs)[1]
    assert agg["resp_buckets"] == [3, 2, 2, 2, 2, 2, 2, 4]
    assert agg["max_bytes_in"] == ta.U32 and agg["bytes_in"] == ta.U32 * len(EDGES)
    assert agg["max_resp_us"] == ta.U32


def test_trace_event_layout():
    u64 = lambda v: np.array(v, dtype=np.uint64)
    rec = ta.api_tran(u64([42, 43]), u64([7, 1 << 33]), u64([1 << 40, 9]), u64([11, (1 << 64) - 1]),
                      u64([0, 2]), np.array([0, 500], dtype=np.int32))
    ev = ta.trace_events(rec, host_idx=3)
    assert ev["type"].tolist() == [8, 8] and ge.EV_TRACE == 8
    assert ev["svc_id"].tolist() == [42, 43] and ev["value"].tolist() == [7, ta.U32] and ev["host_idx"].tolist() == [3, 3]
    assert ev["flow_key"].tolist() == [ta.U32 | (11 << 32), 9 | (ta.U32 << 32)]
    assert ev["flags"].tolist() == [ge.EVF_TRACE_NEWCONN, ge.EVF_TRACE_ERROR]
    hdr = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert re.search(r"GYSK_EV_TRACE\s*=\s*8,", hdr)
    assert re.search(r"#define GYSK_EVF_TRACE_ERROR\s+0x1u", hdr) and re.search(r"#define GYSK_EVF_TRACE_NEWCONN\s+0x2u", hdr)


def test_config_word_and_entry_points():
    assert C.sizeof(ge.Config) == 64 and ge.Config.max_trace_svcs.offset == 60
    assert C.sizeof(ge.TraceRow) == 320 and C.sizeof(ge.TraceWindow) == 152
    L = ge.load_library()
    cfg = ge.Config()
    L.gysk_config_default(C.byref(cfg))
    assert cfg.max_trace_svcs == 0
    hdr = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    for n in ("gysk_query_traces", "gysk_query_trace_window", "gysk_export_trace_tdigest", "gysk_export_trace_tdigest_pgtext", "gysk_trace_info"):
        assert re.search(r"\bint\s+%s\s*\(" % n, hdr) and hasattr(L, n)
    n, d = C.c_uint32(), C.c_uint64()
    buf = C.create_string_buffer(64)
    assert L.gysk_query_traces(None, None, 0, None) == -22
    assert L.gysk_query_trace_window(None, -1, 0, None, 0, C.byref(n)) == -22
    assert L.gysk_export_trace_tdigest(None, 1, 0, None, None, 0, C.byref(n), None, None) == -22
    assert L.gysk_export_trace_tdigest_pgtext(None, 1, 0, buf, 64) == -22
    assert L.gysk_trace_info(None, C.byref(n), C.byref(d)) == -22


def test_slot_bytes_do_not_count_trace_rows():
    L = ge.load_library()
    out = []
    for rows in (0, 65536):
        cfg = ge.Config()
        L.gysk_config_default(C.byref(cfg))
        cfg.max_trace_svcs = rows
        s, t = C.c_uint64(), C.c_uint64()
        assert L.gysk_slot_bytes(C.byref(cfg), C.byref(s), C.byref(t)) == 0
        out.append((s.value, t.value))
    assert out[0] == out[1]
