"""GYSK_FLAG_MERGE_TRACES without a device: the restatement the GPU tests hold the merged trace rows to, pinned against the trace view's
SQL over the union of the members' raw records; the header's flag, struct layout and entry points against the bindings."""
import ctypes as C
import os
import re

import numpy as np

from gyeeta_b200 import engine as ge
from tests import logical_traces as lt
from tests import trace_agg as ta
from tests.util import td_fold

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVAL = -22


def test_counter_fold_equals_sql_over_the_union_of_the_members():
    """three ranks, two logical services whose members spread over them, one member without requests: the restated counters equal
    tracereq_aggr_info over the union of the members' records grouped by logical id; the digest count equals the samples within the
    validity rule, and the fold of the members' digests is what td_fold gives"""
    rng = np.random.default_rng(4)
    world = 3
    members = {600: [101, 102, 103, 104, 105], 601: [201, 202, 203]}
    host = {g: i for i, g in enumerate(members[600] + members[601])}
    n = 4000
    gid = rng.choice(np.array(members[600] + members[601][:2], dtype=np.uint64), size=n)
    usec = np.exp(rng.normal(8.0, 2.0, size=n)).astype(np.uint64)
    usec[:4] = [0, 999_999, 1_000_001_000, 5_000_000_000]
    rec = ta.api_tran(gid, usec, rng.integers(0, 1 << 33, size=n).astype(np.uint64), rng.integers(0, 1 << 20, size=n).astype(np.uint64),
                      np.where(rng.random(n) < 0.2, 0, 1).astype(np.uint64), rng.choice(np.array([0, 0, 500], dtype=np.int32), size=n))
    ev = ta.trace_events(rec)
    ev["host_idx"] = [host[g] for g in gid.tolist()]
    oracles = [ta.TraceOracle(8) for _ in range(world)]
    for r, to in enumerate(oracles):
        to.ingest(ev[ev["host_idx"] % world == r])
        to.flush()
    lid_of = {g: l for l, gs in members.items() for g in gs}
    sql = ta.sql_aggregate([dict(glob_id=lid_of[int(x["glob_id"])], response=int(x["response_usec"]), reqlen=int(x["reqlen"]),
                                 reslen=int(x["reslen"]), reqnum=int(x["reqnum"]), errorcode=int(x["errorcode"])) for x in rec])
    for lid, gs in members.items():
        w, ntraced = lt.fold_counters(oracles, gs)
        assert ntraced == len(set(gid.tolist()) & set(gs))
        for f in lt.SUMS + lt.MAXES + ("resp_buckets",):
            assert w[f] == sql[lid][f], (lid, f)
        v = usec[np.isin(gid, np.array(gs, dtype=np.uint64))]
        assert w["td_count"] == int((v < ta.VALID_USEC).sum())
        d = lt.merged_digest(oracles, gs)
        assert d.total == w["td_count"] and d.minv == float(v[v < ta.VALID_USEC].min()) and d.maxv == float(v[v < ta.VALID_USEC].max())
        per_rank = [td_fold([lt.window_digest(to, g) for g in gs], lt.DELTA) for to in oracles]
        assert sum(x.total for x in per_rank) == d.total and len(d.cent) <= lt.DELTA
        r, _ = lt.row(oracles, lid, gs)
        assert r.found == 1 and r.ntraced == ntraced and r.last.nreq == sum(r.last.resp_buckets) == sql[lid]["nreq"]
        assert 0 < r.last.p99_resp_us <= d.maxv
    # a logical service without a traced member: found, zero window, NaN p99
    r, d = lt.row(oracles, 602, [301, 302])
    assert r.found == 1 and r.ntraced == 0 and r.last.nreq == 0 and np.isnan(r.last.p99_resp_us) and d.total == 0


def test_flag_and_layout_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert int(re.search(r"#define GYSK_FLAG_MERGE_TRACES\s+(0x[0-9a-fA-F]+)u", hdr).group(1), 16) == ge.FLAG_MERGE_TRACES == 0x40
    flags = [int(v, 16) for v in re.findall(r"#define GYSK_FLAG_\w+\s+(0x[0-9a-fA-F]+)u", hdr)]
    assert len(flags) == len(set(flags))
    body = re.search(r"typedef struct gysk_logical_trace\s*\{(.*?)\}\s*gysk_logical_trace;", hdr, re.S).group(1)
    fields = re.findall(r"^\s*(\w+)\s+(\w+);", body, re.M)
    assert fields == [("uint64_t", "logical_id"), ("int32_t", "found"), ("uint32_t", "ntraced"), ("gysk_trace_window", "last")]
    assert [(f, getattr(ge.LogicalTrace, f).offset) for f, _ in ge.LogicalTrace._fields_] == [("logical_id", 0), ("found", 8), ("ntraced", 12),
                                                                                            ("last", 16)]
    assert C.sizeof(ge.LogicalTrace) == 168 and "/* 168 bytes */" in hdr.split("gysk_logical_trace;")[1].splitlines()[0]


def test_new_symbols_answer_inval_without_an_engine():
    L = ge.load_library()
    n = C.c_uint32()
    ids = np.array([1], dtype=np.uint64)
    out = (ge.LogicalTrace * 1)()
    m, w, d = np.zeros(100), np.zeros(100, dtype=np.uint64), C.c_double()
    assert L.gysk_query_logical_traces(None, ge._p(ids), 1, out) == INVAL
    assert L.gysk_query_logical_traces_all(None, 0, out, 1, C.byref(n)) == INVAL
    assert L.gysk_export_logical_trace_tdigest(None, 1, ge._p(m), ge._p(w), 100, C.byref(n), C.byref(d), C.byref(d)) == INVAL
    assert L.gysk_export_logical_trace_tdigest_pgtext(None, 1, C.create_string_buffer(64), 64) == INVAL
