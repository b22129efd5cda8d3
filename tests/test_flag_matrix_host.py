"""The flag matrix is complete, on the CPU: the flag sets gysk_create accepts are the ones tests/all_flags.py's rule allows (the
configuration check comes before any device is looked for), the GPU matrix of tests/test_gpu_flag_matrix.py reaches every TCP drain_kernel
tuple and every ingest_kernel instance with trace rows on and off, and the instances it covers are the ones the dispatch tables of
gysk_kernels.cu can launch. A new flag that adds kernel instances fails here until the matrix covers them."""
import inspect
import os
import re

import pytest

from gyeeta_b200 import engine as ge
from tests import all_flags as af

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVAL, NODEV = -22, -19
TINY = dict(max_svcs=16, max_tasks=16, cms_depth=1, cms_log2_width=4, hll_p=4, max_batch=1024)


def _lib():
    if not os.path.exists(os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")):
        pytest.skip("library not built")
    return ge.load_library()


def _src():
    with open(os.path.join(ROOT, "gyeeta_b200", "csrc", "gysk_kernels.cu")) as f:
        return f.read()


def _span(src, head):
    """(start, end) of the brace block that follows the first match of head"""
    m = re.search(head, src)
    assert m, head
    i = src.index("{", m.end())
    depth = 0
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return i + 1, j
    raise AssertionError(head)


def _body(src, head):
    a, b = _span(src, head)
    return src[a: b]


def _bools(args):
    return tuple(a.strip() == "true" for a in args.split(","))


def ingest_instances():
    """(TRACE, QRY, TOPK, ERR, CL) of every ingest_kernel instance launch_ingest's tables hold"""
    body = _body(_src(), r"\bint launch_ingest\(")
    out = set()
    for args, cl_ in re.findall(r"ingest_kernel<((?:\s*(?:true|false)\s*,){3}\s*(?:true|false))\s*(,\s*uint8_t \*)?>", body):
        out.add(_bools(args) + (bool(cl_),))
    return out


def drain_tuples():
    """(QRY, RH, TOPK, SLOW, CL, ERR) of every TCP drain_kernel pass launch_drains can reach, the dispatch evaluated from the sources:
    each launch_drain_passes call of launch_drains (its QRY, RH and ERR), both values of CL (launch_drain_passes picks by cl_open), and
    each TCP launch_drain_pass call of launch_drain_passes_t, those inside `if constexpr (RH)` only where RH holds"""
    src = _src()
    drains = _body(src, r"\bint launch_drains\(")
    calls = [_bools(a) for a in re.findall(r"launch_drain_passes<([^>]*)>", drains)]
    assert calls, "no launch_drain_passes call in launch_drains"
    passes = _body(src, r"static int launch_drain_passes_t\(")
    lo, hi = _span(passes, r"if constexpr \(RH\)")
    tcp = [(m.group(1), lo <= m.start() < hi) for m in re.finditer(r"launch_drain_pass<false,\s*([^>]*)>", passes)]
    assert any(r for _, r in tcp) and not all(r for _, r in tcp)
    out = set()
    for call in calls:
        qry, rh = call[0], call[1]
        err = call[2] if len(call) > 2 else False
        for cl_ in (False, True):
            env = {"QRY": qry, "RH": rh, "CL": cl_, "ERR": err, "true": True, "false": False}
            for args, rh_only in tcp:
                if rh_only and not rh:
                    continue
                vals = tuple(env[a.strip()] for a in args.split(","))
                assert len(vals) == 6, args
                out.add(vals)
    return out


def test_accepted_flag_sets_are_the_rule():
    _lib()
    accepted = []
    for f in af.subsets():
        try:
            eng = ge.Engine(**TINY, **f)
        except ge.GyskError as ex:
            assert ex.code in (INVAL, NODEV), (f, ex.code, str(ex))
            if ex.code == NODEV:                # past the configuration check, stopped for want of a device
                accepted.append(f)
            continue
        eng.close()                             # a machine with a device creates it
        accepted.append(f)
    want = [f for f in af.subsets() if af.allowed(f)]
    assert len(want) == 126
    assert accepted == want, [f for f in af.subsets() if (f in accepted) != (f in want)][:4]


def test_dispatch_tables_hold_24_ingest_instances_and_24_tcp_drain_tuples():
    ing = ingest_instances()
    assert len(ing) == 24, sorted(ing)
    # every instance is one a flag set reaches: ERR only with QRY
    reach = {af.ingest_instance(f, tr) for f in af.subsets() if af.allowed(f) for tr in (False, True)}
    assert ing == reach
    tcp = drain_tuples()
    assert len(tcp) == 24, sorted(tcp)
    assert tcp == {af.drain_tuple(f) for f in af.subsets() if af.allowed(f)}


def test_gpu_matrix_covers_every_instance():
    cases = af.matrix()
    assert len(cases) == 48 and len({c[0] for c in cases}) == 48
    assert all(af.allowed(f) for _, f, _ in cases)
    assert {rows for _, _, rows in cases} == {0, 64}
    for rows in (0, 64):
        sub = [f for _, f, r in cases if r == rows]
        assert {af.drain_tuple(f) for f in sub} == drain_tuples(), rows
        assert {af.ingest_instance(f, rows) for f in sub} == {i for i in ingest_instances() if i[0] == bool(rows)}, rows
    for flag in ("flow_level", "flow_query_level", "flow_topk_5min"):
        assert {f[flag] for _, f, _ in cases} == {False, True}, flag
    # the level flags vary inside the cases that can hold them, not only across them
    for flag, need in (("flow_query_level", "flow_queries"), ("flow_topk_5min", "flow_topk")):
        assert {f[flag] for _, f, _ in cases if f[need]} == {False, True}, flag


def test_flag_names_match_the_engine_keywords():
    params = inspect.signature(ge.Engine.__init__).parameters
    assert all(k in params for k in af.FLAGS)
    bits = [ge.FLAG_FLOW_QUERIES, ge.FLAG_FLOW_QUERY_LEVEL, ge.FLAG_FLOW_RESP_HIST, ge.FLAG_FLOW_TOPK, ge.FLAG_FLOW_TOPK_SLOW,
            ge.FLAG_CLIENT_LEVELS, ge.FLAG_FLOW_ERRORS]
    assert len(set(bits)) == len(bits)
