"""The flag matrix is complete, on the CPU: the flag sets gysk_create accepts are the ones tests/all_flags.py's rule allows (the
configuration check comes before any device is looked for), the GPU matrix of tests/test_gpu_flag_matrix.py reaches every TCP drain_kernel
tuple and every ingest_kernel instance with trace rows on and off, and the instances it covers are the ones the built library holds. Each
kernel's dispatch table in gysk_kernels.cu compiles only the instances its flag rules reach, so the library's kernels are the launchable
ones. A new flag that adds kernel instances fails here until the matrix covers them."""
import inspect
import os
import re

import pytest

from gyeeta_b200 import engine as ge
from tests import all_flags as af

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVAL, NODEV = -22, -19
TINY = dict(max_svcs=16, max_tasks=16, cms_depth=1, cms_log2_width=4, hll_p=4, max_batch=1024)
LIB = os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")


def _lib():
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    return ge.load_library()


def _kernels(pattern):
    """the template arguments of every kernel instance the library holds whose mangled name matches pattern: the names its kernel
    registration carries"""
    _lib()
    with open(LIB, "rb") as f:
        return set(re.findall(pattern, f.read()))


def _bools(mangled):
    return tuple(b == b"1" for b in re.findall(rb"Lb([01])E", mangled))


def ingest_instances():
    """(TRACE, QRY, TOPK, ERR, CL) of every ingest_kernel instance in the library (CL: the one-pointer ClOpen pack)"""
    return {_bools(args) + (bool(cl_),) for args, cl_ in _kernels(rb"_ZN4gysk13ingest_kernelI((?:Lb[01]E){4})J(Ph)?EEEv")}


def drain_instances():
    """(TASK, QRY, RH, TOPK, SLOW, CL, ERR) of every drain_kernel instance in the library"""
    return {_bools(args) for args in _kernels(rb"_ZN4gysk12drain_kernelI((?:Lb[01]E){7})EEv")}


def drain_tuples():
    """(QRY, RH, TOPK, SLOW, CL, ERR) of every TCP drain_kernel instance in the library"""
    return {t[1:] for t in drain_instances() if not t[0]}


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


def test_library_holds_24_ingest_instances_and_24_tcp_and_10_task_drain_tuples():
    ing = ingest_instances()
    assert len(ing) == 24, sorted(ing)
    # every instance is one a flag set reaches: ERR only with QRY
    reach = {af.ingest_instance(f, tr) for f in af.subsets() if af.allowed(f) for tr in (False, True)}
    assert ing == reach
    tcp = drain_tuples()
    assert len(tcp) == 24, sorted(tcp)
    assert tcp == {af.drain_tuple(f) for f in af.subsets() if af.allowed(f)}
    # the TASK pass runs beside each TCP pass with the same flags but SLOW and CL
    task = {t[1:] for t in drain_instances() if t[0]}
    assert len(task) == 10, sorted(task)
    assert task == {(q, rh, tk, False, False, err) for q, rh, tk, _, _, err in tcp}


def test_gpu_matrix_covers_every_library_instance():
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
