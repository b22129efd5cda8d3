"""GYSK_FLAG_SVC_TOP_CLIENTS across ranks on the CPU: the two-level fold of tests/logical_top_clients.py (members in map order on each
rank, then the ranks ascending) keeps the four guarantees over the records of every member on every rank, on seeded streams of every
shape split over random members and ranks; the empty summary is the fold's identity; saturation holds through the fold; the header's
declarations and the ctypes binding match."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import logical_top_clients as lt
from tests import svc_top_clients as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = tc.K


def _records(rng, shape, n):
    """(member index, flow key, kbytes) of n records of one logical service with up to 12 members"""
    nm = int(rng.integers(1, 13))
    member = rng.integers(0, nm, n)
    if shape == "zipf":
        keys = rng.zipf(1.3, n) % 5000
    elif shape == "uniform":
        keys = rng.integers(0, 400, n)
    elif shape == "shared":                    # every member sees the same 3K clients
        keys = rng.integers(0, 3 * K, n)
    elif shape == "disjoint":                  # each member its own clients
        keys = member * 1000 + rng.integers(0, 40, n)
    elif shape == "few":                       # at most K clients over every member and rank
        keys = rng.integers(0, K, n)
    elif shape == "ties":
        keys = np.arange(n) % (3 * K)
        return member, keys.astype(np.uint64) + np.uint64(7), np.full(n, 5, dtype=np.int64)
    else:
        raise AssertionError(shape)
    kb = rng.integers(0, 64, n)
    kb[rng.random(n) < 0.1] = 0
    return member, keys.astype(np.uint64) + np.uint64(7), kb


def _sums(keys, kb):
    d = {}
    for k, v in zip(keys.tolist(), kb.tolist()):
        a = d.setdefault(k, [0, 0])
        a[0] += v
        a[1] += 1
    return d


SHAPES = ["zipf", "uniform", "shared", "disjoint", "few", "ties"]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_two_level_fold_keeps_the_guarantees(shape, world):
    """each member's summary from its records in a few batches, on a random rank (some members on every rank: a member can be split
    over ranks, as a recycled id can); the rank folds and the rank fold hold the guarantees over every record"""
    rng = np.random.default_rng(hash((shape, world)) % 2**32)
    for trial in range(4):
        member, keys, kb = _records(rng, shape, 3000)
        nm = int(member.max()) + 1
        rank = rng.integers(0, world, len(keys))
        if trial % 2 == 0:
            rank = rng.integers(0, world, nm)[member]          # each member wholly on one rank
        per_rank = []
        for r in range(world):
            summaries = []
            for m in rng.permutation(nm):                       # any map order
                sel = (member == m) & (rank == r)
                s = tc.EMPTY
                for part in np.array_split(np.flatnonzero(sel), int(rng.integers(1, 4))):
                    s = tc.merge([s], _sums(keys[part], kb[part]))
                summaries.append(s)
            acc = lt.fold(summaries)
            tc.check_guarantees(acc, _sums(keys[rank == r], kb[rank == r]))
            per_rank.append(acc)
        got = lt.fold(per_rank)
        exact = _sums(keys, kb)             # summed over every member on every rank
        tc.check_guarantees(got, exact, n_s=int(kb.sum()))
        if shape == "few":
            assert got[1] == 0 and len(got[0]) == len({k for k, v in exact.items() if v[0] > 0})


def test_empty_summary_is_the_identity():
    rng = np.random.default_rng(3)
    _, keys, kb = _records(rng, "zipf", 2000)
    s = tc.merge([tc.EMPTY], _sums(keys, kb))
    assert tc.merge([s, tc.EMPTY]) == s and tc.merge([tc.EMPTY, s]) == s
    assert lt.fold([tc.EMPTY, s, tc.EMPTY, tc.EMPTY]) == lt.fold([s]) == s
    assert lt.fold([]) == tc.EMPTY


def test_fold_order_is_part_of_the_answer():
    """the merge is not associative: the fold's order is fixed, map order then ranks ascending"""
    a = tc.merge([tc.EMPTY], {i: (10 + i, 1) for i in range(K)})
    b = tc.merge([tc.EMPTY], {100 + i: (11 + i, 1) for i in range(K)})
    c = tc.merge([tc.EMPTY], {i: (30, 1) for i in range(3)})
    assert lt.fold([a, b, c]) != lt.fold([c, a, b])


def test_saturation_through_the_fold():
    big = tc.M32 - 5
    a = (((1, big, 3),), 0)
    b = (((1, big, tc.M32),), 0)
    ents, delta = lt.fold([a, b])
    assert ents == ((1, tc.M32, tc.M32),) and delta == 0


def test_members_of_keeps_map_order():
    g = np.array([5, 9, 3, 7, 1], dtype=np.uint64)
    l = np.array([70, 71, 70, 72, 70], dtype=np.uint64)
    assert lt.members_of(g, l) == {70: [5, 3, 1], 71: [9], 72: [7]}


def test_header_and_binding():
    with open(os.path.join(ROOT, "include", "gysketch.h")) as f:
        h = f.read()
    assert re.search(r"int\s+gysk_query_logical_top_clients\(gysk_engine \*e, const uint64_t \*logical_ids, uint32_t n, int which, "
                     r"gysk_svc_top_clients \*out\);", h)
    assert re.search(r"int\s+gysk_query_logical_top_clients_all\(gysk_engine \*e, uint32_t flags, int which, gysk_svc_top_clients \*out, "
                     r"uint32_t cap, uint32_t \*n\);", h)
    assert re.search(r"#define GYSK_TOPC_LAST\s+1\b", h) and re.search(r"#define GYSK_TOPC_5MIN\s+2\b", h)
    assert ge.TOPC_LAST == 1 and ge.TOPC_5MIN == 2
    if not os.path.exists(os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")):
        pytest.skip("library not built")
    L = ge.load_library()
    vp, u32, i32 = C.c_void_p, C.c_uint32, C.c_int32
    assert L.gysk_query_logical_top_clients.argtypes == [vp, vp, u32, i32, vp]
    assert L.gysk_query_logical_top_clients_all.argtypes == [vp, u32, i32, vp, u32, vp]
    assert L.gysk_query_logical_top_clients.restype == L.gysk_query_logical_top_clients_all.restype == i32
