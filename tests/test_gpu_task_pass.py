"""The TASK pass of drain_kernel on process-record streams that the streams of test_gpu_record_regions.py do not reach, against the
CPU oracle after every batch (every task's three histograms, counters and the whole count-min table).

The pass reads one record per lane and group of 32, applies the group's three histograms with one cell_add each over the whole
warp, and loads the next group of its share while the current one is applied (DESIGN.md §4). The streams here give it groups of
one cell only (the hot table only hits), groups of 32 different tasks, shares that end in a partial group followed by empty
regions, and values of 2^31 and more, which narrow to negative ints, in all three fields."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests.test_gpu_record_regions import TIDS, Geometry, Pair, _tcp

BIG = 1 << 31


@pytest.fixture(scope="module")
def geo():
    import torch
    return Geometry(torch.cuda.get_device_properties(0).multi_processor_count)


def _task_events(n, ids, value, cpu_delay, blkio, rng):
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = ids
    ev["type"] = ge.EV_TASK
    ev["value"] = value
    ev["flow_key"] = np.asarray(cpu_delay, dtype=np.uint64) | (np.asarray(blkio, dtype=np.uint64) << np.uint64(32))
    ev["host_idx"] = rng.integers(0, 64, n)
    ev["tsec"] = 1
    return ev


def _one_cell(rng, n, big=False):
    """every process record of the batch: one task, one bucket per histogram (the same three values)"""
    v = (BIG + 12345, BIG + 7, 0xFFFFFFFF) if big else (150, 40, 3)
    return _task_events(n, TIDS[3], v[0], v[1], v[2], rng)


def _all_different(rng, n):
    """a tasks-only batch: each chunk's records are handed over in order, so every group of 32 records holds 32 consecutive
    events; their task is the event's index mod 32, plus 32 x a block number, so that no two records of a group share a task"""
    i = np.arange(n)
    ids = TIDS[(i % 32) + 32 * ((i // 32) % 12)]
    return _task_events(n, ids, rng.integers(0, 3200, n), rng.integers(0, 100_000, n), rng.integers(0, 100_000, n), rng)


def _big_values(rng, n):
    """all three fields at 2^31 or more for most records: negative after the narrowing to int; the rest small"""
    big = rng.random(n) < 0.8
    f = lambda: np.where(big, rng.integers(BIG, 1 << 32, n, dtype=np.uint64), rng.integers(0, 5000, n, dtype=np.uint64))
    return _task_events(n, TIDS[rng.integers(0, 40, n)], f().astype(np.uint32), f(), f(), rng)


def _sparse_regions(rng, n, geo):
    """connection records everywhere; in the chunks of ingest warp w (chunk c goes to warp c % nwarps) no process record when
    w % 3 == 0, 37 when w % 3 == 1 (one full group and a partial one of 5), a whole chunk's worth otherwise; so the regions are
    empty, end in a partial group, or are full, in turn, and a drain warp's share can end in a partial group followed by empty
    regions"""
    ev = _tcp(rng, n)
    nwarps = geo.regions(n)[0]
    c = np.arange(n) // geo.chunk
    pos = np.arange(n) % geo.chunk
    w = c % nwarps
    k = np.where(w % 3 == 0, 0, np.where(w % 3 == 1, 37, geo.chunk))
    # 37 records per chunk: in a chunk of 64 events the hand-over at 32 leaves 5 for the warp's next chunk or its end
    is_task = pos < k
    t = _task_events(n, TIDS[rng.integers(0, 300, n)], rng.integers(0, 3200, n), rng.integers(0, 100_000, n),
                     rng.integers(0, 100_000, n), rng)
    ev[is_task] = t[is_task]
    return ev


def _run(p, batches):
    for ev in batches:
        p.feed(ev)
        p.check()                           # every task's three histograms after every batch
    p.flush(5)


@pytest.mark.gpu
def test_one_task_one_bucket(geo):
    """all 32 lanes of every group hold the same three cells: the group collapses to one leader per histogram and the hot table
    only hits after its first group; with small values, then with values that narrow to negative ints"""
    n1, n2, n3 = geo.sizes()
    rng = np.random.default_rng(201)
    p = Pair(max_batch=n3)
    _run(p, [_one_cell(rng, n2), _one_cell(rng, n1), _one_cell(rng, n3, big=True), _one_cell(rng, 37)])
    assert p.eng.stats()["events_task"] == n1 + n2 + n3 + 37


@pytest.mark.gpu
def test_every_record_of_a_group_a_different_task(geo):
    """no two lanes of a group share a cell: every cell_add is 32 single-lane groups"""
    n1, n2, n3 = geo.sizes()
    rng = np.random.default_rng(202)
    p = Pair(max_batch=n3)
    _run(p, [_all_different(rng, n) for n in (n1, n3, 32 * 7 + 3)])


@pytest.mark.gpu
def test_shares_end_in_partial_groups_and_empty_regions(geo):
    """regions that are empty, end in a partial group or are full, in turn, at batch sizes from a fraction of one grid of chunks
    (most drain warps get no group or one) to several chunks per ingest warp; the lookahead stops at each warp's last group"""
    n1, n2, n3 = geo.sizes()
    small = (geo.full // 3) * geo.chunk + 5
    rng = np.random.default_rng(203)
    p = Pair(max_batch=n3)
    batches = [_sparse_regions(rng, n, geo) for n in (small, n1, n3, n2, 3 * geo.chunk + 1)]
    for b in batches[1:4]:
        nwarps = geo.regions(len(b))[0]
        per_region = np.bincount((np.arange(len(b)) // geo.chunk) % nwarps, weights=b["type"] == ge.EV_TASK, minlength=nwarps)
        assert per_region.min() == 0 and (per_region % 32 != 0).any()
    _run(p, batches)


@pytest.mark.gpu
def test_values_of_2_31_and_more_in_all_three_fields(geo):
    """values, cpu delays and blkio delays of 2^31 and more: negative ints in the histograms (sums and maxima)"""
    n1, n2, n3 = geo.sizes()
    rng = np.random.default_rng(204)
    p = Pair(max_batch=n3)
    _run(p, [_big_values(rng, n) for n in (n2, n3, 1000)])
