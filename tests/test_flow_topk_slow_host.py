"""The slow-response sets of GYSK_FLAG_FLOW_TOPK_SLOW on the CPU: the threshold-to-bucket rule against the library's own bucket
function, the score's place between the exact slow count and the smallest row sum on keys made to collide, its monotonicity under
saturation, the window guarantee and the 300-s bound of tests/flow_topk_slow.py on seeded streams (a few slow clients hidden in a crowd of
fast heavy ones among them), and the header, the Python constant and the bindings that pin the ABI."""
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import flow_level as fl
from tests import flow_queries as fq
from tests import flow_resp_hist as frh
from tests import flow_topk_slow as fs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, W = 4, 8
CLS_RESP_TIME = 0                 # GYSK_CLS_RESP_TIME
SAMPLE = np.dtype([("flow_key", "<u8"), ("value", "<u4")])


def _lib():
    lib = os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    return ge.load_library()


def samples(keys, msec):
    s = np.zeros(len(keys), dtype=SAMPLE)
    s["flow_key"], s["value"] = np.asarray(keys, dtype=np.uint64), np.asarray(msec, dtype=np.uint32) * 1000 + 999
    return s


def test_threshold_to_first_slow_bucket():
    L = _lib()
    for i, t in enumerate(fs.THR.tolist()):
        bs = fs.b_slow(t)
        assert bs == 2 + i
        assert L.gysk_hist_bucket(CLS_RESP_TIME, t) < bs <= L.gysk_hist_bucket(CLS_RESP_TIME, t + 1), t
        assert frh.buckets(np.array([t * 1000 + 999, (t + 1) * 1000], dtype=np.uint32)).tolist() == \
            [L.gysk_hist_bucket(CLS_RESP_TIME, t), L.gysk_hist_bucket(CLS_RESP_TIME, t + 1)]
    assert fs.b_slow(300) == 9


def test_score_between_exact_count_and_smallest_row_sum():
    """keys that share cells in some rows (width 16): S is at least the exact slow count and at most each row's slow sum"""
    rng = np.random.default_rng(1)
    d, w = 3, 4
    keys = np.unique(rng.integers(1, 1 << 40, 60).astype(np.uint64))
    s = samples(rng.choice(keys, 3000), rng.choice([0, 5, 50, 250, 400, 900, 2000, 20000], 3000))
    table = frh.add_samples(frh.empty(d, w), s, d, w)
    for t in (1, 300, 15000):
        bs = fs.b_slow(t)
        S = fs.scorer(bs)(table, keys, d, w)
        ex = fs.exact_slow(s, keys, bs)
        assert np.all(S >= ex), t
        t3 = table.reshape(d, 1 << w, frh.WORDS)
        cols = fq.columns(keys, d, w)
        row_sums = np.stack([frh.halves(t3[r][cols[r]])[:, bs:frh.NB].astype(np.int64).sum(axis=1) for r in range(d)])
        assert np.all(S <= row_sums.min(axis=0)), t
        assert np.any(S > ex), "the keys collide, so some estimates exceed the exact count"


def test_score_saturates_monotonely():
    bs = 2
    base = np.zeros((1, frh.NB), dtype=np.uint64)
    base[0, 2:] = 0x7FFFFFFF
    s0 = fs.score_of_counts(base, bs)[0]
    assert s0 == fs.SAT
    more = base.copy()
    more[0, 5] += 1
    assert fs.score_of_counts(more, bs)[0] == fs.SAT >= s0
    # below saturation, one more slow sample raises the score by one; mod 2^32 would have wrapped to a small value
    c = np.zeros((1, frh.NB), dtype=np.uint64)
    c[0, 13], c[0, 14] = 0xFFFFFFFF, 0
    assert fs.score_of_counts(c, bs)[0] == fs.SAT
    c[0, 14] = 1
    assert fs.score_of_counts(c, bs)[0] == fs.SAT and (int(c[0].sum()) & fs.SAT) == 0


def _window(rng, fast, slow, nbatches, per_batch, t_ms):
    """batches of samples: a Zipf crowd of fast heavy flows (<= t_ms), and each slow flow a few samples of which most are above t_ms"""
    w = 1.0 / np.arange(1, len(fast) + 1) ** 1.1
    out = []
    for _ in range(nbatches):
        keys = fast[rng.choice(len(fast), per_batch, p=w / w.sum())]
        ms = rng.integers(0, t_ms + 1, per_batch)
        sk = np.repeat(slow, 3)
        sm = np.where(rng.random(len(sk)) < 0.8, rng.integers(t_ms + 1, 4 * t_ms + 2, len(sk)), rng.integers(0, t_ms + 1, len(sk)))
        out.append(samples(np.concatenate([keys, sk]), np.concatenate([ms, sm])))
    return out


@pytest.mark.parametrize("t_ms", [1, 300, 15000])
@pytest.mark.parametrize("k,nslow", [(8, 5), (8, 40), (32, 200)])
def test_window_guarantee_with_slow_clients_in_a_fast_crowd(t_ms, k, nslow):
    rng = np.random.default_rng(k * 100 + nslow + t_ms)
    fast = rng.choice(1 << 40, 2000, replace=False).astype(np.uint64)
    slow = rng.choice(1 << 40, nslow, replace=False).astype(np.uint64) | np.uint64(1 << 41)
    bs = fs.b_slow(t_ms)
    score = fs.scorer(bs)
    sets = fs.Sets(bs, D, W, k)
    table = frh.empty(D, W)
    seen = []
    for b in _window(rng, fast, slow, 4, 400, t_ms):
        table = frh.add_samples(table, b, D, W)
        seen.append(b)
        sets.batch(fs.slow_keys(b, bs), table)
        allb = np.concatenate(seen)
        keys = np.unique(allb["flow_key"])
        assert fs.guarantee_holds(sets.open, table, D, W, score, keys, fs.exact_slow(allb, keys, bs), k)
        # a flow with only fast samples is never listed
        ex_set = fs.exact_slow(allb, np.sort(sets.open), bs)
        assert np.all(ex_set > 0)
    rows = fs.read(sets.open, table, D, W, bs)
    assert np.array_equal(fs.score_of_counts(rows["counts"], bs), score(table, rows["flow_key"], D, W))
    if nslow <= k:
        assert set(slow.tolist()) <= set(sets.open.tolist())


@pytest.mark.parametrize("seq", sorted(fl.SEQUENCES))
def test_level_bound_on_seeded_streams(seq):
    rng = np.random.default_rng(len(seq))
    k, bs = 8, fs.b_slow(300)
    fast = rng.choice(1 << 40, 500, replace=False).astype(np.uint64)
    slow = rng.choice(1 << 40, 60, replace=False).astype(np.uint64) | np.uint64(1 << 41)
    lv = fs.LevelSets(bs, D, W, k)
    tsecs, history = [], []
    for i, t in enumerate(fl.SEQUENCES[seq]):
        sets = fs.Sets(bs, D, W, k)
        table = frh.empty(D, W)
        win = []
        for b in _window(rng, fast, np.roll(slow, 5 * i)[:12], 2, 150, 300):
            table = frh.add_samples(table, b, D, W)
            sets.batch(fs.slow_keys(b, bs), table)
            win.append(b)
        L, B = lv.flush(t, sets.open, table)
        tsecs.append(t)
        history.append(np.concatenate(win))
        held = np.concatenate([history[j] for j in fl.held_windows(tsecs)])
        keys = np.unique(held["flow_key"])
        ex = dict(zip(keys.tolist(), fs.exact_slow(held, keys, bs).tolist()))
        members = set(L.tolist())
        assert all(x <= B for key, x in ex.items() if key not in members), (seq, i)
        assert len(L) <= k


def test_merge_bound():
    rng = np.random.default_rng(9)
    k, world, bs = 8, 3, fs.b_slow(100)
    fast = rng.choice(1 << 40, 800, replace=False).astype(np.uint64)
    slow = rng.choice(1 << 40, 80, replace=False).astype(np.uint64) | np.uint64(1 << 41)
    ranks, tables, allw = [], [], []
    for r in range(world):
        sets, table = fs.Sets(bs, D, W, k), frh.empty(D, W)
        for b in _window(rng, fast, np.roll(slow, 13 * r)[:30], 3, 200, 100):
            table = frh.add_samples(table, b, D, W)
            sets.batch(fs.slow_keys(b, bs), table)
            allw.append(b)
        sets.flush()
        ranks.append(sets.last)
        tables.append(table)
    summed = sum(tables[1:], tables[0].copy())
    g = fs.merged(ranks, summed, D, W, bs, k=k)
    score = fs.scorer(bs)
    thr_sum = sum(fs.thr(s, t, D, W, score, k) for s, t in zip(ranks, tables))
    allw = np.concatenate(allw)
    keys = np.unique(allw["flow_key"])
    union = set(np.concatenate(ranks).tolist())
    for key, x in zip(keys.tolist(), fs.exact_slow(allw, keys, bs).tolist()):
        if x > thr_sum:
            assert key in union
    assert len(g) <= k and set(g.tolist()) <= union


CALLS = ("int		gysk_set_flow_slow(gysk_engine *e, uint32_t above_ms);",
         "int		gysk_topk_flow_slow(gysk_engine *e, int last_window, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout);",
         "int		gysk_topk_flow_slow_global(gysk_engine *e, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout);",
         "int		gysk_topk_flow_slow_5min(gysk_engine *e, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout, uint64_t *bound);",
         "int		gysk_topk_flow_slow_global_5min(gysk_engine *e, uint32_t n, gysk_flow_resp_est *out, uint32_t *nout, uint64_t *bound);")


def test_header_constants_and_bindings():
    with open(os.path.join(ROOT, "include", "gysketch.h")) as f:
        h = f.read()
    assert re.search(r"#define GYSK_FLAG_FLOW_TOPK_SLOW\s+0x1000u", h)
    assert re.search(r"#define GYSK_ABI_VERSION\s+2\b", h)
    for call in CALLS:
        assert call in h, call
    assert "a set scored by the response histograms" not in h
    assert ge.FLAG_FLOW_TOPK_SLOW == 0x1000
    for name in ("set_flow_slow", "topk_flow_slow", "topk_flow_slow_global", "topk_flow_slow_5min", "topk_flow_slow_global_5min"):
        assert callable(getattr(ge.Engine, name))
    with open(os.path.join(ROOT, "gyeeta_b200", "engine.py")) as f:
        src = f.read()
    for sig in ('"gysk_set_flow_slow": (i32, [vp, u32])', '"gysk_topk_flow_slow": (i32, [vp, i32, u32, vp, vp])',
                '"gysk_topk_flow_slow_global": (i32, [vp, u32, vp, vp])', '"gysk_topk_flow_slow_5min": (i32, [vp, u32, vp, vp, vp])',
                '"gysk_topk_flow_slow_global_5min": (i32, [vp, u32, vp, vp, vp])'):
        assert sig in src, sig


def test_library_refuses_the_flag_without_its_prerequisites():
    L = _lib()
    # the configuration check comes before any device is looked for
    for kw, msg in ((dict(flow_queries=True, flow_resp_hist=True), "needs GYSK_FLAG_FLOW_TOPK"),
                    (dict(flow_topk=True, flow_queries=True), "needs GYSK_FLAG_FLOW_RESP_HIST")):
        with pytest.raises(ge.GyskError) as ex:
            ge.Engine(flow_topk_slow=True, **kw)
        assert ex.value.code == -22 and msg in str(ex.value), kw
    assert L.gysk_set_flow_slow(None, 300) == -22
    assert L.gysk_topk_flow_slow(None, 0, 0, None, None) == -22
    assert L.gysk_topk_flow_slow_global(None, 0, None, None) == -22
    for name in ("gysk_topk_flow_slow_5min", "gysk_topk_flow_slow_global_5min"):
        assert getattr(L, name)(None, 0, None, None, None) == -22
