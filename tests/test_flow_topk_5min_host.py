"""The 300-s heaviest-flow rule of GYSK_FLAG_FLOW_TOPK_5MIN on the CPU: the restatement of tests/flow_topk_5min.py on scripted and
seeded count-min streams keeps its stated properties (every flow outside L scores at most B_L over the level, a slot's threshold never
falls within its epoch, the merge's bound), including a steady-client stream that no window ranks and a slot expiry that the rejected
"old L u closing window" rule gets wrong; and the header, the Python constant and the bindings pin the ABI."""
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import flow_level as fl
from tests import flow_topk as ft
from tests import flow_topk_5min as f5

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, W = 4, 10
KB = np.uint64(32)              # the kbytes half: scores are the high half of each increment


class Stream:
    """one level fed window by window: each window a list of batches of (keys, kbytes), its set restated as the engine keeps it"""

    def __init__(self, k, d=D, w=W):
        self.k, self.d, self.w = k, d, w
        self.lv = f5.LevelSets(1, d, w, k)
        self.tsecs, self.windows = [], []

    def window(self, tsec, batches):
        sets = ft.Sets(1, self.d, self.w, self.k)
        table = np.zeros(self.d << self.w, dtype=np.uint64)
        exact = {}
        for keys, kb in batches:
            keys = np.asarray(keys, dtype=np.uint64)
            table = table + f5.table_of(keys, np.asarray(kb, dtype=np.uint64) << KB, self.d, self.w)
            sets.batch(np.unique(keys), table)
            for key, x in zip(keys.tolist(), np.asarray(kb).tolist()):
                exact[key] = exact.get(key, 0) + int(x)
        self.tsecs.append(tsec)
        self.windows.append(exact)
        return self.lv.flush(tsec, sets.open, table), sets.open

    def exact(self):
        return f5.exact_level(self.tsecs, self.windows)

    def check(self, what):
        L, B = self.lv.L, self.lv.B
        assert f5.guarantee_holds(L, B, self.exact()), what
        by_slot = {}
        for s, ep, t in self.lv.slot_thr:                   # a slot's threshold never falls within its epoch
            if by_slot.get(s, (None, 0))[0] == ep:
                assert t >= by_slot[s][1], (what, s, ep)
            by_slot[s] = (ep, t)


def _zipf_batches(rng, flows, nbatches, per_batch):
    w = 1.0 / np.arange(1, len(flows) + 1) ** 1.1
    return [(flows[rng.choice(len(flows), per_batch, p=w / w.sum())], rng.integers(0, 64, per_batch)) for _ in range(nbatches)]


@pytest.mark.parametrize("seq", sorted(fl.SEQUENCES))
@pytest.mark.parametrize("k,nflows", [(8, 300), (32, 4000), (64, 40)])
def test_bound_holds_on_seeded_streams(seq, k, nflows):
    rng = np.random.default_rng(k * 1000 + nflows + len(seq))
    flows = rng.choice(1 << 40, nflows, replace=False).astype(np.uint64)
    st = Stream(k)
    for i, t in enumerate(fl.SEQUENCES[seq]):
        # the heavy flows drift: each window favours a rotated part of the population
        st.window(t, _zipf_batches(rng, np.roll(flows, 7 * i), 3, 200))
        st.check((seq, k, i))
        assert len(st.lv.L) <= k and len(set(st.lv.L.tolist())) == len(st.lv.L)


def test_steady_clients_no_window_ranks():
    """60 windows over 300 s: 40 steady clients send 10 kB each window, and each window brings its own 8 bursts of 50 kB. No window's
    set holds a steady client, so L holds none, yet they are the heaviest of the five minutes: the bound covers them, and is large."""
    k = 8
    steady = np.arange(1, 41, dtype=np.uint64)
    st = Stream(k)
    for i in range(60):
        burst = np.arange(1000 + 8 * i, 1008 + 8 * i, dtype=np.uint64)
        (_, _), win = st.window(5 * (i + 1), [(np.concatenate([steady, burst]), np.r_[np.full(40, 10), np.full(8, 50)])])
        assert not set(win.tolist()) & set(steady.tolist())
        st.check(i)
    ex = st.exact()
    top = max(ex.values())
    assert all(ex[int(s)] == top for s in steady) and top > 50
    assert not set(st.lv.L.tolist()) & set(steady.tolist())
    assert st.lv.B >= top and st.lv.B >= 8 * 50


def _old_rule(L, win, level, k):
    """the rejected rule: the K best of the old L and the closing window's set, on the level"""
    return ft.select(np.concatenate([L, np.asarray(win, dtype=np.uint64)]), level, D, W, 1, k)


def test_expired_leaders_slot_lists_the_flow_cut_beside_them():
    """K = 2. Two leaders send once at 5 s; f sends once at 35 s and is cut from L while they lead; small flows follow. At 305 s the
    leaders' slot expires: this rule lists f, the heaviest of the five minutes, and the old-L-u-window rule has lost it."""
    k = 2
    a1, a2, f, g = 11, 12, 13, 14
    st = Stream(k)
    old = np.zeros(0, dtype=np.uint64)
    script = [(5, [a1, a2], [100, 100]), (35, [f, g], [80, 1])] + \
             [(65 + 30 * i, [100 + 2 * i, 101 + 2 * i], [1, 1]) for i in range(8)] + [(305, [21, 22], [5, 5])]
    for t, keys, kb in script:
        (L, B), win = st.window(t, [(np.asarray(keys, dtype=np.uint64), np.asarray(kb))])
        old = _old_rule(old, win, st.lv.level, k)
        st.check(t)
        if t == 35:
            assert f not in L.tolist() and set(L.tolist()) == {a1, a2}
    ex = st.exact()
    assert max(ex, key=lambda x: ex[x]) == f and a1 not in ex
    assert f in st.lv.L.tolist()
    assert f not in old.tolist()
    # and what the old rule leaves out can exceed any bound it could state from the sets it keeps
    assert ex[f] > f5.thr(old, st.lv.level, D, W, 1, k)


def test_merge_bound():
    """a flow whose exact score over every rank's level exceeds B_G is in G"""
    rng = np.random.default_rng(5)
    k, world = 16, 3
    flows = rng.choice(1 << 40, 2000, replace=False).astype(np.uint64)
    ranks = [Stream(k) for _ in range(world)]
    for i, t in enumerate(fl.SEQUENCES["steps_5s"][:30]):
        for r, st in enumerate(ranks):
            st.window(t, _zipf_batches(rng, np.roll(flows, 11 * i + 100 * r), 2, 150))
    summed = sum((st.lv.level for st in ranks[1:]), ranks[0].lv.level.copy())
    g, bg = f5.merged([st.lv.L for st in ranks], [st.lv.B for st in ranks], summed, D, W, 1, k)
    ex = {}
    for st in ranks:
        for key, x in st.exact().items():
            ex[key] = ex.get(key, 0) + x
    assert len(g) == k and bg >= sum(st.lv.B for st in ranks)
    assert f5.guarantee_holds(g, bg, ex)


def test_header_constants_and_bindings():
    with open(os.path.join(ROOT, "include", "gysketch.h")) as f:
        h = f.read()
    assert re.search(r"#define GYSK_FLAG_FLOW_TOPK_5MIN\s+0x800u", h)
    assert re.search(r"#define GYSK_ABI_VERSION\s+2\b", h)
    for call in ("int		gysk_topk_flows_5min(gysk_engine *e, uint32_t n, gysk_flow_est *out, uint32_t *nout, uint64_t *bound);",
                 "int		gysk_topk_flow_queries_5min(gysk_engine *e, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout, uint64_t *bound);",
                 "int		gysk_topk_flows_global_5min(gysk_engine *e, uint32_t n, gysk_flow_est *out, uint32_t *nout, uint64_t *bound);",
                 "int		gysk_topk_flow_queries_global_5min(gysk_engine *e, uint32_t n, gysk_flow_qry_est *out, uint32_t *nout, uint64_t *bound);"):
        assert call in h, call
    assert "sets for the 300-s levels" not in h
    assert ge.FLAG_FLOW_TOPK_5MIN == 0x800
    names = ("topk_flows_5min", "topk_flow_queries_5min", "topk_flows_global_5min", "topk_flow_queries_global_5min")
    for name in names:
        assert callable(getattr(ge.Engine, name))
    with open(os.path.join(ROOT, "gyeeta_b200", "engine.py")) as f:
        src = f.read()
    for name in names:
        assert f'"gysk_{name}": (i32, [vp, u32, vp, vp, vp])' in src


def test_library_refuses_the_flag_without_its_prerequisites():
    lib = os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    # the configuration check comes before any device is looked for
    for kw, msg in ((dict(flow_level=True), "needs GYSK_FLAG_FLOW_TOPK"), (dict(flow_topk=True), "needs GYSK_FLAG_FLOW_LEVEL or"),
                    (dict(flow_topk=True, flow_queries=True), "needs GYSK_FLAG_FLOW_LEVEL or")):
        with pytest.raises(ge.GyskError) as ex:
            ge.Engine(flow_topk_5min=True, **kw)
        assert ex.value.code == -22 and msg in str(ex.value), kw
    L = ge.load_library()
    for name in ("gysk_topk_flows_5min", "gysk_topk_flow_queries_5min", "gysk_topk_flows_global_5min", "gysk_topk_flow_queries_global_5min"):
        assert getattr(L, name)(None, 0, None, None, None) == -22
