"""Process eviction (gysk_config.task_idle_evict_secs) against the CPU oracle with the rule restated over it (tests/task_evict.py). After
every flush of each script: the evicted ids in their order, gysk_task_evict_count, tasks_in_use, every live id's three histograms bit
for bit, its gysk_query_tasks row restated field by field and byte-equal to its gysk_query_task_window row, found = 0 / GYSK_ERR_NOENT
for every evicted id, and gysk_topn_tasks over the live processes only."""
import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from tests.task_evict import TaskEvict
from tests.test_gpu_merge import _emulate_collectives
from tests.test_gpu_merge_exact import _dev_bytes
from tests.test_gpu_topn_global import Ranks, check_topn
from tests.test_gpu_window_read import _pct
from tests.util import assert_hist_equal

HOSTS = 5
KW = dict(max_svcs=256, max_batch=1 << 14, cms_log2_width=10)
WHICH = (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY)
CLS = (6, 3, 3)                 # HASH_1_3000 (cpu %), DURATION_HASH (delays)


def ids_of(n, base):
    return [int(x) for x in synth.splitmix64(np.arange(1, n + 1, dtype=np.uint64) + np.uint64(base)) >> np.uint64(17)]


def task_events(rng, ids, per_id=3, tsec=0):
    ids = np.repeat(np.array(ids, dtype=np.uint64), per_id)
    ev = np.zeros(len(ids), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = ids; ev["type"] = ge.EV_TASK; ev["tsec"] = tsec
    ev["host_idx"] = (ids % np.uint64(HOSTS)).astype(np.uint32)
    ev["value"] = rng.integers(0, 400, len(ev))
    ev["flow_key"] = rng.integers(0, 5000, len(ev)).astype(np.uint64) | (rng.integers(0, 5000, len(ev)).astype(np.uint64) << np.uint64(32))
    return ev[rng.permutation(len(ev))]


def svc_events(rng, ids, per_id=20, tsec=0):
    ids = np.repeat(np.array(ids, dtype=np.uint64), per_id)
    ev = np.zeros(len(ids), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = ids; ev["type"] = ge.EV_RESP; ev["tsec"] = tsec
    ev["host_idx"] = (ids % np.uint64(HOSTS)).astype(np.uint32)
    ev["value"] = rng.lognormal(9.0, 1.5, len(ev)).astype(np.uint32) + 1
    return ev[rng.permutation(len(ev))]


class Pair:
    """an engine and the restated oracle, fed the same device batches"""

    def __init__(self, max_tasks=64, secs=20, idle_evict_secs=0, **kw):
        self.eng = ge.Engine(max_tasks=max_tasks, task_idle_evict_secs=secs, idle_evict_secs=idle_evict_secs, **{**KW, **kw})
        self.m = TaskEvict(max_tasks, secs, max_svcs=self.eng.cfg.max_svcs, cms_log2_width=KW["cms_log2_width"])
        if idle_evict_secs:
            self.m.orc.set_idle_evict(idle_evict_secs)
        self.gone = set()

    def feed(self, ev, batch=1 << 14):
        for off in range(0, len(ev), batch):
            chunk = ev[off: off + batch]
            self.eng.ingest_events(chunk)
            self.eng.sync()
            self.m.ingest(chunk)

    def flush(self, t):
        self.eng.flush(t)
        want = self.m.flush(t)
        self.gone |= set(want)
        self.gone -= set(self.m.live)
        check(self.eng, self.m, self.gone)
        return want


def expected_row(m, id_):
    hists = [m.hist(id_, w) for w in WHICH]
    last = m.last(id_)
    r = ge.TaskSummary(aggr_task_id=id_, found=1, host_idx=m.host[id_])
    r.p95_cpu_pct, r.p95_cpu_delay_ms, r.p95_blkio_delay_ms = [_pct(c, 1, h, [95])[0] for h, c in zip(hists, CLS)]
    r.nsamples = hists[0][1]
    for k in range(3):
        r.last_count[k] = int(last[2 * k])
        r.last_sum[k] = int(last[2 * k + 1].view(np.int64))
    return bytes(r)


def check(eng, m, gone):
    assert eng.evicted_task_ids().tolist() == m.evicted
    assert eng.task_evict_count() == m.total
    assert eng.capacity()["tasks_in_use"] == len(m.live) == eng.stats()["ntasks"]
    live = sorted(m.live)
    for i in live:
        for w in WHICH:
            a, b = eng.export_hist(i, w), m.hist(i, w)
            assert np.array_equal(a[0], b[0]) and a[1:] == b[1:], (hex(i), w)
    rows = [bytes(r) for r in eng.query_tasks(live)] if live else []
    assert rows == [expected_row(m, i) for i in live]
    wrows, n = eng.query_task_window()
    by_id = dict(zip(live, rows))
    assert n == len(live) and [r.aggr_task_id for r in wrows] == sorted(live, key=lambda i: (m.host[i], i))
    assert all(bytes(r) == by_id[r.aggr_task_id] for r in wrows)
    dead = sorted(gone)
    if dead:
        assert [bytes(r) for r in eng.query_tasks(dead)] == [bytes(ge.TaskSummary(aggr_task_id=i)) for i in dead]
        assert all(eng.export_hist(i, w) is None for i in dead for w in WHICH)
    for k in range(3):
        top = eng.topn_tasks(k, 64)                      # every live process of these scripts fits
        want = {(i, int(m.last(i)[2 * k + 1])) for i in live} - {(i, 0) for i in live}
        assert sorted(top) == sorted(want) and not {i for i, _ in top} & gone, k


@pytest.mark.gpu
def test_quiet_exactly_at_the_limit_one_window_before_and_after():
    """X_w sends in windows up to the one closed at w and goes quiet: with 20 s it leaves at the flush w + 25 (w + 20 < tsec), never at w + 20"""
    rng = np.random.default_rng(1)
    p = Pair(max_tasks=64, secs=20)
    xs = {w: ids_of(3, (1 << 40) + w) for w in range(5, 40, 5)}
    keep = ids_of(4, 1 << 41)
    left = {}
    for t in range(5, 90, 5):
        send = keep + [i for w, ids in xs.items() if t <= w for i in ids]
        p.feed(task_events(rng, send, tsec=t))
        for i in p.flush(t):
            left[i] = t
    for w, ids in xs.items():
        assert all(left[i] == w + 25 for i in ids), w
    assert not set(keep) & set(left)


@pytest.mark.gpu
def test_gap_larger_than_the_limit_and_samples_in_the_evicting_window():
    rng = np.random.default_rng(2)
    p = Pair(max_tasks=64, secs=20)
    a, b, c = ids_of(10, 1 << 42), ids_of(10, 1 << 43), ids_of(5, 1 << 44)
    p.feed(task_events(rng, a + b + c, tsec=5))
    p.flush(5)
    p.feed(task_events(rng, a + c, tsec=10))
    p.flush(10)
    p.feed(task_events(rng, c, tsec=500))            # c sends in the window the flush at 500 closes: kept
    assert p.flush(500) == sorted(a + b)
    assert set(p.m.live) == set(c)
    p.flush(521)                                     # 500 + 20 < 521
    assert not p.m.live


@pytest.mark.gpu
def test_returning_ids_and_new_ids_take_recycled_slots_and_a_full_table_takes_ids_again():
    rng = np.random.default_rng(3)
    p = Pair(max_tasks=32, secs=10)
    a, b, new = ids_of(16, 1 << 45), ids_of(16, 1 << 46), ids_of(24, 1 << 47)
    t = 5
    p.feed(task_events(rng, a + b, tsec=t)); p.flush(t)
    # full: the first 8 new ids are dropped on both sides
    t += 5; p.feed(task_events(rng, b + new[:8], tsec=t)); p.flush(t)
    assert p.eng.stats()["events_dropped"] == p.m.dropped == 8 * 3
    for _ in range(3):
        t += 5; p.feed(task_events(rng, b, tsec=t)); p.flush(t)
    assert set(a) <= p.gone
    # a's 16 slots are free again: a returns (empty histograms) beside 8 new ids, then 8 more find the table full
    t += 5; p.feed(task_events(rng, a[:8] + new[8:16] + b, tsec=t)); p.flush(t)
    t += 5; p.feed(task_events(rng, new[16:24] + b, tsec=t)); p.flush(t)
    assert p.eng.stats()["events_dropped"] == p.m.dropped == 16 * 3
    assert p.eng.capacity()["max_tasks"] == 32


@pytest.mark.gpu
def test_services_and_processes_evicted_by_the_same_flush():
    rng = np.random.default_rng(4)
    p = Pair(max_tasks=64, secs=20, idle_evict_secs=20)
    svcs, tasks = ids_of(30, 1 << 38), ids_of(30, 1 << 39)
    for t in range(5, 120, 5):
        sv = svcs if t < 20 else svcs[:10]
        tk = tasks if t < 20 else tasks[10:]
        p.feed(np.concatenate([svc_events(rng, sv, tsec=t), task_events(rng, tk, tsec=t)]))
        p.flush(t)
        assert sorted(p.eng.evicted_ids().tolist()) == sorted(p.m.orc.evicted_ids()[0].tolist())
        for i in svcs:
            assert_hist_equal(p.eng, p.m.orc, i, ge.HIST_RESP_ALL)
    assert set(tasks[:10]) <= p.gone and p.eng.stats()["svcs_evicted"] == 20


@pytest.mark.gpu
def test_eviction_between_two_batches_of_hot_rows():
    """services hot enough for the dense rows in the batches before and after a flush that evicts processes"""
    rng = np.random.default_rng(5)
    p = Pair(max_tasks=64, secs=10)
    hot, tasks = ids_of(3, 1 << 37), ids_of(20, 1 << 36)
    for t, tk in ((5, tasks), (10, tasks[:5]), (15, tasks[:5]), (20, tasks[:5]), (25, tasks[:5])):
        p.feed(np.concatenate([svc_events(rng, hot, per_id=6000, tsec=t), task_events(rng, tk, tsec=t)]), batch=1 << 14)
        p.flush(t)
    assert p.eng.hot_rows_in_use() > 0 and set(tasks[5:]) <= p.gone
    for i in hot:
        for w in (0, 1, 2):
            assert_hist_equal(p.eng, p.m.orc, i, w)


@pytest.mark.gpu
def test_grow_after_an_eviction_keeps_the_free_stack():
    rng = np.random.default_rng(6)
    p = Pair(max_tasks=32, secs=10)
    a, b, new = ids_of(20, 1 << 35), ids_of(12, 1 << 34), ids_of(40, 1 << 33)
    p.feed(task_events(rng, a + b, tsec=5)); p.flush(5)
    for t in (10, 15, 20):
        p.feed(task_events(rng, b, tsec=t)); p.flush(t)
    assert set(a) <= p.gone and p.eng.capacity()["tasks_in_use"] == 12
    p.eng.grow(max_tasks=64)
    p.m.max_tasks = 64
    check(p.eng, p.m, p.gone)
    p.feed(task_events(rng, b + new, tsec=25)); p.flush(25)          # 20 recycled slots, then 20 fresh ones
    assert p.eng.capacity()["tasks_in_use"] == 52 and p.eng.stats()["events_dropped"] == 0


@pytest.mark.gpu
def test_auto_grow_does_not_fire_when_eviction_freed_the_table():
    rng = np.random.default_rng(7)
    a, b, c = ids_of(20, 1 << 32), ids_of(10, 1 << 31), ids_of(10, 1 << 30)
    caps = {}
    for secs in (0, 10):
        p = Pair(max_tasks=64, secs=secs)
        p.eng.set_auto_grow(0, 256)
        p.feed(task_events(rng, a + b, tsec=5)); p.flush(5)             # 30 of 64
        for t in (10, 15, 20):                                          # a leaves at 20
            p.feed(task_events(rng, b, tsec=t)); p.flush(t)
        for t in (25, 30, 35):                                          # 40 of 64 without the eviction: past half
            p.feed(task_events(rng, b + c, tsec=t)); p.flush(t)
        caps[secs] = p.eng.capacity()
    assert caps[0]["max_tasks"] == 128 and caps[0]["ngrows"] == 1
    assert caps[10]["max_tasks"] == 64 and caps[10]["ngrows"] == 0 and caps[10]["tasks_in_use"] == 20


@pytest.mark.gpu
def test_off_by_default_and_a_rule_that_never_fires_answer_alike():
    """task_idle_evict_secs = 0 against a limit no flush reaches: every task read and merge array byte-equal"""
    import torch
    rng = np.random.default_rng(8)
    e0 = ge.Engine(max_tasks=64, merge_topn=True, **KW)
    e1 = ge.Engine(max_tasks=64, merge_topn=True, task_idle_evict_secs=1 << 30, **KW)
    assert ge.slot_bytes(12)[1] + 20 == ge.slot_bytes(12, 1)[1]
    ids, svcs = ids_of(40, 1 << 30), ids_of(20, 1 << 29)
    for t in (5, 10, 400):
        ev = np.concatenate([svc_events(rng, svcs, tsec=t), task_events(rng, ids[: 40 - t // 20], tsec=t)])
        for e in (e0, e1):
            e.ingest_events(ev); e.sync(); e.flush(t)
        assert [bytes(r) for r in e0.query_task_window()[0]] == [bytes(r) for r in e1.query_task_window()[0]]
        assert [bytes(r) for r in e0.query_tasks(ids)] == [bytes(r) for r in e1.query_tasks(ids)]
        assert all(e0.topn_tasks(k, 64) == e1.topn_tasks(k, 64) for k in range(3))
        assert all(np.array_equal(e0.export_hist(i, w)[0], e1.export_hist(i, w)[0]) for i in ids for w in WHICH)
        assert e1.evicted_task_ids().size == 0 and e1.task_evict_count() == 0 and e0.task_evict_count() == 0
        for e in (e0, e1):
            _emulate_collectives(torch, [e])
        b0, b1 = e0.merge_buffers(), e1.merge_buffers()
        assert [(n, nb, op) for n, _, nb, op in b0] == [(n, nb, op) for n, _, nb, op in b1]
        for (name, p0, nb, _), (_, p1, _, _) in zip(b0, b1):
            assert np.array_equal(_dev_bytes(torch, p0, nb), _dev_bytes(torch, p1, nb)), name
        for k in range(3):
            g0, r0 = e0.topn_global_tasks(k, 64)
            g1, r1 = e1.topn_global_tasks(k, 64)
            assert [bytes(x) for x in g0] == [bytes(x) for x in g1] and [bytes(x) for x in r0] == [bytes(x) for x in r1]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_merged_top_processes_never_list_an_evicted_one(world):
    import torch
    rng = np.random.default_rng(9 + world)
    sh = Ranks(world, task_idle_evict_secs=20, merge_topn=True)
    ids = ids_of(60, 1 << 28)
    gone = set()
    for t in (5, 10, 15, 20, 25, 30, 35, 40, 45):
        send = ids if t <= 10 else ids[: 60 - 4 * (t // 5)]
        ev = task_events(rng, send, tsec=t)
        ev["host_idx"] = (ev["svc_id"] % np.uint64(2 * world + 1)).astype(np.uint32)
        sh.feed(ev)
        sh.flush(t)
        for e in sh.engines:
            gone |= set(e.evicted_task_ids().tolist())
        check_topn(torch, sh.engines)
        for e in sh.engines:
            for k in range(3):
                got, rows = e.topn_global_tasks(k, 64)
                assert not {x.glob_id for x in got} & gone and not {r.aggr_task_id for r in rows} & gone
    assert len(gone) >= 20
