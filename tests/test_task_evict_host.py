"""CPU-side checks (no GPU) of process eviction: the restated rule (tests/task_evict.py) against a restatement of
MCONN_HANDLER::cleanup_partha_unused_aggr_tasks, the configuration field in the ABI, and the new entry points."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests.task_evict import REFERENCE_SECS, TaskEvict, cleanup_rule

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
USEC = 1_000_000


def task_events(ids, hosts, tsec):
    ev = np.zeros(len(ids), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = ids; ev["host_idx"] = hosts; ev["type"] = ge.EV_TASK; ev["tsec"] = tsec; ev["value"] = 7
    return ev


def run(m, script):
    """script: [(tsec, [(id, host)])] -> {tsec: ids evicted by that flush}; also checks each flush against cleanup_rule over the
    model's live processes, their last_tusec_ being the tsec of their last window with samples"""
    out = {}
    for tsec, sends in script:
        if sends:
            ids, hosts = zip(*sends)
            m.ingest(task_events(np.array(ids, dtype=np.uint64), np.array(hosts, dtype=np.uint32), tsec))
        before = dict(m.live)
        host = dict(m.host)
        got = m.flush(tsec)
        # what each partha's walk deletes at now = tsec, with last_tusec_ = the stamp this flush leaves (a window with samples: tsec)
        sent = {i for i, _ in sends}
        parthas = {}
        for i in before:
            parthas.setdefault(host[i], {})[i] = (tsec if i in sent or not before[i] else before[i]) * USEC
        want = sorted(i for ids in cleanup_rule(parthas, tsec * USEC, m.secs).values() for i in ids) if m.secs else []
        assert got == want, tsec
        out[tsec] = got
    return out


def test_the_rule_is_the_reference_walk_thirty_minutes_strict():
    m = TaskEvict(64, REFERENCE_SECS)
    A, B, C_ = 11, 12, 13
    script = [(5, [(A, 0), (B, 0), (C_, 0)]), (10, [(B, 0), (C_, 0)]), (15, [(C_, 0)])]
    script += [(t, [(C_, 0)]) for t in (1800, 1805, 1810, 1815, 1820, 1825)]
    out = run(m, script)
    # A's last window closed at 5: 5 + 1800 < tsec first holds at 1810 (1805 is exactly the limit)
    assert out[1805] == [] and out[1810] == [A]
    assert out[1815] == [B] and out[1820] == [] and out[1825] == []
    assert set(m.live) == {C_}


def test_the_rule_is_per_process_not_per_host():
    """a host whose other process keeps sending does not save its idle ones; an idle host's busy process is not taken with them"""
    m = TaskEvict(64, REFERENCE_SECS)
    script = [(5, [(1, 0), (2, 0), (3, 1), (4, 1)])]
    script += [(t, [(2, 0), (3, 1)]) for t in range(10, 1830, 5)]
    out = run(m, script)
    assert [t for t, ids in out.items() if ids] == [1810] and out[1810] == [1, 4]


def test_gaps_samples_in_the_evicting_window_and_returning_ids():
    m = TaskEvict(4, 20)
    out = run(m, [(5, [(1, 0), (2, 0), (3, 0), (4, 0)]), (10, [(5, 1)]), (400, [(4, 0)]), (405, [(5, 2), (1, 3)])])
    assert m.dropped == 1 and out[400] == [1, 2, 3]
    # 1 returns as a new incarnation: the oracle sees another id with empty histograms, on the host of its new first event
    assert m.oracle_id(1) != 1 and m.host[1] == 3 and int(m.last(1)[0]) == 1 and m.hist(1, ge.HIST_TASK_CPU_PCT)[1] == 1
    assert sorted(m.live) == [1, 4, 5]


def test_zero_never_evicts():
    m = TaskEvict(8, 0)
    out = run(m, [(5, [(1, 0)]), (100000, []), (10 ** 9, [])])
    assert not any(out.values()) and list(m.live) == [1]


def test_config_field_takes_a_reserved_word_and_the_entry_points_exist():
    hdr = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    assert re.search(r"#define GYSK_ABI_VERSION\s+2\b", hdr)
    assert C.sizeof(ge.Config) == 4 * 16
    assert ge.Config.task_idle_evict_secs.offset == ge.Config.idle_evict_secs.offset + 4
    cfg = ge.Config()
    L = ge.load_library()
    L.gysk_config_default(C.byref(cfg))
    assert cfg.task_idle_evict_secs == 0
    for n in ("gysk_evicted_task_ids", "gysk_task_evict_count"):
        assert re.search(r"\bint\s+%s\s*\(" % n, hdr) and hasattr(L, n)
    n = C.c_uint32()
    assert L.gysk_evicted_task_ids(None, None, 0, C.byref(n)) == -22
    assert L.gysk_task_evict_count(None, None) == -22


@pytest.mark.parametrize("hll_p", [4, 12])
def test_slot_bytes_count_the_eviction_arrays_only_when_set(hll_p):
    s0, t0 = ge.slot_bytes(hll_p)
    s1, t1 = ge.slot_bytes(hll_p, 1800)
    assert s1 == s0 and t1 == t0 + 4 + 4 + 8 + 4          # last-active stamp, eviction list slot and id, free stack entry
