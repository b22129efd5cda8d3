"""CPU-side checks (no GPU) of table growth: the new entry points are exported and declared, answer GYSK_ERR_INVAL without an engine, and
gysk_slot_bytes equals the sum of the per-slot arrays gysk_create allocates, restated here array by array."""
import ctypes as C
import os
import re

import pytest

from gyeeta_b200 import engine as ge

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("gysk_grow", "gysk_set_auto_grow", "gysk_capacity_info", "gysk_slot_bytes")

# bytes per service slot of each array gysk_create sizes by max_svcs + 1 (the level ring: by max_svcs, NLEVELS x NSLOTS rows of 16 cells)
HIST = 16 * 16                       # one histogram: 16 cells of {u64 count, i64 sum}
SVC_ARRAYS = dict(slot_id=8, slot_host=4, slot_first_seen=4, slot_last_active=4, evict_list=4, evict_ids=8, free_slots=4,
                  hist_cur=HIST, hist_last=HIST, hist_all=HIST, level_ring=2 * 10 * HIST, conn_cur=8, conn_last=8, conn_all_cnt=8,
                  conn_all_kb=8, bm_cur=16 * 4, bm_last=16 * 4, td_cent=256 * 16, td_head=32, slot_batch=16, slot_aux=40, qps_hist=HIST,
                  act_hist=HIST, slot_state=8, sort_touched=4, sort_segs=16)
TASK_ARRAYS = dict(task_hist=3 * HIST, task_prev=3 * 16, task_last=3 * 16, task_slot_id=8, task_slot_host=4)


def test_growth_symbols_are_exported_and_declared():
    hdr = open(os.path.join(ROOT, "include", "gysketch.h")).read()
    L = C.CDLL(ge.LIB_PATH)
    for n in NEW:
        assert re.search(r"\b%s\s*\(" % n, hdr), n
        assert hasattr(L, n), n
    assert "typedef struct gysk_capacity" in hdr and C.sizeof(ge.Capacity) == 32
    L = ge.load_library()
    assert L.gysk_grow(None, 1, 1) == -22
    assert L.gysk_set_auto_grow(None, 0, 0) == -22
    assert L.gysk_capacity_info(None, None) == -22
    assert L.gysk_slot_bytes(None, None, None) == -22


@pytest.mark.parametrize("hll_p", [4, 12, 16])
def test_slot_bytes_are_the_sum_of_the_per_slot_allocations(hll_p):
    svc, task = ge.slot_bytes(hll_p)
    assert svc == sum(SVC_ARRAYS.values()) + (1 << hll_p)
    assert task == sum(TASK_ARRAYS.values())
    # the defaults of gysk_config_default (NULL configuration): hll_p 12, about 15 KB a service slot
    s, t = C.c_uint64(), C.c_uint64()
    assert ge.load_library().gysk_slot_bytes(None, C.byref(s), C.byref(t)) == 0
    assert (s.value, t.value) == ge.slot_bytes(12) and 14_000 < s.value < 16_000


def test_slot_bytes_rejects_a_bad_configuration():
    cfg = ge.Config()
    L = ge.load_library()
    L.gysk_config_default(C.byref(cfg))
    s, t = C.c_uint64(), C.c_uint64()
    cfg.hll_p = 17
    assert L.gysk_slot_bytes(C.byref(cfg), C.byref(s), C.byref(t)) == -22
    cfg.hll_p, cfg.struct_size = 12, 8
    assert L.gysk_slot_bytes(C.byref(cfg), C.byref(s), C.byref(t)) == -22
