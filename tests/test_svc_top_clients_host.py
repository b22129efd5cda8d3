"""GYSK_FLAG_SVC_TOP_CLIENTS on the CPU: the restated merge (tests/svc_top_clients.py) keeps its four guarantees on seeded streams of
every shape, for any split of a stream into batches and windows, and saturates as the header says; the header's constants and row
layout, and the ctypes binding, match."""
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import svc_top_clients as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = tc.K


def _stream(rng, shape, n=4000):
    """(flow keys, kbytes) of n records of one service"""
    if shape == "zipf":
        keys = rng.zipf(1.3, n) % 5000
    elif shape == "uniform":
        keys = rng.integers(0, 400, n)
    elif shape == "single":
        keys = np.zeros(n, dtype=np.int64)
    elif shape.startswith("clients_"):
        keys = rng.integers(0, int(shape[len("clients_"):]), n)
    elif shape == "ties":
        keys = np.arange(n) % (3 * K)           # every client the same volume
        return keys.astype(np.uint64) + np.uint64(7), np.full(n, 5, dtype=np.int64)
    else:
        raise AssertionError(shape)
    kb = rng.integers(0, 64, n)
    kb[rng.random(n) < 0.1] = 0                 # records below one kbyte
    return keys.astype(np.uint64) + np.uint64(7), kb


SHAPES = ["zipf", "uniform", "single", f"clients_{K - 1}", f"clients_{K}", f"clients_{K + 1}", f"clients_{3 * K}", "ties"]


def _sums(keys, kb):
    d = {}
    for k, v in zip(keys.tolist(), kb.tolist()):
        a = d.setdefault(k, [0, 0])
        a[0] += v
        a[1] += 1
    return d


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("nbatch", [1, 3, 17])
def test_guarantees_over_any_batch_split(shape, nbatch):
    rng = np.random.default_rng(hash((shape, nbatch)) % 2**32)
    keys, kb = _stream(rng, shape)
    cuts = np.sort(rng.choice(np.arange(1, len(keys)), nbatch - 1, replace=False)) if nbatch > 1 else []
    s = tc.EMPTY
    for a, b in zip([0, *cuts], [*cuts, len(keys)]):
        s = tc.merge([s], _sums(keys[a:b], kb[a:b]))
        tc.check_guarantees(s, _sums(keys[:b], kb[:b]))
    ents, delta = s
    assert list(ents) == sorted(ents, key=lambda e: (-e[1], e[0])) and len(ents) <= K
    assert all(e[1] > 0 for e in ents)


@pytest.mark.parametrize("shape", SHAPES)
def test_window_merges_keep_the_guarantees(shape):
    """summaries of several windows merged (a ring slot, the level) keep the guarantees over the union of their records"""
    rng = np.random.default_rng(11)
    parts = [_stream(rng, shape, 1500) for _ in range(5)]
    sums = [tc.merge([tc.EMPTY], _sums(k, v)) for k, v in parts]
    allk = np.concatenate([k for k, _ in parts])
    allv = np.concatenate([v for _, v in parts])
    tc.check_guarantees(tc.merge(sums), _sums(allk, allv))
    tc.check_guarantees(tc.merge([tc.merge(sums[:2]), tc.merge(sums[2:])]), _sums(allk, allv))


def test_few_clients_are_exact():
    d = {5: (10, 2), 9: (10, 1), 3: (4, 3)}
    ents, delta = tc.merge([tc.EMPTY], d)
    assert delta == 0 and ents == ((5, 10, 2), (9, 10, 1), (3, 4, 3))


def test_merge_rule_on_k_plus_one():
    d = {i: (100 + i, 1) for i in range(K + 1)}                 # K + 1 clients: c = the smallest, 100
    ents, delta = tc.merge([tc.EMPTY], d)
    assert delta == 100 and len(ents) == K and ents[0] == (K, K, 1) and ents[-1] == (1, 1, 1)


def test_zero_kbyte_pairs_enter_only_with_an_old_entry():
    s = tc.merge([tc.EMPTY], {1: (5, 1)})
    s = tc.merge([s], {1: (0, 4), 2: (0, 9)})
    assert s == (((1, 5, 5),), 0)


def test_saturation():
    big = 3 << 32
    ents, delta = tc.merge([tc.EMPTY], {1: (big, 1), 2: (big + 1, (1 << 33))})
    assert ents == ((2, tc.M32, tc.M32), (1, tc.M32, 1)) and delta == 0


def test_ring_restatement_follows_the_level_rule():
    """TopClients: a slot holding an older epoch is replaced, the level merges the live slots only"""
    t = tc.TopClients()
    ev = np.zeros(2, dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["type"], ev["flow_key"], ev["value"] = 77, ge.EV_CONNECT, [1, 2], [4096, 2048]
    t.batch(ev)
    t.flush(30)
    assert t.get(ge.TOPC_LAST, 77) == (((1, 4, 1), (2, 2, 1)), 0) and t.get(ge.TOPC_5MIN, 77) == t.get(ge.TOPC_LAST, 77)
    t.flush(35)
    assert t.get(ge.TOPC_LAST, 77) == tc.EMPTY and t.get(ge.TOPC_5MIN, 77) == (((1, 4, 1), (2, 2, 1)), 0)
    t.flush(30 + 300)                   # epoch 11 takes slot 1 from epoch 1
    assert t.get(ge.TOPC_5MIN, 77) == tc.EMPTY


def test_header_and_binding():
    with open(os.path.join(ROOT, "include", "gysketch.h")) as f:
        h = f.read()
    assert re.search(r"#define GYSK_FLAG_SVC_TOP_CLIENTS\s+0x8000u", h)
    assert re.search(r"#define GYSK_SVC_TOPC_K\s+16u", h)
    for name, v in (("OPEN", 0), ("LAST", 1), ("5MIN", 2)):
        assert re.search(rf"#define GYSK_TOPC_{name}\s+{v}\b", h)
        assert getattr(ge, f"TOPC_{name}") == v
    body = re.search(r"typedef struct gysk_svc_top_clients\s*\{(.*?)\}", h, re.S).group(1)
    fields = re.findall(r"^\s*(\w+)\s+(\w+)", body, re.M)
    assert [f for _, f in fields] == list(ge.SVC_TOP_CLIENTS_DTYPE.names)
    ent = re.search(r"typedef struct gysk_topc_entry\s*\{(.*?)\}", h, re.S).group(1)
    assert [f for _, f in re.findall(r"^\s*(\w+)\s+(\w+)", ent, re.M)] == list(ge.TOPC_ENTRY_DTYPE.names)
    assert ge.TOPC_ENTRY_DTYPE.itemsize == 16 and ge.SVC_TOP_CLIENTS_DTYPE.itemsize == 8 + 4 + 4 + 8 + K * 16
    assert ge.FLAG_SVC_TOP_CLIENTS == 0x8000 and ge.TOPC_K == 16
    for fn in ("gysk_query_svc_top_clients", "gysk_query_top_clients_window"):
        assert re.search(rf"\bint\s+{fn}\(", h)


def _lib():
    if not os.path.exists(os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")):
        pytest.skip("library not built")
    return ge.load_library()


def test_flag_passes_the_configuration_check_and_counts_its_slot_bytes():
    L = _lib()
    import ctypes as C
    try:
        ge.Engine(max_svcs=16, max_tasks=16, max_batch=1024, cms_log2_width=4, svc_top_clients=True).close()
    except ge.GyskError as ex:
        assert ex.code == -19                   # NODEV: past the configuration check
    cfg = ge.Config()
    L.gysk_config_default(C.byref(cfg))
    a, b, a2, b2 = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
    assert L.gysk_slot_bytes(C.byref(cfg), C.byref(a), C.byref(b)) == 0
    cfg.flags |= ge.FLAG_SVC_TOP_CLIENTS
    assert L.gysk_slot_bytes(C.byref(cfg), C.byref(a2), C.byref(b2)) == 0
    assert a2.value - a.value == 13 * 264 and b2.value == b.value
