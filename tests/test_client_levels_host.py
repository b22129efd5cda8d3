"""GYSK_FLAG_CLIENT_LEVELS on the CPU: the fold of p-registers to p = 8 against the oracle's registers at 8, the accuracy bound the GPU
tests hold the estimates to, the restatement's window and level rule, and the header and ctypes layout of the new calls."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests.client_levels import BOUND, NREG, P, History, fold_registers, window_keys
from tests.flow_level import SEQUENCES

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "gysketch.h")


def _keysets(seed):
    rng = np.random.default_rng(seed)
    rand = rng.integers(1, 1 << 64, 20000, dtype=np.uint64)
    ip = (np.uint64(0x0A000000) + rng.integers(0, 300, 20000).astype(np.uint64)) << np.uint64(32)
    ipport = ip | rng.integers(1024, 65536, 20000).astype(np.uint64)
    return {"random": rand, "ip_port": ipport}


def _capped_keys(p):
    """keys whose mixed hash leaves the bits after the top p all zero or nearly so: the rank cap 64 - p + 1 and its neighbours"""
    out = []
    lib = po.lib()
    idx, rank = C.c_uint32(), C.c_uint8()
    # search a small space for keys of high rank at p (rank > 20 is rare, so take the highest ranks found)
    keys = np.random.default_rng(p).integers(1, 1 << 64, 400000, dtype=np.uint64)
    for k in keys:
        lib.gyo_hll_idx_rank(C.c_uint64(int(k)), p, C.byref(idx), C.byref(rank))
        if rank.value >= 14:
            out.append(k)
    return np.array(out, dtype=np.uint64)


@pytest.mark.parametrize("p", [8, 12, 16])
@pytest.mark.parametrize("kind", ["random", "ip_port"])
def test_fold_equals_the_registers_at_8(p, kind):
    keys = _keysets(p)[kind]
    for n in (1, 10, 300, 5000, 20000):
        a = po.hll_registers(keys[:n], p)
        assert fold_registers(a, p).tobytes() == po.hll_registers(keys[:n], P).tobytes(), (p, kind, n)


@pytest.mark.parametrize("p", [8, 12, 16])
def test_fold_at_high_ranks(p):
    keys = _capped_keys(p)
    assert len(keys) > 0
    a = po.hll_registers(keys, p)
    assert a.max() >= 14
    assert fold_registers(a, p).tobytes() == po.hll_registers(keys, P).tobytes()


def test_fold_at_the_rank_cap():
    """a register at the cap 64 - p + 1 (the hash's bits after the top p all zero) folds to the cap at 8, 57"""
    for p in (12, 16):
        regs = np.zeros(1 << p, np.uint8)
        regs[5 << (p - P)] = 64 - p + 1                 # child x = 0 of register 5
        regs[(7 << (p - P)) | 1] = 64 - p + 1           # child x = 1 of register 7: its rank at 8 is p - 8
        f = fold_registers(regs, p)
        assert f[5] == 57 and f[7] == p - P and f.sum() == 57 + p - P


def test_estimate_bound_at_8():
    """every estimate from 1 to 10^5 exact distinct keys, three key streams: within BOUND = 4 sigma of the exact count"""
    for seed in range(3):
        keys = np.random.default_rng(seed).integers(1, 1 << 62, 100000, dtype=np.uint64)
        regs = np.zeros(NREG, np.uint8)
        prev = 0
        for n in list(range(1, 200)) + list(np.unique(np.geomspace(200, 100000, 200).astype(int))):
            po.hll_registers(keys[prev:n], P, regs)
            prev = n
            est = po.hll_estimate(regs, P)
            assert abs(est - n) <= BOUND * n, (seed, n, est)


def test_window_keys_count_connections_only():
    ev = np.zeros(8, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = [1, 1, 1, 1, 1, 2, 2, 0]
    ev["flow_key"] = [10, 11, 12, 13, 14, 20, 21, 30]
    ev["type"] = [ge.EV_CONNECT, ge.EV_ACCEPT, ge.EV_CLOSE_CLI, ge.EV_RESP, ge.EV_ACTIVE, ge.EV_CLOSE_SER, ge.EV_TRACE, ge.EV_CONNECT]
    got = window_keys(ev)
    assert sorted(got) == [1, 2] and got[1].tolist() == [10, 11, 12, 14] and got[2].tolist() == [20]


@pytest.mark.parametrize("name", sorted(SEQUENCES))
def test_level_is_the_maximum_of_the_held_windows(name):
    """the restatement's level equals a ring kept slot by slot (max-merge into slot (tsec / 30) % 10, a slot of another epoch replaced,
    the level the maximum of the slots of the last 10 epochs)"""
    rng = np.random.default_rng(len(name))
    h = History()
    ring, epochs = np.zeros((10, NREG), np.uint8), [None] * 10
    for t in SEQUENCES[name]:
        ev = np.zeros(300, dtype=ge.EVENT_DTYPE)
        ev["svc_id"], ev["type"] = 7, ge.EV_ACCEPT
        ev["flow_key"] = rng.integers(1, 1 << 62, 300, dtype=np.uint64)
        h.flush(t, ev)
        ep, k = t // 30, (t // 30) % 10
        if epochs[k] != ep:
            ring[k], epochs[k] = 0, ep
        np.maximum(ring[k], po.hll_registers(ev["flow_key"], P), out=ring[k])
        level = np.zeros(NREG, np.uint8)
        for j in range(10):
            if epochs[j] is not None and ep - 10 < epochs[j] <= ep:
                np.maximum(level, ring[j], out=level)
        assert h.level(7).tobytes() == level.tobytes(), (name, t)


def _header():
    return open(HEADER).read()


def test_header_pins():
    h = _header()
    assert re.search(r"#define GYSK_FLAG_CLIENT_LEVELS\s+0x2000u", h)
    assert re.search(r"#define GYSK_HLL_WINDOW_P\s+8u", h)
    assert re.search(r"#define GYSK_CLIENTS_LAST\s+0\b", h) and re.search(r"#define GYSK_CLIENTS_5MIN\s+1\b", h)
    body = re.search(r"typedef struct gysk_svc_clients\s*\{(.*?)\}\s*gysk_svc_clients;", h, re.S).group(1)
    fields = re.findall(r"(uint64_t|int32_t|uint32_t|double)\s+(\w+);", body)
    assert fields == [("uint64_t", "glob_id"), ("int32_t", "found"), ("uint32_t", "pad"), ("double", "last_5s"), ("double", "last_5min")]
    for decl in ("int\t\tgysk_query_svc_clients(gysk_engine *e, const uint64_t *ids, uint32_t n, gysk_svc_clients *out);",
                 "int\t\tgysk_export_hll_window(gysk_engine *e, uint64_t glob_id, int which, uint8_t regs[256]);",
                 "int\t\tgysk_query_logical_clients(gysk_engine *e, const uint64_t *logical_ids, uint32_t n, gysk_svc_clients *out);",
                 "int\t\tgysk_export_logical_hll_window(gysk_engine *e, uint64_t logical_id, int which, uint8_t regs[256]);"):
        assert decl in h, decl
    assert "int\t\tgysk_query_clients_window(gysk_engine *e, int32_t host_idx, uint32_t flags, gysk_svc_clients *out, uint32_t *hosts," in h


def test_ctypes_binding():
    assert ge.FLAG_CLIENT_LEVELS == 0x2000 and ge.HLL_WINDOW_P == 8 and (ge.CLIENTS_LAST, ge.CLIENTS_5MIN) == (0, 1)
    assert C.sizeof(ge.SvcClients) == 32
    assert [(n, getattr(ge.SvcClients, n).offset) for n, _ in ge.SvcClients._fields_] == \
        [("glob_id", 0), ("found", 8), ("pad", 12), ("last_5s", 16), ("last_5min", 24)]


def test_slot_bytes_with_the_flag():
    L = ge.load_library()
    cfg = ge.Config()
    L.gysk_config_default(C.byref(cfg))
    svc, task = C.c_uint64(), C.c_uint64()
    assert L.gysk_slot_bytes(C.byref(cfg), C.byref(svc), C.byref(task)) == 0
    base = svc.value
    cfg.flags |= ge.FLAG_CLIENT_LEVELS
    assert L.gysk_slot_bytes(C.byref(cfg), C.byref(svc), C.byref(task)) == 0
    assert (base, svc.value) == (14904, 18232) and svc.value - base == (2 + 10 + 1) * 256
