"""The HyperLogLog definition (oracle/gysk_oracle.c gyo_hll_hash / gyo_hll_idx_rank, the device's hll_idx_rank2 bit for bit)
against exact distinct counts, on the keys the library builds and not only on pre-mixed random ones.

Raw connection events key a flow as (client ip << 32) | client port, a caller may pass a 64-bit fold of the 5-tuple, and wire
records carry small sequential client-process ids. Such keys are far from random: an index and rank taken from the two
one-round lookup2 words directly left whole register ranges empty and undercounted them by up to 65 %. Every (p, n) here is
run over 24 key sets (8 shapes x 3 bases, each stream with duplicates), with these bounds on the relative error e = est/n - 1,
sigma = 1.04 / sqrt(m):
  - n <= 10: |est - n| <= 1 (at p <= 8, where ten keys often share registers: the error of three shared keys, or the
    linear-counting bound below)
  - n <= 2.5 m (linear counting): |e| <= 4 sqrt(m (e^t - t - 1)) / n, t = n / m (Whang et al. 1990)
  - 2.5 m < n < 5 m: |e| <= 6 sigma; the raw estimator's own bias reaches 2.5 sigma here (Heule et al. 2013 correct it; the
    engine does not)
  - n >= 5 m: |e| <= 4 sigma, 6 sigma at p = 4, where the m = 16 estimate has a long upper tail
  - per (p, n > 10) over the 24 sets: RMS(e) <= 1.5 sigma (3 sigma between 2.5 m and 5 m) and |mean(e)| <= 3 sigma / sqrt(24)
    (not between 2.5 m and 5 m)"""
import math

import numpy as np
import pytest

from oracle import pyoracle as po

M64 = (1 << 64) - 1
PS = (4, 8, 12, 14, 16)
PORTS_PER_IP = (1, 8, 64, 1024, 28232)          # 28 232: the whole default Linux ephemeral range, 32768..60999
SHAPES = ("random",) + tuple(f"ip_port_{k}" for k in PORTS_PER_IP) + ("tuple5", "seq")
BASES = 3
NMAX = 1_000_000


def fmix64(h):
    h ^= h >> 33
    h = (h * 0xFF51AFD7ED558CCD) & M64
    h ^= h >> 33
    h = (h * 0xC4CEB9FE1A85EC53) & M64
    return h ^ (h >> 33)


def ip_port_keys(n, per_ip, ip_base, port_base):
    i = np.arange(n, dtype=np.uint64)
    ip = np.uint64(ip_base) + i // np.uint64(per_ip)
    return (ip << np.uint64(32)) | (np.uint64(port_base) + i % np.uint64(per_ip))


def tuple5_keys(n, cli_base, srv_ip, srv_port):
    """a caller's 64-bit fold of {client ip, client port, server ip, server port, TCP}: (cip ^ sip) << 32 | (cport << 16 | sport) ^ 6,
    64 client ports per client address"""
    i = np.arange(n, dtype=np.uint64)
    cip, cport = np.uint64(cli_base) + i // np.uint64(64), np.uint64(32768) + i % np.uint64(64)
    return ((cip ^ np.uint64(srv_ip)) << np.uint64(32)) | (((cport << np.uint64(16)) | np.uint64(srv_port)) ^ np.uint64(6))


def distinct_keys(shape, n, rng):
    """n keys of one shape at bases drawn from rng; distinct except for the random shape, which may (never in practice) repeat"""
    if shape == "random":
        return rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False)
    if shape.startswith("ip_port_"):
        k = int(shape.rsplit("_", 1)[1])
        ip_base = (10 << 24) | int(rng.integers(0, 1 << 16)) << 8
        return ip_port_keys(n, k, ip_base, int(rng.integers(1024, 65536 - k + 1)))
    if shape == "tuple5":
        return tuple5_keys(n, (172 << 24) | (16 << 16) | int(rng.integers(0, 1 << 12)) << 4, (10 << 24) | int(rng.integers(1, 1 << 24)),
                           int(rng.choice([80, 443, 5432, 8080])))
    assert shape == "seq"                                       # cli_task_aggr_id_ of a test or a small deployment
    return np.uint64(int(rng.integers(1, 1000))) + np.arange(n, dtype=np.uint64)


def stream(keys, rng):
    """the keys with a third of them again, shuffled: the exact answer is the number of distinct keys, not the stream length"""
    if not len(keys):
        return keys
    s = np.concatenate([keys, keys[rng.integers(0, len(keys), len(keys) // 3)]])
    return s[rng.permutation(len(s))]


def cardinalities(p):
    m = 1 << p
    return sorted({0, 1, 2, 10, m // 2, 2 * m, 3 * m, 5 * m, min(100 * m, NMAX), NMAX})


def sigma(p):
    return 1.04 / math.sqrt(1 << p)


def lc_rel_sd(n, m):
    t = n / m
    return math.sqrt(m * (math.expm1(t) - t)) / n


def bound(p, n):
    """largest |est/n - 1| one key set may show (the module docstring)"""
    m, s = 1 << p, sigma(p)
    if n <= 10:
        # only keys that share a register move the estimate: at p <= 8 allow three such keys (at m = 256 and n = 10, more happen
        # with probability 1e-4) or the linear-counting bound, whichever is wider
        three = abs(m * math.log(m / (m - max(n - 3, 0))) - n) / n
        return 1.0 / n if p >= 12 else max(1.0 / n, three, 4 * lc_rel_sd(n, m))
    if n <= 2.5 * m:
        return 4 * lc_rel_sd(n, m)
    if n < 5 * m:
        return 6 * s
    return (6 if p == 4 else 4) * s


def estimate(keys, p):
    return po.hll_estimate(po.hll_registers(keys, p), p)


def test_hash_is_fmix64_of_the_two_lookup2_words():
    """the device's hll_idx_rank2 states the same definition; the GPU parity tests compare its registers with this one"""
    import ctypes as C
    L = po.lib()
    rng = np.random.default_rng(1)
    keys = [0, 1, M64, 1 << 32, (10 << 56) | 443] + [int(k) for k in rng.integers(0, 1 << 64, 200, dtype=np.uint64, endpoint=False)]
    for k in keys:
        h1, h2 = C.c_uint32(), C.c_uint32()
        L.gyo_flow_hashes(k, C.byref(h1), C.byref(h2))
        h = fmix64((h2.value << 32) | h1.value)
        assert L.gyo_hll_hash(k) == h, hex(k)
        for p in PS:
            idx, rank = C.c_uint32(), C.c_uint8()
            L.gyo_hll_idx_rank(k, p, C.byref(idx), C.byref(rank))
            w = (h << p) & M64
            assert idx.value == h >> (64 - p) and rank.value == (64 - w.bit_length() + 1 if w else 64 - p + 1), (hex(k), p)


def test_batch_registers_equal_the_per_key_entry():
    import ctypes as C
    L = po.lib()
    rng = np.random.default_rng(2)
    keys = np.concatenate([ip_port_keys(3000, 64, 0x0A000000, 32768), rng.integers(0, 1 << 63, 3000, dtype=np.uint64)])
    for p in PS:
        want = np.zeros(1 << p, dtype=np.uint8)
        for k in keys.tolist():
            idx, rank = C.c_uint32(), C.c_uint8()
            L.gyo_hll_idx_rank(k, p, C.byref(idx), C.byref(rank))
            want[idx.value] = max(want[idx.value], rank.value)
        assert np.array_equal(po.hll_registers(keys, p), want), p
        # in two calls: the registers are raised, not reset
        regs = po.hll_registers(keys[:1000], p)
        assert np.array_equal(po.hll_registers(keys[1000:], p, regs), want), p


def test_structured_keys_reach_every_register():
    """20 000 keys, 64 ports per client address, p = 12: a uniform index leaves m (1 - 1/m)^n = 31 registers empty (sd 5.5)"""
    p, n, m = 12, 20_000, 4096
    regs = po.hll_registers(ip_port_keys(n, 64, 0x0A000000, 32768), p)
    empty = int((regs == 0).sum())
    want = m * (1 - 1 / m) ** n
    assert abs(empty - want) <= 6 * math.sqrt(want), (empty, want)
    assert abs(estimate(ip_port_keys(n, 64, 0x0A000000, 32768), p) / n - 1) <= 4 * sigma(p)


@pytest.mark.parametrize("p", PS)
def test_estimate_against_exact_count(p):
    m, s = 1 << p, sigma(p)
    rng = np.random.default_rng(1000 + p)
    fails, stats = [], {}
    for n in cardinalities(p):
        errs = []
        for shape in SHAPES:
            for b in range(BASES):
                keys = stream(distinct_keys(shape, n, rng), rng)
                exact = len(np.unique(keys))
                est = estimate(keys, p)
                if exact == 0:
                    assert est == 0.0, (shape, b)
                    continue
                e = est / exact - 1
                errs.append(e)
                if abs(e) > bound(p, exact):
                    fails.append((shape, b, exact, round(est, 1), round(e / s, 2)))
        if n <= 10:
            continue
        errs = np.array(errs)
        rms, mean = float(np.sqrt(np.mean(errs ** 2))), float(np.mean(errs))
        stats[n] = (round(rms / s, 2), round(mean / s, 2))
        between = 2.5 * m < n < 5 * m
        if rms > (3.0 if between else 1.5) * s or (not between and abs(mean) > 3 * s / math.sqrt(len(errs))):
            fails.append(("rms/mean over sets", n, stats[n]))
    assert not fails, (p, fails, stats)
