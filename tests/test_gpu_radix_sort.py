"""The engine's stable LSD radix sort (gysk::launch_radix_sort: os_hist_kernel + os_pass_kernel<6|7|8|9>) and its top-N pick
(gysk::launch_topn_pick) on their own, through a small nvcc-built harness (tests/cpp/sort_harness.cu) linked against libgysketch.so.

Every output buffer is compared byte for byte with a CPU stable sort, keys[argsort((keys >> lo) & mask, kind="stable")]. Where the
sort field has ties, the bits outside the field carry the input position, so a lost tie order is a mismatch. Covered: every field
width 0 to 64 at three placements (every plan the planner makes, 1 to 8 passes, each kernel instantiation, the 9-bit carry, both
histogram kernels); tile edges, partial tiles and sizes at which every CTA takes two tile tickets; digit distributions that put
each kernel on both rank paths (ballot and match.any) in full and partial tiles; a key count on the device below the grid's size;
the look-back status words reused across sorts of other widths and tile counts; the epoch wrap; the refusals; the top-N pick's
order and its zero fill."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

from gyeeta_b200 import engine as ge

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SORT_TILE = 4096                    # keys per tile (gysk_kernels.cuh)
RADIX_MAX = 512
OS_MAX_PASSES = 8
OS_GHIST_WORDS = OS_MAX_PASSES * RADIX_MAX + OS_MAX_PASSES
CTAS_PER_SM = 4                     # os_pass_kernel's __launch_bounds__: the persistent grid is min(tiles, 4 x SMs)
SENTINEL = np.uint64(0xA5A5_5A5A_C3C3_3C3C)
U64 = 0xFFFF_FFFF_FFFF_FFFF


def plain_sort_plan(lo, hi):
    """gysk_kernels.cu plain_sort_plan restated: [(shift, bits)] of the passes, or None where launch_radix_sort refuses the range.
    8-bit digits from lo upwards, the last one short, the first ones 9 bits wide where that saves a whole pass."""
    if lo < 0 or hi > 64 or lo > hi:
        return None
    t = hi - lo
    p8, p9 = (t + 7) // 8, (t + 8) // 9
    wide = t - 8 * p9 if p9 < p8 else 0
    plan, at = [], lo
    while at < hi:
        if len(plan) == OS_MAX_PASSES:
            return None
        b = min(9 if wide > 0 else 8, hi - at)
        wide -= 1
        plan.append((at, b))
        at += b
    return plan


def next_epoch(e):
    """gysk_kernels.cu next_epoch restated: the epoch of the next pass; 0 is skipped (the status words are cleared there)"""
    e = (e + 1) & 0xFFFF_FFFF
    return e or 1


def seed_of(*what):
    return zlib.crc32(repr(what).encode())


def kernel_of(bits):
    """the os_pass_kernel instantiation a digit of `bits` runs in"""
    return 6 if bits <= 6 else bits


def cpu_sort(keys, lo, hi):
    mask = np.uint64((1 << (hi - lo)) - 1)
    return keys[np.argsort((keys >> np.uint64(lo)) & mask if hi > lo else np.zeros(len(keys), np.uint8), kind="stable")]


def deposit(idx, field, lo, hi):
    """the key with `field` in bits [lo, hi) and the input position idx in the other bits, low bits first"""
    idx = idx.astype(np.uint64)
    low = idx & np.uint64((1 << lo) - 1)
    key = low | (field << np.uint64(lo)) if hi > lo else low
    if hi < 64:
        key |= (idx >> np.uint64(lo)) << np.uint64(hi)
    return key


# ---------------------------------------------------------------------------------------------------------------------------
# key distributions: each fills every pass's digit of the field; the bits outside the field carry the input position
# ---------------------------------------------------------------------------------------------------------------------------
def _digits(dist, rng, n, plan):
    field = np.zeros(n, dtype=np.uint64)
    lo = plan[0][0] if plan else 0
    for p, (shift, bits) in enumerate(plan):
        r = 1 << bits
        if dist == "field_const":
            d = np.full(n, (0x5B + 37 * p) % r, dtype=np.uint64)
        elif dist == "tile_const":          # one value in each tile, another in the next
            d = ((np.arange(n, dtype=np.uint64) // np.uint64(SORT_TILE)) * np.uint64(0x9E37) + np.uint64(13 + 97 * p)) % np.uint64(r)
        elif dist in ("ten", "eleven"):     # exactly k equally frequent digit values
            k = min(10 if dist == "ten" else 11, r)
            vals = rng.choice(r, k, replace=False).astype(np.uint64)
            d = vals[rng.permutation(np.arange(n) % k)]
        elif dist == "zipf":
            d = (rng.zipf(1.3, n).astype(np.uint64) - np.uint64(1) + np.uint64(29 * p)) % np.uint64(r)
        else:                               # uniform field
            d = rng.integers(0, r, n, dtype=np.uint64)
        field |= d << np.uint64(shift - lo)
    return field


DISTS = ("uniform64", "all_equal", "field_const", "tile_const", "ten", "eleven", "zipf", "sorted", "reversed")


def make_keys(dist, n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    plan = plain_sort_plan(lo, hi)
    if dist == "uniform64":                 # every bit random, the field's and the others'
        return rng.integers(0, U64, n, dtype=np.uint64, endpoint=True)
    if dist == "all_equal":
        return np.full(n, 0x0123_4567_89AB_CDEF, dtype=np.uint64)
    field = _digits("uniform" if dist in ("sorted", "reversed") else dist, rng, n, plan)
    keys = deposit(np.arange(n), field, lo, hi)
    if dist in ("sorted", "reversed"):
        keys = cpu_sort(keys, lo, hi)
        if dist == "reversed":
            keys = keys[::-1].copy()
    return keys


def rank_paths(keys, lo, hi):
    """per pass: (kernel, ballot ranking?) as os_pass_kernel decides it, from the pass's global digit histogram: the expected number of
    distinct digits among 32 keys, sum over digits of 1 - (1 - count / n)^32 in float, > 10 ranks by ballots"""
    out = []
    for shift, bits in plain_sort_plan(lo, hi):
        cnt = np.bincount(((keys >> np.uint64(shift)) & np.uint64((1 << bits) - 1)).astype(np.int64), minlength=1 << bits)
        q = np.float32(1) - cnt.astype(np.float32) / np.float32(len(keys))
        for _ in range(5):
            q = q * q
        out.append((kernel_of(bits), float(np.sum(np.float32(1) - q, dtype=np.float32)) > 10.0))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# the harness
# ---------------------------------------------------------------------------------------------------------------------------
class Sorter:
    """one set of sort buffers (torch CUDA tensors) and a host epoch counter, shared by every sort of the module"""

    def __init__(self, so, cap):
        import torch
        self.torch = torch
        self.L = C.CDLL(so)
        vp, u32, u64, ci = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
        self.L.st_radix_sort.argtypes = [vp, vp, vp, u32, vp, C.POINTER(u32), vp, u64, ci, ci, C.POINTER(ci), vp]
        self.L.st_topn_pick.argtypes = [vp, vp, vp, u32, vp, C.POINTER(u32), vp, u32, vp, vp, u32, vp, vp, vp]
        self.L.st_radix_sort.restype = self.L.st_topn_pick.restype = ci
        dev = torch.device("cuda", 0)
        self.cap = cap
        self.max_tiles = (cap + SORT_TILE - 1) // SORT_TILE
        # A pass that misplaces keys leaves the next pass's digit counts unlike the histogram of the input, and that pass's writes can
        # then reach 2n + a tile: the slack past the keys turns such a regression into a reported mismatch instead of a fault.
        self.a = torch.zeros(2 * cap + SORT_TILE, dtype=torch.int64, device=dev)
        self.b = torch.zeros_like(self.a)
        self.status = torch.zeros(self.max_tiles * RADIX_MAX, dtype=torch.int64, device=dev)
        self.ghist = torch.zeros(OS_GHIST_WORDS, dtype=torch.int32, device=dev)
        self.dn = torch.zeros(1, dtype=torch.int64, device=dev)
        self.epoch = C.c_uint32(0)
        self.sm = torch.cuda.get_device_properties(0).multi_processor_count

    def _t(self, x):
        return self.torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(self.a.device)

    def _np(self, t):
        return t.cpu().numpy().view(np.uint64)

    def stream(self):
        return C.c_void_p(self.torch.cuda.current_stream().cuda_stream)

    def _buffers(self):
        return (C.c_void_p(self.a.data_ptr()), C.c_void_p(self.b.data_ptr()), C.c_void_p(self.status.data_ptr()), self.max_tiles,
                C.c_void_p(self.ghist.data_ptr()), C.byref(self.epoch))

    def raw_sort(self, lo, hi, n_max, d_n):
        self.dn.fill_(d_n)
        which = C.c_int(-7)
        rc = self.L.st_radix_sort(*self._buffers(), C.c_void_p(self.dn.data_ptr()), n_max, lo, hi, C.byref(which), self.stream())
        self.torch.cuda.synchronize()
        return rc, which.value

    def sort(self, keys, lo, hi, what, n_max=None):
        """sorts keys on [lo, hi) with *d_n = len(keys) and a grid for n_max >= len(keys); checks the whole output, the launch count,
        the output buffer and that nothing in [n, max(n_max, 2n + a tile)) moved in either buffer"""
        n = len(keys)
        n_max = n if n_max is None else n_max
        guard = min(max(n_max, 2 * n + SORT_TILE), len(self.a))
        self.a[n:guard].fill_(int(SENTINEL.view(np.int64)))
        self.b[:guard].fill_(int(SENTINEL.view(np.int64)))
        if n:
            self.a[:n].copy_(self._t(keys))
        plan = plain_sort_plan(lo, hi)
        e = self.epoch.value
        for _ in plan:
            e = next_epoch(e)
        rc, which = self.raw_sort(lo, hi, n_max, n)
        assert rc == 1 + len(plan), (what, rc)
        assert which == len(plan) % 2, (what, which)
        assert self.epoch.value == e, (what, "one epoch per pass")
        out, other = (self.b, self.a) if which else (self.a, self.b)
        got = self._np(out[:guard])
        want = cpu_sort(keys, lo, hi)
        if not np.array_equal(got[:n], want):
            bad = np.flatnonzero(got[:n] != want)
            raise AssertionError(f"{what}: {len(bad)} of {n} keys misplaced, first at {bad[0]}: {int(got[bad[0]]):#x} != {int(want[bad[0]]):#x}")
        assert (got[n:] == SENTINEL).all(), (what, "a key written past n in the output buffer")
        assert (self._np(other[n:guard]) == SENTINEL).all(), (what, "a key written past n in the other buffer")
        return got[:n]


@pytest.fixture(scope="module")
def sorter(tmp_path_factory):
    import torch
    ge.load_library()
    libdir = os.path.dirname(ge.LIB_PATH)
    so = str(tmp_path_factory.mktemp("sort_harness") / "sort_harness.so")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    cmd = [nvcc if os.path.exists(nvcc) else "nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-Xcompiler", "-fPIC",
           "-shared", "-I", os.path.join(ROOT, "gyeeta_b200", "csrc"), os.path.join(ROOT, "tests", "cpp", "sort_harness.cu"), "-o", so,
           "-L", libdir, "-lgysketch", "-Xlinker", f"-rpath,{libdir}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return Sorter(so, big_n(sm))


def big_n(sm):
    """every CTA of the persistent grid takes at least two tile tickets"""
    return 2 * CTAS_PER_SM * sm * SORT_TILE + 1


# ---------------------------------------------------------------------------------------------------------------------------
# the planner restated
# ---------------------------------------------------------------------------------------------------------------------------
def test_plan_restatement_reaches_every_plan_shape():
    """the widths below name the plans they reach: one pass of 1 to 9 bits, 9-bit passes with their carry, 1 to 8 passes"""
    bits = {t: [b for _, b in plain_sort_plan(0, t)] for t in range(65)}
    assert bits[0] == [] and all(bits[t] == [t] for t in range(1, 10))
    assert bits[17] == [9, 8] and bits[18] == [9, 9] and bits[19] == [8, 8, 3] and bits[26] == [9, 9, 8] and bits[27] == [9, 9, 9]
    assert bits[31] == [8, 8, 8, 7] and bits[63] == [9] * 7 and bits[64] == [8] * 8
    assert {len(b) for b in bits.values()} == set(range(9))
    assert {kernel_of(x) for b in bits.values() for x in b} == {6, 7, 8, 9}
    assert plain_sort_plan(0, 73) is None and plain_sort_plan(0, 72) is None and plain_sort_plan(-1, 8) is None and plain_sort_plan(9, 8) is None


# ---------------------------------------------------------------------------------------------------------------------------
# every width at three placements
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", range(65))
def test_every_width(sorter, width):
    los = sorted({0, 64 - width} | ({32} if width <= 32 else set()))
    for lo in los:
        for n in (33, 4097, 3 * SORT_TILE + 5):
            for dist in ("uniform", "field_const", "uniform64"):
                keys = make_keys(dist, n, lo, lo + width, seed_of(width, lo, n, dist))
                got = sorter.sort(keys, lo, lo + width, f"[{lo}, {lo + width}) n={n} {dist}")
                if width == 0:
                    assert np.array_equal(got, keys)


# ---------------------------------------------------------------------------------------------------------------------------
# sizes x distributions for one plan of each kernel and shape
# ---------------------------------------------------------------------------------------------------------------------------
PLANS = {                                   # (lo, hi): what the plan exercises
    "w5_6bit_narrow": (32, 37),
    "w6_6bit": (0, 6),
    "w7": (32, 39),
    "w8": (0, 8),
    "w9_carry": (32, 41),
    "w17_9_8": (0, 17),
    "w31_8887": (32, 63),
    "w63_9x7": (1, 64),
}
SIZES = (1, 2, 31, 32, 33, 511, 512, 513, 4095, 4096, 4097, 8191, 8193)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("plan", PLANS)
def test_sizes_and_distributions(sorter, plan, dist):
    lo, hi = PLANS[plan]
    for n in SIZES:
        keys = make_keys(dist, n, lo, hi, seed_of(plan, dist, n))
        sorter.sort(keys, lo, hi, f"plan {plan} [{lo}, {hi}) n={n} {dist}")


def test_matrix_puts_every_kernel_on_both_rank_paths():
    """the distributions above send each kernel instantiation down both rank paths, in a partial tile and in full tiles (the rule of
    os_pass_kernel restated; the 10 / 11 value distributions sit either side of its threshold)"""
    seen = set()
    for plan, (lo, hi) in PLANS.items():
        for dist in DISTS:
            for n in (511, 4096, 4097):
                keys = make_keys(dist, n, lo, hi, seed_of(plan, dist, n))
                for kern, ballot in rank_paths(keys, lo, hi):
                    seen.add((kern, ballot, n % SORT_TILE != 0))
    assert seen == {(k, b, p) for k in (6, 7, 8, 9) for b in (False, True) for p in (False, True)}, seen
    for plan, (lo, hi) in PLANS.items():
        for n in SIZES[2:]:
            ten, eleven = (rank_paths(make_keys(d, n, lo, hi, seed_of(plan, d, n)), lo, hi) for d in ("ten", "eleven"))
            assert not any(b for _, b in ten) and all(b for _, b in eleven), (plan, n)


@pytest.mark.parametrize("plan,dist", [("w17_9_8", "uniform64"), ("w17_9_8", "tile_const"), ("w9_carry", "eleven"), ("w8", "ten"),
                                       ("w31_8887", "zipf"), ("w5_6bit_narrow", "field_const")])
def test_every_cta_takes_two_tickets(sorter, plan, dist):
    """2 x 4 x SMs tiles and one key: every CTA of the persistent grid loops to a second ticket, the last tile holds one key"""
    lo, hi = PLANS[plan]
    n = big_n(sorter.sm)
    sorter.sort(make_keys(dist, n, lo, hi, seed_of(plan, dist)), lo, hi, f"plan {plan} n={n} {dist}")


def test_key_count_below_the_grid(sorter):
    """*d_n = 0 and *d_n far below n_max: the surplus CTAs leave at once, nothing past *d_n moves"""
    for lo, hi in ((0, 9), (32, 64), (0, 17), (32, 38)):
        sorter.sort(np.zeros(0, dtype=np.uint64), lo, hi, f"[{lo}, {hi}) d_n=0", n_max=50_000)
        for n in (1, 4097, 20_001):
            sorter.sort(make_keys("uniform64", n, lo, hi, seed_of(lo, hi, n)), lo, hi, f"[{lo}, {hi}) d_n={n} n_max=300001", n_max=300_001)


# ---------------------------------------------------------------------------------------------------------------------------
# the look-back status words: reused across sorts, and the epoch wrap
# ---------------------------------------------------------------------------------------------------------------------------
def test_status_words_reused_across_widths_and_tile_counts(sorter):
    """one set of status words for a 9-bit sort of many tiles, a 6-bit sort of a few, an 8-bit sort of another size and back: the
    words each pass leaves (at its own stride tile * RADIX + d) are stale for the next sort"""
    seq = [((0, 9), 600_001), ((10, 16), 9_000), ((0, 8), 123_457), ((32, 41), 40_000), ((3, 9), 700_000), ((0, 17), 5)]
    for rep in range(2):
        for (lo, hi), n in seq:
            sorter.sort(make_keys("uniform", n, lo, hi, seed_of(lo, hi, n, rep)), lo, hi, f"reuse {rep} [{lo}, {hi}) n={n}")


@pytest.mark.parametrize("start", [2**32 - 1, 2**32 - 3])
def test_epoch_wrap(sorter, start):
    """the epoch counter wraps inside a 64-bit sort of 8 passes: next_epoch clears the status words and restarts at 1.
    Every word is first set to {epoch 1 | inclusive prefix | count 0}, the word the first pass after the wrap would accept from a
    predecessor tile that has not published yet; without the clear that pass takes a prefix of 0 and misplaces keys. A pass meets
    such a word only while it looks back at a predecessor that has not published, which the first wave of a many-tile pass does often;
    and only the pass right after the wrap meets them before the sort's own passes overwrite every word, so one case wraps at the
    first pass (the other, two passes later, checks the wrap between passes of one sort)."""
    n = big_n(sorter.sm)
    poison = (1 << 32) | (2 << 30)
    sorter.status.fill_(poison)
    sorter.epoch.value = start
    sorter.sort(make_keys("uniform64", n, 0, 64, seed_of(start)), 0, 64, f"epoch wrap from {start:#x}")
    assert sorter.epoch.value == (start + 8 + 1) & 0xFFFF_FFFF          # 8 passes and the skipped epoch 0
    sorter.sort(make_keys("field_const", 70_000, 32, 41, seed_of(start, 1)), 32, 41, "the sort after the wrap")


def test_refusals_launch_nothing(sorter):
    """no plan for the range (nine passes, or bits outside the key) and n_max >= 2^30: -1, before the first memset or epoch"""
    sorter.ghist.fill_(-1)
    sorter.a[:8].fill_(5); sorter.b[:8].fill_(6)
    for lo, hi, n_max in ((0, 73, 10), (0, 72, 10), (60, 72, 10), (-1, 8, 10), (9, 8, 10), (0, 64, 1 << 30), (32, 40, (1 << 30) + 5)):
        e0 = sorter.epoch.value
        rc, which = sorter.raw_sort(lo, hi, n_max, 5)
        assert (rc, which) == (-1, 0), (lo, hi, n_max)
        assert sorter.epoch.value == e0
    assert (sorter.ghist == -1).all()
    assert (sorter.a[:8] == 5).all() and (sorter.b[:8] == 6).all()
    # n_max = 0: nothing to sort, no launch
    assert sorter.raw_sort(0, 64, 0, 0) == (0, 0)
    # the largest accepted n_max sizes the grid only; *d_n keys are sorted
    rc, _ = sorter.raw_sort(32, 40, (1 << 30) - 1, 0)
    assert rc == 2


# ---------------------------------------------------------------------------------------------------------------------------
# the top-N pick
# ---------------------------------------------------------------------------------------------------------------------------
ENTRY = np.dtype([("glob_id", "<u8"), ("score", "<u8"), ("host_idx", "<u4"), ("pad", "<u4")])


def cpu_pick(scores, ids, hosts, want):
    """descending score, the later index first on equal scores; zero entries and slot 0 past the keys"""
    order = np.lexsort((-np.arange(len(scores)), -scores.astype(np.int64)))[:want]
    out = np.zeros(want, dtype=ENTRY)
    slots = np.zeros(want, dtype=np.uint64)
    for j, i in enumerate(order):
        out[j] = (ids[i], scores[i], hosts[i] if hosts is not None else 0, 0)
        slots[j] = i
    return out, slots


@pytest.mark.parametrize("n", [1, 7, 64, 100, 4097, 70_000])
def test_topn_pick_order(sorter, n):
    torch = sorter.torch
    rng = np.random.default_rng(n)
    ids = rng.integers(1, U64, n, dtype=np.uint64, endpoint=True)
    hosts = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    for scores in (rng.integers(0, 4, n, dtype=np.uint64),                                  # heavy ties
                   np.where(rng.random(n) < 0.5, np.uint64(0xFFFF_FFFF), rng.integers(0, 1 << 32, n, dtype=np.uint64)),
                   np.zeros(n, dtype=np.uint64)):
        keys = (scores << np.uint64(32)) | np.arange(n, dtype=np.uint64)
        d_ids = sorter._t(ids)
        d_hosts = torch.from_numpy(hosts.view(np.int32)).to(sorter.a.device)
        for want in sorted({1, 10, 64, min(n + 3, 64)}):
            for with_hosts in (True, False):
                sorter.a[:n].copy_(sorter._t(keys))
                sorter.dn.fill_(n)
                out = torch.full((64 * ENTRY.itemsize // 8,), -1, dtype=torch.int64, device=sorter.a.device)
                slots = torch.full((64,), -1, dtype=torch.int64, device=sorter.a.device)
                rc = sorter.L.st_topn_pick(*sorter._buffers(), C.c_void_p(sorter.dn.data_ptr()), n, C.c_void_p(d_ids.data_ptr()),
                                           C.c_void_p(d_hosts.data_ptr() if with_hosts else 0), want, C.c_void_p(out.data_ptr()),
                                           C.c_void_p(slots.data_ptr()), sorter.stream())
                torch.cuda.synchronize()
                assert rc == 2 + len(plain_sort_plan(32, 64))
                raw = out.cpu().numpy().view(np.uint8)
                exp, exp_slots = cpu_pick(scores, ids, hosts if with_hosts else None, want)
                what = (n, want, with_hosts, int(scores.max()))
                assert raw[: want * ENTRY.itemsize].tobytes() == exp.tobytes(), what
                assert (raw[want * ENTRY.itemsize:] == 0xFF).all(), what
                s = slots.cpu().numpy().view(np.uint64)
                assert np.array_equal(s[:want], exp_slots) and (s[want:] == U64).all(), what
