"""The connection / process record queue of ingest_kernel at batch sizes where every warp takes several chunks, and every launch
shape and sort switch of the library, against the CPU oracle.

ingest_kernel deals its chunks of 32 x EPT events to the warps round-robin. Each warp owns one region of the batch's record queue,
rcap = ceil(chunks / warps) x CHUNK entries: connection (TCP) records grow from its front, process (TASK) records from its back, and
the drain_kernel passes find each region's groups of 32 records through a table built from the per-warp counts (DESIGN.md §4). Below
one full grid of chunks (nsm x MIN_CTAS x WARPS of them, about 200 000 events for the default shape on an H100) every region holds
at most one chunk, so the batches here are sized in chunks relative to that grid, from the device's SM count and the active shape.

The shape and the sort switches are read once per process, so test_every_shape_and_switch re-runs these tests and a set of parity
tests in a child process per setting; test_switch_list_is_complete (no GPU) keeps that list in step with the sources."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from tests.util import assert_hist_equal, make_pair

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gyeeta_b200", "csrc")

# GYSK_INGEST_VARIANT -> (WARPS, MIN_CTAS, EPT, TMA): the `switch (ingest_variant())` of launch_ingest; unset or unknown = 832
SHAPES = {832: (8, 3, 2, False), 842: (8, 4, 2, False), 852: (8, 5, 2, False), 834: (8, 3, 4, False), 844: (8, 4, 4, False),
          482: (4, 8, 2, False), 1832: (8, 3, 2, True), 1834: (8, 3, 4, True)}
DEFAULT_VARIANT = 832

# every launch shape and sort switch; test_every_shape_and_switch runs the tests below once per entry
SETTINGS = [{"GYSK_INGEST_VARIANT": str(v)} for v in (832, 842, 852, 834, 844, 482, 1832, 1834)] + [
    {"GYSK_KEY_DIGIT_MAX": "9"},                                   # 9-bit digits: os_pass_kernel<9>, ingest_kernel with DH = 512
    {"GYSK_KEY_DIGIT_MAX": "9", "GYSK_INGEST_VARIANT": "1834"},    # ... in ingest_kernel's largest shared-memory layout
    {"GYSK_OS_RANK": "1"}, {"GYSK_OS_RANK": "2"},                  # one ranking code in every radix tile (the default picks per tile)
    {"GYSK_OS_NARROW": "0"}, {"GYSK_OS_PERSIST": "0"}, {"GYSK_RM_THREADS": "512"}, {"GYSK_MERGE_SMEM_N": "512"},
]
# switches that are not in SETTINGS, and why
NOT_RUN = {
    "GYSK_EXP_ABLATE": "timing runs only: each bit skips part of the work, so the results are wrong by definition",
    "GYSK_HOT_ROWS": "read per engine, so a test can set it: tests/test_gpu_hot_rows.py",
    "GYSK_HOT_MIN": "read per engine, so a test can set it: tests/test_gpu_hot_rows.py",
    "GYSK_HOT_MAX": "read per engine, so a test can set it: tests/test_gpu_hot_rows.py",
    "GYSK_HOT_BIN_MAX": "read per engine, so a test can set it: tests/test_gpu_hot_rows.py",
}
# what each child process runs besides this file's region tests
PARITY_TESTS = ["tests/test_gpu_parity.py::test_mixed_stream_bit_exact", "tests/test_gpu_parity.py::test_full_value_range_keys",
                "tests/test_gpu_parity.py::test_topn_services_last_window",
                "tests/test_gpu_hot_rows.py::test_hot_rows_are_taken_and_every_batch_is_bit_exact"]
CHILD_TIMEOUT_S = 1800

NSVC, NTASK = 2000, 500
TIDS = synth.task_ids(NTASK)
CMS_DEPTH, CMS_LOG2W = 4, 16
M32 = 0xFFFFFFFF
COUNTERS = (("events_in", "in"), ("events_dropped", "dropped"), ("events_resp", "resp"), ("events_tcp", "tcp"),
            ("events_task", "task"), ("nsvcs", "nsvcs"), ("ntasks", "ntasks"))
TASK_HISTS = (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY)


def _setting_id(s):
    return ",".join(f"{k}={v}" for k, v in s.items())


# ---------------------------------------------------------------------------------------------------------------------------
# geometry of the record regions, as launch_ingest_variant and ingest_kernel compute it
# ---------------------------------------------------------------------------------------------------------------------------
class Geometry:
    def __init__(self, nsm, variant):
        self.nsm = nsm
        self.warps, self.min_ctas, self.ept, self.tma = SHAPES.get(variant, SHAPES[DEFAULT_VARIANT])
        self.chunk = 32 * self.ept
        self.full = nsm * self.min_ctas * self.warps           # warps of a full grid (N)

    def regions(self, n):
        """(nwarps, rcap) of an n-event batch"""
        nchunks = -(-n // self.chunk)
        grid = min(-(-n // (self.chunk * self.warps)), self.nsm * self.min_ctas)
        nwarps = grid * self.warps
        return nwarps, -(-nchunks // nwarps) * self.chunk

    def sizes(self):
        N, C = self.full, self.chunk
        n1 = N * C + C // 2 + 1          # N + 1 chunks, the last one partial: exactly one warp takes a second chunk
        n2 = 2 * N * C                   # every region exactly two chunks
        n3 = (7 * N // 2) * C + 7        # 3.5 N chunks and a few events: regions of four chunks, the last warps with three
        assert n1 % C and self.regions(n1) == (N, 2 * C)
        assert self.regions(n2) == (N, 2 * C)
        assert n3 % C and self.regions(n3) == (N, 4 * C)
        return n1, n2, n3


def _variant():
    try:
        return int(os.environ.get("GYSK_INGEST_VARIANT", "0"))
    except ValueError:
        return 0


@pytest.fixture(scope="module")
def geo():
    import torch
    return Geometry(torch.cuda.get_device_properties(0).multi_processor_count, _variant())


# ---------------------------------------------------------------------------------------------------------------------------
# streams
# ---------------------------------------------------------------------------------------------------------------------------
def _negative_task_values(rng, ev):
    """process values of 2^31 and more narrow to negative ints in the histograms; four tasks get nothing else, so their histogram
    maxima stay negative"""
    task = ev["type"] == ge.EV_TASK
    sel = task & (np.isin(ev["svc_id"], TIDS[4:8]) | (rng.random(len(ev)) < 0.03))
    k = int(sel.sum())
    big = lambda: rng.integers(1 << 31, 1 << 32, k, dtype=np.uint64)
    ev["value"][sel] = big().astype(np.uint32)
    ev["flow_key"][sel] = big() | (big() << np.uint64(32))


def _tasks(rng, n):
    """n process samples with the formulas of synth.gen_mixed"""
    ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = TIDS[np.searchsorted(synth.zipf_cdf(NTASK, 1.05), rng.random(n), side="left")]
    ev["type"] = ge.EV_TASK
    ev["value"] = np.minimum(rng.gamma(1.2, 20.0, n), 3200).astype(np.uint32)
    cpu_delay = np.minimum(np.exp(rng.normal(np.log(30.0), 2.0, n)), 1.0e5).astype(np.uint64)
    blkio = np.minimum(np.exp(rng.normal(np.log(5.0), 2.5, n)), 1.0e5).astype(np.uint64)
    ev["flow_key"] = cpu_delay | (blkio << np.uint64(32))
    ev["host_idx"] = rng.integers(0, 64, n)
    ev["tsec"] = 1
    _negative_task_values(rng, ev)
    return ev


def _tcp(rng, n):
    return synth.gen_tcp(rng, n, NSVC, zipf_s=1.05, nclients=20_000, nhosts=64)


def _mixed(rng, n):
    """70 / 20 / 10 RESP / TCP / TASK; 2 % of the connection events are ACTIVE_CONN_STATS records"""
    ev = synth.gen_mixed(rng, n, NSVC, ntask=NTASK, nhosts=64, nclients=20_000, zipf_s=1.05)
    act = (ev["type"] >= ge.EV_CONNECT) & (ev["type"] <= ge.EV_CLOSE_SER) & (rng.random(n) < 0.02)
    k = int(act.sum())
    ev["type"][act] = ge.EV_ACTIVE
    ev["flags"][act] = rng.integers(1, 200, k)                                       # active connections
    ev["value"][act] = rng.integers(0, 1 << 16, k)                                   # kbytes
    ev["tsec"][act] = (rng.random(k) * 500).astype(np.float32).view(np.uint32)       # max rtt, msec
    _negative_task_values(rng, ev)
    return ev


def _records_only(rng, n):
    """TCP and TASK events only, no RESP; blocks of 128 events alternate between 80 % TASK and 80 % TCP, so many chunks bring 32
    or more process records and hand them over inside the loop, not only at its end"""
    ev = _tcp(rng, n)
    heavy = (np.arange(n) // 128) % 2 == 0
    is_task = rng.random(n) < np.where(heavy, 0.8, 0.2)
    ev[is_task] = _tasks(rng, n)[is_task]
    return ev


def _resp_only(rng, n):
    ev = _tcp(rng, n)
    ev["type"] = ge.EV_RESP
    ev["value"] = np.minimum(np.exp(rng.normal(np.log(2000.0), 1.5, n)), 9.0e8).astype(np.uint32)
    return ev


# ---------------------------------------------------------------------------------------------------------------------------
# engine + oracle on identical device batches
# ---------------------------------------------------------------------------------------------------------------------------
def _device_batch(eng, ev):
    """the events as ONE device batch (the engine's max_batch is at least len(ev))"""
    import torch
    d = torch.from_numpy(np.ascontiguousarray(ev).view(np.uint8)).to("cuda:0")
    torch.cuda.synchronize()
    eng.ingest_device_ptr(d.data_ptr(), len(ev))
    eng.sync()


class Pair:
    """an engine and the oracle with the same configuration, fed the same batches; all integer state compared after every batch"""

    def __init__(self, max_batch, max_svcs=4096, max_tasks=1024, rank=0, world=1):
        self.eng, self.orc = make_pair(max_svcs=max_svcs, max_tasks=max_tasks, max_batch=max_batch, cms_depth=CMS_DEPTH,
                                       cms_log2_width=CMS_LOG2W, rank=rank, world=world)
        self.max_batch, self.rank, self.world = max_batch, rank, world
        self.svcs, self.tasks = set(), set()
        self.win_cnt = self.win_kb = 0          # connection events and kbytes of the open window (this shard's)

    def feed(self, ev):
        assert len(ev) <= self.max_batch
        b0 = self.eng.stats()["batches"]
        _device_batch(self.eng, ev)
        self.orc.ingest(ev)
        assert self.eng.stats()["batches"] == b0 + 1
        own = ev[ev["host_idx"] % self.world == self.rank]
        t = own["type"]
        tcp, act = (t >= ge.EV_CONNECT) & (t <= ge.EV_CLOSE_SER), t == ge.EV_ACTIVE
        self.win_cnt += int(tcp.sum()) + int(own["flags"][act].astype(np.int64).sum())
        self.win_kb += int((own["value"][tcp] >> 10).astype(np.int64).sum()) + int(own["value"][act].astype(np.int64).sum())
        self.svcs |= set(np.unique(own["svc_id"][t != ge.EV_TASK]).tolist())
        self.tasks |= set(np.unique(own["svc_id"][t == ge.EV_TASK]).tolist())
        self.check(every_id=False)

    def check(self, every_id=True):
        """counters and the whole count-min table; with every_id, the state of every service and task seen so far as well (it
        carries every earlier batch: a record lost or applied twice in any of them stays visible)"""
        eng, orc = self.eng, self.orc
        s, o = eng.stats(), orc.counters()
        for k, ko in COUNTERS:
            assert s[k] == o[ko], (k, s[k], o[ko])
        cms = eng.export_cms()
        # independent of the oracle: every count-min row holds each connection event once (count 1, bytes >> 10 kbytes) and each
        # ACTIVE_CONN_STATS record with its connections and kbytes; a lost or doubled record changes these sums
        for r, row in enumerate(cms.reshape(CMS_DEPTH, -1)):
            got = (int((row & np.uint64(M32)).sum()), int((row >> np.uint64(32)).sum()))
            assert got == (self.win_cnt, self.win_kb), (r, got, (self.win_cnt, self.win_kb))
        assert np.array_equal(cms, orc.cms())
        if not every_id:
            return
        for id_ in sorted(self.svcs):
            assert_hist_equal(eng, orc, id_, ge.HIST_RESP_CUR)
            assert np.array_equal(eng.export_hll(id_), orc.export_hll(id_)), hex(id_)
            g, w = eng.export_conn_bitmap(id_), orc.export_conn_bitmap(id_)
            assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]), hex(id_)
            (means, weights, mn, mx), td = eng.export_tdigest(id_), orc.export_tdigest(id_)
            om, ow = td.centroids()
            assert np.array_equal(weights, ow) and np.array_equal(means, om), hex(id_)
            if len(ow):
                assert (mn, mx) == (td.minv, td.maxv), hex(id_)
        for id_ in sorted(self.tasks):
            for which in TASK_HISTS:
                assert_hist_equal(eng, orc, id_, which)

    def flush(self, tsec):
        """every id's state of the window, then the flush and the window's connection and active-connection totals per service"""
        self.check()
        self.eng.flush(tsec)
        self.orc.flush(tsec)
        self.win_cnt = self.win_kb = 0
        ids = np.array(sorted(self.svcs), dtype=np.uint64)
        for s_, id_ in zip(self.eng.query_svcs(ids), ids.tolist()):
            assert s_["found"] == 1, hex(id_)
            _cur, last, all_cnt, all_kb = self.orc.export_conn(id_)
            assert (s_["nconns_5s"], s_["kbytes_5s"]) == (last & M32, last >> 32), hex(id_)
            assert (s_["nconns_all"], s_["kbytes_all"]) == (all_cnt, all_kb), hex(id_)
            a = self.orc.export_aux(id_)
            assert (s_["nconns_active"], s_["active_kbytes"]) == (a["act_last"] & M32, a["act_last"] >> 32), hex(id_)
            assert s_["max_rtt_msec"] == a["rtt_last"], hex(id_)
        self.check(every_id=False)


# ---------------------------------------------------------------------------------------------------------------------------
# the region tests
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_mixed_stream_several_chunks_per_warp(geo):
    """(a) the mixed stream in batches of N + 1, 2 N and 3.5 N chunks, flushed between windows. 65 536 services: 26 sort-key bits,
    so GYSK_KEY_DIGIT_MAX=9 sorts in 9/9/8-bit passes (8-bit digits: 7/7/6/6)."""
    n1, n2, n3 = geo.sizes()
    rng = np.random.default_rng(101)
    p = Pair(max_batch=n3, max_svcs=1 << 16)
    for n in (n1, n2):
        p.feed(_mixed(rng, n))
    p.flush(5)
    for n in (n3, n1):                   # the largest batch is max_batch: the record queue's bound holds exactly
        p.feed(_mixed(rng, n))
    p.flush(10)
    p.feed(_mixed(rng, n2))
    p.flush(15)
    assert p.eng.stats()["batches"] == 5


@pytest.mark.gpu
def test_records_only_regions_fill_from_both_ends(geo):
    """(b) every event a connection or process record: at 2 N chunks each region is exactly full, the TCP records from its front
    and the TASK records from its back meet at its last entry"""
    n1, n2, n3 = geo.sizes()
    rng = np.random.default_rng(102)
    p = Pair(max_batch=n3)
    for n in (n2, n1, n3, n2):
        p.feed(_records_only(rng, n))
    p.flush(5)
    st = p.eng.stats()
    assert st["events_resp"] == 0 and st["events_dropped"] == 0 and st["events_tcp"] > 0 and st["events_task"] > 0


@pytest.mark.gpu
def test_tcp_only_then_task_only(geo):
    """(c) batches of connection records only fill the regions from the front, then batches of process records only from the back"""
    sizes = geo.sizes()
    rng = np.random.default_rng(103)
    p = Pair(max_batch=sizes[2])
    for n in sizes:
        p.feed(_tcp(rng, n))
    for n in sizes:
        p.feed(_tasks(rng, n))
    p.flush(5)


@pytest.mark.gpu
def test_grid_shrinks_and_grows_between_batches(geo):
    """(d) a record-heavy batch of 3.5 N chunks, then one of fewer than N chunks (a smaller grid: the counts of the warps beyond
    it still hold the last batch's), then responses only (every region empty), then 3.5 N chunks again: no record is applied twice"""
    n1, n2, n3 = geo.sizes()
    small = (geo.full // 3) * geo.chunk + 5
    assert geo.regions(small)[0] < geo.full
    rng = np.random.default_rng(104)
    p = Pair(max_batch=n3)
    p.feed(_records_only(rng, n3))
    p.feed(_records_only(rng, small))
    p.feed(_resp_only(rng, n2))
    p.feed(_records_only(rng, n3))
    p.feed(_mixed(rng, small))
    p.flush(5)


@pytest.mark.gpu
def test_sharded_mixed_stream_skips_empty_regions(geo):
    """(e) the mixed stream on the two engines of a world of 2: each drops the other's events, so many regions are partly or
    wholly empty and the drain passes' forward walk skips them"""
    n1, n2, n3 = geo.sizes()
    rng = np.random.default_rng(105)
    batches = [_mixed(rng, n) for n in (n1, n2, n3)]
    for i in (0, 2):
        # each shard's events in runs of a few thousand, as one host's messages arrive: whole chunks, and so whole regions, are foreign
        b = batches[i]
        block = np.cumsum(rng.random(len(b)) < 1 / 8192)
        batches[i] = b[np.argsort(block * 2 + b["host_idx"] % 2, kind="stable")]
    for b in (batches[0], batches[2]):
        nwarps = geo.regions(len(b))[0]
        for r in range(2):
            rec = (b["type"] <= ge.EV_CLOSE_SER) & (b["host_idx"] % 2 == r)          # this shard's connection records
            per_region = np.bincount((np.arange(len(b)) // geo.chunk) % nwarps, weights=rec, minlength=nwarps)
            assert per_region.min() == 0 < per_region.max()
    pairs = [Pair(max_batch=n3, max_svcs=1 << 16, rank=r, world=2) for r in range(2)]
    for p in pairs:
        for b in batches[:2]:
            p.feed(b)
        p.flush(5)
        p.feed(batches[2])
        p.flush(10)
    assert sum(p.eng.stats()["events_in"] for p in pairs) == sum(len(b) for b in batches)


# ---------------------------------------------------------------------------------------------------------------------------
# every launch shape and sort switch
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("setting", SETTINGS, ids=[_setting_id(s) for s in SETTINGS])
def test_every_shape_and_switch(setting):
    """the region tests above and the parity tests of PARITY_TESTS in a child process with the setting in its environment (the
    library reads these switches once per process); one run, the child's output in the failure message"""
    env = {k: v for k, v in os.environ.items() if not k.startswith("GYSK_")}
    env.update(setting)
    env["PYTHONDONTWRITEBYTECODE"] = "1"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_record_regions.py", "-k", "not every_shape"] + PARITY_TESTS
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=CHILD_TIMEOUT_S)
    assert r.returncode == 0, f"{_setting_id(setting)}: the child exited with {r.returncode}\n{r.stdout[-12000:]}\n{r.stderr[-4000:]}"


def _sources():
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if ".cu" in f or f.endswith(".h"):
            with open(os.path.join(CSRC, f)) as fh:
                out[f] = fh.read()
    return out


def _variant_cases(src):
    """{label: (WARPS, MIN_CTAS, EPT, TMA)} of the case lines of `switch (ingest_variant())`, and the default's shape"""
    i = src.index("switch (ingest_variant())")
    body = src[i: src.index("default", i)]
    line = r"\s*:\s*GYSK_LI\(\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*,\s*(true|false)\s*\)"
    cases = {int(c): (int(w), int(m), int(e), t == "true") for c, w, m, e, t in re.findall(r"case\s+(\d+)" + line, body)}
    assert len(cases) == body.count("case "), "a case line of the switch does not have the expected form"
    w, m, e, t = re.search(r"default" + line, src[i:]).groups()
    return cases, (int(w), int(m), int(e), t == "true")


def _selecting_values(src):
    """switch -> the values that select its other code path, read off the line that reads it (`== 9` selects 9, `!= 0` is
    switched off by 0); for GYSK_OS_RANK the modes other than 0 (auto) that the radix pass's rank_mode parameter documents"""
    out = {}
    for ln in src.splitlines():
        m = re.search(r'getenv\("(GYSK_\w+)"\)', ln)
        if m and re.findall(r"[!=]= (\d+)", ln[m.end():]):
            out[m.group(1)] = set(re.findall(r"[!=]= (\d+)", ln[m.end():]))
    modes = re.search(r"int rank_mode\s*/\*([^*]*)\*/", src)
    assert modes and "GYSK_OS_RANK" in src
    out["GYSK_OS_RANK"] = set(re.findall(r"(\d+) ", modes.group(1))) - {"0"}
    return out


def test_switch_list_is_complete():
    """every ingest shape (case label) and every GYSK_ switch the library reads is in SETTINGS or, with its reason, in NOT_RUN;
    SHAPES equals the template arguments of the case lines"""
    srcs = _sources()
    allsrc = "\n".join(srcs.values())
    run = {}
    for s in SETTINGS:
        for k, v in s.items():
            run.setdefault(k, set()).add(v)
    # launch shapes
    cases, default = _variant_cases(srcs["gysk_kernels.cu"])
    assert cases == SHAPES, (cases, SHAPES)
    assert default == SHAPES[DEFAULT_VARIANT]
    missing = [v for v in cases if {"GYSK_INGEST_VARIANT": str(v)} not in SETTINGS]
    assert not missing, f"ingest shapes not run on their own: {sorted(missing)}"
    assert {int(v) for v in run["GYSK_INGEST_VARIANT"]} <= set(cases)
    # switches: every name in a string literal of the sources is an environment switch (getenv and the engine's envl helper)
    names = set(re.findall(r'"(GYSK_[A-Z0-9_]+)"', allsrc))
    assert "GYSK_INGEST_VARIANT" in names and len(names) >= 10
    unlisted = names - set(run) - set(NOT_RUN)
    assert not unlisted, f"switches neither run nor excluded: {sorted(unlisted)}"
    assert not set(run) & set(NOT_RUN)
    assert set(run) | set(NOT_RUN) <= names, f"listed switches the library does not read: {sorted(set(run) | set(NOT_RUN) - names)}"
    # each switch is run with every value that changes what the library does
    for name, vals in _selecting_values(allsrc).items():
        if name in NOT_RUN:
            continue
        assert vals <= run.get(name, set()), f"{name}: values {sorted(vals - run.get(name, set()))} never run"
        assert all({name: v} in SETTINGS for v in vals), f"{name} is not run on its own"
    # 9-bit digits also with the TMA-staged shape of the widest chunks: ingest_kernel's largest shared-memory layout
    widest_tma = max((v for v, s in SHAPES.items() if s[3]), key=lambda v: SHAPES[v][2])
    assert {"GYSK_KEY_DIGIT_MAX": "9", "GYSK_INGEST_VARIANT": str(widest_tma)} in SETTINGS, "9-bit digits with the largest ingest layout"
