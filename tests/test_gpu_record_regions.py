"""The connection / process record queue of ingest_kernel at batch sizes where every warp takes several chunks, against the CPU
oracle.

ingest_kernel deals its chunks of 32 x EPT events to the warps round-robin. Each warp owns one region of the batch's record queue,
rcap = ceil(chunks / warps) x CHUNK entries: connection (TCP) records grow from its front, process (TASK) records from its back, and
the drain_kernel passes find each region's groups of 32 records through a table built from the per-warp counts (DESIGN.md §4). Below
one full grid of chunks (nsm x MIN_CTAS x WARPS of them, about 200 000 events on an H100) every region holds at most one chunk, so
the batches here are sized in chunks relative to that grid, from the device's SM count and the launch shape (IngestShape)."""
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import synth
from tests.util import assert_hist_equal, make_pair

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gyeeta_b200", "csrc")

# ingest_kernel's launch shape, IngestShape in gysk_kernels.cuh (test_ingest_shape_matches_the_sources keeps the two equal)
WARPS, MIN_CTAS, EPT = 8, 3, 2

# every GYSK_ string the library reads from the environment, and why no test here sets it
NOT_RUN = {
    "GYSK_HOT_ROWS": "read per engine, so a test can set it: tests/test_gpu_hot_rows.py",
    "GYSK_HOT_MIN": "read per engine, so a test can set it: tests/test_gpu_hot_rows.py",
    "GYSK_HOT_MAX": "read per engine, so a test can set it: tests/test_gpu_hot_rows.py",
    "GYSK_HOT_BIN_MAX": "read per engine, so a test can set it: tests/test_gpu_hot_rows.py",
}

NSVC, NTASK = 2000, 500
TIDS = synth.task_ids(NTASK)
CMS_DEPTH, CMS_LOG2W = 4, 16
M32 = 0xFFFFFFFF
COUNTERS = (("events_in", "in"), ("events_dropped", "dropped"), ("events_resp", "resp"), ("events_tcp", "tcp"),
            ("events_task", "task"), ("nsvcs", "nsvcs"), ("ntasks", "ntasks"))
TASK_HISTS = (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY)


# ---------------------------------------------------------------------------------------------------------------------------
# geometry of the record regions, as launch_ingest and ingest_kernel compute it
# ---------------------------------------------------------------------------------------------------------------------------
class Geometry:
    def __init__(self, nsm):
        self.nsm = nsm
        self.warps, self.min_ctas, self.chunk = WARPS, MIN_CTAS, 32 * EPT
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


@pytest.fixture(scope="module")
def geo():
    import torch
    return Geometry(torch.cuda.get_device_properties(0).multi_processor_count)


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
    sorted in 7/7/6/6-bit passes."""
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


# the sources
# ---------------------------------------------------------------------------------------------------------------------------
def _sources():
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if ".cu" in f or f.endswith(".h"):
            with open(os.path.join(CSRC, f)) as fh:
                out[f] = fh.read()
    return out


def test_ingest_shape_matches_the_sources():
    """the shape Geometry sizes the batches with is IngestShape, so they still hit N + 1, 2 N and 3.5 N chunks"""
    m = re.search(r"struct IngestShape\s*\{([^}]*)\}", _sources()["gysk_kernels.cuh"])
    assert m, "IngestShape not found in gysk_kernels.cuh"
    shape = {k: int(v) for k, v in re.findall(r"\b(WARPS|MIN_CTAS|EPT)\s*=\s*(\d+)", m.group(1))}
    assert shape == {"WARPS": WARPS, "MIN_CTAS": MIN_CTAS, "EPT": EPT}, shape
    assert re.search(r"\bCHUNK\s*=\s*32\s*\*\s*EPT\b", m.group(1))
    Geometry(132).sizes()                # the batch sizes of an H100 land where the region tests want them


def test_every_switch_is_listed_with_its_reason():
    """every GYSK_ string literal of the sources (getenv and the engine's envl helper) is in NOT_RUN with its reason: a new
    process-wide switch fails here until it comes with one"""
    names = set(re.findall(r'"(GYSK_[A-Z0-9_]+)"', "\n".join(_sources().values())))
    assert names, "no GYSK_ switch found in the sources"
    assert names == set(NOT_RUN), f"unlisted: {sorted(names - set(NOT_RUN))}, no longer read: {sorted(set(NOT_RUN) - names)}"
    assert all(NOT_RUN.values())
