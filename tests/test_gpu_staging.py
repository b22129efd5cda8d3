"""The host-to-device staging every production event passes through (gysk_engine.cu, "staging: per-thread page-locked buffers"),
in the two states no other test puts it in:

- the copy stream backed up behind the compute stream, so that a staged chunk's H2D copy is still queued when its thread (or the
  thread that adopts its stage) touches the chunk again: every ordered pair of entry paths, and a stage handed from an exited thread
  to a new one, against the oracle fed the same events;
- a tick thread flushing, reading and merging while eight threads ingest through every path and a reader thread queries: every
  event lands in exactly one window, calls split only as a prefix before a flush and the rest after it, windows follow each thread's
  call order and the host clock, and every closed window equals the oracle re-fed window by window with the membership observed."""
import itertools
import os
import threading
import time

import numpy as np
import pytest
import torch

from gyeeta_b200 import engine as ge, synth
from gyeeta_b200.wire import API_TRAN, TCP_CONN, build_msg
from oracle import pyoracle as po
from tests.test_gpu_ingest_paths import _packed, _pinned, _same
from tests.test_gpu_merge import _emulate_collectives
from tests.util import M32, MergeRestatement, assert_hist_equal

pytestmark = pytest.mark.gpu

RAW_BULK_MIN = 16384
CFG = dict(max_svcs=2048, max_tasks=512, cms_log2_width=12)
TASK_HISTS = (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY)
# a bounded spin on the engine's stream: 2.5e8 SM cycles, about 0.13 s at the H100's boost clock and 0.25 s at 1 GHz
SPIN_CYCLES = 250_000_000


def _tcp_conn_msg(rng, n, svc_id, host):
    """one NOTIFY_TCP_CONN message of n accepted connections of svc_id, and the GYSK_EV_CLOSE_SER events it stages, in order"""
    recs, ev = [], np.zeros(n, dtype=ge.EVENT_DTYPE)
    for i in range(n):
        r = np.zeros(1, dtype=TCP_CONN)
        r["ser_glob_id"], r["cli_task_aggr_id"] = svc_id, 5000 + int(rng.integers(0, 500))
        r["is_accept"], r["tusec_close"], r["tusec_start"] = 1, 9_000_000, 1_000_000
        r["bytes_sent"], r["bytes_rcvd"] = int(rng.integers(0, 1 << 20)), int(rng.integers(0, 1 << 20))
        recs.append((r, b"x" * int(rng.integers(0, 9))))
        ev[i]["svc_id"], ev[i]["flow_key"], ev[i]["type"], ev[i]["host_idx"] = svc_id, r["cli_task_aggr_id"][0], ge.EV_CLOSE_SER, host
        ev[i]["value"] = int(r["bytes_sent"][0]) + int(r["bytes_rcvd"][0])
    return build_msg(ge.NOTIFY_TCP_CONN, recs), ev


def _api_tran(resp):
    """API_TRAN records carrying the response events resp (tsec 0, no error): what gysk_ingest_raw(GYSK_RAW_API_TRAN) turns back into
    resp when the engine keeps no trace rows"""
    rec = np.zeros(len(resp), dtype=API_TRAN)
    rec["glob_id"], rec["response_usec"], rec["cliport"], rec["reqnum"] = resp["svc_id"], resp["value"], resp["flow_key"], 1
    return rec


def _resp16(resp):
    return _packed(resp)[1][0][1]


def _tcp24(tcp):
    return _packed(tcp)[1][1][1]


def _task24(task):
    return _packed(task)[1][2][1]


# ---- a. the copy stream backed up ---------------------------------------------------------------------------------------

S_A = RAW_BULK_MIN          # stage_batch: a pageable RESP16 bulk of S_A records is one piece, of S_A + 1 two
PATHS = ("bulk pageable 1 piece", "bulk pageable 2 pieces", "bulk page-locked", "raw pieces", "API_TRAN", "wire message",
         "event32 pageable", "gysk_ingest_pinned", "gysk_ingest_device")


class _Feed:
    """one engine, the oracle, and every entry path as a call on pre-built inputs (input buffers kept alive until the end)"""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        ev = synth.gen_mixed(self.rng, 200_000, 64, ntask=16, nhosts=8, nclients=2000)
        ev["flow_key"][ev["type"] == ge.EV_RESP] &= np.uint64(0xFF)      # RESP16 keeps 8 bits of the client port
        ev["tsec"] = 0
        self.resp, self.tcp = ev[ev["type"] == ge.EV_RESP], ev[(ev["type"] >= 1) & (ev["type"] <= 4)]
        self.task, self.mixed = ev[ev["type"] == ge.EV_TASK], ev
        self.off = dict(resp=0, tcp=0, task=0, mixed=0)
        self.eng = ge.Engine(max_batch=1 << 16, stage_batch=S_A, **CFG)
        self.fed, self.keep = [], []

    def take(self, what, n):
        a = getattr(self, what)
        o = self.off[what]
        assert o + n <= len(a), what
        self.off[what] = o + n
        return np.ascontiguousarray(a[o: o + n])

    def call(self, path):
        """the ingest of one path, to be run on the calling thread; its events go to the oracle's list now"""
        e = self.eng
        if path.startswith("bulk pageable"):
            r = self.take("resp", S_A if path.endswith("1 piece") else S_A + 3000)
            raw = _resp16(r)
            self.fed.append(r)
            return lambda: e.ingest_raw(ge.RAW_RESP16, raw, len(raw))
        if path == "bulk page-locked":
            t = self.take("tcp", RAW_BULK_MIN + 1000)
            self.keep.append(_pinned(_tcp24(t)))
            self.fed.append(t)
            buf = self.keep[-1]
            return lambda: e.ingest_raw_ptr(ge.RAW_TCP24, buf.data_ptr(), len(t))
        if path == "raw pieces":
            r, k = self.take("resp", 700), self.take("task", 500)
            r16, k24 = _resp16(r), _task24(k)
            self.fed += [r, k]
            return lambda: (e.ingest_raw(ge.RAW_RESP16, r16, len(r16)), e.ingest_raw(ge.RAW_TASK24, k24, len(k24)))
        if path == "API_TRAN":
            r = self.take("resp", 600).copy()
            r["host_idx"] = 3
            rec = _api_tran(r)
            self.fed.append(r)
            return lambda: e.ingest_raw(ge.RAW_API_TRAN, rec, len(rec), host_idx=3)
        if path == "wire message":
            msg, mev = _tcp_conn_msg(self.rng, 150, 1000 + int(self.rng.integers(0, 60)), 2)
            self.fed.append(mev)
            return lambda: self._ok(e.ingest_msg(msg, host_idx=2))
        m = self.take("mixed", 3000)
        self.fed.append(m)
        if path == "event32 pageable":
            return lambda: e.ingest_events(m)
        if path == "gysk_ingest_pinned":
            self.keep.append(_pinned(m))
            buf = self.keep[-1]
            return lambda: e.ingest_pinned_ptr(buf.data_ptr(), len(m))
        assert path == "gysk_ingest_device"
        self.keep.append(torch.from_numpy(m.view(np.uint8).copy()).cuda())
        torch.cuda.synchronize()
        buf = self.keep[-1]
        return lambda: e.ingest_device_ptr(buf.data_ptr(), len(m))

    @staticmethod
    def _ok(rc):
        assert rc == 0

    def hold(self):
        """a bounded spin on the engine's stream, then two device buffers' worth of page-locked events and one more: both buffers'
        batches queue behind the spin, and the copy stream waits for the first of them before its next copy"""
        m = self.take("mixed", 2 * S_A + 1)
        buf = _pinned(m)
        self.keep.append(buf)
        self.fed.append(m)
        stream = torch.cuda.ExternalStream(self.eng.stream())
        with torch.cuda.stream(stream):
            torch.cuda._sleep(SPIN_CYCLES)
        self.eng.ingest_pinned_ptr(buf.data_ptr(), len(m))
        assert not stream.query(), "the spin ended before the paths ran: the copies were never held back"

    def check(self):
        """sync, then every counter, the whole count-min table, every service's histogram, HLL registers and connection bitmap and
        every process's three histograms against the oracle fed the same events"""
        e = self.eng
        e.sync()
        ev = np.concatenate(self.fed)
        orc = po.OracleEngine(**CFG)
        orc.ingest(ev)
        st, oc = e.stats(), orc.counters()
        assert st["events_in"] == len(ev)
        for k, ok in dict(events_in="in", events_dropped="dropped", events_resp="resp", events_tcp="tcp", events_task="task",
                          nsvcs="nsvcs", ntasks="ntasks").items():
            assert st[k] == oc[ok], k
        assert np.array_equal(e.export_cms(), orc.cms())
        for s in np.unique(ev["svc_id"][ev["type"] != ge.EV_TASK]).tolist():
            assert_hist_equal(e, orc, s, ge.HIST_RESP_CUR)
            assert np.array_equal(e.export_hll(s), orc.export_hll(s)), hex(s)
            assert _same(e.export_conn_bitmap(s), orc.export_conn_bitmap(s)), hex(s)
        for t in np.unique(ev["svc_id"][ev["type"] == ge.EV_TASK]).tolist():
            for w in TASK_HISTS:
                assert_hist_equal(e, orc, t, w)


@pytest.mark.parametrize("first,then", list(itertools.product(PATHS, PATHS)))
def test_path_after_path_with_the_copy_stream_held(first, then):
    """Path `first` then path `then` on one thread while every copy waits behind the spin. A stage write into a chunk whose copy is
    still queued (ThreadStage's invariant broken) overwrites bytes the copy has not read yet."""
    f = _Feed(31)
    a, b = f.call(first), f.call(then)
    f.hold()
    a()
    b()
    f.check()


def _exited(native_id):
    """the thread is gone from the process, its thread_local destructors (which orphan its stages) run"""
    for _ in range(2000):
        if not os.path.exists(f"/proc/self/task/{native_id}"):
            return True
        time.sleep(0.001)
    return False


def test_adopted_stage_after_a_bulk_with_the_copy_stream_held():
    """a thread does a two-piece pageable bulk and exits; a new thread adopts its stage and stages events into it at once"""
    f = _Feed(32)
    bulk = f.call("bulk pageable 2 pieces")
    staged = [f.call(p) for p in ("event32 pageable", "raw pieces", "wire message", "API_TRAN")]
    f.hold()
    errs, ids = [], []

    def run(fns):
        ids.append(threading.get_native_id())
        try:
            for fn in fns:
                fn()
        except Exception as ex:               # noqa: BLE001 - reported below
            errs.append(ex)

    t1 = threading.Thread(target=run, args=([bulk],))
    t1.start(); t1.join()
    assert _exited(ids[0])
    t2 = threading.Thread(target=run, args=(staged,))
    t2.start(); t2.join()
    assert not errs, errs
    f.check()


# ---- b, c. flushes, reads and merges during ingest ----------------------------------------------------------------------

NTHR = 8
S_B = 2048                  # stage_batch: a thread chunk holds 2048 events, so staged calls of a few thousand events span chunks
KINDS = ("event32", "bulk pageable", "bulk page-locked", "raw pieces", "API_TRAN", "wire message", "gysk_ingest_pinned",
         "gysk_ingest_device")
ATOMIC = ("gysk_ingest_pinned", "gysk_ingest_device")     # one call under the engine mutex, after every stage is drained


class _Call:
    """one ingest call with a service of its own: its events in the order the engine stages them, is_resp[i] telling whether event i
    counts in the service's nqrys_5s (a response sample) or in its nconns_5s (a connection event); process events of its own
    processes only in the atomic paths, where no flush can split them"""

    def __init__(self, rng, thr, k, kind, svc_id, task_base):
        self.thr, self.k, self.kind, self.svc = thr, k, kind, svc_id
        self.keep = None
        host = thr

        def resp(n):
            ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
            ev["svc_id"], ev["type"], ev["host_idx"] = svc_id, ge.EV_RESP, host
            ev["value"] = np.minimum(np.exp(rng.normal(np.log(2000.0), 1.5, n)), 9.0e8).astype(np.uint32)
            ev["flow_key"] = rng.integers(0, 256, n)
            return ev

        def tcp(n):
            ev = np.zeros(n, dtype=ge.EVENT_DTYPE)
            ev["svc_id"], ev["host_idx"] = svc_id, host
            ev["type"] = rng.integers(1, 5, n)
            ev["flow_key"] = rng.integers(0, 1 << 63, n, dtype=np.uint64)
            ev["value"] = rng.integers(0, 1 << 22, n)
            return ev

        def alternate(n):
            """response and connection events in turn, starting with a response sample"""
            ev = np.empty(2 * n, dtype=ge.EVENT_DTYPE)
            ev[0::2], ev[1::2] = resp(n), tcp(n)
            return ev

        if kind == "event32":
            self.ev = alternate(int(rng.integers(400, 3000)))
        elif kind == "bulk pageable":
            self.ev = resp(RAW_BULK_MIN + int(rng.integers(0, 3000)))
        elif kind == "bulk page-locked":
            self.ev = tcp(RAW_BULK_MIN + int(rng.integers(0, 3000)))
            self.keep = _pinned(_tcp24(self.ev))
        elif kind == "raw pieces":
            self.ev = resp(int(rng.integers(300, 1500)))
        elif kind == "API_TRAN":
            self.ev = resp(int(rng.integers(300, 1500)))
        elif kind == "wire message":
            self.msg, self.ev = _tcp_conn_msg(rng, int(rng.integers(20, 120)), svc_id, host)
        else:
            task = np.zeros(int(rng.integers(20, 200)), dtype=ge.EVENT_DTYPE)
            task["svc_id"] = task_base + rng.integers(0, 4, len(task)).astype(np.uint64)
            task["type"], task["host_idx"] = ge.EV_TASK, host
            task["value"] = rng.integers(0, 3200, len(task))
            task["flow_key"] = rng.integers(0, 1 << 16, len(task)).astype(np.uint64) | (rng.integers(0, 1 << 16, len(task)).astype(np.uint64) << np.uint64(32))
            self.ev = np.concatenate([alternate(int(rng.integers(200, 1500))), task])
            if kind == "gysk_ingest_pinned":
                self.keep = _pinned(self.ev)
            else:
                self.keep = torch.from_numpy(self.ev.view(np.uint8).copy()).cuda()
        self.is_resp = self.ev["type"] == ge.EV_RESP
        self.counted = self.ev["type"] != ge.EV_TASK
        self.nresp, self.nconn = int(self.is_resp.sum()), int((self.counted & ~self.is_resp).sum())
        self.t0 = self.t1 = None
        self.pause = float(rng.uniform(0.0, 0.05))      # spreads each thread's calls over several ticks

    def run(self, e):
        if self.kind == "event32":
            e.ingest_events(self.ev)
        elif self.kind == "bulk pageable":
            r16 = _resp16(self.ev)
            e.ingest_raw(ge.RAW_RESP16, r16, len(r16))
        elif self.kind == "bulk page-locked":
            e.ingest_raw_ptr(ge.RAW_TCP24, self.keep.data_ptr(), len(self.ev))
        elif self.kind == "raw pieces":
            r16 = _resp16(self.ev)
            e.ingest_raw(ge.RAW_RESP16, r16, len(r16))
        elif self.kind == "API_TRAN":
            rec = _api_tran(self.ev)
            e.ingest_raw(ge.RAW_API_TRAN, rec, len(rec), host_idx=self.thr)
        elif self.kind == "wire message":
            assert e.ingest_msg(self.msg, host_idx=self.thr) == 0
        elif self.kind == "gysk_ingest_pinned":
            e.ingest_pinned_ptr(self.keep.data_ptr(), len(self.ev))
        else:
            e.ingest_device_ptr(self.keep.data_ptr(), len(self.ev))

    def segments(self, counts):
        """counts[w] = (responses, connections) of the call's service in window w -> [(w, start, end)]: the call's events as
        consecutive runs in window order, each run's mix of kinds checked against the layout"""
        out, pos = [], 0
        for w, (r, c) in enumerate(counts):
            if r == 0 and c == 0:
                continue
            seg = slice(pos, pos + r + c)
            assert pos + r + c <= int(self.counted.sum()), (self.kind, self.svc, counts)
            assert int(self.is_resp[seg].sum()) == r, ("not a run of the call's events", self.kind, hex(self.svc), counts)
            out.append((w, pos, pos + r + c))
            pos += r + c
        assert pos == int(self.counted.sum()), ("events lost or counted twice", self.kind, hex(self.svc), counts)
        return out


def test_tick_flushes_reads_and_merges_while_eight_threads_ingest():
    rng = np.random.default_rng(41)
    eng = ge.Engine(max_batch=1 << 16, stage_batch=S_B, **CFG)
    calls = []
    for t in range(NTHR):
        mine = []
        for k in range(32):
            kind = KINDS[(k + t) % len(KINDS)]
            mine.append(_Call(rng, t, k, kind, 0x51000000 + t * 1000 + k, np.uint64(0x71000000 + t * 1000 + 4 * k)))
        calls.append(mine)
    flat = [c for mine in calls for c in mine]
    ids = np.array([c.svc for c in flat], dtype=np.uint64)
    logical = np.array([1000 + c.thr * 8 + KINDS.index(c.kind) for c in flat], dtype=np.uint64)
    lids = np.unique(logical)
    eng.set_logical_map(ids, logical)
    torch.cuda.synchronize()

    errs, done = [], [0] * NTHR
    running = threading.Event()
    running.set()

    def ingest(t):
        try:
            for c in calls[t]:
                time.sleep(c.pause)
                c.t0 = time.monotonic_ns()
                c.run(eng)
                c.t1 = time.monotonic_ns()
                done[t] += 1
        except Exception as ex:               # noqa: BLE001 - reported below
            errs.append(ex)

    flushes = []                              # (tsec, t0, t1, snapshot)

    def snapshot():
        rows = {r["glob_id"]: r for r in eng.query_svcs(ids) if r["found"]}
        return dict(rows=rows, cms=eng.export_cms(last_window=True),
                    last={s: eng.export_hist(s, ge.HIST_RESP_LAST) for s in rows},
                    all={s: eng.export_hist(s, ge.HIST_RESP_ALL) for s in rows},
                    bm={s: eng.export_conn_bitmap(s, last_window=True) for s in rows})

    def flush(tsec):
        t0 = time.monotonic_ns()
        eng.flush(tsec)
        t1 = time.monotonic_ns()
        snap = snapshot()
        _emulate_collectives(torch, [eng])
        snap["logical"] = {r["glob_id"]: r for r in eng.query_logical(lids)}
        flushes.append((tsec, t0, t1, snap))

    def tick():
        try:
            while running.is_set():
                time.sleep(0.01)
                flush(5 * (len(flushes) + 1))
        except Exception as ex:               # noqa: BLE001 - reported below
            errs.append(ex)

    reads = []

    def reader():
        """all-time response counts (the t-digest's weight, kept per batch) never fall, and hold every sample of a call that returned
        before the read started; every read call succeeds"""
        try:
            prev, regs = {}, {}
            keys = np.unique(np.concatenate([c.ev["flow_key"][~c.is_resp & c.counted] for c in flat]))[:512]
            while running.is_set() or len(reads) < 3:
                during = running.is_set()
                ret = [c for t in range(NTHR) for c in calls[t][: done[t]]]
                rows = {r["glob_id"]: r for r in eng.query_svcs(ids)}
                for c in ret:
                    assert rows[c.svc]["found"] and rows[c.svc]["td_count"] == c.nresp, (c.kind, hex(c.svc))
                for s, r in rows.items():
                    assert r["td_count"] >= prev.get(s, 0), hex(s)
                    prev[s] = r["td_count"]
                win, n = eng.query_window()
                assert len(win) <= n <= len(ids)          # a service may register between the count call and the rows call
                eng.export_cms()
                eng.query_flows(keys)
                for c in ret[:: 7]:
                    h = eng.export_hll(c.svc)
                    assert np.all(h >= regs.get(c.svc, h)), hex(c.svc)
                    regs[c.svc] = h
                reads.append((time.monotonic_ns(), during))
        except Exception as ex:               # noqa: BLE001 - reported below
            errs.append(ex)

    ths = [threading.Thread(target=ingest, args=(t,)) for t in range(NTHR)]
    aux = [threading.Thread(target=tick), threading.Thread(target=reader)]
    for th in aux + ths:
        th.start()
    for th in ths:
        th.join()
    running.clear()
    for th in aux:
        th.join()
    assert not errs, errs
    flush(5 * (len(flushes) + 1))             # the last window: whatever is still staged
    last_call = max(c.t1 for c in flat)
    assert sum(f[1] < last_call for f in flushes) >= 2, (len(flushes), last_call)
    assert sum(d for _t, d in reads) >= 1, (reads, last_call)

    # membership: each call's per-window counts, read from its service's closed window after every flush
    nw = len(flushes)
    member = {}
    for c in flat:
        counts = []
        for _tsec, _t0, _t1, snap in flushes:
            r = snap["rows"].get(c.svc)
            counts.append((r["nqrys_5s"], r["nconns_5s"] & M32) if r else (0, 0))
        seg = c.segments(counts)
        member[c.svc] = seg
        ws = [w for w, _a, _b in seg]
        if c.kind in ATOMIC:
            assert len(ws) == 1, (c.kind, hex(c.svc), counts)
        for w, (_tsec, f0, f1, _snap) in enumerate(flushes):
            if c.t1 < f0:
                assert ws[-1] <= w, ("returned before flush", w, c.kind, hex(c.svc), ws)
            if c.t0 > f1:
                assert ws[0] > w, ("started after flush", w, c.kind, hex(c.svc), ws)
    # per thread, windows follow call order; page-locked raw input is the exception the header states (gysk_ingest_raw: its records
    # may reach the device ahead of records the thread staged before the call)
    for mine in calls:
        hi = 0
        for c in mine:
            ws = [w for w, _a, _b in member[c.svc]]
            if c.kind != "bulk page-locked":
                assert ws[0] >= hi, ("window order", c.kind, hex(c.svc), ws, hi)
            hi = max(hi, ws[-1])

    # the oracle re-fed window by window with that membership
    orc = po.OracleEngine(**CFG)
    restate = MergeRestatement([orc], ids, logical, 200, 12)
    for w, (tsec, _t0, _t1, snap) in enumerate(flushes):
        parts = []
        for c in flat:
            counted = c.ev[c.counted]
            for ww, a, b in member[c.svc]:
                if ww == w:
                    parts.append(counted[a:b])
                    if c.kind in ATOMIC:
                        parts.append(c.ev[~c.counted])
        if parts:
            orc.ingest(np.concatenate(parts))
        orc.flush(tsec)
        assert np.array_equal(snap["cms"], orc.cms(last_window=True)), w
        for s in ids.tolist():
            ol, oa = orc.export_hist(s, ge.HIST_RESP_LAST), orc.export_hist(s, ge.HIST_RESP_ALL)
            if ol is None:                     # nothing of it closed yet; it may be registered by events of the open window
                assert s not in snap["rows"] or (snap["last"][s][1] == 0 and snap["all"][s][1] == 0), (w, hex(s))
                continue
            assert s in snap["rows"], (w, hex(s))
            for got, want in ((snap["last"][s], ol), (snap["all"][s], oa)):
                assert np.array_equal(got[0]["count"], want[0]["count"]) and np.array_equal(got[0]["sum"], want[0]["sum"]), (w, hex(s))
                assert got[1:] == want[1:], (w, hex(s), got[1:], want[1:])
            assert _same(snap["bm"][s], orc.export_conn_bitmap(s, last_window=True)), (w, hex(s))
            row, (_cur, cl, _ac, _ak) = snap["rows"][s], orc.export_conn(s)
            assert (row["nconns_5s"], row["kbytes_5s"]) == (cl & M32, (cl >> 32) & M32), (w, hex(s))
            st = orc.export_state(s)
            assert (row["curr_state"], row["curr_issue"], row["issue_bit_hist"], row["high_resp_bit_hist"]) == st[:4], (w, hex(s))
        for lid in lids.tolist():
            cells, got = restate.cells(lid), snap["logical"][lid]
            assert got["nqrys_5s"] == int(cells["last"]["count"].sum()) & M32, (w, lid)
            assert got["total_resp_5sec"] == int(cells["last"]["sum"].sum()), (w, lid)
            assert (got["nconns_5s"], got["kbytes_5s"]) == (cells["conn"][0] & M32, cells["conn"][1] & M32), (w, lid)

    # what keeps growing inside a window, once everything has landed: HLL registers, process histograms, t-digest weights (the
    # centroids depend on how the events were cut into batches), the counters
    st, oc = eng.stats(), orc.counters()
    for k, ok in dict(events_in="in", events_resp="resp", events_tcp="tcp", events_task="task", nsvcs="nsvcs", ntasks="ntasks").items():
        assert st[k] == oc[ok], k
    rows = {r["glob_id"]: r for r in eng.query_svcs(ids)}
    for c in flat:
        assert np.array_equal(eng.export_hll(c.svc), orc.export_hll(c.svc)), hex(c.svc)
        td = orc.export_tdigest(c.svc)
        assert rows[c.svc]["td_count"] == c.nresp == (td.total if td is not None else 0), hex(c.svc)
        if c.kind in ATOMIC:
            for p in np.unique(c.ev["svc_id"][~c.counted]).tolist():
                for w in TASK_HISTS:
                    assert_hist_equal(eng, orc, p, w)
