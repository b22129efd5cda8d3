"""One model of an engine with any set of the flow and client flags (tests only): the Engine, the CPU oracle and one instance of every
restatement the flags turn on, fed the same device batches and flushes. check() reads every answer family the flags enable and compares
it with its restatement by that family's own rule, so that a feature is held to the truth while the others run beside it (every
ingest_kernel and drain_kernel instance, the shared sort buffers and the per-slot arrays that grow and eviction move). The flag rules of
gysk_create and the GPU matrix of tests/test_gpu_flag_matrix.py are stated here too, so that the CPU test can hold them to the library and
to the dispatch tables of gysk_kernels.cu."""
import itertools

import numpy as np

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests import client_levels as cl
from tests import flow_errors as fe
from tests import flow_level as fl
from tests import flow_queries as fq
from tests import flow_resp_hist as frh
from tests import flow_topk as ft
from tests import flow_topk_5min as ft5
from tests import flow_topk_slow as fs
from tests import logical_traces as lt
from tests import trace_agg as ta
from tests.task_evict import TaskEvict

# the nine flow and client flags, as Engine keywords
FLAGS = ("flow_level", "flow_queries", "flow_query_level", "flow_resp_hist", "flow_topk", "flow_topk_5min", "flow_topk_slow",
         "client_levels", "flow_errors")
K = ft.K
HIST_SVC = (ge.HIST_RESP_CUR, ge.HIST_RESP_LAST, ge.HIST_RESP_ALL)
HIST_TASK = (ge.HIST_TASK_CPU_PCT, ge.HIST_TASK_CPU_DELAY, ge.HIST_TASK_BLKIO_DELAY)
B_SLOW = fs.b_slow(300)                 # the default slow threshold


def allowed(f):
    """gysk_create's flag rules restated: f maps each of FLAGS to a bool"""
    if (f["flow_query_level"] or f["flow_resp_hist"] or f["flow_errors"]) and not f["flow_queries"]:
        return False
    if f["flow_topk_5min"] and not (f["flow_topk"] and (f["flow_level"] or f["flow_query_level"])):
        return False
    if f["flow_topk_slow"] and not (f["flow_topk"] and f["flow_resp_hist"]):
        return False
    return True


def subsets():
    """every one of the 2^9 flag sets, as {flag: bool}"""
    return [dict(zip(FLAGS, bits)) for bits in itertools.product((False, True), repeat=len(FLAGS))]


def drain_tuple(f):
    """(QRY, RH, TOPK, SLOW, CL, ERR) of the TCP drain_kernel pass launch_drains runs for flag set f"""
    return (f["flow_queries"], f["flow_queries"] and f["flow_resp_hist"], f["flow_topk"], f["flow_topk"] and f["flow_topk_slow"],
            f["client_levels"], f["flow_queries"] and f["flow_errors"])


def ingest_instance(f, trace):
    """(TRACE, QRY, TOPK, ERR, CL) of the ingest_kernel launch_ingest picks"""
    return (bool(trace), f["flow_queries"], f["flow_topk"], f["flow_errors"], f["client_levels"])


TRACE_ROWS = (0, 64)


def matrix():
    """the GPU matrix: [(name, flags, max_trace_svcs)], one case per reachable TCP drain tuple and trace setting. The level flags
    (FLOW_LEVEL, FLOW_QUERY_LEVEL, FLOW_TOPK_5MIN) follow a pattern over the cases, so that each is on in some and off in others."""
    tuples = sorted({drain_tuple(f) for f in subsets() if allowed(f)})
    out = []
    for i, (qry, rh, topk, slow, cl_, err) in enumerate(tuples):
        for j, rows in enumerate(TRACE_ROWS):
            f = dict(flow_queries=qry, flow_resp_hist=rh, flow_topk=topk, flow_topk_slow=slow, client_levels=cl_, flow_errors=err)
            f["flow_level"] = (i + j) % 2 == 0
            f["flow_query_level"] = qry and (i // 2 + j) % 2 == 0
            f["flow_topk_5min"] = topk and (f["flow_level"] or f["flow_query_level"]) and (i + 2 * j) % 3 != 2
            assert allowed(f), f
            name = "-".join(k[5:] if k.startswith("flow_") else k for k in FLAGS if f[k]) or "none"
            out.append((f"{name}-tr{rows}", f, rows))
    return out


def flag_name(kw):
    return "+".join(k for k in FLAGS if kw.get(k)) or "no flow flags"


class Mismatch(AssertionError):
    pass


def _first_diff(got, want):
    """the index of the first differing record of two arrays of one dtype (or the shorter length)"""
    got, want = np.asarray(got), np.asarray(want)
    n = min(len(got), len(want))
    if got.dtype.fields is None:
        d = np.flatnonzero(got[:n] != want[:n])
    else:
        gb, wb = got[:n].view(np.uint8).reshape(n, -1), want[:n].view(np.uint8).reshape(n, -1)
        d = np.flatnonzero((gb != wb).any(axis=1))
    return int(d[0]) if len(d) else n


class Model:
    """an Engine of one configuration and the restatement of everything it answers

    kw: the Engine keywords (flags, sizes, max_trace_svcs, rank / world, idle_evict_secs, task_idle_evict_secs); cap_svcs / cap_tasks:
    the oracles' capacities (the auto-grow ceilings where the engine starts small), so that no restatement drops an id the engine
    keeps. The stream must never fill the engine's tables: the tests assert the oracle's counters against the engine's."""

    def __init__(self, cap_svcs=None, cap_tasks=None, **kw):
        self.f = {k: bool(kw.get(k)) for k in FLAGS}
        self.eng = ge.Engine(**kw)
        c = self.eng.cfg
        self.d, self.w = c.cms_depth, c.cms_log2_width
        self.name = flag_name(kw) + (f", {kw['max_trace_svcs']} trace rows" if kw.get("max_trace_svcs") else "")
        if kw.get("rank") is not None and kw.get("world", 1) > 1:
            self.name += f", rank {kw['rank']}/{kw['world']}"
        self.orc = po.OracleEngine(max_svcs=cap_svcs or c.max_svcs, max_tasks=cap_tasks or c.max_tasks, cms_depth=self.d,
                                   cms_log2_width=self.w, hll_p=c.hll_p, td_compression=c.td_compression,
                                   flags=1 if kw.get("auto_register", True) else 0)        # fed this rank's shard only
        if c.idle_evict_secs:
            self.orc.set_idle_evict(c.idle_evict_secs)
        self.tasks = TaskEvict(cap_tasks or c.max_tasks, c.task_idle_evict_secs, cms_log2_width=4) if c.task_idle_evict_secs else None
        self.trace = ta.TraceOracle(c.max_trace_svcs, max_windows=1 << 16) if c.max_trace_svcs else None     # a long run's windows
        f, d, w = self.f, self.d, self.w
        empty1 = lambda: fe.empty(d, w)
        self.qry = [empty1(), empty1()] if f["flow_queries"] else None                   # [open, last]
        self.resp = [frh.empty(d, w), frh.empty(d, w)] if f["flow_resp_hist"] else None
        self.err = [empty1(), empty1()] if f["flow_errors"] else None
        cells = d << w
        self.ring = {}                                                                  # the 300-s levels of the tables
        if f["flow_level"]:
            self.ring["conn"] = fl.FlowLevelRing(cells)
        if f["flow_query_level"]:
            self.ring["qry"] = fl.FlowLevelRing(cells)
            if self.resp is not None:
                self.ring["resp"] = fl.FlowLevelRing(cells * frh.WORDS)
            if self.err is not None:
                self.ring["err"] = fl.FlowLevelRing(cells)
        self.sets, self.lv = {}, {}
        if f["flow_topk"]:
            self.sets["conn"] = ft.Sets(1, d, w)
            if f["flow_queries"]:
                self.sets["qry"] = ft.Sets(0, d, w)
            if f["flow_topk_slow"]:
                self.sets["slow"] = fs.Sets(B_SLOW, d, w)
            if f["flow_errors"]:
                self.sets["err"] = fe.Sets(d, w)
            if f["flow_topk_5min"]:
                if f["flow_level"]:
                    self.lv["conn"] = ft5.LevelSets(1, d, w)
                if f["flow_query_level"]:
                    self.lv["qry"] = ft5.LevelSets(0, d, w)
                    if "slow" in self.sets:
                        self.lv["slow"] = fs.LevelSets(B_SLOW, d, w)
                    if "err" in self.sets:
                        self.lv["err"] = fe.LevelSets(d, w)
        self.clients = cl.History() if f["client_levels"] else None
        self.win = []                       # the open window's batches (trace events left out)
        self.samples = []                   # the open window's counted response samples
        self.last_win = np.zeros(0, dtype=ge.EVENT_DTYPE)
        self.nflush, self.nbatch = 0, 0
        self.evicted = set()
        self.host_of = None                 # id -> host of the service's slot, where the stream fixes it
        self.exact_windows = {name: [] for name in self.lv}     # per flush {flow key: exact score} of the closed window, each level set
        self.tsecs = []
        self.ids = set()                    # every service id the stream has named
        self.task_ids = set()
        self.trace_host = {}

    # ---- feeding ----
    def ingest(self, ev, ingest=None, what=None):
        """one device batch: ev as the library expands it (a raw route's records already as events); ingest(eng) ingests it when the
        route is not ingest_events"""
        (ingest or (lambda e: e.ingest_events(ev)))(self.eng)
        self.eng.sync()
        self.nbatch += 1
        if self.trace is not None:
            self.trace.ingest(ev)
        ev = ev[ev["type"] != ge.EV_TRACE]
        if self.tasks is not None:
            is_task = ev["type"] == ge.EV_TASK
            self.tasks.ingest(ev[is_task])
            self.orc.ingest(ev[~is_task])
        else:
            self.orc.ingest(ev)
        self.ids |= set(np.unique(ev["svc_id"][ev["type"] != ge.EV_TASK]).tolist())
        self.task_ids |= set(np.unique(ev["svc_id"][ev["type"] == ge.EV_TASK]).tolist())
        self.win.append(ev)
        s = fq.counted(ev, None)
        self.samples.append(s)
        d, w = self.d, self.w
        if self.qry is not None:
            fq.add_samples(self.qry[0], s, d, w)
        if self.resp is not None:
            frh.add_samples(self.resp[0], s, d, w)
        if self.err is not None:
            fe.add_samples(self.err[0], s, d, w)
        if "conn" in self.sets:
            self.sets["conn"].batch(ft.batch_keys(ev, ft.CONN), self.orc.cms(False))
        if "qry" in self.sets:
            self.sets["qry"].batch(np.unique(s["flow_key"]), self.qry[0])
        if "slow" in self.sets:
            self.sets["slow"].batch(fs.slow_keys(s, B_SLOW), self.resp[0])
        if "err" in self.sets:
            self.sets["err"].batch(fe.ser_keys(s), self.err[0])

    def register(self, ids):
        ids = np.asarray(ids, dtype=np.uint64)
        self.eng.register_ids(ids)
        self.orc.register_ids(ids)
        self.ids |= set(ids.tolist())

    def grow(self, max_svcs=None, max_tasks=None):
        self.eng.grow(max_svcs, max_tasks)

    def flush(self, tsec):
        closing = dict(conn=self.orc.cms(False))
        for name, tab in (("qry", self.qry), ("resp", self.resp), ("err", self.err)):
            if tab is not None:
                closing[name] = tab[0]
        self.eng.flush(tsec)
        self.orc.flush(tsec)
        self.nflush += 1
        got, (want, _tot) = np.sort(self.eng.evicted_ids()), self.orc.evicted_ids()
        if not np.array_equal(got, np.sort(want)):
            raise Mismatch(f"[{self.name}] evicted_ids at flush {self.nflush} (tsec {tsec}): {got[:8]} != {np.sort(want)[:8]}")
        self.evicted = set(got.tolist())
        if self.tasks is not None:
            te = self.tasks.flush(tsec)
            gt = self.eng.evicted_task_ids().tolist()
            if gt != te:
                raise Mismatch(f"[{self.name}] evicted_task_ids at flush {self.nflush}: {gt[:8]} != {te[:8]}")
        for name, ring in self.ring.items():
            ring.flush(tsec, closing[name])
        for name, lv in self.lv.items():
            lv.flush(tsec, self.sets[name].open, closing[self.LEVEL_TABLE[name]])
        for s in self.sets.values():
            s.flush()
        for tab in (self.qry, self.resp, self.err):
            if tab is not None:
                tab[1], tab[0] = tab[0], np.zeros_like(tab[0])
        win = np.concatenate(self.win) if self.win else np.zeros(0, dtype=ge.EVENT_DTYPE)
        if self.clients is not None:
            self.clients.flush(tsec, win)
            for regs in self.clients.windows:           # an evicted service's sets go with its slot
                for sid in self.evicted:
                    regs.pop(int(sid), None)
        if self.trace is not None:
            self.trace.flush()
            self.trace.evict(self.evicted)
        self.last_win, self.last_samples = win, (np.concatenate(self.samples) if self.samples else fq.counted(win, None))
        self.tsecs.append(tsec)
        for name in self.lv:
            keys, ex = self.exact_scores(name, win, self.last_samples)
            self.exact_windows[name].append(dict(zip(keys.tolist(), ex.tolist())))
        self.win, self.samples = [], []

    # ---- checking ----
    def _fail(self, what, call, detail):
        raise Mismatch(f"[{self.name}] {call} at {what} (flush {self.nflush}, batch {self.nbatch}): {detail}")

    def _same(self, what, call, got, want, keys=None):
        got, want = np.asarray(got), np.asarray(want)
        if got.dtype == want.dtype and got.shape == want.shape and got.tobytes() == want.tobytes():
            return
        if got.dtype != want.dtype or got.shape != want.shape:
            if got.dtype.itemsize == want.dtype.itemsize and got.size == want.size and got.tobytes() == want.tobytes():
                return
            self._fail(what, call, f"shape {got.shape} {got.dtype} != {want.shape} {want.dtype}")
        i = _first_diff(got.reshape(-1) if got.dtype.fields is None else got, want.reshape(-1) if want.dtype.fields is None else want)
        g = got.reshape(-1)[i] if got.dtype.fields is None else (got[i] if i < len(got) else None)
        wv = want.reshape(-1)[i] if want.dtype.fields is None else (want[i] if i < len(want) else None)
        key = f" key {int(np.asarray(keys)[i]):#x}" if keys is not None and i < len(keys) else ""
        self._fail(what, call, f"first difference at {i}{key}: {g} != {wv} (lengths {len(got)} / {len(want)})")

    def probe_keys(self):
        """the flow keys the point queries read: the open and last windows' keys (a sample of them) and keys never seen"""
        parts = [w["flow_key"][:1500] for w in self.win[-2:]] + [self.last_win["flow_key"][:1500],
                                                                  np.arange(7, 70, dtype=np.uint64) << np.uint64(40)]
        return np.unique(np.concatenate(parts))

    def check(self, what, keys=None, nids=64):
        keys = self.probe_keys() if keys is None else np.unique(np.asarray(keys, dtype=np.uint64))
        self.check_always(what, keys, nids)
        self.check_flows(what, keys)
        if self.sets:
            self.check_sets(what)
        if self.clients is not None:
            self.check_clients(what)
        if self.trace is not None:
            self.check_traces(what)

    def live_ids(self, nids):
        ids = sorted(i for i in self.ids if i not in (0, (1 << 64) - 1))
        if len(ids) > nids:
            step = len(ids) / nids
            ids = [ids[int(j * step)] for j in range(nids)]
        return ids

    def check_always(self, what, keys, nids):
        e, o = self.eng, self.orc
        for lw in (False, True):
            self._same(what, f"export_cms(last_window={lw})", e.export_cms(lw).reshape(-1), o.cms(lw))
        s, c = e.stats(), o.counters()
        pairs = [("events_resp", "resp"), ("events_tcp", "tcp")]
        if not self.eng.cfg.idle_evict_secs:          # with eviction the evicted ids, and every id's answers, are checked instead
            pairs.append(("nsvcs", "nsvcs"))
        if self.tasks is None:
            pairs += [("events_task", "task"), ("ntasks", "ntasks")]
        for a, b in pairs:
            if s[a] != c[b]:
                self._fail(what, "stats()", f"{a} {s[a]} != oracle {b} {c[b]}")
        if self.tasks is not None and s["ntasks"] != len(self.tasks.live):
            self._fail(what, "stats()", f"ntasks {s['ntasks']} != {len(self.tasks.live)} live processes")
        for id_ in self.live_ids(nids):
            for which in HIST_SVC:
                a, b = e.export_hist(id_, which), o.export_hist(id_, which)
                if (a is None) != (b is None) or (a is not None and (a[0].tobytes() != b[0].tobytes() or a[1:] != b[1:])):
                    self._fail(what, f"export_hist({id_:#x}, {which})", f"{None if a is None else a[1:]} != {None if b is None else b[1:]}")
            a, b = e.export_hll(id_), o.export_hll(id_)
            if (a is None) != (b is None) or (a is not None and a.tobytes() != b.tobytes()):
                self._fail(what, f"export_hll({id_:#x})", "registers differ")
            td, otd = e.export_tdigest(id_), o.export_tdigest(id_)
            if (td is None) != (otd is None):
                self._fail(what, f"export_tdigest({id_:#x})", f"{td is None} != {otd is None}")
            if td is not None:
                m, wt = otd.centroids()
                if td[0].tobytes() != m.tobytes() or td[1].tobytes() != wt.astype(td[1].dtype).tobytes() or \
                        (len(m) and (td[2], td[3]) != (otd.minv, otd.maxv)):
                    self._fail(what, f"export_tdigest({id_:#x})", f"{len(td[0])} centroids != {len(m)}")
            for lw in (False, True):
                a, b = e.export_conn_bitmap(id_, lw), o.export_conn_bitmap(id_, lw)
                if (a is None) != (b is None) or (a is not None and not (np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]))):
                    self._fail(what, f"export_conn_bitmap({id_:#x}, {lw})", "differs")
        tids = sorted(self.task_ids)[:16]
        for id_ in tids:
            for which in HIST_TASK:
                a = e.export_hist(id_, which)
                b = self.tasks.hist(id_, which) if self.tasks is not None else o.export_hist(id_, which)
                if (a is None) != (b is None) or (a is not None and (a[0].tobytes() != b[0].tobytes() or a[1:] != b[1:])):
                    self._fail(what, f"export_hist(task {id_:#x}, {which})", f"{None if a is None else a[1:]} != {None if b is None else b[1:]}")

    def _flow_rows(self, table, keys):
        lo, hi = fq.point_query(table, keys, self.d, self.w)
        out = np.zeros(len(keys), dtype=ge.FLOW_EST_DTYPE)
        out["flow_key"], out["count"], out["kbytes"] = keys, lo, hi
        return out

    def _qry_rows(self, table, keys):
        return self._flow_rows(table, keys).view(ge.FLOW_QRY_EST_DTYPE)

    def check_flows(self, what, keys):
        e, d, w = self.eng, self.d, self.w
        for lw in (False, True):
            self._same(what, f"query_flows(last_window={lw})", e.query_flows(keys, lw), self._flow_rows(self.orc.cms(lw), keys), keys)
            if self.qry is not None:
                q = self.qry[lw]
                self._same(what, f"export_cms_queries(last_window={lw})", e.export_cms_queries(lw).reshape(-1), q)
                self._same(what, f"query_flow_queries(last_window={lw})", e.query_flow_queries(keys, lw), self._qry_rows(q, keys), keys)
            if self.resp is not None:
                self._same(what, f"export_cms_resp(last_window={lw})", e.export_cms_resp(lw).reshape(-1), self.resp[lw])
                self._same(what, f"query_flow_resp(last_window={lw})", e.query_flow_resp(keys, lw), frh.point_query(self.resp[lw], keys, d, w),
                           keys)
            if self.err is not None:
                self._same(what, f"export_cms_errors(last_window={lw})", e.export_cms_errors(lw).reshape(-1), self.err[lw])
                self._same(what, f"query_flow_errors(last_window={lw})", e.query_flow_errors(keys, lw),
                           fe.point_query(self.err[lw], self.qry[lw], keys, d, w), keys)
        if "conn" in self.ring:
            lv = self.ring["conn"].level
            self._same(what, "export_cms_5min", e.export_cms_5min().reshape(-1), lv)
            self._same(what, "query_flows_5min", e.query_flows_5min(keys), self._flow_rows(lv, keys), keys)
        if "qry" in self.ring:
            lv = self.ring["qry"].level
            self._same(what, "export_cms_queries_5min", e.export_cms_queries_5min().reshape(-1), lv)
            self._same(what, "query_flow_queries_5min", e.query_flow_queries_5min(keys), self._qry_rows(lv, keys), keys)
        if "resp" in self.ring:
            lv = self.ring["resp"].level
            self._same(what, "export_cms_resp_5min", e.export_cms_resp_5min().reshape(-1), lv)
            self._same(what, "query_flow_resp_5min", e.query_flow_resp_5min(keys), frh.point_query(lv, keys, d, w), keys)
        if "err" in self.ring:
            lv = self.ring["err"].level
            self._same(what, "export_cms_errors_5min", e.export_cms_errors_5min().reshape(-1), lv)
            self._same(what, "query_flow_errors_5min", e.query_flow_errors_5min(keys), fe.point_query(lv, self.ring["qry"].level, keys, d, w),
                       keys)

    def _read(self, name, keys, lw=None, level=False):
        """the restated read of a set (keys) on the table it is scored on: the window's (lw) or the level's"""
        d, w = self.d, self.w
        if name == "conn":
            t = self.ring["conn"].level if level else self.orc.cms(lw)
            return ft.read(keys, t, d, w, 1)
        if name == "qry":
            t = self.ring["qry"].level if level else self.qry[lw]
            return ft.read(keys, t, d, w, 0)
        if name == "slow":
            t = self.ring["resp"].level if level else self.resp[lw]
            return fs.read(keys, t, d, w, B_SLOW)
        t, q = (self.ring["err"].level, self.ring["qry"].level) if level else (self.err[lw], self.qry[lw])
        return fe.read(keys, t, q, d, w)

    LEVEL_TABLE = {"conn": "conn", "qry": "qry", "slow": "resp", "err": "err"}       # the table each set is scored on
    READS = {"conn": ("topk_flows", "topk_flows_5min"), "qry": ("topk_flow_queries", "topk_flow_queries_5min"),
             "slow": ("topk_flow_slow", "topk_flow_slow_5min"), "err": ("topk_flow_errors", "topk_flow_errors_5min")}

    def check_sets(self, what):
        e = self.eng
        for name, s in self.sets.items():
            call, call5 = self.READS[name]
            for lw, keys in ((False, s.open), (True, s.last)):
                got = getattr(e, call)(K, lw)
                want = self._read(name, keys, lw)
                self._same(what, f"{call}(last_window={lw})", got.view(want.dtype) if got.dtype != want.dtype else got, want, want["flow_key"])
            if name in self.lv:
                rows, bound = getattr(e, call5)(K)
                lv = self.lv[name]
                want = self._read(name, lv.L, level=True)
                self._same(what, call5, rows.view(want.dtype) if rows.dtype != want.dtype else rows, want, want["flow_key"])
                if bound != lv.B:
                    self._fail(what, call5, f"bound {bound} != {lv.B}")
        self.check_guarantees(what)

    @staticmethod
    def exact_scores(name, ev, s):
        """(flow keys, their exact scores) of set name over the events ev of a window and its counted samples s"""
        if name == "conn":
            ev = ev[np.isin(ev["type"], ft.TCP_TYPES) & (ev["svc_id"] != 0)]
            allk = np.unique(ev["flow_key"])
            return allk, ft.exact_scores(allk, ev["flow_key"], ft.conn_increments(ev), 1)
        allk = np.unique(s["flow_key"])
        if name == "qry":
            return allk, ft.exact_scores(allk, s["flow_key"], fq.increments(s), 0)
        if name == "slow":
            return allk, fs.exact_slow(s, allk, B_SLOW)
        return allk, fe.exact(s, allk)[:, 1]

    def check_guarantees(self, what):
        """each set's guarantee against exact scores: the open window's set (while the window holds batches), the last window's set,
        and every level set with its bound against the exact scores over the windows its level holds"""
        d, w = self.d, self.w
        views = []
        if self.win:
            views.append((False, np.concatenate(self.win), np.concatenate(self.samples)))
        if self.nflush:
            views.append((True, self.last_win, self.last_samples))
        for name, sets in self.sets.items():
            for lw, ev, s in views:
                keys = sets.last if lw else sets.open
                tab = {"conn": lambda: self.orc.cms(lw), "qry": lambda: self.qry[lw], "slow": lambda: self.resp[lw],
                       "err": lambda: self.err[lw]}[name]()
                allk, ex = self.exact_scores(name, ev, s)
                if name == "conn":
                    ok = ft.guarantee_holds(keys, tab, d, w, 1, allk, ex)
                elif name == "qry":
                    ok = ft.guarantee_holds(keys, tab, d, w, 0, allk, ex)
                elif name == "slow":
                    ok = fs.guarantee_holds(keys, tab, d, w, sets.score, allk, ex)
                else:
                    t = fs.thr(keys, tab, d, w, fe.ser_score) if len(keys) == K else 0
                    members = set(keys.tolist())
                    ok = all(k in members for k, x in zip(allk.tolist(), ex.tolist()) if x > t)
                if not ok:
                    self._fail(what, f"{self.READS[name][0]}(last_window={lw}) guarantee", "a flow above the set's floor is missing")
            if name in self.lv and self.tsecs:
                lv = self.lv[name]
                exact = ft5.exact_level(self.tsecs, self.exact_windows[name])
                if not ft5.guarantee_holds(lv.L, lv.B, exact):
                    self._fail(what, f"{self.READS[name][1]} bound", f"a flow outside the level set scores above the bound {lv.B}")

    def check_clients(self, what):
        e, h = self.eng, self.clients
        ids = np.array(self.live_ids(64), dtype=np.uint64)
        rows = e.query_svc_clients(ids)
        lastkeys = cl.window_keys(self.last_win) if self.clients.windows else {}
        for sid, r in zip(ids.tolist(), rows):
            last, lvl = e.export_hll_window(sid, ge.CLIENTS_LAST), e.export_hll_window(sid, ge.CLIENTS_5MIN)
            if last is None:
                if r.found:
                    self._fail(what, f"export_hll_window({sid:#x})", "None for a service query_svc_clients finds")
                continue
            self._same(what, f"export_hll_window({sid:#x}, CLIENTS_LAST)", last, h.last(sid))
            self._same(what, f"export_hll_window({sid:#x}, CLIENTS_5MIN)", lvl, h.level(sid))
            est = (e.L.gysk_hll_estimate(ge._p(last), cl.P), e.L.gysk_hll_estimate(ge._p(lvl), cl.P))
            if not r.found or (r.last_5s, r.last_5min) != est:
                self._fail(what, f"query_svc_clients({sid:#x})", f"{(r.found, r.last_5s, r.last_5min)} != {est}")
            exact = len(np.unique(lastkeys.get(sid, np.zeros(0, np.uint64))))
            if exact >= 64 and abs(r.last_5s - exact) > cl.BOUND * exact:
                self._fail(what, f"query_svc_clients({sid:#x})", f"last_5s {r.last_5s} not within {cl.BOUND} of {exact} distinct clients")

    def check_traces(self, what):
        e, to = self.eng, self.trace
        ids = sorted(to.in_use)
        probe = ids + [0xDEAD0000BEEF]
        for id_, r in zip(probe, e.query_traces(probe)):
            # the row's host is its service slot's; the stream fixes it where host_of is set
            want = to.row(id_, self.host_of(id_) if self.host_of and id_ in to.in_use else r.host_idx)
            if ta.row_bytes(r) != ta.row_bytes(want):
                self._fail(what, f"query_traces({id_:#x})", f"{r.asdict()} != {want.asdict()}")
        for id_ in ids[:16]:
            for lw in (False, True):
                m, wt, mn, mx = e.export_trace_tdigest(id_, lw)
                om, ow, omn, omx = to.digest(id_, lw)
                if m.tobytes() != np.asarray(om, dtype=np.float64).tobytes() or not np.array_equal(wt, ow) or \
                        (len(m) and (mn, mx) != (omn, omx)):
                    self._fail(what, f"export_trace_tdigest({id_:#x}, {lw})", f"{len(m)} centroids != {len(om)}")
        if e.trace_info() != (len(to.in_use), to.dropped):
            self._fail(what, "trace_info", f"{e.trace_info()} != {(len(to.in_use), to.dropped)}")


def check_merged(models, what):
    """the _global reads of every rank after a merge, restated from the per-rank models: the summed tables and levels, and the merge of
    each module's sets"""
    m0 = models[0]
    d, w, f = m0.d, m0.w, m0.f
    total = lambda get: sum((get(m) for m in models[1:]), get(models[0]).copy())
    keys = np.unique(np.concatenate([m.last_win["flow_key"][:1500] for m in models] + [np.arange(1, 50, dtype=np.uint64)]))
    conn = total(lambda m: m.orc.cms(True))
    qry = total(lambda m: m.qry[1]) if f["flow_queries"] else None
    resp = total(lambda m: m.resp[1]) if f["flow_resp_hist"] else None
    err = total(lambda m: m.err[1]) if f["flow_errors"] else None
    lv = {name: total(lambda m: m.ring[name].level) for name in m0.ring}
    want = {"query_flows_global": m0._flow_rows(conn, keys)}
    if qry is not None:
        want["query_flow_queries_global"] = m0._qry_rows(qry, keys)
    if resp is not None:
        want["query_flow_resp_global"] = frh.point_query(resp, keys, d, w)
    if err is not None:
        want["query_flow_errors_global"] = fe.point_query(err, qry, keys, d, w)
    want5 = {}
    if "conn" in lv:
        want5["query_flows_global_5min"] = m0._flow_rows(lv["conn"], keys)
    if "qry" in lv:
        want5["query_flow_queries_global_5min"] = m0._qry_rows(lv["qry"], keys)
    if "resp" in lv:
        want5["query_flow_resp_global_5min"] = frh.point_query(lv["resp"], keys, d, w)
    if "err" in lv:
        want5["query_flow_errors_global_5min"] = fe.point_query(lv["err"], lv["qry"], keys, d, w)
    sets = {}
    if f["flow_topk"]:
        last = lambda name: [m.sets[name].last for m in models]
        sets["topk_flows_global"] = ft.read(ft.merged(last("conn"), conn, d, w, 1), conn, d, w, 1)
        if "qry" in m0.sets:
            sets["topk_flow_queries_global"] = ft.read(ft.merged(last("qry"), qry, d, w, 0), qry, d, w, 0)
        if "slow" in m0.sets:
            sets["topk_flow_slow_global"] = fs.read(fs.merged(last("slow"), resp, d, w, B_SLOW), resp, d, w, B_SLOW)
        if "err" in m0.sets:
            sets["topk_flow_errors_global"] = fe.read(fe.merged(last("err"), err, d, w), err, qry, d, w)
    sets5 = {}
    Ls, Bs = (lambda name: [m.lv[name].L for m in models]), (lambda name: [m.lv[name].B for m in models])
    if "conn" in m0.lv:
        g, b = ft5.merged(Ls("conn"), Bs("conn"), lv["conn"], d, w, 1)
        sets5["topk_flows_global_5min"] = (ft.read(g, lv["conn"], d, w, 1), b)
    if "qry" in m0.lv:
        g, b = ft5.merged(Ls("qry"), Bs("qry"), lv["qry"], d, w, 0)
        sets5["topk_flow_queries_global_5min"] = (ft.read(g, lv["qry"], d, w, 0), b)
    if "slow" in m0.lv:
        g, b = fs.merged(Ls("slow"), lv["resp"], d, w, B_SLOW, bounds=Bs("slow"))
        sets5["topk_flow_slow_global_5min"] = (fs.read(g, lv["resp"], d, w, B_SLOW), b)
    if "err" in m0.lv:
        g, b = fe.merged(Ls("err"), lv["err"], d, w, bounds=Bs("err"))
        sets5["topk_flow_errors_global_5min"] = (fe.read(g, lv["err"], lv["qry"], d, w), b)
    for m in models:
        for call, rows in want.items():
            m._same(what, call, getattr(m.eng, call)(keys, True), rows, keys)
        for call, rows in want5.items():
            m._same(what, call, getattr(m.eng, call)(keys), rows, keys)
        for call, rows in sets.items():
            got = getattr(m.eng, call)()
            m._same(what, call, got.view(rows.dtype) if got.dtype != rows.dtype else got, rows, rows["flow_key"])
        for call, (rows, b) in sets5.items():
            got, bound = getattr(m.eng, call)()
            m._same(what, call, got.view(rows.dtype) if got.dtype != rows.dtype else got, rows, rows["flow_key"])
            if bound != b:
                m._fail(what, call, f"bound {bound} != {b}")


def check_logical(models, glob, logical, what):
    """the logical services' merged reads on every rank after a merge, restated from the ranks' models: gysk_query_logical against
    LevelRestatement over the ranks' oracles (every field but the listener state, which the merge takes from the state decision),
    the merged client registers and their estimates against the maximum of the members' restated registers, and
    gysk_query_logical_traces against tests/logical_traces.py over the ranks' trace restatements"""
    from tests.test_gpu_merge_exact import DOUBLE_FIELDS, INT_FIELDS
    from tests.test_gpu_merge_levels import STATE_FIELDS, LevelRestatement
    from tests.util import same_double
    m0 = models[0]
    c = m0.eng.cfg
    lib = ge.load_library()
    members = lt.members_of(glob, logical)
    lids = list(members)
    rs = LevelRestatement([m.orc for m in models], glob, logical, c.td_compression, c.hll_p)
    want = {lid: rs.summary(lid, lib) for lid in lids}
    ints = [f for f in INT_FIELDS if f not in STATE_FIELDS]
    regs = {}
    if m0.clients is not None:
        for lid, gs in members.items():
            for which, get in ((ge.CLIENTS_LAST, lambda h, g: h.last(g)), (ge.CLIENTS_5MIN, lambda h, g: h.level(g))):
                acc = np.zeros(cl.NREG, np.uint8)
                for m in models:
                    for g in gs:
                        np.maximum(acc, get(m.clients, g), out=acc)
                regs[lid, which] = acc
    traces = {lid: lt.row_bytes(lt.row([m.trace for m in models], lid, gs)[0]) for lid, gs in members.items()} if m0.trace else {}
    for m in models:
        for lid, got in zip(lids, m.eng.query_logical(lids)):
            got = got.asdict() if hasattr(got, "asdict") else got
            for f in ints:
                if got[f] != want[lid][f]:
                    m._fail(what, f"query_logical({lid})", f"{f} {got[f]} != {want[lid][f]}")
            for f in DOUBLE_FIELDS:
                if not same_double(got[f], want[lid][f]):
                    m._fail(what, f"query_logical({lid})", f"{f} {got[f]} != {want[lid][f]}")
        if regs:
            for lid, r in zip(lids, m.eng.query_logical_clients(np.array(lids, dtype=np.uint64))):
                est = []
                for which in (ge.CLIENTS_LAST, ge.CLIENTS_5MIN):
                    w = regs[lid, which]
                    m._same(what, f"export_logical_hll_window({lid}, {which})", m.eng.export_logical_hll_window(lid, which), w)
                    est.append(lib.gysk_hll_estimate(ge._p(w), cl.P))
                if not r.found or [r.last_5s, r.last_5min] != est:
                    m._fail(what, f"query_logical_clients({lid})", f"{(r.found, r.last_5s, r.last_5min)} != {est}")
        if traces:
            for lid, r in zip(lids, m.eng.query_logical_traces(lids)):
                if lt.row_bytes(r) != traces[lid]:
                    m._fail(what, f"query_logical_traces({lid})", f"{r.asdict()}")
