"""The trace rows restated (tests only): what the engine keeps per traced service and 5-s window, from the raw request traces.

- The counters are the columns of the reference's trace view, tracereq_aggr_info (common/gy_json_field_maps.h:2628-2664), summed per
  service over the samples that arrived in the window.
- The digest of a window is the CPU oracle's own t-digest at compression 100: each (service, window) pair is a service of its own in an
  oracle engine created with td_compression = 100, fed the window's samples within the RESP validity rule as GYSK_EV_RESP events, one
  oracle batch per device batch. The device compresses its trace keys with the same value bins and merge step, so its centroids are
  the oracle's bit for bit.
- A service takes a row with its first trace event while rows are left (freed rows first); without one its events are dropped."""
import ctypes as C

import numpy as np

from gyeeta_b200 import engine as ge
from gyeeta_b200.wire import API_TRAN
from oracle import pyoracle as po

U32 = 0xFFFFFFFF
VALID_USEC = 1000001000          # GYSK_EV_RESP validity rule: response msec <= 1 000 000
BUCKET_EDGES = (300, 1000, 10000, 30000, 100000, 300000, 1000000)
COLS = ("nreq", "nerr", "nconns", "sum_resp_us", "max_resp_us", "bytes_in", "bytes_out", "max_bytes_in", "max_bytes_out")


def api_tran(glob_id, usec, reqlen=0, reslen=0, reqnum=1, errorcode=0, cliport=0):
    n = len(np.atleast_1d(glob_id))
    rec = np.zeros(n, dtype=API_TRAN)
    rec["tupd_usec"] = 1_700_000_000_000_000 + np.arange(n)
    rec["glob_id"], rec["response_usec"], rec["reqlen"], rec["reslen"] = glob_id, usec, reqlen, reslen
    rec["reqnum"], rec["errorcode"], rec["cliport"] = reqnum, errorcode, cliport
    return rec


def trace_events(rec, host_idx=0):
    """the GYSK_EV_TRACE event of each API_TRAN record (gysketch.h)"""
    ev = np.zeros(len(rec), dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = rec["glob_id"]
    ev["flow_key"] = np.minimum(rec["reqlen"], U32) | (np.minimum(rec["reslen"], U32) << np.uint64(32))
    ev["value"] = np.minimum(rec["response_usec"], U32)
    ev["host_idx"] = host_idx
    ev["tsec"] = rec["tupd_usec"] // 1_000_000
    ev["type"] = ge.EV_TRACE
    ev["flags"] = np.where(rec["errorcode"] != 0, ge.EVF_TRACE_ERROR, 0) | np.where(rec["reqnum"] == 0, ge.EVF_TRACE_NEWCONN, 0)
    return ev


def resp_events(rec, host_idx=0):
    """the GYSK_EV_RESP event the engine stages for each API_TRAN record beside its trace event"""
    ev = np.zeros(len(rec), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"], ev["value"] = rec["glob_id"], rec["cliport"], np.minimum(rec["response_usec"], U32)
    ev["host_idx"], ev["tsec"], ev["type"] = host_idx, rec["tupd_usec"] // 1_000_000, ge.EV_RESP
    err = rec["errorcode"]
    ev["flags"] = np.where(err == 0, 0, np.where(err >= 500, ge.EVF_SER_ERROR, ge.EVF_CLI_ERROR))
    return ev


def sql_aggregate(records):
    """tracereq_aggr_info over a list of API_TRAN dicts {glob_id, response, reqlen, reslen, reqnum, errorcode}, grouped by glob_id: the
    SQL of each column stated on its own, one record at a time; bytesin / bytesout are the 32-bit saturated reqlen_ / reslen_ the event
    carries"""
    out = {}
    for r in records:
        g = out.setdefault(r["glob_id"], dict(nreq=0, nerr=0, nconns=0, sum_resp_us=0, max_resp_us=0, bytes_in=0, bytes_out=0,
                                              max_bytes_in=0, max_bytes_out=0, resp_buckets=[0] * 8))
        resp, bin_, bout = min(r["response"], U32), min(r["reqlen"], U32), min(r["reslen"], U32)
        g["nreq"] += 1                                           # count(*)
        g["nerr"] += r["errorcode"] != 0                         # count(*) filter (where errorcode != 0)
        g["nconns"] += r["reqnum"] == 0                          # count(*) filter (where reqnum = 0)
        g["sum_resp_us"] += resp                                 # avg(response) = sum / nreq
        g["max_resp_us"] = max(g["max_resp_us"], resp)
        g["bytes_in"] += bin_
        g["bytes_out"] += bout
        g["max_bytes_in"] = max(g["max_bytes_in"], bin_)
        g["max_bytes_out"] = max(g["max_bytes_out"], bout)
        if resp < 300: g["resp_buckets"][0] += 1                 # resplt300us
        elif resp < 1000: g["resp_buckets"][1] += 1              # resplt1ms
        elif resp < 10000: g["resp_buckets"][2] += 1             # resplt10ms
        elif resp < 30000: g["resp_buckets"][3] += 1             # resplt30ms
        elif resp < 100000: g["resp_buckets"][4] += 1            # resplt100ms
        elif resp < 300000: g["resp_buckets"][5] += 1            # resplt300ms
        elif resp < 1000000: g["resp_buckets"][6] += 1           # resplt1sec
        else: g["resp_buckets"][7] += 1                          # respgt1sec
    return out


def empty_window():
    return dict(nreq=0, nerr=0, nconns=0, sum_resp_us=0, max_resp_us=0, bytes_in=0, bytes_out=0, max_bytes_in=0, max_bytes_out=0,
                resp_buckets=[0] * 8)


class TraceOracle:
    """the trace rows of an engine with `rows` trace rows, fed the same device batches and flushes"""

    def __init__(self, rows, max_windows=4096):
        self.rows, self.in_use, self.dropped = rows, set(), 0
        self.cur, self.last = {}, {}
        self.win = 0
        self.orc = po.OracleEngine(max_svcs=max_windows, max_tasks=16, cms_log2_width=4, hll_p=4, td_compression=100)
        self.shadow = {}             # (glob_id, window number) -> oracle service id
        self.win_of = {}             # glob_id -> (number of its open window, of its last window)
        self.L = ge.load_library()

    def _shadow(self, id_, w):
        return self.shadow.setdefault((id_, w), len(self.shadow) + 1)

    def ingest(self, ev):
        """one device batch: its GYSK_EV_TRACE events, in order"""
        tr = ev[ev["type"] == ge.EV_TRACE]
        keep = np.zeros(len(tr), dtype=bool)
        for i, id_ in enumerate(tr["svc_id"].tolist()):
            if id_ in (0, (1 << 64) - 1):
                continue
            if id_ not in self.in_use:
                if len(self.in_use) >= self.rows:
                    self.dropped += 1
                    continue
                self.in_use.add(id_)
                self.cur[id_], self.last[id_] = empty_window(), empty_window()
            keep[i] = True
        tr = tr[keep]
        for e in tr:
            id_, v = int(e["svc_id"]), int(e["value"])
            fk, fl = int(e["flow_key"]), int(e["flags"])
            w = self.cur[id_]
            w["nreq"] += 1; w["nerr"] += fl & 1; w["nconns"] += (fl >> 1) & 1
            w["sum_resp_us"] += v; w["max_resp_us"] = max(w["max_resp_us"], v)
            w["bytes_in"] += fk & U32; w["bytes_out"] += fk >> 32
            w["max_bytes_in"] = max(w["max_bytes_in"], fk & U32); w["max_bytes_out"] = max(w["max_bytes_out"], fk >> 32)
            w["resp_buckets"][int(np.searchsorted(BUCKET_EDGES, v, side="right"))] += 1
        dig = tr[tr["value"] < VALID_USEC]
        if len(dig):
            sev = np.zeros(len(dig), dtype=po.EVENT_DTYPE)
            sev["svc_id"] = [self._shadow(int(i), self.win) for i in dig["svc_id"].tolist()]
            sev["value"], sev["type"] = dig["value"], ge.EV_RESP
            self.orc.ingest(sev)

    def flush(self):
        self.last = self.cur
        self.cur = {i: empty_window() for i in self.in_use}
        self.win += 1

    def evict(self, ids):
        for i in ids:
            if i in self.in_use:
                self.in_use.discard(i)
                del self.cur[i], self.last[i]
                for w in (self.win, self.win - 1):          # a returning id starts from empty windows
                    self.shadow.pop((i, w), None)

    def digest(self, id_, last_window):
        """(means, weights, min, max) of a window's digest, or None for an id without a row"""
        if id_ not in self.in_use:
            return None
        key = (id_, self.win - (1 if last_window else 0))
        td = self.orc.export_tdigest(self.shadow[key]) if key in self.shadow else None
        if td is None:
            return np.zeros(0), np.zeros(0, dtype=np.uint64), float("inf"), float("-inf")
        means, weights = td.centroids()
        return means, weights.astype(np.uint64), td.minv, td.maxv

    def window(self, id_, last_window):
        w = dict((self.last if last_window else self.cur)[id_])
        means, weights, mn, mx = self.digest(id_, last_window)
        w["td_count"] = int(weights.sum())
        w["p99_resp_us"] = self.L.gysk_tdigest_quantile(ge._p(np.ascontiguousarray(means)), ge._p(np.ascontiguousarray(weights)),
                                                         len(means), mn, mx, 0.99) if len(means) else float("nan")
        return w

    def row(self, id_, host_idx=0):
        """the gysk_trace_row of id_ as a TraceRow"""
        r = ge.TraceRow()
        r.glob_id = id_
        if id_ not in self.in_use:
            return r
        r.found, r.host_idx = 1, host_idx
        for name, last in (("cur", False), ("last", True)):
            w, tw = self.window(id_, last), getattr(r, name)
            for f in COLS + ("td_count", "p99_resp_us"):
                setattr(tw, f, w[f])
            tw.resp_buckets[:] = w["resp_buckets"]
        return r


def row_bytes(r):
    return bytes(C.string_at(C.addressof(r), C.sizeof(r)))
