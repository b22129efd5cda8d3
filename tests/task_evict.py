"""The process eviction of gysk_config.task_idle_evict_secs, restated over the CPU oracle, which keeps every process for good.

TaskEvict drives one oracle engine and decides the rule itself: a live process is stamped with the tsec of every flush whose closed
window held its samples (gyo_task_last), and by the first flush that sees it; the flush at tsec evicts it when stamp + secs < tsec.
Each eviction starts a new incarnation of the id: from then on its events reach the oracle under another id (oracle_id), so the oracle
builds the returning process from empty histograms, as the engine's recycled slot must. The table holds max_tasks live processes:
an event of a new id finds no slot while max_tasks are live and is dropped (the engine's free stack makes an evicted slot usable by the
next new id, so the live count is what fills the table).

cleanup_rule restates MCONN_HANDLER::cleanup_partha_unused_aggr_tasks (server/gy_mconnhdlr.cc:16492-16541) in its own terms, per
partha: every MAGGR_TASK of task_aggr_tbl_ whose last_tusec_ < now - 30 min is deleted."""
import numpy as np

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po

REFERENCE_SECS = 1800                  # 30 * GY_USEC_PER_MINUTE
INC_SHIFT = 48                         # incarnation k of id x reaches the oracle as x | k << 48 (test ids stay below 2^48)


def cleanup_rule(parthas, now_usec, secs=REFERENCE_SECS):
    """{partha: {aggr_task_id: last_tusec}} -> the ids each partha's walk deletes, per partha (the reference: secs = 30 min)"""
    min_upd_tusec = now_usec - secs * 1_000_000
    return {p: sorted(i for i, last in tbl.items() if last < min_upd_tusec) for p, tbl in parthas.items()}


class TaskEvict:
    def __init__(self, max_tasks, secs, max_svcs=1 << 10, oracle_tasks=1 << 14, **ocfg):
        self.orc = po.OracleEngine(max_svcs=max_svcs, max_tasks=oracle_tasks, **ocfg)
        self.max_tasks, self.secs = max_tasks, secs
        self.live = {}                  # id -> stamp (0: no flush has seen it yet)
        self.inc = {}                   # id -> incarnation
        self.host = {}                  # id -> host of the event that created its slot
        self.dropped = 0
        self.total = 0
        self.evicted = []

    def oracle_id(self, id_):
        return int(id_) | (self.inc.get(int(id_), 0) << INC_SHIFT)

    def admit(self, ev):
        """the events the engine applies, process ids renamed to their incarnation; new ids take slots in event order"""
        ev = np.array(ev, copy=True)
        keep = np.ones(len(ev), dtype=bool)
        for k in np.flatnonzero(ev["type"] == ge.EV_TASK):
            i = int(ev["svc_id"][k])
            if i not in self.live:
                if len(self.live) >= self.max_tasks:
                    keep[k] = False
                    self.dropped += 1
                    continue
                self.live[i] = 0
                self.host[i] = int(ev["host_idx"][k])
            ev["svc_id"][k] = self.oracle_id(i)
        return ev[keep]

    def ingest(self, ev):
        out = self.admit(ev)
        self.orc.ingest(out)
        return out

    def register(self, ids):
        for i in ids:
            i = int(i)
            if i not in self.live and len(self.live) < self.max_tasks:
                self.live[i] = 0
                self.host[i] = 0
                self.orc.register_ids(np.array([self.oracle_id(i)], dtype=np.uint64), is_task=True)

    def flush(self, tsec):
        self.orc.flush(tsec)
        ev = []
        for i in sorted(self.live):
            last = self.orc.task_last(self.oracle_id(i))
            if int(last[0]) or not self.live[i]:
                self.live[i] = tsec or 1
            if self.secs and self.live[i] + self.secs < tsec:
                ev.append(i)
        for i in ev:
            del self.live[i]
            self.inc[i] = self.inc.get(i, 0) + 1
        self.total += len(ev)
        self.evicted = ev
        return ev

    def hist(self, id_, which):
        return self.orc.export_hist(self.oracle_id(id_), which) if int(id_) in self.live else None

    def last(self, id_):
        return self.orc.task_last(self.oracle_id(id_)) if int(id_) in self.live else None
