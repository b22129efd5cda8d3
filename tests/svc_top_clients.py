"""Each service's heaviest clients of GYSK_FLAG_SVC_TOP_CLIENTS restated on the CPU. batch_sums gives the exact per-(service, client)
sums {kbytes, conns} of the records of one device batch that feed the service's exact {count, kbytes} cell: the connection events
(CONNECT, ACCEPT, CLOSE_CLI, CLOSE_SER), each adding value >> 10 kbytes and one connection. merge is the weighted Misra-Gries merge of
include/gysketch.h. TopClients keeps the open and last summaries and the ring of 30-s slots as the engine keeps them, flush by flush and
slot by slot: the merge is not associative, so the level is not a merge of the held windows at once."""
import numpy as np

from gyeeta_b200 import engine as ge

K = ge.TOPC_K
NSLOTS, WIDTH = 10, 30
M32 = 0xFFFFFFFF
COUNTED = (ge.EV_CONNECT, ge.EV_ACCEPT, ge.EV_CLOSE_CLI, ge.EV_CLOSE_SER)
EMPTY = ((), 0)                     # a summary: (entries ((flow_key, kbytes, conns), ...) best first, delta)


def batch_sums(ev):
    """{svc_id: {flow_key: [kbytes, conns]}} of the counted records of one batch"""
    ev = ev[np.isin(ev["type"], COUNTED) & (ev["svc_id"] != 0) & (ev["svc_id"] != np.uint64(0xFFFFFFFFFFFFFFFF))]
    out = {}
    for s, k, v in zip(ev["svc_id"].tolist(), ev["flow_key"].tolist(), (ev["value"] >> 10).tolist()):
        d = out.setdefault(s, {}).setdefault(k, [0, 0])
        d[0] += v
        d[1] += 1
    return out


def merge(summaries, sums=None):
    """the merge of summaries and (optional) exact sums {flow_key: (kbytes, conns)}"""
    g = {}
    for ents, _ in summaries:
        for k, kb, c in ents:
            a = g.setdefault(k, [0, 0])
            a[0] += kb
            a[1] += c
    for k, (kb, c) in (sums or {}).items():
        a = g.setdefault(k, [0, 0])
        a[0] += kb
        a[1] += c
    groups = sorted(((k, kb, c) for k, (kb, c) in g.items() if kb > 0), key=lambda t: (-t[1], t[0]))
    cut = groups[K][1] if len(groups) > K else 0
    kept = tuple((k, min(kb - cut, M32), min(c, M32)) for k, kb, c in groups[:K] if kb > cut)
    return kept, sum(d for _, d in summaries) + cut


def row(summary):
    """(n, delta, entries as a K x 3 array) of a summary, as gysk_svc_top_clients holds it"""
    ents, delta = summary
    a = np.zeros((K, 3), dtype=np.uint64)
    for i, e in enumerate(ents):
        a[i] = e
    return len(ents), delta, a


class TopClients:
    """the summaries of every service: open, last, the ring slots with their epochs, and the level"""

    def __init__(self):
        self.open, self.last, self.level = {}, {}, {}
        self.ring = [{} for _ in range(NSLOTS)]
        self.epoch = [None] * NSLOTS

    def batch(self, ev):
        for s, d in batch_sums(ev).items():
            self.open[s] = merge([self.open.get(s, EMPTY)], d)

    def evict(self, ids):
        """the summaries of evicted services cleared (before the flush's roll, as the engine's eviction runs first)"""
        for s in ids:
            for m in [self.open, self.last, self.level] + self.ring:
                m.pop(int(s), None)

    def flush(self, tsec):
        ep = tsec // WIDTH
        k = ep % NSLOTS
        fresh = self.epoch[k] != ep
        if fresh:
            self.ring[k] = {}
            self.epoch[k] = ep
        for s in set(self.open) | set(self.ring[k]):
            self.ring[k][s] = merge([self.open.get(s, EMPTY), self.ring[k].get(s, EMPTY)])
        live = [j for j in range(NSLOTS) if self.epoch[j] is not None and ep - NSLOTS < self.epoch[j] <= ep]
        self.level = {}
        for s in set().union(*(self.ring[j] for j in live)):
            self.level[s] = merge([self.ring[j][s] for j in live if s in self.ring[j]])
        self.last, self.open = self.open, {}

    def get(self, which, sid):
        m = (self.open, self.last, self.level)[which]
        return m.get(int(sid), EMPTY)


def check_guarantees(summary, exact, n_s=None):
    """the four guarantees of a summary against exact {flow_key: (kbytes, conns)} over the records it covers; n_s: the service's exact
    kbytes (the sum of exact's kbytes by default)"""
    ents, delta = summary
    est = {k: (kb, c) for k, kb, c in ents}
    n_s = sum(kb for kb, _ in exact.values()) if n_s is None else n_s
    for k, (kb, c) in exact.items():
        e = est.get(k, (0, 0))[0]
        assert e <= kb <= e + delta, (k, e, kb, delta)
    for k, (kb, c) in est.items():
        assert k in exact and c <= exact[k][1], (k, c, exact.get(k))
    assert sum(kb for kb, _ in est.values()) + (K + 1) * delta <= n_s, (sum(kb for kb, _ in est.values()), delta, n_s)
    pos = {k: v for k, v in exact.items() if v[0] > 0}
    if len(pos) <= K and max((v[0] for v in pos.values()), default=0) <= M32:
        assert delta == 0 and {k: kb for k, (kb, _) in est.items()} == {k: kb for k, (kb, _) in pos.items()}, (est, pos, delta)
