"""The rolling 300-s count-min level of GYSK_FLAG_FLOW_LEVEL restated on the CPU, two ways. FlowLevelRing keeps the ring as the engine
keeps it: ring slot (tsec / 30) % 10, a slot holding another epoch replaced, the level the sum of the slots whose epochs lie in the last
10 of the last flush's. held_windows states which flushes the level holds from the whole flush history. Both take the table of each
window a flush closes: the oracle's cms(last_window=True) or the engine's export_cms(last_window=True) right after the flush. The
scripted flush sequences and the flow stream are shared by the CPU and the GPU tests."""
import numpy as np

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po

NSLOTS, WIDTH = 10, 30
M32 = 0xFFFFFFFF

# flush tsec sequences: 5-s steps across more than 300 s; gaps of 29, 30, 31 and 301 s; the same tsec twice; a first flush at 0; and a
# step back, which takes a ring slot from a later epoch
SEQUENCES = {
    "steps_5s": list(range(5, 405, 5)),
    "gaps": [1000, 1005, 1034, 1064, 1095, 1396, 1401, 1430, 1460, 1491, 1792, 1797],
    "same_tsec": [600, 605, 605, 610, 610, 640, 640, 645],
    "first_at_0": [0, 5, 30, 300, 305, 329, 330],
    "step_back": [900, 930, 960, 620, 930, 935, 1200],
}


class FlowLevelRing:
    def __init__(self, ncell):
        self.ring = np.zeros((NSLOTS, ncell), dtype=np.uint64)
        self.epoch = [None] * NSLOTS
        self.level = np.zeros(ncell, dtype=np.uint64)

    def flush(self, tsec, closed):
        """the window closed at tsec, whose table is `closed`, joins the ring; returns the level"""
        ep = tsec // WIDTH
        k = ep % NSLOTS
        if self.epoch[k] != ep:
            self.ring[k] = 0
            self.epoch[k] = ep
        self.ring[k] += closed                          # uint64: mod 2^64 per cell
        self.level = np.zeros_like(self.level)
        for j in range(NSLOTS):
            if self.epoch[j] is not None and ep - NSLOTS < self.epoch[j] <= ep:
                self.level += self.ring[j]
        return self.level


def held_windows(tsecs):
    """indices of the flushes the level holds after the last of tsecs: the epoch lies in the last NSLOTS epochs of the last flush's,
    and no later flush took its ring slot for another epoch (which only a step back in tsec can do)"""
    ep = [t // WIDTH for t in tsecs]
    last = ep[-1]
    return [i for i, e in enumerate(ep)
            if last - NSLOTS < e <= last and all(ep[j] % NSLOTS != e % NSLOTS or ep[j] == e for j in range(i + 1, len(ep)))]


def level_of_history(tsecs, tables):
    out = np.zeros_like(tables[0])
    for i in held_windows(tsecs):
        out += tables[i]
    return out


def flow_events(rng, n, keys, nsvc=64, huge=0):
    """n connection events over the flow keys: connect / accept / close events (count 1, kbytes = bytes >> 10) and ACTIVE_CONN_STATS
    records (count = active connections, kbytes = value). huge: that many more close events of 4 GB - 1 bytes on keys[0], so that the
    kbytes half of its cells wraps"""
    ev = np.zeros(n + huge, dtype=ge.EVENT_DTYPE)
    ev["svc_id"] = rng.integers(1, nsvc + 1, len(ev)).astype(np.uint64) * np.uint64(2654435761)
    ev["host_idx"] = rng.integers(0, 16, len(ev))
    ev["flow_key"] = keys[rng.integers(0, len(keys), len(ev))]
    ev["type"] = rng.choice(np.array([ge.EV_CONNECT, ge.EV_ACCEPT, ge.EV_CLOSE_CLI, ge.EV_CLOSE_SER, ge.EV_ACTIVE], dtype=np.uint16), len(ev))
    ev["value"] = rng.integers(0, 1 << 24, len(ev))
    act = ev["type"] == ge.EV_ACTIVE
    ev["flags"][act] = rng.integers(1, 100, int(act.sum()))
    ev["value"][act] = rng.integers(0, 1 << 16, int(act.sum()))
    if huge:
        ev["flow_key"][n:], ev["type"][n:], ev["value"][n:], ev["flags"][n:] = keys[0], ge.EV_CLOSE_SER, M32, 0
    return ev


def exact_flows(ev, keys):
    """the exact (connections, kbytes) of each key in the events, each as a Python int"""
    act = ev["type"] == ge.EV_ACTIVE
    cnt = np.where(act, ev["flags"].astype(np.uint64), np.uint64(1))
    kb = np.where(act, ev["value"].astype(np.uint64), (ev["value"] >> np.uint32(10)).astype(np.uint64))
    out = {}
    for k in np.asarray(keys, dtype=np.uint64).tolist():
        m = ev["flow_key"] == np.uint64(k)
        out[k] = (int(cnt[m].sum()), int(kb[m].sum()))
    return out


def point_query(table, keys, depth, log2w):
    """gysk_query_flows restated on a table: per key the minimum over rows of each half"""
    L = po.lib()
    t = table.reshape(depth, 1 << log2w)
    out = []
    for k in np.asarray(keys, dtype=np.uint64).tolist():
        cells = [int(t[r, L.gyo_cms_index(k, r, log2w)]) for r in range(depth)]
        out.append((min(c & M32 for c in cells), min(c >> 32 for c in cells)))
    return out
