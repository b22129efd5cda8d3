"""The windowed client registers of GYSK_FLAG_CLIENT_LEVELS restated on the CPU. A window's set of a service is the oracle's
gyo_hll_registers(keys, 8) of the flow keys of the records that reached the service in it: connection events and ACTIVE_CONN_STATS
records, never response samples or trace events. The 300-s level is the registerwise maximum of the sets of the windows the flow level's
ring holds (tests/flow_level.held_windows): max-merging a window into a ring slot and the slots into the level is one maximum over the
held windows. fold_registers restates how the registers of a precision p >= 8 fold to p = 8, which gives the invariants against the
all-time registers."""
import numpy as np

from gyeeta_b200 import engine as ge
from oracle import pyoracle as po
from tests.flow_level import held_windows

P = ge.HLL_WINDOW_P
NREG = 1 << P
SIGMA = 1.04 / 16                    # the raw range's standard error at p = 8
BOUND = 4 * SIGMA                    # the accuracy bound every estimate is held to, linear counting range included
COUNTED = (ge.EV_CONNECT, ge.EV_ACCEPT, ge.EV_CLOSE_CLI, ge.EV_CLOSE_SER, ge.EV_ACTIVE)


def window_keys(ev):
    """{svc_id: flow keys} of the records of one window that raise a service's registers"""
    ev = ev[np.isin(ev["type"], COUNTED) & (ev["svc_id"] != 0) & (ev["svc_id"] != np.uint64(0xFFFFFFFFFFFFFFFF))]
    out = {}
    if not len(ev):
        return out
    order = np.argsort(ev["svc_id"], kind="stable")
    sid, keys = ev["svc_id"][order], ev["flow_key"][order]
    cut = np.flatnonzero(np.diff(sid)) + 1
    for s, k in zip(np.split(sid, cut), np.split(keys, cut)):
        out[int(s[0])] = np.ascontiguousarray(k, dtype=np.uint64)
    return out


def window_regs(ev):
    """{svc_id: its 256 registers} of one window"""
    return {s: po.hll_registers(k, P) for s, k in window_keys(ev).items()}


class History:
    """the closed windows' sets of every service, by flush: last(s) and level(s) as the engine must answer after the last flush"""

    def __init__(self):
        self.tsecs, self.windows = [], []

    def flush(self, tsec, ev):
        self.tsecs.append(tsec)
        self.windows.append(window_regs(ev))

    def last(self, sid):
        return self.windows[-1].get(int(sid), np.zeros(NREG, np.uint8)) if self.windows else np.zeros(NREG, np.uint8)

    def level(self, sid):
        out = np.zeros(NREG, np.uint8)
        for i in held_windows(self.tsecs) if self.tsecs else []:
            r = self.windows[i].get(int(sid))
            if r is not None:
                np.maximum(out, r, out=out)
        return out


def fold_registers(regs, p):
    """the 1 << p registers of precision p >= 8 folded to p = 8: register j is the maximum over its children c = j << (p - 8) | x of
    the rank the child's hash has at p = 8. An empty child adds nothing; for x != 0 that rank is clz(x) + 1 within p - 8 bits (the
    bits after the top 8 decide it), for x = 0 it is reg[c] + (p - 8)."""
    assert p >= P and len(regs) == 1 << p
    d = p - P
    if d == 0:
        return np.asarray(regs, dtype=np.uint8).copy()
    r = np.asarray(regs, dtype=np.int64).reshape(NREG, 1 << d)
    x = np.arange(1 << d)
    xr = np.where(x > 0, d - np.floor(np.log2(np.maximum(x, 1))).astype(np.int64), 0)      # clz(x) + 1 within d bits
    rank = np.where(x[None, :] > 0, xr[None, :], r + d)
    rank = np.where(r > 0, rank, 0)
    return rank.max(axis=1).astype(np.uint8)
