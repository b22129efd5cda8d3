"""Times the window read of every service (gysk_query_window) against the by-id read of the same ids (gysk_query_svcs), at
100 K and 1 M services: ms per call, bytes copied device to host, and svc_summary_kernel's bytes read over its time (torch.profiler)
against the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM. Also the tick's whole read path, the steps of the shim's
window_listener_states: one gysk_query_window_hosts call, then every host's rows encoded into LISTENER_STATE_NOTIFY batches of at
most 512 records. Prints one JSON line per size, with the card's name and power limit.

    python scripts/window_read_probe.py [--sizes 100000 1000000] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import engine as ge  # noqa: E402

ROW_BYTES = C.sizeof(ge.SvcSummary)
HBM_TBS = 3.35


def kernel_bytes_per_slot(hll_p, live0=1, live1=1):
    """words svc_summary_kernel reads per listed slot: cur / last / all histograms, both CONN_BITMAPs, the live
    ring slots of both levels, the qps / active-conn histograms (16 cells of 16 B each), conn counters, t-digest head, aux, state,
    all TD_CAP centroids, the HLL registers, the slot's id and its list entry; plus the 208-byte row it writes"""
    hist = 16 * 16
    return 3 * hist + 2 * 64 + (live0 + live1) * hist + 2 * hist + 4 * 8 + 32 + 40 + 8 + 256 * 16 + (1 << hll_p) + 8 + 8 + ROW_BYTES


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as ex:          # noqa: BLE001
        return f"unknown ({ex})"


def fill(eng, n, rng):
    """n services, 8 response samples and 2 connection events each, over 64 hosts, in device batches of 4 M events"""
    ids = (rng.choice(1 << 40, n, replace=False) + 1).astype(np.uint64)
    per = 10
    for off in range(0, n, (1 << 22) // per):
        part = ids[off: off + (1 << 22) // per]
        ev = np.zeros(len(part) * per, dtype=ge.EVENT_DTYPE)
        ev["svc_id"] = np.repeat(part, per)
        ev["type"] = np.tile(np.array([ge.EV_RESP] * 8 + [ge.EV_ACCEPT] * 2, dtype=np.uint16), len(part))
        ev["value"] = rng.lognormal(9.0, 1.5, len(ev)).astype(np.uint32) + 1
        ev["flow_key"] = rng.integers(0, 1 << 62, len(ev), dtype=np.uint64)
        ev["host_idx"] = (ev["svc_id"] % 64).astype(np.uint32)
        eng.ingest_events(ev)
    eng.flush(5)
    return ids


def timed(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t)), [round(x, 3) for x in t]


def probe(n, name):
    import torch
    from torch.profiler import ProfilerActivity, profile

    rng = np.random.default_rng(n)
    eng = ge.Engine(max_svcs=n, max_tasks=1024, max_batch=1 << 22)
    fill(eng, n, rng)
    out = (ge.SvcSummary * n)()
    win = (ge.SvcSummary * n)()
    k = C.c_uint32()

    def window():
        assert eng.L.gysk_query_window(eng.h, -1, 0, win, n, C.byref(k)) == 0 and k.value == n

    window()
    ids = np.frombuffer(win, dtype=np.uint64).reshape(n, ROW_BYTES // 8)[:, 0].copy()

    def by_id():
        assert eng.L.gysk_query_svcs(eng.h, ids.ctypes.data_as(C.c_void_p), n, out) == 0

    hosts = np.zeros(n, dtype=np.uint32)
    recs = C.create_string_buffer(512 * 88)
    nrecs, nbytes = C.c_uint32(), C.c_uint32()
    batches = [0]

    def tick():
        assert eng.L.gysk_query_window_hosts(eng.h, -1, 0, win, hosts.ctypes.data_as(C.c_void_p), n, C.byref(k)) == 0 and k.value == n
        cuts = np.flatnonzero(np.diff(hosts)) + 1
        nb = 0
        for a, b in zip(np.concatenate([[0], cuts]).tolist(), np.concatenate([cuts, [n]]).tolist()):
            for off in range(a, b, 512):
                m = min(512, b - off)
                assert eng.L.gysk_encode_listener_state(C.byref(win, off * ROW_BYTES), m, recs, len(recs), C.byref(nrecs), C.byref(nbytes)) == 0
                nb += 1
        batches[0] = nb

    ms_tick, t_tick = timed(tick, 5)
    ms_win, t_win = timed(window, 5)
    ms_ids, t_ids = timed(by_id, 2)
    same = bytes(win) == bytes(out)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        window()
        torch.cuda.synchronize()
    kus = 0.0
    for e in prof.key_averages():
        if "svc_summary_kernel" in e.key:
            kus += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    kb = kernel_bytes_per_slot(eng.cfg.hll_p) * n
    eng.close()
    return dict(services=n, card=name, window_ms=round(ms_win, 3), window_runs_ms=t_win, tick_read_ms=round(ms_tick, 3), tick_runs_ms=t_tick,
                tick_batches=batches[0], by_id_ms=round(ms_ids, 3), by_id_runs_ms=t_ids,
                rows_equal=same, window_d2h_bytes=n * (ROW_BYTES + 16) + 8, by_id_d2h_bytes=n * ROW_BYTES,
                by_id_launches=-(-n // 1024), window_kernel_ms=round(kus / 1e3, 3), window_kernel_bytes=kb,
                window_kernel_tbs=round(kb / (kus * 1e-6) / 1e12, 3) if kus else None,
                window_kernel_share_of_3_35_tbs=round(kb / (kus * 1e-6) / 1e12 / HBM_TBS, 3) if kus else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--out", help="also write the JSON lines to DIR/window_read_probe.jsonl")
    a = ap.parse_args()
    name = card()
    lines = []
    for n in a.sizes:
        r = probe(n, name)
        print(json.dumps(r), flush=True)
        lines.append(json.dumps(r))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "window_read_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
