"""Times the listener walk's two reads, gysk_query_day_stats (every listener's LISTENER_DAY_STATS row) and gysk_query_host_listen (per-host
listener counts), next to gysk_query_window in the same session, at 100 K and 1 M services: ms per call, bytes copied device to host, and
day_stats_kernel's bytes read over its time (torch.profiler) against the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM. The services
are flushed once in each of ten 43 200-s slots of the 5-day level, so every row reads all ten ring slots. Prints one JSON line per size,
with the card's name and power limit.

    python scripts/day_stats_probe.py [--sizes 100000 1000000] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gyeeta_b200 import engine as ge  # noqa: E402
from scripts.window_read_probe import HBM_TBS, card, fill, timed  # noqa: E402

DAY_BYTES = C.sizeof(ge.ListenerDayStats)
HOST_BYTES = C.sizeof(ge.HostListen)


def day_kernel_bytes_per_row(live1=10):
    """what day_stats_kernel reads per listed slot: 16 cells of 16 B of every live 5-day ring slot, of qps_hist_ and of
    active_conn_hist_, the slot's id and its list entry; plus the 48-byte row it writes"""
    return live1 * 256 + 2 * 256 + 8 + 8 + DAY_BYTES


def probe(n, name):
    import torch
    from torch.profiler import ProfilerActivity, profile

    rng = np.random.default_rng(n)
    eng = ge.Engine(max_svcs=n, max_tasks=1024, max_batch=1 << 22)
    fill(eng, n, rng)                                       # first flush at 5
    for k in range(1, 10):                                  # one flush in each further slot of the 5-day level
        eng.flush(5 + 43200 * k)
    day = (ge.ListenerDayStats * n)()
    dhosts = np.zeros(n, dtype=np.uint32)
    win = (ge.SvcSummary * n)()
    hl = (ge.HostListen * 4096)()
    k = C.c_uint32()

    def day_stats():
        assert eng.L.gysk_query_day_stats(eng.h, -1, day, dhosts.ctypes.data_as(C.c_void_p), n, C.byref(k)) == 0 and k.value == n

    def host_listen():
        assert eng.L.gysk_query_host_listen(eng.h, hl, 4096, C.byref(k)) == 0 and k.value == 64

    def window():
        assert eng.L.gysk_query_window(eng.h, -1, 0, win, n, C.byref(k)) == 0 and k.value == n

    ms_day, t_day = timed(day_stats, 5)
    ms_hl, t_hl = timed(host_listen, 5)
    ms_win, t_win = timed(window, 5)
    nlisten = sum(hl[i].nlisten for i in range(64))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        day_stats()
        host_listen()
        torch.cuda.synchronize()
    kus = {"day_stats_kernel": 0.0, "host_listen_count_kernel": 0.0, "host_listen_rows_kernel": 0.0}
    for e in prof.key_averages():
        for kn in kus:
            if kn in e.key:
                kus[kn] += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    kb = day_kernel_bytes_per_row() * n
    kd = kus["day_stats_kernel"]
    eng.close()
    return dict(services=n, card=name, day_stats_ms=round(ms_day, 3), day_stats_runs_ms=t_day, host_listen_ms=round(ms_hl, 3),
                host_listen_runs_ms=t_hl, window_ms=round(ms_win, 3), window_runs_ms=t_win, nlisten_total=nlisten,
                day_d2h_bytes=n * (DAY_BYTES + 16) + 8, host_listen_d2h_bytes=64 * HOST_BYTES + 8,
                day_kernel_ms=round(kd / 1e3, 3), day_kernel_bytes=kb, day_kernel_tbs=round(kb / (kd * 1e-6) / 1e12, 3) if kd else None,
                day_kernel_share_of_3_35_tbs=round(kb / (kd * 1e-6) / 1e12 / HBM_TBS, 3) if kd else None,
                host_listen_count_kernel_ms=round(kus["host_listen_count_kernel"] / 1e3, 3),
                host_listen_rows_kernel_ms=round(kus["host_listen_rows_kernel"] / 1e3, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--out", help="also write the JSON lines to DIR/day_stats_probe.jsonl")
    a = ap.parse_args()
    name = card()
    lines = []
    for n in a.sizes:
        r = probe(n, name)
        print(json.dumps(r), flush=True)
        lines.append(json.dumps(r))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "day_stats_probe.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
