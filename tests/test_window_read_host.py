"""CPU side of the window reads: the Python mirrors of gysk_task_summary and AGGR_TASK_HIST_STATS have the layout the C
compiler gives the structs, and the shim's read side (window_listener_states, handle_aggr_task_hist_stats) compiles against the
C ABI and reports failure without a GPU, leaving the records untouched."""
import ctypes as C
import os
import subprocess

import pytest

from gyeeta_b200 import engine as ge
from gyeeta_b200 import wire

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LAYOUT_SRC = r"""
#include <cstddef>
#include <cstdio>
#include "gysketch.h"
#include "gysk_wire.h"
#define F(T, f) std::printf(#T " " #f " %zu %zu\n", offsetof(T, f), sizeof(((T *)0)->f));
int main()
{
	using gysk::wire::AGGR_TASK_HIST_STATS;
	std::printf("gysk_task_summary sizeof %zu 0\n", sizeof(gysk_task_summary));
	std::printf("AGGR_TASK_HIST_STATS sizeof %zu 0\n", sizeof(AGGR_TASK_HIST_STATS));
	F(gysk_task_summary, aggr_task_id) F(gysk_task_summary, found) F(gysk_task_summary, host_idx) F(gysk_task_summary, p95_cpu_pct)
	F(gysk_task_summary, p95_cpu_delay_ms) F(gysk_task_summary, p95_blkio_delay_ms) F(gysk_task_summary, pad) F(gysk_task_summary, nsamples)
	F(gysk_task_summary, last_count) F(gysk_task_summary, last_sum)
	F(AGGR_TASK_HIST_STATS, aggr_task_id_) F(AGGR_TASK_HIST_STATS, starttimeusec_) F(AGGR_TASK_HIST_STATS, p95_cpu_pct_)
	F(AGGR_TASK_HIST_STATS, p95_cpu_delay_ms_) F(AGGR_TASK_HIST_STATS, p95_blkio_delay_ms_) F(AGGR_TASK_HIST_STATS, nprocs_)
	F(AGGR_TASK_HIST_STATS, nthreads_) F(AGGR_TASK_HIST_STATS, max_cores_allowed_) F(AGGR_TASK_HIST_STATS, cpu_cg_pct_limit_)
	F(AGGR_TASK_HIST_STATS, max_mem_cg_pct_rss_)
	return 0;
}
"""


def _compile(tmp_path, src, name, link=False):
    exe = os.path.join(str(tmp_path), name)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "gyeeta_b200", "host"),
           "-I", os.path.join(ROOT, "gyeeta_b200", "csrc"), src, "-o", exe]
    if link:
        libdir = os.path.dirname(ge.LIB_PATH)
        cmd += ["-L", libdir, "-lgysketch", f"-Wl,-rpath,{libdir}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_task_summary_and_hist_stats_layouts_match_the_compiler(tmp_path):
    src = os.path.join(str(tmp_path), "layout.cc")
    with open(src, "w") as f:
        f.write(LAYOUT_SRC)
    out = subprocess.run([_compile(tmp_path, src, "layout")], capture_output=True, text=True, check=True).stdout.split("\n")
    c = {(t, f): (int(o), int(s)) for t, f, o, s in (line.split() for line in out if line)}
    assert c[("gysk_task_summary", "sizeof")][0] == C.sizeof(ge.TaskSummary) == 88
    for f, t in ge.TaskSummary._fields_:
        assert c[("gysk_task_summary", f)] == (getattr(ge.TaskSummary, f).offset, C.sizeof(t)), f
    dt = wire.AGGR_TASK_HIST_STATS
    assert c[("AGGR_TASK_HIST_STATS", "sizeof")][0] == dt.itemsize == 40
    for f in dt.names:
        assert c[("AGGR_TASK_HIST_STATS", f + "_")] == (dt.fields[f][1], dt.fields[f][0].itemsize), f


def _shim(tmp_path):
    return _compile(tmp_path, os.path.join(ROOT, "tests", "cpp", "window_shim.cc"), "window_shim", link=True)


def test_shim_read_side_fails_loudly_without_gpu(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([_shim(tmp_path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "rc=-19" in r.stdout and "window: 0 batches: 0 tasks: 0 unchanged: 1" in r.stdout


@pytest.mark.gpu
def test_shim_read_side_on_gpu(tmp_path):
    r = subprocess.run([_shim(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "window rows: 1810 batches: 6 max records: 512 order errors: 0 same bytes: 1" in r.stdout and "task fill: 1" in r.stdout
