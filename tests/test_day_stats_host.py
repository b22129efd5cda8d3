"""CPU side of the listener walk's day stats and host counts: gysk_classify_host against a restatement of host_status_update's state
rule (common/gy_socket_stat.cc:4455-4528) over every combination of its inputs plus one hand-derived case per branch, the layouts of the
new ABI structs and wire records, and the shim's host_state / window_listener_day_stats failing loudly without a GPU."""
import ctypes as C
import itertools
import os
import subprocess

import pytest

from gyeeta_b200 import engine as ge

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDLE, GOOD, OK, BAD, SEVERE = ge.STATE_IDLE, ge.STATE_GOOD, ge.STATE_OK, ge.STATE_BAD, ge.STATE_SEVERE


def host_state(cpu_issue, mem_issue, severe_cpu_issue, severe_mem_issue, cpu_idle, ntasks_issue, ntasks_severe, nlisten_issue, nlisten_severe):
    """gyo_host_state: host_status_update's rule, statement for statement"""
    if (ntasks_severe or nlisten_severe) and (severe_cpu_issue or severe_mem_issue):
        return SEVERE
    if not cpu_issue and not mem_issue and not ntasks_issue and not nlisten_issue:
        return IDLE if cpu_idle else GOOD
    if (ntasks_issue or nlisten_issue) and (cpu_issue or mem_issue):
        if ntasks_issue > 5 or nlisten_issue > 5:
            return SEVERE
        return BAD
    elif cpu_issue or mem_issue:
        if severe_cpu_issue or severe_mem_issue:
            return BAD
        return OK
    if nlisten_issue:
        if nlisten_severe or ntasks_issue:
            if nlisten_issue > 5:
                return SEVERE
            return BAD
        elif nlisten_issue > 2:
            return BAD
        else:
            return OK
    if ntasks_issue:
        if ntasks_severe:
            return BAD
        elif ntasks_issue > 5:
            return BAD
    return OK


FLAGS = ("cpu_issue", "mem_issue", "severe_cpu_issue", "severe_mem_issue", "cpu_idle")
COUNTS = ("ntasks_issue", "ntasks_severe", "nlisten_issue", "nlisten_severe")


def test_classify_host_equals_the_restatement_everywhere():
    for flags in itertools.product((0, 1), repeat=5):
        for counts in itertools.product((0, 1, 2, 3, 5, 6), repeat=4):
            kw = dict(zip(FLAGS + COUNTS, flags + counts))
            assert ge.classify_host(**kw) == host_state(**kw), kw


@pytest.mark.parametrize("kw,want", [
    (dict(nlisten_severe=1, severe_mem_issue=1), SEVERE),                         # :4462 severe listeners on a severely loaded host
    (dict(ntasks_severe=1, severe_cpu_issue=1, cpu_issue=1), SEVERE),
    (dict(cpu_idle=1), IDLE),                                                      # :4467 nothing wrong, idle cpu
    (dict(), GOOD),
    (dict(nlisten_issue=6, cpu_issue=1), SEVERE),                                  # :4479 issues on a loaded host, more than 5
    (dict(nlisten_issue=5, mem_issue=1), BAD),
    (dict(cpu_issue=1, severe_cpu_issue=1), BAD),                                  # :4488 host load alone
    (dict(mem_issue=1, cpu_idle=1), OK),
    (dict(nlisten_issue=6, nlisten_severe=1), SEVERE),                             # :4498 listener issues with severe ones
    (dict(nlisten_issue=2, ntasks_issue=1), BAD),
    (dict(nlisten_issue=3), BAD),
    (dict(nlisten_issue=2, cpu_idle=1), OK),
    (dict(ntasks_issue=1, ntasks_severe=1), BAD),                                  # :4518 process issues alone
    (dict(ntasks_issue=6), BAD),
    (dict(ntasks_issue=5), OK),
])
def test_classify_host_branches(kw, want):
    assert ge.classify_host(**kw) == want == host_state(**{k: kw.get(k, 0) for k in FLAGS + COUNTS})


LAYOUT_SRC = r"""
#include <cstddef>
#include <cstdio>
#include "gysketch.h"
#include "gysk_wire.h"
#define F(T, f) std::printf(#T " " #f " %zu %zu\n", offsetof(T, f), sizeof(((T *)0)->f));
#define S(T) std::printf(#T " sizeof %zu 0\n", sizeof(T));
int main()
{
	using gysk::wire::LISTENER_DAY_STATS; using gysk::wire::HOST_STATE_NOTIFY;
	S(gysk_listener_day_stats) S(gysk_host_listen) S(gysk_host_state_in) S(LISTENER_DAY_STATS) S(HOST_STATE_NOTIFY)
	F(gysk_listener_day_stats, glob_id) F(gysk_listener_day_stats, tcount_5d) F(gysk_listener_day_stats, tsum_5d)
	F(gysk_listener_day_stats, p95_5d_respms) F(gysk_listener_day_stats, p25_5d_respms) F(gysk_listener_day_stats, p95_qps)
	F(gysk_listener_day_stats, p25_qps) F(gysk_listener_day_stats, p95_nactive) F(gysk_listener_day_stats, p25_nactive)
	F(gysk_host_listen, host_idx) F(gysk_host_listen, nlisten) F(gysk_host_listen, nlisten_issue) F(gysk_host_listen, nlisten_severe)
	F(gysk_host_state_in, cpu_issue) F(gysk_host_state_in, mem_issue) F(gysk_host_state_in, severe_cpu_issue)
	F(gysk_host_state_in, severe_mem_issue) F(gysk_host_state_in, cpu_idle) F(gysk_host_state_in, pad) F(gysk_host_state_in, ntasks_issue)
	F(gysk_host_state_in, ntasks_severe) F(gysk_host_state_in, nlisten_issue) F(gysk_host_state_in, nlisten_severe)
	F(HOST_STATE_NOTIFY, nlisten_issue_) F(HOST_STATE_NOTIFY, nlisten_severe_) F(HOST_STATE_NOTIFY, nlisten_) F(HOST_STATE_NOTIFY, curr_state_)
	F(HOST_STATE_NOTIFY, issue_bit_hist_) F(HOST_STATE_NOTIFY, total_cpu_delayms_)
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


def test_struct_layouts_match_the_compiler(tmp_path):
    src = os.path.join(str(tmp_path), "layout.cc")
    with open(src, "w") as f:
        f.write(LAYOUT_SRC)
    out = subprocess.run([_compile(tmp_path, src, "layout")], capture_output=True, text=True, check=True).stdout.split("\n")
    c = {(t, f): (int(o), int(s)) for t, f, o, s in (line.split() for line in out if line)}
    for name, st, size in (("gysk_listener_day_stats", ge.ListenerDayStats, 48), ("gysk_host_listen", ge.HostListen, 16),
                           ("gysk_host_state_in", ge.HostStateIn, 24)):
        assert c[(name, "sizeof")][0] == C.sizeof(st) == size, name
        for f, t in st._fields_:
            assert c[(name, f)] == (getattr(st, f).offset, C.sizeof(t)), (name, f)
    assert c[("LISTENER_DAY_STATS", "sizeof")][0] == 48 and c[("HOST_STATE_NOTIFY", "sizeof")][0] == 56
    assert [c[("HOST_STATE_NOTIFY", f)][0] for f in ("nlisten_issue_", "nlisten_severe_", "nlisten_", "curr_state_", "issue_bit_hist_",
                                                      "total_cpu_delayms_")] == [20, 24, 28, 32, 33, 40]


def _shim(tmp_path):
    return _compile(tmp_path, os.path.join(ROOT, "tests", "cpp", "day_stats_shim.cc"), "day_stats_shim", link=True)


def test_shim_listener_walk_fails_loudly_without_gpu(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    r = subprocess.run([_shim(tmp_path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "rc=-19" in r.stdout and "day: 0 batches: 0 host_state: 0 unchanged: 1" in r.stdout


@pytest.mark.gpu
def test_shim_listener_walk_on_gpu(tmp_path):
    r = subprocess.run([_shim(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "day rows: 3110 early batches: 0 batches: 4 max records: 2048 order errors: 0 same bytes: 1" in r.stdout
    assert "host_state: 5 of 5" in r.stdout and "one read per window: 1 next window nlisten: 2510" in r.stdout
