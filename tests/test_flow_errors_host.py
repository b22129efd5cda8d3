"""The flow error tables and server-error sets of GYSK_FLAG_FLOW_ERRORS on the CPU: the counting rule (both bits, no bit, samples the
query tables do not count) and the two invariants on seeded streams restated with tests/flow_errors.py, the point query's place above the
exact counts on keys made to collide, the window guarantee with a few failing clients hidden in a crowd of heavy healthy ones, the 300-s
bound over the level's flush sequences, and the header, the Python constants and the bindings that pin the ABI."""
import os
import re

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import flow_errors as fe
from tests import flow_level as fl
from tests import flow_queries as fq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, W = 4, 8


def _lib():
    if not os.path.exists(os.path.join(ROOT, "gyeeta_b200", "libgysketch.so")):
        pytest.skip("library not built")
    return ge.load_library()


def events(keys, flags, usec=20_500, svc=1000003):
    ev = np.zeros(len(keys), dtype=ge.EVENT_DTYPE)
    ev["svc_id"], ev["flow_key"], ev["type"], ev["value"], ev["flags"] = svc, keys, ge.EV_RESP, usec, flags
    return ev


def test_counting_rule():
    keys = np.array([11, 12, 13, 14, 15, 16, 17], dtype=np.uint64)
    ev = events(keys, [0, 1, 2, 3, 3, 2, 1])
    ev["value"][4] = fq.VALID_USEC                    # beyond the validity rule: no sample
    ev["type"][5] = ge.EV_TRACE                       # a trace event: no sample
    ev["svc_id"][6] = 0                               # no slot: no sample
    s = fq.counted(ev, None)
    s = s[s["svc_id"] != 0]
    t = fe.add_samples(fe.empty(D, W), s, D, W)
    rows = fe.point_query(t, fe.empty(D, W), keys, D, W)
    assert rows["cli_errors"].tolist() == [0, 1, 0, 1, 0, 0, 0]
    assert rows["ser_errors"].tolist() == [0, 0, 1, 1, 0, 0, 0]
    assert fe.exact(s, keys).tolist() == [[0, 0], [1, 0], [0, 1], [1, 1], [0, 0], [0, 0], [0, 0]]
    assert fe.ser_keys(s).tolist() == [13, 14]


def _stream(rng, n, nkeys, share):
    keys = rng.integers(1, 1 << 40, nkeys).astype(np.uint64)
    ev = events(rng.choice(keys, n), np.where(rng.random(n) < share, rng.integers(1, 4, n), 0), usec=rng.integers(0, 1_100_000_000, n))
    ev["svc_id"] = rng.integers(1, 30, n).astype(np.uint64)
    return ev


@pytest.mark.parametrize("share", [0.0, 0.01, 0.3, 1.0])
def test_invariants_on_seeded_streams(share):
    """per row the error halves sum to the services' error counts (mod 2^32); cell by cell each error half is at most the query half"""
    rng = np.random.default_rng(int(share * 100))
    d, w = 3, 5
    ev = _stream(rng, 20_000, 400, share)
    s = fq.counted(ev, None)
    err, qry = fe.add_samples(fe.empty(d, w), s, d, w), fq.add_samples(np.zeros(d << w, dtype=np.uint64), s, d, w)
    cli = int((s["flags"] & 1).sum()) & fe.U32
    ser = int(((s["flags"] >> 1) & 1).sum()) & fe.U32
    assert fe.row_sums(err, d, w) == [(cli, ser)] * d
    assert np.all((err & np.uint64(fe.U32)) <= (qry & np.uint64(fe.U32)))
    assert np.all((err >> np.uint64(32)) <= (qry & np.uint64(fe.U32)))
    if share == 0.0:
        assert not err.any()


def test_point_query_at_least_exact_on_colliding_keys():
    rng = np.random.default_rng(2)
    d, w = 3, 4
    ev = _stream(rng, 5000, 80, 0.5)
    s = fq.counted(ev, None)
    err = fe.add_samples(fe.empty(d, w), s, d, w)
    keys = np.unique(s["flow_key"])
    rows = fe.point_query(err, fe.empty(d, w), keys, d, w)
    ex = fe.exact(s, keys)
    assert np.all(rows["cli_errors"] >= ex[:, 0]) and np.all(rows["ser_errors"] >= ex[:, 1])
    assert np.any(rows["ser_errors"] > ex[:, 1]), "the keys collide, so some estimates exceed the exact count"


def _window(rng, healthy, failing, nbatches, per_batch):
    """batches of counted samples: a Zipf crowd of heavy healthy flows with rare client errors, and each failing flow a few 5xx"""
    wts = 1.0 / np.arange(1, len(healthy) + 1) ** 1.1
    out = []
    for _ in range(nbatches):
        keys = healthy[rng.choice(len(healthy), per_batch, p=wts / wts.sum())]
        fk = np.repeat(failing, 3)
        ev = np.concatenate([events(keys, np.where(rng.random(per_batch) < 0.02, 1, 0)), events(fk, 2)])
        out.append(fq.counted(ev, None))
    return out


@pytest.mark.parametrize("k,nfail", [(8, 5), (8, 40), (32, 200)])
def test_window_guarantee_with_failing_clients_in_a_crowd(k, nfail):
    rng = np.random.default_rng(k * 100 + nfail)
    healthy = rng.choice(1 << 40, 2000, replace=False).astype(np.uint64)
    failing = rng.choice(1 << 40, nfail, replace=False).astype(np.uint64) | np.uint64(1 << 41)
    sets, table, seen = fe.Sets(D, W, k), fe.empty(D, W), []
    for b in _window(rng, healthy, failing, 4, 400):
        table = fe.add_samples(table, b, D, W)
        seen.append(b)
        sets.batch(fe.ser_keys(b), table)
        allb = np.concatenate(seen)
        keys = np.unique(allb["flow_key"])
        ex = fe.exact(allb, keys)[:, 1]
        members = set(sets.open.tolist())
        t = fe.fs.thr(sets.open, table, D, W, fe.ser_score, k)
        assert all(key in members for key, x in zip(keys.tolist(), ex.tolist()) if x > (t if len(sets.open) == k else 0))
        assert np.all(fe.exact(allb, np.sort(sets.open))[:, 1] > 0)          # a client-error-only flow is never listed
    if nfail <= k:
        assert set(failing.tolist()) <= set(sets.open.tolist())


@pytest.mark.parametrize("seq", sorted(fl.SEQUENCES))
def test_level_bound_on_seeded_streams(seq):
    rng = np.random.default_rng(len(seq))
    k = 8
    healthy = rng.choice(1 << 40, 500, replace=False).astype(np.uint64)
    failing = rng.choice(1 << 40, 60, replace=False).astype(np.uint64) | np.uint64(1 << 41)
    lv = fe.LevelSets(D, W, k)
    tsecs, history = [], []
    for i, t in enumerate(fl.SEQUENCES[seq]):
        sets, table, win = fe.Sets(D, W, k), fe.empty(D, W), []
        for b in _window(rng, healthy, np.roll(failing, 5 * i)[:12], 2, 150):
            table = fe.add_samples(table, b, D, W)
            sets.batch(fe.ser_keys(b), table)
            win.append(b)
        L, B = lv.flush(t, sets.open, table)
        tsecs.append(t)
        history.append(np.concatenate(win))
        held = np.concatenate([history[j] for j in fl.held_windows(tsecs)])
        keys = np.unique(held["flow_key"])
        members = set(L.tolist())
        assert all(x <= B for key, x in zip(keys.tolist(), fe.exact(held, keys)[:, 1].tolist()) if key not in members), (seq, i)
        assert len(L) <= k


CALLS = ("int		gysk_query_flow_errors(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_err_est *out);",
         "int		gysk_query_flow_errors_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_err_est *out);",
         "int		gysk_query_flow_errors_global(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, int last_window, gysk_flow_err_est *out);",
         "int		gysk_query_flow_errors_global_5min(gysk_engine *e, const uint64_t *flow_keys, uint32_t n, gysk_flow_err_est *out);",
         "int		gysk_export_cms_errors(gysk_engine *e, int last_window, uint64_t *cells /* depth << log2_width entries */);",
         "int		gysk_export_cms_errors_5min(gysk_engine *e, uint64_t *cells /* depth << log2_width entries */);",
         "int		gysk_topk_flow_errors(gysk_engine *e, int last_window, uint32_t n, gysk_flow_err_est *out, uint32_t *nout);",
         "int		gysk_topk_flow_errors_global(gysk_engine *e, uint32_t n, gysk_flow_err_est *out, uint32_t *nout);",
         "int		gysk_topk_flow_errors_5min(gysk_engine *e, uint32_t n, gysk_flow_err_est *out, uint32_t *nout, uint64_t *bound);",
         "int		gysk_topk_flow_errors_global_5min(gysk_engine *e, uint32_t n, gysk_flow_err_est *out, uint32_t *nout, uint64_t *bound);",
         "int64_t		gysk_last_batch_flow_err_direct(gysk_engine *e);")


def test_header_constants_and_bindings():
    with open(os.path.join(ROOT, "include", "gysketch.h")) as f:
        h = f.read()
    assert re.search(r"#define GYSK_FLAG_FLOW_ERRORS\s+0x4000u", h)
    assert re.search(r"#define GYSK_EVF_CLI_ERROR\s+0x1u", h) and re.search(r"#define GYSK_EVF_SER_ERROR\s+0x2u", h)
    assert re.search(r"typedef struct gysk_flow_err_est\s*\{\s*uint64_t\s+flow_key;\s*uint32_t\s+queries;[^}]*uint32_t\s+cli_errors;[^}]*"
                     r"uint32_t\s+ser_errors;[^}]*uint32_t\s+pad;[^}]*\}", h)
    for call in CALLS:
        assert call in h, call
    assert ge.FLAG_FLOW_ERRORS == 0x4000
    assert ge.FLOW_ERR_EST_DTYPE.itemsize == 24 and ge.FLOW_ERR_EST_DTYPE.names == ("flow_key", "queries", "cli_errors", "ser_errors", "pad")
    for name in ("query_flow_errors", "query_flow_errors_5min", "query_flow_errors_global", "query_flow_errors_global_5min",
                 "export_cms_errors", "export_cms_errors_5min", "topk_flow_errors", "topk_flow_errors_global", "topk_flow_errors_5min",
                 "topk_flow_errors_global_5min", "last_batch_flow_err_direct"):
        assert callable(getattr(ge.Engine, name)), name


def test_library_refuses_the_flag_without_flow_queries_and_null_engines():
    L = _lib()
    with pytest.raises(ge.GyskError) as ex:               # the configuration check comes before any device is looked for
        ge.Engine(flow_errors=True)
    assert ex.value.code == -22 and "needs GYSK_FLAG_FLOW_QUERIES" in str(ex.value)
    assert L.gysk_query_flow_errors(None, None, 0, 0, None) == -22
    assert L.gysk_export_cms_errors(None, 0, None) == -22
    assert L.gysk_topk_flow_errors(None, 0, 0, None, None) == -22
    assert L.gysk_topk_flow_errors_global(None, 0, None, None) == -22
    for name in ("gysk_topk_flow_errors_5min", "gysk_topk_flow_errors_global_5min"):
        assert getattr(L, name)(None, 0, None, None, None) == -22
    assert L.gysk_last_batch_flow_err_direct(None) == -22
