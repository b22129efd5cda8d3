"""Every ingest_kernel and TCP drain_kernel instance with its answers checked: one engine per reachable drain tuple and trace setting
(tests/all_flags.py: matrix, held to the dispatch tables by tests/test_flag_matrix_host.py), each fed mixed events with error bits on a
few percent of the response samples, slow samples, ACTIVE records and API_TRAN trace records, one batch whose colliding flows take the
direct path of every batch flow table, one batch on the hot-row route, and flushes at 5, 10, 40, 300 and 305. After every batch and flush
tests/all_flags.Model.check reads every answer family the flags enable and compares it with its restatement."""
import functools
import zlib

import numpy as np
import pytest

from gyeeta_b200 import engine as ge
from tests import all_flags as af
from tests import flow_queries as fq
from tests import flow_resp_hist as frh
from tests.test_gpu_flow_errors import _err_mixed
from tests.trace_agg import api_tran, resp_events, trace_events

pytestmark = pytest.mark.gpu

CFG = dict(max_svcs=512, max_tasks=64, max_batch=1 << 16, cms_depth=4)
HOT_MIN = 64
FLOW_PROBES = 16                # gysk_kernels.cuh: the linear probe limit of a batch flow table


def _host_of(ids):
    return (np.asarray(ids, dtype=np.uint64) % np.uint64(16)).astype(np.uint32)


def _stream(rng, n, nsvc=200):
    """_err_mixed with slow samples (above the 300-ms threshold) on a set of clients"""
    ev = _err_mixed(rng, n, nsvc=nsvc, nclients=4000)
    svc = ev["type"] != ge.EV_TASK
    ev["host_idx"][svc] = _host_of(ev["svc_id"][svc])         # one host per service: its slot's host, which its trace row shows
    r = np.flatnonzero(ev["type"] == ge.EV_RESP)
    slow = r[rng.random(len(r)) < 0.03]
    ev["value"][slow] = rng.integers(301_000, 5_000_000, len(slow))
    return ev


def _api_tran(rng, ids, n):
    """API_TRAN records: a response sample and a trace event each, errors among them. Of at most 48 services, so that every one takes
    a trace row (which services win the last rows when they run out depends on the order the device meets them in)"""
    rec = api_tran(rng.choice(ids[:48], n), rng.integers(100, 3_000_000, n).astype(np.uint64), reqlen=100, reslen=200,
                   reqnum=rng.integers(0, 3, n), errorcode=rng.choice([0, 0, 0, 1, 500], n), cliport=rng.integers(40000, 40400, n))
    ev = np.concatenate([resp_events(rec), trace_events(rec)])
    return ev, (lambda e: e.ingest_raw(ge.RAW_API_TRAN, rec, len(rec)))


@functools.lru_cache(maxsize=None)
def _colliding_keys(n_events, count, log2w=None, usec=None):
    """count flow keys whose entries in a batch flow table sized for n_events (launch_drains: the smallest power of two >= 2 n_events)
    all start at one position: table_hash(key) & mask. The key of the connection, query and error flow tables is h2:h1, the flow's
    lookup2 words; with log2w and usec it is the response flow table's key of a sample of usec (flow_resp_hist.packed_keys), and the
    flows found have distinct ones"""
    mask = np.uint64((1 << int(np.ceil(np.log2(2 * n_events)))) - 1)
    cand = np.arange(1, 4 * count * (int(mask) + 1), dtype=np.uint64) + np.uint64(1 << 44)
    if log2w is None:
        h1, h2 = fq.flow_hashes(cand)
        key = (h2.astype(np.uint64) << np.uint64(32)) | h1.astype(np.uint64)
    else:
        key = frh.packed_keys(cand, frh.buckets(np.full(len(cand), usec, dtype=np.uint32)), log2w)
    key, first = np.unique(key, return_index=True)
    cand = cand[first]
    with np.errstate(over="ignore"):
        pos = ((key * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(32)) & mask
    vals, cnt = np.unique(pos, return_counts=True)
    keys = cand[pos == vals[np.argmax(cnt)]][:count]
    assert len(keys) == count
    return keys


def _direct(rng, ids, log2w):
    """records on more flows than FLOW_PROBES that share one flow table position: past the probe limit they update the count-min cells
    directly. Connection records and response samples with error bits whose flows collide in the connection, query and error flow tables,
    and response samples of one response time whose flows collide in the response flow table"""
    n, nf, per, usec = 8000, 3 * FLOW_PROBES, 30, 50_000
    ev = _stream(rng, n)
    total = n + (2 * nf + 8) * per
    z = np.zeros(nf * per, dtype=ge.EVENT_DTYPE)
    z["flow_key"] = np.repeat(_colliding_keys(total, nf), per)
    z["type"] = np.where(np.arange(len(z)) % 3 == 0, ge.EV_ACCEPT, ge.EV_RESP)
    z["value"] = rng.integers(1000, 400_000, len(z))
    z["flags"] = np.where(z["type"] == ge.EV_RESP, rng.integers(1, 4, len(z)), 0)
    r = np.zeros((FLOW_PROBES + 8) * per, dtype=ge.EVENT_DTYPE)
    r["flow_key"] = np.repeat(_colliding_keys(total, FLOW_PROBES + 8, log2w, usec), per)
    r["type"], r["value"] = ge.EV_RESP, usec
    out = np.concatenate([z, r])
    out["svc_id"] = rng.choice(ids, len(out))
    out["host_idx"] = _host_of(out["svc_id"])
    return np.concatenate([ev, out])


def _hot(rng, ids):
    """a batch in which a few services take far more than GYSK_HOT_MIN response samples"""
    ev = _stream(rng, 30_000)
    r = np.flatnonzero(ev["type"] == ge.EV_RESP)
    ev["svc_id"][r[: len(r) // 2]] = rng.choice(ids[:4], len(r) // 2)
    return ev


@pytest.mark.parametrize("name,flags,rows", af.matrix(), ids=[c[0] for c in af.matrix()])
def test_every_instance_answers_as_restated(name, flags, rows, monkeypatch):
    monkeypatch.setenv("GYSK_HOT_MIN", str(HOT_MIN))
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    log2w = 10 + len(name) % 3
    m = af.Model(**CFG, cms_log2_width=log2w, max_trace_svcs=rows, **flags)
    m.host_of = lambda i: int(_host_of([i])[0])
    ev0 = _stream(rng, 20_000)
    ids = np.unique(ev0["svc_id"][ev0["type"] == ge.EV_RESP])
    m.ingest(ev0)
    m.check(("batch", 0))
    steps = ["api", 5, "direct", 10, "hot", "b", 40, "b", 300, "api", 305]
    for i, step in enumerate(steps, 1):
        if step == "api":
            ev, ingest = _api_tran(rng, ids, 4000)
            m.ingest(ev, ingest=ingest)
        elif step == "direct":
            m.ingest(_direct(rng, ids, log2w))
            assert m.eng.last_batch_flow_direct() > 0, name
            if flags["flow_queries"]:
                assert m.eng.last_batch_flow_query_direct() > 0, name
            if flags["flow_resp_hist"]:
                assert m.eng.last_batch_flow_resp_direct() > 0, name
            if flags["flow_errors"]:
                assert m.eng.last_batch_flow_err_direct() > 0, name
        elif step == "hot":
            m.ingest(_hot(rng, ids))
            assert m.eng.hot_rows_in_use() > 0, name
        elif step == "b":
            m.ingest(_stream(rng, int(rng.integers(10_000, 40_000))))
        else:
            m.flush(step)
        m.check((step, i))
    if rows:
        assert m.eng.trace_info()[0] > 0
