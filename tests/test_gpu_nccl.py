"""2-GPU NCCL run of the merge step (skipped on a 1-GPU box): one process per GPU, host-sharded ingest, gyeeta_b200.dist.merge_global
over NCCL, and the merged logical-service answers compared with the CPU oracle over the whole stream."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    from gyeeta_b200 import dist as gd
    from gyeeta_b200 import engine as ge
    from gyeeta_b200 import synth
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        rng = np.random.default_rng(5)
        nsvc = 256
        ev = synth.gen_mixed(rng, 120_000, nsvc, ntask=16, nhosts=32, nclients=3000)
        eng = ge.Engine(device=rank, max_svcs=1024, max_tasks=64, max_batch=1 << 17, cms_log2_width=14, rank=rank, world=world)
        eng.ingest_events(ev); eng.sync(); eng.flush(5)
        ids = synth.service_ids(nsvc)
        logical = np.arange(nsvc, dtype=np.uint64) // np.uint64(16) + np.uint64(7000)
        eng.set_logical_map(ids, logical)
        ms = gd.merge_global(eng, torch, dist, torch.device("cuda", rank))
        out = eng.query_logical(np.unique(logical))
        # the same step with NCCL INSIDE the library (gysk_merge_global): identical answers
        gd.nccl_comm_init(eng, dist)
        eng.merge_global()
        out2 = eng.query_logical(np.unique(logical))
        same = all(a == b or (a != a and b != b) for o1, o2 in zip(out, out2) for a, b in zip(o1.values(), o2.values()))
        keys = np.unique(ev["flow_key"][(ev["type"] >= 1) & (ev["type"] <= 4)])[:500]
        flows = eng.query_flows_global(keys, last_window=True)
        if rank == 0:
            from oracle import pyoracle as po
            orc = po.OracleEngine(max_svcs=1024, max_tasks=64, cms_log2_width=14)
            orc.ingest(ev); orc.flush(5)
            ok = bool(same)
            for o, lid in zip(out, np.unique(logical)):
                members = ids[logical == lid]
                hs = [orc.export_hist(int(m), 1) for m in members]
                tot = sum(h[1] for h in hs if h is not None)
                ok &= (o["nqrys_5s"] == tot)
                regs = np.zeros(4096, dtype=np.uint8)
                for m in members:
                    r = orc.export_hll(int(m))
                    if r is not None:
                        regs = np.maximum(regs, r)
                ok &= (o["distinct_clients"] == po.lib().gyo_hll_estimate(po._p(regs), 12))
            tbl = orc.cms(last_window=True).reshape(4, -1)
            for k, f in zip(keys[:100], flows[:100]):
                cells = [tbl[r, po.lib().gyo_cms_index(int(k), r, 14)] for r in range(4)]
                ok &= (f["count"] == min(int(c) & 0xFFFFFFFF for c in cells))
            q.put((bool(ok), float(ms)))
        elif not same:
            raise AssertionError('library NCCL merge differs from the torch.distributed merge')
    finally:
        dist.destroy_process_group()


def test_nccl_two_gpu_merge():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    ok, ms = q.get(timeout=5)
    assert ok is True


def test_two_engines_on_two_devices_in_one_process():
    """the deployment INTEGRATION.md describes: ONE process owns an engine per GPU. cudaFuncSetAttribute is per device, so the
    second engine must get its own opt-in for the large dynamic shared memory of ingest_kernel / os_pass_kernel<9> — drive the
    batch's key sort (max_svcs 2^17 -> 7 + 7 + 7 + 6-bit digits) and a plain top-N sort on BOTH devices and compare with the
    oracle; then merge the two engines with a caller-made communicator (ncclCommInitAll equivalent: two comms from one unique id,
    one per thread); last, a group-by of more than 2^16 samples on both devices (17 group bits: a 9-bit and an 8-bit pass)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import threading
    from gyeeta_b200 import engine as ge
    from gyeeta_b200 import synth
    from oracle import pyoracle as po
    rng = np.random.default_rng(12)
    nsvc = 400
    ev = synth.gen_mixed(rng, 150_000, nsvc, ntask=16, nhosts=32, nclients=3000)
    engs = [ge.Engine(device=d, max_svcs=1 << 17, max_tasks=64, max_batch=1 << 18, cms_log2_width=14, rank=d, world=2) for d in (1, 0)]
    engs = [engs[1], engs[0]]                                  # created on device 1 FIRST, then device 0
    orcs = [po.OracleEngine(max_svcs=1 << 17, max_tasks=64, cms_log2_width=14, rank=d, world=2) for d in range(2)]
    for e_, o_ in zip(engs, orcs):
        e_.ingest_events(ev); e_.sync(); o_.ingest(ev)
        e_.flush(5); o_.flush(5)
    resp = ev[ev["type"] == ge.EV_RESP]
    ids, first = np.unique(resp["svc_id"], return_index=True)
    checked = 0
    for id_, h in zip(ids, resp["host_idx"][first]):
        e_, o_ = engs[int(h) % 2], orcs[int(h) % 2]
        a, b = e_.export_hist(int(id_), ge.HIST_RESP_LAST), o_.export_hist(int(id_), ge.HIST_RESP_LAST)
        assert (a is None) == (b is None)
        if a is None:
            continue
        assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]
        td = o_.export_tdigest(int(id_)); means, weights, mn, mx = e_.export_tdigest(int(id_))
        om, ow = td.centroids()
        assert np.array_equal(means, om) and np.array_equal(weights, ow)
        checked += 1
    assert checked > 300
    for e_ in engs:
        assert len(e_.topn(0, 10)) == 10
    # library-side NCCL across the two engines of this process: one thread per engine (ncclCommInitRank blocks until all joined)
    logical = np.arange(nsvc, dtype=np.uint64) // np.uint64(16) + np.uint64(7000)
    sids = synth.service_ids(nsvc)
    uid = engs[0].nccl_unique_id()
    for e_ in engs:
        e_.set_logical_map(sids, logical)
    errs = []

    def run(r):
        try:
            engs[r].nccl_comm_init(uid, 2, r)
            engs[r].merge_global()
            engs[r].sync()
        except Exception as ex:      # noqa: BLE001
            errs.append(ex)
    th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errs, errs
    one = po.OracleEngine(max_svcs=1 << 17, max_tasks=64, cms_log2_width=14)
    one.ingest(ev); one.flush(5)
    for r in range(2):
        for o, lid in zip(engs[r].query_logical(np.unique(logical)), np.unique(logical)):
            members = sids[logical == lid]
            tot = sum(h[1] for h in (one.export_hist(int(m), 1) for m in members) if h is not None)
            assert o["nqrys_5s"] == tot
    from gyeeta_b200 import wire
    from tests.test_gpu_boundary import _proc_samples
    s = _proc_samples(rng, 100_000, 20_000)                    # n <= max_batch (2^18)
    want = po.task_groupby(s, wire.TASK)
    for e_ in engs:
        got, ng = e_.task_groupby(s)
        assert ng == len(want) and got.tobytes() == want.tobytes()
