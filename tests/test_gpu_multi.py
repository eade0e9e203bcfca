"""Multi-GPU parity (needs >= 2 H100s; skipped on a 1-GPU box): two ranks, one process per GPU, NCCL inside
libcco_b200.so; the merged row slices must equal the oracle's (= the single-GPU) model bit for bit."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, names, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import row_paths
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import synth
        import universal_recommender_b200 as ur
        from oracle import oracle as orc
        from universal_recommender_b200 import distributed as D
        ctx = D.context_from_env(dist)
        ok = True
        for name in names:
            w = synth.make(name)
            local = ctx.train_csr(w.mats, w.params, seed=42)
            merged = D.gather_indicators(dist, local)
            ref = orc.train([orc.Csr(*m) for m in w.mats], [orc.Params(*p) for p in w.params], 42)
            bar = 2.0 * row_paths.llr_error_bound(w.mats[0][0])       # each LLR within eps(N) of the real value
            for (n_rows, n_cols, rp, ci, ll, cn), r in zip(merged, ref):
                ok &= n_rows == r.n_rows and np.array_equal(rp, r.row_ptr) and np.array_equal(ci, r.col_idx)
                ok &= np.array_equal(cn, r.count) and len(ll) == len(r.llr) and bool((np.abs(ll - r.llr) <= bar).all())
            ok &= sum(local[i][1] - local[i][0] for i in range(len(local))) > 0     # this rank really owns rows
        ctx.close()
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_parity():
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), ["tiny", "small", "C3-tenth"], ret), nprocs=world, join=True)
    assert dict(ret) == {0: True, 1: True}


def _oracle_equal(orc, mats, params, seed, got):
    from oracle import parity as par
    ref = orc.train([orc.Csr(*m) for m in mats], [orc.Params(*p) for p in params], seed)
    p = par.compare(ref, got)
    assert p["ok"], p


def test_group_context_on_one_gpu(orc):
    """cco_create_group with a single device: the threaded group path (member context, merged result) on the 1-GPU box"""
    import synth
    import universal_recommender_b200 as ur
    g = ur.CcoContext(devices=[0])
    try:
        for name in ("tiny", "small"):
            w = synth.make(name)
            got = g.train_csr(w.mats, w.params, seed=42)
            assert all(x[0] == 0 and x[1] == w.n_items for x in got)           # full row range, one merged model
            _oracle_equal(orc, w.mats, w.params, 42, got)
        got = g.train_csr(w.mats, w.params, seed=42, flags=ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR)
        assert all(len(x[5]) == 0 and len(x[6]) == 0 and len(x[4]) == x[3][-1] for x in got)
    finally:
        g.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_group_context_all_gpus(orc):
    """one process, one context, every GPU of the box (what the JNI shim creates): merged model == oracle, including
    unsorted / duplicated input rows (each GPU canonicalises its own block of users)"""
    import synth
    import universal_recommender_b200 as ur
    n = torch.cuda.device_count()
    g = ur.CcoContext(devices=list(range(n)))
    try:
        for name in ("tiny", "small", "C3-tenth"):
            w = synth.make(name)
            got = g.train_csr(w.mats, w.params, seed=42)
            assert all(x[0] == 0 and x[1] == w.n_items for x in got)
            _oracle_equal(orc, w.mats, w.params, 42, got)
        rng = np.random.default_rng(4)
        w = synth.make("small")
        messy = []
        for (nr, nc, rp, ci) in w.mats:
            rows = [list(ci[rp[r]:rp[r + 1]]) for r in range(nr)]
            rows = [list(rng.permutation(r + r[: len(r) // 2])) for r in rows]
            nrp = np.zeros(nr + 1, dtype=np.int64)
            np.cumsum([len(r) for r in rows], out=nrp[1:])
            messy.append((nr, nc, nrp, np.array([c for r in rows for c in r], dtype=np.int32)))
        _oracle_equal(orc, w.mats, w.params, 8, g.train_csr(messy, w.params, seed=8))
    finally:
        g.close()
