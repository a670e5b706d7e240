"""GPU, multi-device paths against the single-rank oracle.

  * 2 ranks, one process per GPU (skipped on boxes with one GPU): the collective INSIDE the library
    (wva_comm_init: totals all-gather + rank-order sum in wva_allocate_by_type, packed candidate-row
    all-gather in the limited wva_solve), and the host-driven variant over torch.distributed;
  * wva_group: ONE process driving the devices (2 when present; the 1-device group runs everywhere and
    still goes through NCCL with a 1-rank communicator)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import wva_import
    wva = wva_import.load()
    from inferno_autoscaler_b200 import binding, distributed as D
    import oracle
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import rank_emulation
    dev = torch.device("cuda", rank)
    img = wva.synth.make_system(61, 4, seed=93, n_types=2, max_pair_batch=128)
    pairs_all, feas_all, _ = oracle.analyze_pairs(img, threads=4)
    acc_u, ch_u = oracle.solve(img, pairs_all, feas_all, unlimited=True)
    wva.synth.set_capacity_from_demand(img, ch_u.acc, ch_u.num_replicas, fraction=0.6)
    ctx = binding.Context(rank)
    first, count = D.shard_range(img.S, rank, world)
    ok = True
    # unlimited: shard-local solve + one all-reduce
    ctx.upload(img); ctx.set_shard(first, count)
    ctx.analyze_pairs(download=False)
    acc, chosen = ctx.solve(unlimited=True)
    ctx.allocate_by_type()
    cnt, cst = D.allreduce_totals_device(ctx, img.T, dev)
    torch.cuda.synchronize()
    w_cnt, w_cst = rank_emulation.expected_totals(oracle, img, acc_u, ch_u, world)     # rank-order sum of the shard partials
    ok = ok and np.array_equal(cnt.cpu().numpy(), w_cnt) and cst.cpu().numpy().tobytes() == w_cst.tobytes()
    ok = ok and np.array_equal(acc[first:first + count], acc_u[first:first + count])
    # limited: gather rows in place, identical greedy everywhere
    ctx.upload(img); ctx.set_shard(first, count)
    ctx.analyze_pairs(download=False)
    D.gather_pair_rows_device(ctx, img.S, img.A, world, dev)
    torch.cuda.synchronize()
    acc, chosen = ctx.solve(unlimited=False, policy=wva.abi.POLICY_PRIORITY_ROUND_ROBIN)
    w_acc, w_chosen = oracle.solve(img, pairs_all, feas_all, unlimited=False, policy=wva.abi.POLICY_PRIORITY_ROUND_ROBIN)
    ok = ok and np.array_equal(acc, w_acc) and chosen.equal_bits(w_chosen)[0]
    ctx.allocate_by_type()
    cnt, cst = D.allreduce_totals_device(ctx, img.T, dev)
    torch.cuda.synchronize()
    w_cnt, w_cst = rank_emulation.expected_totals(oracle, img, w_acc, w_chosen, world)
    ok = ok and np.array_equal(cnt.cpu().numpy(), w_cnt) and cst.cpu().numpy().tobytes() == w_cst.tobytes()
    # ---- the same two modes with the collective inside the library --------------------------------
    D.attach_library_comm(ctx, dev)
    ctx.upload(img); ctx.comm_shard()
    ok = ok and (ctx.first, ctx.count) == (first, count)
    ctx.analyze_pairs(download=False)
    acc, chosen = ctx.solve(unlimited=True)
    cnt, cst = ctx.allocate_by_type()                       # GLOBAL totals, exchanged by the library
    w_cnt, w_cst = rank_emulation.expected_totals(oracle, img, acc_u, ch_u, world)
    ok = ok and np.array_equal(cnt, w_cnt) and cst.tobytes() == w_cst.tobytes()
    ok = ok and np.array_equal(acc[first:first + count], acc_u[first:first + count])
    box = [cst.tobytes()]
    dist.broadcast_object_list(box, src=0)
    ok = ok and box[0] == cst.tobytes()                     # bit-equal on every rank (rank-order sum)
    for policy in (wva.abi.POLICY_PRIORITY_ROUND_ROBIN, wva.abi.POLICY_PRIORITY_EXHAUSTIVE):
        ctx.upload(img); ctx.comm_shard()
        ctx.analyze_pairs(download=False)
        acc, chosen = ctx.solve(unlimited=False, policy=policy)          # gathers the rows itself (one ncclAllGather)
        w_acc, w_chosen = oracle.solve(img, pairs_all, feas_all, unlimited=False, policy=policy)
        ok = ok and np.array_equal(acc, w_acc) and chosen.equal_bits(w_chosen)[0]
        cnt, cst = ctx.allocate_by_type()
        w_cnt, w_cst = rank_emulation.expected_totals(oracle, img, w_acc, w_chosen, world)
        ok = ok and np.array_equal(cnt, w_cnt) and cst.tobytes() == w_cst.tobytes()
    q.put((rank, bool(ok)))
    ctx.comm_destroy()
    ctx.close()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_nccl():
    c = mp.get_context("spawn")
    q = c.Queue()
    port = 29700 + (os.getpid() % 1000)
    procs = [c.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]


def _group_case(n_dev):
    import wva_import
    wva = wva_import.load()
    from inferno_autoscaler_b200 import binding
    import oracle
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import rank_emulation
    img = wva.synth.make_system(61, 4, seed=93, n_types=2, max_pair_batch=128)
    pairs_all, feas_all, _ = oracle.analyze_pairs(img, threads=4)
    acc_u, ch_u = oracle.solve(img, pairs_all, feas_all, unlimited=True)
    wva.synth.set_capacity_from_demand(img, ch_u.acc, ch_u.num_replicas, fraction=0.6)
    g = binding.Group(list(range(n_dev)))
    try:
        g.upload(img)
        g.analyze(8, 32)
        pairs, feas = g.pairs_fetch()
        assert np.array_equal(feas, feas_all) and pairs.equal_bits(pairs_all)[0]
        best = g.grid_fetch()
        o_best, _, _, _ = oracle.analyze_grid(img, 8, 32, want_cube=False, threads=4)
        assert best.tobytes() == o_best.tobytes()
        acc, chosen = g.solve(unlimited=True)
        assert np.array_equal(acc, acc_u) and chosen.equal_bits(ch_u)[0]
        cnt, cst = g.allocate_by_type()
        w_cnt, w_cst = rank_emulation.expected_totals(oracle, img, acc_u, ch_u, n_dev)   # rank-order sum of the shard partials
        assert np.array_equal(cnt, w_cnt) and cst.tobytes() == w_cst.tobytes()
        for policy in (wva.abi.POLICY_NONE, wva.abi.POLICY_ROUND_ROBIN):
            g.upload(img)
            g.analyze()
            acc, chosen = g.solve(unlimited=False, policy=policy)
            w_acc, w_chosen = oracle.solve(img, pairs_all, feas_all, unlimited=False, policy=policy)
            assert np.array_equal(acc, w_acc) and chosen.equal_bits(w_chosen)[0]
            cnt, cst = g.allocate_by_type()
            w_cnt, w_cst = rank_emulation.expected_totals(oracle, img, w_acc, w_chosen, n_dev)
            assert np.array_equal(cnt, w_cnt) and cst.tobytes() == w_cst.tobytes()
            assert (cnt <= img.type_capacity).all()
    finally:
        g.close()


def test_group_one_device():
    """one-device group: same code path as N devices (NCCL communicator of one rank, shard = everything)"""
    _group_case(1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_group_two_devices_one_process():
    _group_case(2)
