"""SURVEY.md 8(e) on hardware: the batch sharded over 2 GPUs (one process per GPU, NCCL) against the single-GPU run, per batch item.
No kernel mixes batch items and no data-path collective exists; the only batch-global decisions (all items rejected -> retry, the
linear-solve failure flag) are all-reduced, so every per-item quantity must be BITWISE the single-process one -- dense and sparse.
Needs >= 2 GPUs (skipped on a machine with one)."""
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, solver, out):
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here)); sys.path.insert(0, here)
    import torch.distributed as dist
    import theseus_b200 as th
    from theseus_b200.datasets import build_pose_graph_objective, pose_graph_synthetic_3d
    from theseus_b200.distributed import batch_shard
    torch.cuda.set_device(rank)
    device = torch.device("cuda", rank)
    pg = None
    if world > 1:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
        pg = dist.group.WORLD
    try:
        B = 37                                                   # ragged shards: 19 + 18
        data = pose_graph_synthetic_3d(48, B, seed=5)
        sl = batch_shard(B, rank, world)
        objective, poses = build_pose_graph_objective(th, data, device, batch_slice=sl)
        skw = dict(linear_solver_cls=th.CholeskyDenseSolver) if solver == "dense" else dict(
            linear_solver_cls=th.BaspachoSparseSolver, linearization_cls=th.SparseLinearization, linear_solver_kwargs=dict(layout=solver))
        opt = th.LevenbergMarquardt(objective, max_iterations=8, step_size=1.0, abs_err_tolerance=0, rel_err_tolerance=0, process_group=pg, **skw)
        with torch.no_grad():
            info = opt.optimize(track_err_history=True, damping=1e-3, adaptive_damping=True, ellipsoidal_damping=True)
        out[(world, rank)] = (sl.start, sl.stop, info.err_history.cpu().numpy().copy(), np.stack([p.tensor.cpu().numpy() for p in poses], 0))
    finally:
        if world > 1:
            dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("solver", ["dense", "front", "lane"])
def test_two_gpu_sharded_lm_is_bitwise_the_single_gpu_run(solver):
    mgr = mp.Manager()
    out = mgr.dict()
    port = 29500 + (os.getpid() % 400)
    mp.spawn(_worker, args=(1, port, solver, out), nprocs=1, join=True)
    mp.spawn(_worker, args=(2, port + 1, solver, out), nprocs=2, join=True)
    _, _, hist1, poses1 = out[(1, 0)]
    covered = 0
    for r in range(2):
        s0, s1, hist, poses = out[(2, r)]
        np.testing.assert_array_equal(hist, hist1[s0:s1])
        np.testing.assert_array_equal(poses, poses1[:, s0:s1])
        covered += s1 - s0
    assert covered == hist1.shape[0]
