"""Shared by tests/test_motion_planning_costs.py (CPU: torch restatements, host emulation of the kernels) and
tests/test_gpu_motion_planning.py: the motion-planning problems of tests/golden/make_golden_motion_planning.py (motion_planning_problem,
motion_planning_cost_states, motion_planning_cost_functions) and the helpers that run them through the engine."""
import importlib.util
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def golden_module():
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "golden", "make_golden_motion_planning.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def cost_states(g):
    """The per-cost states the fixture was generated from (stored in it as S_*; the maps come from motion_planning_data.npz, item b
    uses map b % 2 as in make_golden_motion_planning.motion_planning_cost_states)."""
    S = {k[2:]: torch.from_numpy(g[k].copy()) for k in g.files if k.startswith("S_")}
    maps = np.load(os.path.join(HERE, "golden", "motion_planning_data.npz"))["sdf"]
    S["sdf"] = torch.from_numpy(maps[[b % 2 for b in range(S["xy"].shape[0])]].copy())
    return S


def cost_functions(th, g, device="cpu", dtype=torch.float64):
    """name -> the fixture's cost functions built with `th` (on `device`, in `dtype`)."""
    G = golden_module()
    S = {k: v.to(device=device, dtype=dtype) for k, v in cost_states(g).items()}
    cfs = G.motion_planning_cost_functions(th, torch, S, eps_at_dist=torch.from_numpy(g["eps_at_dist"]).to(device=device, dtype=dtype))
    if dtype != torch.float64:
        for cf in cfs.values():
            for v in cf.optim_vars + cf.aux_vars + cf.weight.aux_vars:
                v.tensor = v.tensor.to(dtype)
    return cfs


def linearize_one(th, cf, dtype=torch.float64):
    """(weighted Jacobian blocks, weighted error) of ONE cost function through the engine (fused kernel if it has one), read back from
    A_val / b; A_val is filled with NaN first so that an entry the kernel does not write shows up."""
    objective = th.Objective(dtype=dtype)
    objective.add(cf)
    objective.to(cf.optim_vars[0].device)
    eng = objective.engine()
    B, S = eng.batch_size, eng.structure
    A_val = torch.full((B, eng.nnz), float("nan"), dtype=dtype, device=eng.device)
    b = torch.full((B, eng.m), float("nan"), dtype=dtype, device=eng.device)
    eng.linearize_sparse(A_val, b)
    d, st, off = int(S.cost_dims[0]), int(S.stride[0]), int(S.row_block_starts[0])
    blk = A_val[:, off:off + d * st].view(B, d, st)
    jacs = []
    for q, v in enumerate(cf.optim_vars):
        p0 = int(S.block_pointers[0][q])
        jacs.append(blk[:, :, p0:p0 + v.dof()].cpu())
    return jacs, -b[:, :d].cpu(), eng, objective


def run_planner(th, case, solver="dense", device="cpu", iters=None, inputs=None, cuda_graph=False, **lm_kwargs):
    """LM on MP_CASES[case] as the fixture ran it (damping 0.1, the case's step size; `lm_kwargs` added to optimize()); returns
    (errs, deltas, poses_final)."""
    G = golden_module()
    pose, n_it, step, *_ = G.MP_CASES[case]
    inputs = inputs if inputs is not None else G.motion_planning_inputs(torch, case)
    objective, poses, vels, leaves = G.motion_planning_problem(th, torch, inputs, pose, device=device)
    if solver == "dense":
        skw = dict(linear_solver_cls=th.CholeskyDenseSolver)
    else:
        skw = dict(linear_solver_cls=th.BaspachoSparseSolver, linearization_cls=th.SparseLinearization, linear_solver_kwargs=dict(layout=solver))
    opt = th.LevenbergMarquardt(objective, max_iterations=iters or n_it, step_size=step, abs_err_tolerance=0, rel_err_tolerance=0, **skw)
    errs, deltas = [], []

    def cb(optimizer, info, delta, it):
        errs.append(info.last_err.detach().cpu().numpy().copy()); deltas.append(delta.detach().cpu().numpy().copy())
    kw = dict(damping=0.1, end_iter_callback=cb, **lm_kwargs)
    if cuda_graph:
        kw["cuda_graph"] = True
    with torch.no_grad():
        opt.optimize(**kw)
    return np.stack(errs, 0), np.stack(deltas, 0), np.stack([p.tensor.detach().cpu().numpy() for p in poses], 0)


def check_trace(g, case, errs, deltas, rtol_err=1e-8, rtol_delta=1e-5):
    from helpers import decisive_iterations
    ref_err, ref_delta = g[f"{case}_trace_err"], g[f"{case}_trace_delta"]
    k = decisive_iterations(g[f"{case}_err0"], ref_err)
    assert k >= 3, k
    np.testing.assert_allclose(errs[:k], ref_err[:k], rtol=rtol_err)
    for it in range(k):
        rel = np.linalg.norm(deltas[it] - ref_delta[it], axis=1) / np.linalg.norm(ref_delta[it], axis=1)
        assert rel.max() < rtol_delta, (case, it, rel)
    return k
