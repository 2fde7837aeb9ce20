"""Timing of config C4 (tactile pose estimation: the planar-pushing objective of tests/golden/make_golden.py:tactile_problem, T = 25 steps,
the states of tests/golden/tactile_c4_kat.npz at batch 512, tiled along the batch to 2048 and 4096) with the fused QuasiStaticPushingPlanar
and EffectorObjectContactPlanar kernels and with the same objective with those two re-classed onto the torch route (a local subclass whose
schema() returns None).  The two are alternated in the same process.  Per batch size and solver it prints LM it/s over 8 iterations, the
time of one linearization, one error_metric and one solve (CUDA events), the time of one full C4 step (TheseusLayer forward + IMPLICIT
backward), the number of cost functions on the torch route (MovingFrameBetween stays there in both), plus the GPU's name and power limit.

    python tools/tactile_bench.py [--batches 512 2048 4096] [--solvers dense front] [--iters 8] [--json OUT]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

LM = dict(damping=1e-2, adaptive_damping=True, ellipsoidal_damping=True)
_KEYS = ("obj", "eff", "eff_meas", "mfb_meas", "c_square", "eff_radius", "sdf", "sdf_origin", "sdf_cell")
_BATCHED = ("obj", "eff", "eff_meas", "mfb_meas")     # [T or T-1, B, 4]; the other inputs are batch-1


def c4_inputs(torch, g, B):
    reps = -(-B // g["obj"].shape[1])
    out = {}
    for k in _KEYS:
        t = torch.from_numpy(g[k])
        out[k] = t.repeat(1, reps, 1)[:, :B].contiguous() if k in _BATCHED else t
    return out


def to_torch_route(th, objective):
    """QuasiStaticPushingPlanar and EffectorObjectContactPlanar re-classed into local subclasses without a CUDA schema."""
    subs = {}
    for cf in objective.cost_functions.values():
        cls = type(cf)
        if cls not in (th.eb.QuasiStaticPushingPlanar, th.eb.EffectorObjectContactPlanar):
            continue
        if cls not in subs:
            subs[cls] = type("TorchRoute" + cls.__name__, (cls,), {"schema": lambda self, _c=cls: (None, _c.schema(self)[1])})
        cf.__class__ = subs[cls]
    objective._engine = None


def _optimizer(th, objective, solver, iters):
    skw = dict(linear_solver_cls=th.CholeskyDenseSolver) if solver == "dense" else dict(
        linear_solver_cls=th.BaspachoSparseSolver, linearization_cls=th.SparseLinearization, linear_solver_kwargs=dict(layout=solver))
    return th.LevenbergMarquardt(objective, max_iterations=iters, step_size=1.0, abs_err_tolerance=0, rel_err_tolerance=0, **skw)


def _build(th, torch, G, inputs, torch_route, device):
    objective, objs, effs, leaves = G.tactile_problem(th, torch, inputs, device=device)
    if torch_route:
        to_torch_route(th, objective)
    return objective, objs, effs, leaves


def run(torch, th, G, g, B, solver, iters, torch_route, device):
    inputs = c4_inputs(torch, g, B)
    objective, objs, effs, _ = _build(th, torch, G, inputs, torch_route, device)
    opt = _optimizer(th, objective, solver, iters)
    eng = objective.engine()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        opt.optimize(**LM)                                   # warm-up: plans, first launches, library loads
        torch.cuda.synchronize()
        e0, e1 = ev(), ev()
        e0.record()
        opt.optimize(**LM)
        e1.record()
        torch.cuda.synchronize()
        total = e0.elapsed_time(e1) / 1e3
        # phases, each timed alone over 3 calls: linearize (fused kernels / torch route), error_metric, one solve of the linear system
        lin = opt.linear_solver.linearization
        e = [ev() for _ in range(4)]
        e[0].record()
        for _ in range(3):
            lin.linearize()
        e[1].record()
        for _ in range(3):
            objective.error_metric()
        e[2].record()
        for _ in range(3):
            opt.linear_solver.solve(damping=LM["damping"])
        e[3].record()
        torch.cuda.synchronize()
    # one full C4 step: TheseusLayer forward (iters LM iterations) + IMPLICIT backward to the learnable cost parameters
    step_s = []
    for rep in range(2):                                     # the first one is the warm-up
        objective, objs, effs, leaves = _build(th, torch, G, inputs, torch_route, device)
        for v in leaves.values():
            v.tensor.requires_grad_(True)
        layer = th.TheseusLayer(_optimizer(th, objective, solver, iters))
        proj = torch.randn(len(objs), B, 4, generator=torch.Generator().manual_seed(5), dtype=torch.float64).to(device)
        torch.cuda.synchronize()
        s0, s1 = ev(), ev()
        s0.record()
        sol, _ = layer.forward({v.name: v.tensor.clone() for v in objs + effs}, optimizer_kwargs=dict(LM, backward_mode="implicit"))
        (torch.stack([sol[o.name] for o in objs], 0) * proj).sum().backward()
        s1.record()
        torch.cuda.synchronize()
        step_s.append(s0.elapsed_time(s1) / 1e3)
    return dict(batch=B, solver=solver, route="torch" if torch_route else "fused", lm_it_per_s=iters / total,
                linearize_ms=e[0].elapsed_time(e[1]) / 3, error_metric_ms=e[1].elapsed_time(e[2]) / 3, solve_ms=e[2].elapsed_time(e[3]) / 3,
                step_fwd_implicit_bwd_s=step_s[-1], groups=len(eng.groups), torch_route_costs=len(eng.generic))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[512, 2048, 4096])
    ap.add_argument("--solvers", nargs="+", default=["dense", "front"])
    ap.add_argument("--iters", type=int, default=8)
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "tactile_bench.py needs a CUDA device"
    import theseus_b200 as th
    from front_solve_phases import gpu_description
    from test_gpu_backward import _golden_module
    G = _golden_module()
    g = np.load(os.path.join(ROOT, "tests", "golden", "tactile_c4_kat.npz"))
    device = "cuda:0"
    name, plim = gpu_description()
    print(f"GPU: {name}, power limit {plim}")
    rows = []
    for B in args.batches:
        for solver in args.solvers:
            for torch_route in (False, True):         # alternated in the same process
                r = run(torch, th, G, g, B, solver, args.iters, torch_route, device)
                rows.append(r)
                print(json.dumps(r), flush=True)
    out = dict(gpu=name, power_limit=plim, results=rows)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
