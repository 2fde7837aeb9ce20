"""Timing of the SE2 motion planner (the reference's examples/se2_planning.py objective: 100 steps, Collision2D + GPMotionModel +
Nonholonomic + HingeCost per step, boundary costs) on per-item seeded 128x128 SDF maps, with the fused kernels and with the same objective
on the torch route (a local subclass of every motion-planning cost function whose schema() returns None).  The two are alternated in the
same process.  Per batch size and solver it prints LM it/s and the linearize and solve time per iteration (CUDA events), plus the GPU's
name and power limit.

    python tools/motion_planning_bench.py [--batches 256 1024 4096] [--solvers dense front] [--iters 5] [--torch-iters 2] [--json OUT]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def random_maps(torch, B, seed, device, size=128, n_obstacles=8):
    """B SDF grids [B, size, size] over [-5, 5]^2: min over per-item random discs of (distance to centre - radius)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    centres = (torch.rand(B, n_obstacles, 2, generator=g, dtype=torch.float64) * 8.0 - 4.0).to(device)
    radii = (0.3 + 0.7 * torch.rand(B, n_obstacles, generator=g, dtype=torch.float64)).to(device)
    cell = 10.0 / size
    ax = -5.0 + cell * torch.arange(size, dtype=torch.float64, device=device)
    yy, xx = torch.meshgrid(ax, ax, indexing="ij")                      # row = y, col = x
    pts = torch.stack([xx, yy], -1).view(1, 1, size, size, 2)
    dist = (pts - centres.view(B, n_obstacles, 1, 1, 2)).norm(dim=-1) - radii.view(B, n_obstacles, 1, 1)
    return dist.min(dim=1).values.contiguous()


def se2_inputs(torch, B, device, T=100, seed=0):
    d = torch.float64
    g = torch.Generator(device="cpu").manual_seed(seed + 1)
    start = torch.tensor([-4.0, -4.0], dtype=d) + 0.5 * torch.rand(B, 2, generator=g, dtype=d)
    goal = torch.tensor([4.0, 4.0], dtype=d) - 0.5 * torch.rand(B, 2, generator=g, dtype=d)
    s = torch.linspace(0, 1, T + 1, dtype=d)
    line = start[None] + (goal - start)[None] * s[:, None, None]
    poses0 = torch.cat([line, torch.ones(T + 1, B, 1, dtype=d), torch.zeros(T + 1, B, 1, dtype=d)], 2)
    vels0 = torch.cat([((goal - start) / 10.0)[None].expand(T + 1, B, 2), torch.zeros(T + 1, B, 1, dtype=d)], 2)
    return dict(sdf=random_maps(torch, B, seed, device).cpu(), origin=torch.full((B, 2), -5.0, dtype=d), cell=torch.full((B, 1), 10.0 / 128, dtype=d),
                start=poses0[0].clone(), goal=goal, poses0=poses0.contiguous(), vels0=vels0.contiguous(), eps=torch.tensor([[1.75]], dtype=d),
                coll_w=torch.tensor([[20.0]], dtype=d), qc_inv=torch.eye(3, dtype=d)[None], dt=torch.tensor([[10.0 / T]], dtype=d),
                nh_w=torch.tensor([[10.0]], dtype=d), pv_w=torch.tensor([[5.0]], dtype=d))


def to_torch_route(objective):
    """Every motion-planning cost function re-classed into a local subclass without a CUDA schema (the engine's torch route)."""
    import theseus_b200 as th
    subs = {}
    for cf in objective.cost_functions.values():
        cls = type(cf)
        if cls.__module__ != th.eb.__name__ or cls not in (th.eb.Collision2D, th.eb.GPMotionModel, th.eb.Nonholonomic, th.eb.HingeCost):
            continue
        if cls not in subs:
            subs[cls] = type("TorchRoute" + cls.__name__, (cls,), {"schema": lambda self, _c=cls: (None, _c.schema(self)[1])})
        cf.__class__ = subs[cls]
    objective._engine = None


def run(torch, th, G, B, solver, iters, torch_route, device):
    inputs = se2_inputs(torch, B, device)
    objective, poses, vels, _ = G.motion_planning_problem(th, torch, inputs, "se2", device=device)
    if torch_route:
        to_torch_route(objective)
    skw = dict(linear_solver_cls=th.CholeskyDenseSolver) if solver == "dense" else dict(
        linear_solver_cls=th.BaspachoSparseSolver, linearization_cls=th.SparseLinearization, linear_solver_kwargs=dict(layout=solver))
    opt = th.LevenbergMarquardt(objective, max_iterations=iters, step_size=0.25, abs_err_tolerance=0, rel_err_tolerance=0, **skw)
    eng = objective.engine()
    with torch.no_grad():
        opt.optimize(damping=0.1)                            # warm-up: plans, first launches, library loads
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        opt.optimize(damping=0.1)
        ev[1].record()
        torch.cuda.synchronize()
        total = ev[0].elapsed_time(ev[1]) / 1e3
        # phases: linearize (fused kernels / torch route) and one solve of the linear system, each timed alone
        lin = opt.linear_solver.linearization
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        for _ in range(3):
            lin.linearize()
        e1.record()
        for _ in range(3):
            opt.linear_solver.solve(damping=0.1)
        e2.record()
        torch.cuda.synchronize()
    return dict(batch=B, solver=solver, route="torch" if torch_route else "fused", lm_it_per_s=iters / total,
                linearize_ms=e0.elapsed_time(e1) / 3, solve_ms=e1.elapsed_time(e2) / 3, groups=len(eng.groups), torch_route_costs=len(eng.generic))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[256, 1024, 4096])
    ap.add_argument("--solvers", nargs="+", default=["dense", "front"])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--torch-iters", type=int, default=2, help="LM iterations of the torch-route runs (slow: one vmap(jacrev) per cost)")
    ap.add_argument("--json", help="also write the results to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "motion_planning_bench.py needs a CUDA device"
    import theseus_b200 as th
    from front_solve_phases import gpu_description
    from motion_planning_cases import golden_module
    G = golden_module()
    device = "cuda:0"
    name, plim = gpu_description()
    print(f"GPU: {name}, power limit {plim}")
    rows = []
    for B in args.batches:
        for solver in args.solvers:
            for torch_route in (False, True):         # alternated in the same process
                r = run(torch, th, G, B, solver, args.torch_iters if torch_route else args.iters, torch_route, device)
                rows.append(r)
                print(json.dumps(r), flush=True)
    out = dict(gpu=name, power_limit=plim, results=rows)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
