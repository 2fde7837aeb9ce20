"""The fused motion-planning kernels (Collision2D, DoubleIntegrator / GPMotionModel with GPCostWeight, HingeCost, Nonholonomic) on the GPU:
A_val / b against the reference (tests/golden/motion_planning_kat.npz) and against the torch route, masking, broadcasting, batch
independence, both planners' LM traces on every solver, backward-mode gradients and CUDA-graph replay.  Tolerances as DESIGN.md §5.
Dry run on the CPU:  THB_SIMT_EMULATION=1 python -m pytest tests/test_gpu_motion_planning.py -m gpu"""
import os

import numpy as np
import pytest
import torch

import theseus_b200 as th
from helpers import load
from motion_planning_cases import check_trace, cost_functions, cost_states, golden_module, linearize_one, run_planner

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def g():
    return load("motion_planning_kat")


def _torch_route(cf):
    """Re-class `cf` into a test-local subclass without a CUDA schema: the engine evaluates it on the torch route."""
    cls = type(cf)
    sub = type("TorchRoute" + cls.__name__, (cls,), {"schema": lambda self: (None, cls.schema(self)[1])})
    cf.__class__ = sub
    return cf


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(np.asarray(b)), 1e-300))


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-12), (torch.float32, 1e-5)])
def test_fused_linearize_matches_reference(g, dtype, tol):
    for name, cf in cost_functions(th, g, device=DEV, dtype=dtype).items():
        jacs, err, _, _ = linearize_one(th, cf, dtype=dtype)
        assert not torch.isnan(err).any() and all(not torch.isnan(J).any() for J in jacs), name
        # item 3 sits exactly at dist == cost_eps in fp64: in fp32 the rounded inputs fall on either side of the hinge
        sel = [0, 1, 2, 4, 5] if dtype == torch.float32 and name in ("coll_point2", "coll_se2") else slice(None)
        assert _rel(err.double().numpy()[sel], g[f"c_{name}_we"][sel]) < tol, name
        for q, J in enumerate(jacs):
            assert _rel(J.double().numpy()[sel], g[f"c_{name}_wJ{q}"][sel]) < tol, (name, q)


def test_fused_linearize_and_error_match_the_torch_route(g):
    fused = cost_functions(th, g, device=DEV)
    routed = {k: _torch_route(cf) for k, cf in cost_functions(th, g, device=DEV).items()}
    for name in fused:
        jf, ef, _, of = linearize_one(th, fused[name])
        jt, et, eng, ot = linearize_one(th, routed[name])
        assert eng.generic == [0] and not eng.groups, name
        assert _rel(ef.numpy(), et.numpy()) < 1e-12, name
        for a, b in zip(jf, jt):
            assert _rel(a.numpy(), b.numpy()) < 1e-12, name
        # (collision item 3 sits on the hinge, dist == cost_eps: there a one-ulp difference in dist leaves e ~ 1e-16 instead of 0)
        em_f, em_t = of.error_metric().cpu().numpy(), ot.error_metric().cpu().numpy()
        np.testing.assert_allclose(em_f, em_t, rtol=1e-12, atol=1e-24 * max(1.0, float(np.abs(em_t).max())))


def test_zero_weights_mask_the_cost_function(g):
    S = {k: v.to(DEV) for k, v in cost_states(g).items()}
    B = S["xy"].shape[0]
    w = torch.linspace(0.5, 2.0, B, dtype=torch.float64, device=DEV).view(B, 1)
    w[1] = 0.0
    w[3] = 0.0
    sdf = S["sdf"].clone()
    sdf[3] = float("nan")          # a masked item's inputs are not read
    cf = th.eb.Collision2D(th.Point2(tensor=S["xy"]), S["origin"], sdf, th.Variable(S["cell"]), th.Variable(S["eps"]), th.ScaleCostWeight(w))
    jacs, err, _, objective = linearize_one(th, cf)
    assert (err[[1, 3]] == 0).all() and (jacs[0][[1, 3]] == 0).all()
    assert torch.isfinite(err).all() and torch.isfinite(jacs[0]).all()
    em = objective.error_metric().cpu()
    assert em[1] == 0 and em[3] == 0 and torch.isfinite(em).all()
    di = cost_functions(th, g, device=DEV)["di_point2_diag"]
    dw = di.weight.diagonal.tensor.clone()
    dw[2] = 0.0
    di.weight.diagonal.tensor = dw
    jacs, err, _, _ = linearize_one(th, di)
    assert (err[2] == 0).all() and all((J[2] == 0).all() for J in jacs)


def test_batch1_aux_tensors_equal_per_item_copies(g):
    cfs = cost_functions(th, g, device=DEV)
    one = cfs["coll_point2_b1"]
    B = one.pose.tensor.shape[0]
    per_item = th.eb.Collision2D(th.Point2(tensor=one.pose.tensor.clone()), one.sdf_origin.tensor.expand(B, 2).clone(),
                                 one.sdf_data.tensor.expand(B, -1, -1).clone(), th.Variable(one.sdf_cell_size.tensor.expand(B, 1).clone()),
                                 th.Variable(one.cost_eps.tensor.expand(B, 1).clone()), th.ScaleCostWeight(one.weight.scale.tensor.clone()))
    ja, ea, _, _ = linearize_one(th, one)
    jb, eb, _, _ = linearize_one(th, per_item)
    assert torch.equal(ea, eb) and torch.equal(ja[0], jb[0])
    gp = cfs["di_point2_gp"]
    gp_b = th.eb.GPMotionModel(*[type(v)(tensor=v.tensor.clone()) for v in gp.optim_vars], th.Variable(gp.dt.tensor.expand(B, 1).clone()),
                               th.eb.GPCostWeight(gp.weight.Qc_inv.tensor.expand(B, 2, 2).clone(), th.Variable(gp.weight.dt.tensor.expand(B, 1).clone())))
    ja, ea, _, _ = linearize_one(th, gp)
    jb, eb, _, _ = linearize_one(th, gp_b)
    assert torch.equal(ea, eb) and all(torch.equal(a, b) for a, b in zip(ja, jb))


def _slice_inputs(inputs, idx):
    out = {}
    for k, v in inputs.items():
        if k in ("poses0", "vels0"):
            out[k] = v[:, idx].contiguous()
        elif v.shape[0] > 1:
            out[k] = v[idx].contiguous()
        else:
            out[k] = v
    return out


@pytest.mark.parametrize("case", ["point2", "se2"])
def test_items_are_independent_of_the_batch(case):
    G = golden_module()
    full = G.motion_planning_inputs(torch, case)
    e4, d4, p4 = run_planner(th, case, device=DEV, iters=4, inputs=full)
    for idx in ([1, 2], [3]):
        e, dl, p = run_planner(th, case, device=DEV, iters=4, inputs=_slice_inputs(full, idx))
        assert np.array_equal(e, e4[:, idx]) and np.array_equal(dl, d4[:, idx]) and np.array_equal(p, p4[:, idx]), (case, idx)


@pytest.mark.parametrize("case", ["point2", "se2"])
@pytest.mark.parametrize("solver", ["dense", "front", "lane"])
def test_planner_lm_traces_match_reference(g, case, solver):
    errs, deltas, final = run_planner(th, case, solver, device=DEV)
    check_trace(g, case, errs, deltas)


@pytest.mark.parametrize("mode", ["unroll", "truncated", "implicit"])
def test_backward_mode_gradients_match_reference(g, mode):
    G = golden_module()
    inputs = G.motion_planning_inputs(torch, "point2")
    objective, poses, vels, leaves = G.motion_planning_problem(th, torch, inputs, "point2", device=DEV)
    for v in leaves.values():
        v.tensor.requires_grad_(True)
    init = {p.name: p.tensor.clone().requires_grad_(True) for p in poses}
    opt = th.LevenbergMarquardt(objective, linear_solver_cls=th.CholeskyDenseSolver, max_iterations=3, step_size=0.3, abs_err_tolerance=0,
                                rel_err_tolerance=0)
    sol, info = th.TheseusLayer(opt).forward(dict(init), optimizer_kwargs=dict(G.MP_GRAD_MODES[mode], damping=0.1))
    gen = torch.Generator().manual_seed(7)
    Pz = torch.stack([sol[p.name] for p in poses], 0)
    (Pz * torch.randn(Pz.shape, generator=gen, dtype=torch.float64).to(DEV)).sum().backward()
    for k, v in leaves.items():
        ref = g[f"grad_{mode}_{k}"]
        assert _rel(v.tensor.grad.cpu().numpy(), ref) < 1e-6, (mode, k)
    gi = np.stack([(init[p.name].grad if init[p.name].grad is not None else torch.zeros_like(init[p.name])).cpu().numpy() for p in poses], 0)
    ref = g[f"grad_{mode}_init"]
    if np.abs(ref).max() == 0:
        assert np.abs(gi).max() == 0, mode
    else:
        assert _rel(gi, ref) < 1e-6, mode


@pytest.mark.skipif(os.environ.get("THB_SIMT_EMULATION") == "1", reason="CUDA streams and graphs have no host emulation")
@pytest.mark.parametrize("case", ["point2", "se2"])
def test_cuda_graph_is_bitwise_equal_to_eager(case):
    # adaptive damping: the damping is a device tensor in both modes (a python-float damping becomes one only in the captured loop)
    a = run_planner(th, case, device=DEV, iters=5, adaptive_damping=True)
    b = run_planner(th, case, device=DEV, iters=5, cuda_graph=True, adaptive_damping=True)
    for x, y in zip(a, b):
        assert np.array_equal(x, y), case
