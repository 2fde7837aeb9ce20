"""th.eb motion-planning cost functions (Collision2D, SignedDistanceField2D, DoubleIntegrator / GPMotionModel + GPCostWeight, HingeCost,
Nonholonomic) on the CPU: constructor checks as the reference makes them, the torch restatements against the reference's analytic values
(tests/golden/motion_planning_kat.npz), and the fused kernels of thb_costs.cu on the host emulation (tests/simt) -- A_val / b per cost
function and both planners' LM traces."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import theseus_b200 as th
from helpers import load
from motion_planning_cases import check_trace, cost_functions, cost_states, linearize_one, run_planner

HERE = os.path.dirname(os.path.abspath(__file__))
d = torch.float64


@pytest.fixture(scope="module")
def g():
    return load("motion_planning_kat")


# ------------------------------------------------------------------------------------------------ constructor checks
def test_collision2d_constructor_checks():
    sdf = torch.zeros(1, 4, 5, dtype=d)
    w = th.ScaleCostWeight(1.0)
    with pytest.raises(ValueError, match="Collision2D only accepts Point2 or SE2 poses."):
        th.eb.Collision2D(th.Vector(tensor=torch.zeros(1, 2, dtype=d)), torch.zeros(1, 2, dtype=d), sdf, 0.1, 0.5, w)
    with pytest.raises(ValueError, match="must be either a tensor or a Point2 variable"):
        th.eb.Collision2D(th.Point2(tensor=torch.zeros(1, 2, dtype=d)), [0.0, 0.0], sdf, 0.1, 0.5, w)
    with pytest.raises(ValueError, match="must be a batch of 2D tensors"):
        th.eb.Collision2D(th.Point2(tensor=torch.zeros(1, 2, dtype=d)), torch.zeros(1, 3, dtype=d), sdf, 0.1, 0.5, w)
    with pytest.raises(ValueError, match="sdf_data to SignedDistanceField2D must be a batch of matrices"):
        th.eb.Collision2D(th.Point2(tensor=torch.zeros(1, 2, dtype=d)), torch.zeros(1, 2, dtype=d), sdf[0], 0.1, 0.5, w)
    with pytest.raises(ValueError, match="cell_size must be either a Variable, tensor, or float"):
        th.eb.Collision2D(th.Point2(tensor=torch.zeros(1, 2, dtype=d)), torch.zeros(1, 2, dtype=d), sdf, 1, 0.5, w)
    with pytest.raises(ValueError, match="cell_size must be a batch of 0D or 1D tensors"):
        th.eb.Collision2D(th.Point2(tensor=torch.zeros(1, 2, dtype=d)), torch.zeros(1, 2, dtype=d), sdf, th.Variable(torch.ones(1, 2, dtype=d)), 0.5, w)
    cf = th.eb.Collision2D(th.SE2(tensor=torch.tensor([[0.0, 0.0, 1.0, 0.0]], dtype=d)), torch.zeros(1, 2, dtype=d), sdf, 0.1, 0.5, w)
    assert cf.dim() == 1 and cf.num_optim_vars() == 1 and cf.num_aux_vars() == 4
    assert [v.tensor.shape for v in cf.aux_vars] == [(1, 2), (1, 4, 5), (1, 1), (1, 1)]
    c2 = cf.copy(new_name="c2")
    assert type(c2) is th.eb.Collision2D and c2.name == "c2" and c2.pose is not cf.pose and c2.sdf_data is not cf.sdf_data
    new_data = th.Variable(torch.ones(1, 4, 5, dtype=d))
    cf.set_aux_var_at(1, new_data)
    assert cf.sdf.sdf_data is new_data


def test_gp_cost_weight_and_double_integrator_constructor_checks():
    with pytest.raises(ValueError, match="dt must be greater than 0."):
        th.eb.GPCostWeight(torch.eye(2, dtype=d), 0.0)
    with pytest.raises(ValueError, match="dt must be a 0-D or 1-D tensor."):
        th.eb.GPCostWeight(torch.eye(2, dtype=d), torch.ones(2, 2, dtype=d))
    with pytest.raises(ValueError, match="Qc_inv must be a single matrix or a batch of matrices."):
        th.eb.GPCostWeight(torch.ones(1, 1, 2, 2, dtype=d), 0.1)
    with pytest.raises(ValueError, match="Qc_inv must contain square matrices."):
        th.eb.GPCostWeight(torch.ones(2, 3, dtype=d), 0.1)
    with pytest.raises(ValueError, match="Qc_inv must be positive definite."):
        th.eb.GPCostWeight(-torch.eye(2, dtype=d), 0.1)
    w = th.eb.GPCostWeight(torch.eye(2, dtype=d), 0.1)
    assert w.Qc_inv.shape == (1, 2, 2) and w.dt.shape == (1, 1) and not w.is_zero().any()
    assert [v.name for v in w.aux_vars] == [w.Qc_inv.name, w.dt.name]
    w2 = w.copy(new_name="w2")
    assert type(w2) is th.eb.GPCostWeight and w2.Qc_inv is not w.Qc_inv and w2.name == "w2"
    p = lambda n: th.Point2(tensor=torch.zeros(1, 2, dtype=d))
    with pytest.raises(ValueError, match="All variables for a DoubleIntegrator must have the same dimension."):
        th.eb.DoubleIntegrator(p(0), th.Vector(tensor=torch.zeros(1, 3, dtype=d)), p(1), p(2), 0.1, w)
    with pytest.raises(ValueError, match="dt data must be a 0-D or 1-D tensor"):
        th.eb.DoubleIntegrator(p(0), p(0), p(1), p(2), torch.ones(2, 2, dtype=d), w)
    with pytest.raises(ValueError, match="GPMotionModel only accepts cost weights of type GPCostWeight."):
        th.eb.GPMotionModel(p(0), p(0), p(1), p(2), 0.1, th.ScaleCostWeight(1.0))
    cf = th.eb.GPMotionModel(p(0), p(0), p(1), p(2), 0.1, w)
    assert cf.dim() == 4 and cf.num_optim_vars() == 4 and cf.num_aux_vars() == 1
    assert type(cf.copy()) is th.eb.GPMotionModel and type(th.eb.DoubleIntegrator(p(0), p(0), p(1), p(2), 0.1, w).copy()) is th.eb.DoubleIntegrator


def test_hinge_and_nonholonomic_constructor_checks():
    v = th.Vector(tensor=torch.zeros(1, 3, dtype=d))
    w = th.ScaleCostWeight(1.0)
    with pytest.raises(ValueError, match=r"Limit and threshold must be 1D variables with dimension equal to `vector.dof\(\)` \(3\)."):
        th.eb.HingeCost(v, torch.zeros(1, 2, dtype=d), 1.0, 0.1, w)
    with pytest.raises(ValueError, match="All down_limit must be <= than up_limit."):
        th.eb.HingeCost(v, 1.0, -1.0, 0.1, w)
    with pytest.raises(ValueError, match="Threshold values must be positive numbers."):
        th.eb.HingeCost(v, -1.0, 1.0, -0.1, w)
    cf = th.eb.HingeCost(v, -1.0, 1.0, 0.1, w, name="h")
    assert cf.dim() == 3 and [a.name for a in cf.aux_vars] == ["h__downlimit", "h__uplimit", "h__thres"]
    assert all(a.dtype == d for a in cf.aux_vars)
    with pytest.raises(ValueError, match="Nonholonomic only accepts 3D velocity or poses"):
        th.eb.Nonholonomic(th.Point2(tensor=torch.zeros(1, 2, dtype=d)), v, w)
    with pytest.raises(ValueError, match="Nonholonomic only accepts 3D velocity or poses"):
        th.eb.Nonholonomic(v, th.Point2(tensor=torch.zeros(1, 2, dtype=d)), w)
    nh = th.eb.Nonholonomic(th.SE2(tensor=torch.tensor([[0.0, 0.0, 1.0, 0.0]], dtype=d)), v, w)
    assert nh.dim() == 1 and type(nh.copy()) is th.eb.Nonholonomic


def test_schemas_pick_the_fused_kinds():
    from theseus_b200 import core
    z = lambda n: torch.zeros(1, n, dtype=d)
    w = th.ScaleCostWeight(1.0)
    se2 = lambda: th.SE2(tensor=torch.tensor([[0.0, 0.0, 1.0, 0.0]], dtype=d))
    gp = th.eb.GPCostWeight(torch.eye(3, dtype=d), 0.1)
    assert th.eb.GPMotionModel(se2(), th.Vector(tensor=z(3)), se2(), th.Vector(tensor=z(3)), 0.1, gp).schema()[0] == core.COST_DOUBLE_INTEGRATOR_SE2
    so2 = lambda: th.SO2(theta=torch.zeros(1, 1, dtype=d))
    assert th.eb.DoubleIntegrator(so2(), th.Vector(tensor=z(1)), so2(), th.Vector(tensor=z(1)), 0.1, w).schema()[0] is None   # torch route
    assert th.eb.HingeCost(th.Vector(tensor=z(4)), -1.0, 1.0, 0.1, w).schema()[0] is None
    assert th.eb.Nonholonomic(th.Vector(tensor=z(3)), th.Vector(tensor=z(3)), w).schema()[0] == core.COST_NONHOLONOMIC_VECTOR
    robust = th.RobustCostFunction(th.eb.Nonholonomic(se2(), th.Vector(tensor=z(3)), w), th.HuberLoss, th.Variable(torch.zeros(1, 1, dtype=d)))
    assert robust.schema()[0] is None


# ------------------------------------------------------------------------------------------------ torch restatements vs the reference
def test_signed_distance_field_matches_reference(g):
    S = cost_states(g)
    sdf = th.eb.SignedDistanceField2D(th.Point2(tensor=S["origin"]), th.Variable(S["cell"]), th.Variable(S["sdf"]))
    dist, jac = sdf.signed_distance(S["xy"].view(-1, 2, 1))
    np.testing.assert_allclose(dist.numpy(), g["sd_dist"], rtol=1e-13, atol=1e-14)
    np.testing.assert_allclose(jac.numpy(), g["sd_jac"], rtol=1e-13, atol=1e-14)
    assert dist[2].item() == 0.0 and (jac[2] == 0).all()           # out of the grid: boundary value 0
    row, col, oob = sdf.convert_points_to_cell(S["xy"].view(-1, 2, 1))
    assert oob[:, 0].tolist() == [False, False, True, False, False, False]


def test_torch_restatements_match_reference_analytic_values(g):
    for name, cf in cost_functions(th, g).items():
        J, e = cf.jacobians()
        np.testing.assert_allclose(e.numpy(), g[f"c_{name}_e"], rtol=1e-12, atol=1e-13, err_msg=name)
        wJ, we = cf.weighted_jacobians_error()
        np.testing.assert_allclose(we.numpy(), g[f"c_{name}_we"], rtol=1e-11, atol=1e-12, err_msg=name)
        for q in range(cf.num_optim_vars()):
            # autograd differentiates SE2's log exactly; the reference's analytic jlog is a series below 1e-3
            np.testing.assert_allclose(J[q].numpy(), g[f"c_{name}_J{q}"], rtol=1e-9, atol=1e-11, err_msg=f"{name} J{q}")
            np.testing.assert_allclose(wJ[q].numpy(), g[f"c_{name}_wJ{q}"], rtol=1e-9, atol=1e-11, err_msg=f"{name} wJ{q}")


def test_effector_object_contact_uses_the_shared_sdf_lookup():
    """EffectorObjectContactPlanar's lookup now goes through SignedDistanceField2D.interpolate: same ops, same bits as the inline copy."""
    rng = torch.Generator().manual_seed(3)
    o = torch.randn(5, 3, generator=rng, dtype=d)
    obj = torch.stack([o[:, 0], o[:, 1], o[:, 2].cos(), o[:, 2].sin()], 1)
    eff = torch.cat([0.3 * torch.randn(5, 2, generator=rng, dtype=d), obj[:, 2:]], 1)
    sdf = torch.randn(5, 16, 16, generator=rng, dtype=d)
    origin, cell, radius = torch.full((5, 2), -0.375, dtype=d), torch.full((5, 1), 0.05, dtype=d), torch.full((5, 1), 0.05, dtype=d)
    cf = th.eb.EffectorObjectContactPlanar(th.SE2(tensor=obj), th.SE2(tensor=eff), origin, sdf, th.Variable(cell), radius, th.ScaleCostWeight(1.0))
    got = cf._torch_error((obj, eff), (origin, sdf, cell, radius))
    # the inline lookup it replaced
    dx, dy = eff[..., 0] - obj[..., 0], eff[..., 1] - obj[..., 1]
    px, py = obj[..., 2] * dx + obj[..., 3] * dy, -obj[..., 3] * dx + obj[..., 2] * dy
    c = cell.view(-1)
    oob = (px < origin[..., 0]) | (px > origin[..., 0] + 15.0 * c) | (py < origin[..., 1]) | (py > origin[..., 1] + 15.0 * c)
    col, row = (px - origin[..., 0]) / c, (py - origin[..., 1]) / c
    lr, lc = torch.floor(row), torch.floor(col)
    hr, hc = lr + 1.0, lc + 1.0
    lri, lci, hri, hci = lr.long().clamp(0, 15), lc.long().clamp(0, 15), hr.long().clamp(0, 15), hc.long().clamp(0, 15)
    bi = torch.arange(5)
    G = lambda r, cc: sdf[bi, r, cc]
    dist = (hr - row) * (hc - col) * G(lri, lci) + (row - lr) * (hc - col) * G(hri, lci) + (hr - row) * (col - lc) * G(lri, hci) \
        + (row - lr) * (col - lc) * G(hri, hci)
    dist = torch.where(oob, torch.zeros_like(dist), dist)
    assert torch.equal(got, (dist - radius.view(-1)).abs().unsqueeze(-1))


# ------------------------------------------------------------------------------------------------ fused kernels on the host emulation
def _emulation_mode():
    spec = importlib.util.spec_from_file_location("emulation_mode", os.path.join(HERE, "simt", "emulation_mode.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def emu_lib():
    return _emulation_mode().load_emulated_lib()


@pytest.fixture
def emulated(monkeypatch, emu_lib):
    _emulation_mode().patch_host(monkeypatch.setattr, emu_lib)
    return emu_lib


def test_fused_kernels_match_reference_on_the_emulated_library(emulated, g):
    for name, cf in cost_functions(th, g).items():
        kind, _ = cf.schema()
        assert kind is not None, name
        jacs, err, _, _ = linearize_one(th, cf)
        np.testing.assert_allclose(err.numpy(), g[f"c_{name}_we"], rtol=1e-12, atol=1e-13, err_msg=name)
        for q, J in enumerate(jacs):
            assert not torch.isnan(J).any(), name
            np.testing.assert_allclose(J.numpy(), g[f"c_{name}_wJ{q}"], rtol=1e-9, atol=1e-11, err_msg=f"{name} J{q}")


def test_fused_error_metric_on_the_emulated_library(emulated, g):
    for name, cf in cost_functions(th, g).items():
        objective = th.Objective(dtype=d)
        objective.add(cf)
        np.testing.assert_allclose(objective.error_metric().numpy(), 0.5 * (g[f"c_{name}_we"] ** 2).sum(1), rtol=1e-12, atol=1e-14, err_msg=name)


@pytest.mark.parametrize("case", ["point2", "se2"])
def test_planner_lm_traces_on_the_emulated_library(emulated, g, case):
    errs, deltas, final = run_planner(th, case, "dense")
    check_trace(g, case, errs, deltas)
