"""th.eb planar-pushing cost functions (QuasiStaticPushingPlanar, EffectorObjectContactPlanar) on the CPU: which schema they pick, the
torch restatements against the reference's analytic values (tests/golden/tactile_costs_kat.npz), and the fused kernels of thb_costs.cu on
the host emulation (tests/simt) -- A_val / b per cost function and the error metric."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import theseus_b200 as th
from helpers import load
from motion_planning_cases import linearize_one
from tactile_cases import cost_functions, cost_states

HERE = os.path.dirname(os.path.abspath(__file__))
d = torch.float64


@pytest.fixture(scope="module")
def g():
    return load("tactile_costs_kat")


def test_fixture_covers_the_edge_cases(g):
    S = cost_states(g)
    dist, r = g["eoc_dist"][:, 0], S["radius"][:, 0].numpy()
    assert dist[0] > r[0] and dist[1] < r[1] and dist[2] == r[2]
    assert (dist[5:9] == 0).all()                                              # outside on each side
    assert (S["obj"][2:5] == torch.tensor([0.0, 0.0, 1.0, 0.0], dtype=d)).all()          # p = t_eff exactly: on grid nodes, far edge
    assert S["cell"][4, 0] * 14 + S["origin"][4, 0] == S["eff"][4, 0]
    w = torch.atan2(S["o1"][:, 2] * S["o2"][:, 3] - S["o1"][:, 3] * S["o2"][:, 2], S["o1"][:, 2] * S["o2"][:, 2] + S["o1"][:, 3] * S["o2"][:, 3])
    t1, t2 = torch.atan2(S["o1"][:, 3], S["o1"][:, 2]), torch.atan2(S["o2"][:, 3], S["o2"][:, 2])
    assert abs(w[0]) < 1 and (t2 - t1)[0] < -np.pi and abs(w[1]) < 1 and (t2 - t1)[1] > np.pi      # theta2 - theta1 wraps across -pi / +pi
    assert torch.equal(S["e2"][2, :2], S["o2"][2, :2]) and S["c2"][3, 0] == 0


def test_schemas_pick_the_fused_kinds():
    from theseus_b200 import core
    se2 = lambda: th.SE2(tensor=torch.tensor([[0.0, 0.0, 1.0, 0.0]], dtype=d))
    w = th.ScaleCostWeight(1.0)
    qsp = th.eb.QuasiStaticPushingPlanar(se2(), se2(), se2(), se2(), 0.3, w)
    kind, aux = qsp.schema()
    assert kind == core.COST_QUASI_STATIC_PUSHING_PLANAR == 15 and aux == [qsp.c_square]
    eoc = th.eb.EffectorObjectContactPlanar(se2(), se2(), torch.zeros(1, 2, dtype=d), torch.zeros(1, 4, 5, dtype=d), 0.1, 0.05, w)
    kind, aux = eoc.schema()
    assert kind == core.COST_EFF_OBJ_CONTACT_PLANAR == 16 and aux == [eoc.sdf_origin, eoc.sdf_data, eoc.sdf_cell_size, eoc.eff_radius]
    # other pose types: torch route
    se3 = lambda: th.SE3(tensor=torch.eye(3, 4, dtype=d).unsqueeze(0))
    assert th.eb.QuasiStaticPushingPlanar(se2(), se2(), se2(), se3(), 0.3, w).schema() == (None, [])
    assert th.eb.EffectorObjectContactPlanar(se3(), se2(), torch.zeros(1, 2, dtype=d), torch.zeros(1, 4, 5, dtype=d), 0.1, 0.05, w).schema() == (None, [])
    # robust-wrapped: torch route
    lr = th.Variable(torch.zeros(1, 1, dtype=d))
    assert th.RobustCostFunction(qsp, th.HuberLoss, lr).schema()[0] is None
    assert th.RobustCostFunction(eoc, th.WelschLoss, lr).schema()[0] is None
    with pytest.raises(NotImplementedError, match="Jacobians for huber loss are not yet implemented."):
        th.eb.EffectorObjectContactPlanar(se2(), se2(), torch.zeros(1, 2, dtype=d), torch.zeros(1, 4, 5, dtype=d), 0.1, 0.05, w, use_huber_loss=True)


def test_torch_restatements_match_reference_analytic_values(g):
    for name, cf in cost_functions(th, g).items():
        J, e = cf.jacobians()
        np.testing.assert_allclose(e.numpy(), g[f"c_{name}_e"], rtol=1e-12, atol=1e-13, err_msg=name)
        wJ, we = cf.weighted_jacobians_error()
        np.testing.assert_allclose(we.numpy(), g[f"c_{name}_we"], rtol=1e-12, atol=1e-13, err_msg=name)
        # autograd of |dist - r| is 0 at dist == r (item 2), where the reference keeps the +1 sign
        sel = [b for b in range(J[0].shape[0]) if not (name.startswith("eoc") and name != "eoc_b1" and b == 2)]
        for q in range(cf.num_optim_vars()):
            np.testing.assert_allclose(J[q].numpy()[sel], g[f"c_{name}_J{q}"][sel], rtol=1e-10, atol=1e-12, err_msg=f"{name} J{q}")
            np.testing.assert_allclose(wJ[q].numpy()[sel], g[f"c_{name}_wJ{q}"][sel], rtol=1e-10, atol=1e-12, err_msg=f"{name} wJ{q}")


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
        jacs, err, eng, _ = linearize_one(th, cf)
        assert not eng.generic and len(eng.groups) == 1, name
        np.testing.assert_allclose(err.numpy(), g[f"c_{name}_we"], rtol=1e-12, atol=1e-13, err_msg=name)
        for q, J in enumerate(jacs):
            assert not torch.isnan(J).any(), name
            np.testing.assert_allclose(J.numpy(), g[f"c_{name}_wJ{q}"], rtol=1e-12, atol=1e-13, err_msg=f"{name} J{q}")


def test_fused_error_metric_on_the_emulated_library(emulated, g):
    for name, cf in cost_functions(th, g).items():
        objective = th.Objective(dtype=d)
        objective.add(cf)
        np.testing.assert_allclose(objective.error_metric().numpy(), 0.5 * (g[f"c_{name}_we"] ** 2).sum(1), rtol=1e-12, atol=1e-14, err_msg=name)
