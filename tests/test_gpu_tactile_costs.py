"""The fused planar-pushing kernels (QuasiStaticPushingPlanar, EffectorObjectContactPlanar) on the GPU: A_val / b against the reference
(tests/golden/tactile_costs_kat.npz) and against the torch route on config C4's states (tests/golden/tactile_c4_kat.npz, batch 512),
masking, broadcasting, batch independence, and which cost functions of C4 still take the torch route.
Dry run on the CPU:  THB_SIMT_EMULATION=1 python -m pytest tests/test_gpu_tactile_costs.py -m gpu"""
import numpy as np
import pytest
import torch

import theseus_b200 as th
from helpers import load
from motion_planning_cases import linearize_one
from tactile_cases import cost_functions, cost_states, golden_module, torch_route
from test_gpu_backward import _golden_module

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_C4_KEYS = ("obj", "eff", "eff_meas", "mfb_meas", "c_square", "eff_radius", "sdf", "sdf_origin", "sdf_cell")


@pytest.fixture(scope="module")
def g():
    return load("tactile_costs_kat")


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(np.asarray(b)), 1e-300))


def _c4(route):
    """Config C4's objective at batch 512 (make_golden.tactile_problem); route == "torch": QSP and EOC re-classed onto the torch route."""
    c4 = load("tactile_c4_kat")
    objective, objs, effs, leaves = _golden_module().tactile_problem(th, torch, {k: torch.from_numpy(c4[k]) for k in _C4_KEYS}, device=DEV)
    if route == "torch":
        for cf in objective.cost_functions.values():
            if type(cf) in (th.eb.QuasiStaticPushingPlanar, th.eb.EffectorObjectContactPlanar):
                torch_route(cf)
        objective._engine = None
    return objective


def _linearize(objective):
    eng = objective.engine()
    A_val = torch.full((eng.batch_size, eng.nnz), float("nan"), dtype=torch.float64, device=eng.device)
    b = torch.full((eng.batch_size, eng.m), float("nan"), dtype=torch.float64, device=eng.device)
    eng.linearize_sparse(A_val, b)
    return eng, A_val.cpu(), b.cpu()


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-12), (torch.float32, 1e-5)])
def test_fused_linearize_matches_reference(g, dtype, tol):
    for name, cf in cost_functions(th, g, device=DEV, dtype=dtype).items():
        jacs, err, eng, _ = linearize_one(th, cf, dtype=dtype)
        assert not eng.generic and len(eng.groups) == 1, name
        assert not torch.isnan(err).any() and all(not torch.isnan(J).any() for J in jacs), name
        assert _rel(err.double().numpy(), g[f"c_{name}_we"]) < tol, name
        for q, J in enumerate(jacs):
            assert _rel(J.double().numpy(), g[f"c_{name}_wJ{q}"]) < tol, (name, q)


def test_fused_matches_the_torch_route_on_c4():
    fused, routed = _c4("fused"), _c4("torch")
    ef, Af, bf = _linearize(fused)
    et, At, bt = _linearize(routed)
    assert len(et.generic) == 24 + 25 + 24 and len(ef.generic) == 24
    assert ef.nnz == et.nnz and ef.m == et.m
    assert not torch.isnan(Af).any() and not torch.isnan(bf).any()
    assert _rel(Af.numpy(), At.numpy()) < 1e-12 and _rel(bf.numpy(), bt.numpy()) < 1e-12
    np.testing.assert_allclose(fused.error_metric().cpu().numpy(), routed.error_metric().cpu().numpy(), rtol=1e-12)


def test_c4_groups_take_the_fused_kinds():
    eng = _c4("fused").engine()
    names = [eng.costs[f].name for f in eng.generic]
    assert len(names) == 24 and all(n.startswith("mfb_") for n in names)
    kinds = {grp.kind: grp.K for grp in eng.groups}
    assert kinds[15] == 24 and kinds[16] == 25


def test_zero_weights_mask_the_cost_function(g):
    G = golden_module()
    # (cost function, its items with all-zero weights, an input of theirs set to NaN: a masked item's inputs are not read)
    for name, items, key in (("eoc", [10], "sdf"), ("eoc_diag", [7], "radius"), ("qsp", [6], "c2"), ("qsp_scale", [10], "c2")):
        S = cost_states(g, device=DEV)
        S[key][items] = float("nan")
        jacs, err, _, objective = linearize_one(th, G.tactile_cost_functions(th, torch, S)[name])
        assert (err[items] == 0).all() and all((J[items] == 0).all() for J in jacs), name
        assert torch.isfinite(err).all() and all(torch.isfinite(J).all() for J in jacs), name
        em = objective.error_metric().cpu()
        assert (em[items] == 0).all() and torch.isfinite(em).all(), name
    jacs, err, _, _ = linearize_one(th, cost_functions(th, g, device=DEV)["qsp"])
    assert err[5, 1] == 0 and all((J[5, 1] == 0).all() for J in jacs) and (err[5, [0, 2]] != 0).all()   # one zero row


def test_batch1_aux_tensors_equal_per_item_copies(g):
    cfs = cost_functions(th, g, device=DEV)
    B = cfs["eoc"].obj.tensor.shape[0]
    one = cfs["eoc_b1"]
    ex = lambda v: v.tensor.expand((B,) + tuple(v.tensor.shape[1:])).clone()
    per_item = th.eb.EffectorObjectContactPlanar(th.SE2(tensor=one.obj.tensor.clone()), th.SE2(tensor=one.eff.tensor.clone()), ex(one.sdf_origin),
                                                 ex(one.sdf_data), th.Variable(ex(one.sdf_cell_size)), ex(one.eff_radius),
                                                 th.DiagonalCostWeight(ex(one.weight.diagonal)))
    ja, ea, _, _ = linearize_one(th, one)
    jb, eb, _, _ = linearize_one(th, per_item)
    assert torch.equal(ea, eb) and all(torch.equal(a, b) for a, b in zip(ja, jb))
    one = cfs["qsp_b1"]
    per_item = th.eb.QuasiStaticPushingPlanar(*[th.SE2(tensor=v.tensor.clone()) for v in one.optim_vars], th.Variable(ex(one.c_square)),
                                              th.ScaleCostWeight(ex(one.weight.scale)))
    ja, ea, _, _ = linearize_one(th, one)
    jb, eb, _, _ = linearize_one(th, per_item)
    assert torch.equal(ea, eb) and all(torch.equal(a, b) for a, b in zip(ja, jb))


def test_items_are_independent_of_the_batch(g):
    full = cost_states(g, device=DEV)
    G = golden_module()
    ref = {name: linearize_one(th, cf)[:2] for name, cf in G.tactile_cost_functions(th, torch, full).items()}
    for idx in ([1, 2, 7], [11]):
        S = {k: v[idx].contiguous() for k, v in full.items()}
        for name, cf in G.tactile_cost_functions(th, torch, S).items():
            if "b1" in name:
                continue                     # its aux tensors are one item's: not the sliced problem's
            jacs, err = linearize_one(th, cf)[:2]
            assert torch.equal(err, ref[name][1][idx]) and all(torch.equal(a, b[idx]) for a, b in zip(jacs, ref[name][0])), (name, idx)
