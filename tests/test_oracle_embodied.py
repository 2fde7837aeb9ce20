"""oracle/embodied.py (+ its glue in oracle/nls.py) against the reference's own values of the motion-planning and planar-pushing cost
functions (tests/golden/motion_planning_kat.npz, tactile_costs_kat.npz): every cost function of the fixtures, weighted error and weighted
Jacobians, to 1e-12 componentwise relative to each array's largest entry.  The fixtures hold the edge cases these kinds switch on: points
outside the grid, on a grid node, on the far corner and far column (index clamping), dist == eps and dist == radius, +-inf hinge limits,
theta2 - theta1 across +-pi, p = 0 and c^2 = 0, zero-weight items and rows.  CPU only."""
import os

import numpy as np
import pytest

from helpers import load
from oracle import embodied, nls

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def mp():
    g = load("motion_planning_kat")
    S = {k[2:]: g[k] for k in g.files if k.startswith("S_")}
    maps = np.load(os.path.join(HERE, "golden", "motion_planning_data.npz"))["sdf"]
    S["sdf"] = maps[[b % 2 for b in range(S["xy"].shape[0])]]
    return g, S


@pytest.fixture(scope="module")
def tc():
    g = load("tactile_costs_kat")
    return g, {k[2:]: g[k] for k in g.files if k.startswith("S_")}


V = lambda kind, dof: dict(kind=kind, dof=dof)


def _eval(vars_, values, cost):
    spec = dict(dtype=np.dtype(np.float64), vars=vars_, costs=[dict(cost, vars=tuple(range(len(vars_))))])
    return nls.eval_costs(spec, values)[0], spec


def _check(g, name, out, nvars):
    jacs, e = out
    assert len(jacs) == nvars
    for got, key in [(e, f"c_{name}_we")] + [(J, f"c_{name}_wJ{q}") for q, J in enumerate(jacs)]:
        ref = g[key]
        assert got.shape == ref.shape, (key, got.shape, ref.shape)
        scale = max(np.abs(ref).max(), 1e-300)
        np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12 * scale, err_msg=key)


def _mp_costs(g, S):
    """name -> (oracle variables, values, cost dict) of tests/golden/make_golden_motion_planning.motion_planning_cost_functions."""
    B = S["xy"].shape[0]
    c = lambda v: np.array([[v]])
    coll = lambda eps: dict(origin=S["origin"], sdf=S["sdf"], cell=S["cell"], eps=eps)
    di_vars2 = [V("Vector", 2)] * 4
    di_vals2 = [S["p1"], S["v1"], S["p2"], S["v2"]]
    di_vars3 = [V("SE2", 3), V("Vector", 3), V("SE2", 3), V("Vector", 3)]
    di_vals3 = [S["s1"], S["w1"], S["s2"], S["w2"]]
    return {
        "coll_point2": ([V("Vector", 2)], [S["xy"]], dict(kind="collision", aux=coll(g["eps_at_dist"]), weight=("scale", c(3.0)))),
        "coll_se2": ([V("SE2", 3)], [S["se2"]], dict(kind="collision", aux=coll(g["eps_at_dist"]), weight=("scale", c(2.0)))),
        "coll_point2_b1": ([V("Vector", 2)], [S["xy"]], dict(kind="collision", aux=dict(origin=S["origin"][:1], sdf=S["sdf"][:1], cell=S["cell"][:1],
                                                                                      eps=S["eps"][:1]), weight=("scale", np.linspace(0.5, 2.0, B)[:, None]))),
        "di_point2_gp": (di_vars2, di_vals2, dict(kind="double_integrator", aux=dict(dt=c(0.1)),
                                                  weight=("gp", np.array([[[1.5, 0.3], [0.3, 0.8]]]), c(0.1)))),
        "di_point2_gp_b": (di_vars2, di_vals2, dict(kind="double_integrator", aux=dict(dt=S["dt_b"]), weight=("gp", S["qc2_b"], S["dt_b"]))),
        "di_point2_diag": (di_vars2, di_vals2, dict(kind="double_integrator", aux=dict(dt=S["dt_b"]), weight=("diag", S["diag_w"]))),
        "di_se2_gp": (di_vars3, di_vals3, dict(kind="double_integrator", aux=dict(dt=c(0.1)), weight=("gp", np.eye(3)[None], c(0.1)))),
        "di_se2_gp_b": (di_vars3, di_vals3, dict(kind="double_integrator", aux=dict(dt=S["dt_b"]), weight=("gp", S["qc3_b"], S["dt_b"]))),
        "di_se2_scale": (di_vars3, di_vals3, dict(kind="double_integrator", aux=dict(dt=c(0.2)), weight=("scale", c(1.7)))),
        "hinge": ([V("Vector", 3)], [S["hv"]], dict(kind="hinge", aux=dict(down=S["h_down"], up=S["h_up"], threshold=S["h_thr"]),
                                                   weight=("scale", c(4.0)))),
        "hinge_float": ([V("Vector", 3)], [S["hv"]], dict(kind="hinge", aux=dict(down=np.full((1, 3), -0.5), up=np.full((1, 3), 0.5),
                                                                                 threshold=np.full((1, 3), 0.25)), weight=("scale", c(1.0)))),
        "nh_se2": ([V("SE2", 3), V("Vector", 3)], [S["s1"], S["w1"]], dict(kind="nonholonomic", weight=("scale", c(10.0)))),
        "nh_vector": ([V("Vector", 3), V("Vector", 3)], [S["nh_pose"], S["w1"]], dict(kind="nonholonomic", weight=("scale", c(3.0)))),
    }


def _tc_costs(S):
    """name -> (oracle variables, values, cost dict) of tests/golden/make_golden_tactile.tactile_cost_functions."""
    sdf = dict(origin=S["origin"], sdf=S["sdf"], cell=S["cell"], radius=S["radius"])
    se2x2, se2x4 = [V("SE2", 3)] * 2, [V("SE2", 3)] * 4
    qv = [S["o1"], S["o2"], S["e1"], S["e2"]]
    return {
        "eoc": (se2x2, [S["obj"], S["eff"]], dict(kind="eoc", aux=sdf, weight=("scale", S["scale_w"]))),
        "eoc_diag": (se2x2, [S["obj"], S["eff"]], dict(kind="eoc", aux=sdf, weight=("diag", S["diag_w1"]))),
        "eoc_b1": (se2x2, [S["obj"], S["eff"]], dict(kind="eoc", aux={k: v[:1] for k, v in sdf.items()}, weight=("diag", np.array([[1.7]])))),
        "qsp": (se2x4, qv, dict(kind="qsp", aux=dict(c_square=S["c2"]), weight=("diag", S["diag_w3"]))),
        "qsp_scale": (se2x4, qv, dict(kind="qsp", aux=dict(c_square=S["c2"]), weight=("scale", S["scale_w"]))),
        "qsp_b1": (se2x4, qv, dict(kind="qsp", aux=dict(c_square=np.array([[0.3]])), weight=("scale", np.array([[2.0]])))),
        "qsp_b1_diag": (se2x4, qv, dict(kind="qsp", aux=dict(c_square=S["c2"][3:4]), weight=("diag", np.array([[1.0, 0.0, 2.5]])))),
    }


MP_NAMES = ["coll_point2", "coll_se2", "coll_point2_b1", "di_point2_gp", "di_point2_gp_b", "di_point2_diag", "di_se2_gp", "di_se2_gp_b",
            "di_se2_scale", "hinge", "hinge_float", "nh_se2", "nh_vector"]
TC_NAMES = ["eoc", "eoc_diag", "eoc_b1", "qsp", "qsp_scale", "qsp_b1", "qsp_b1_diag"]


@pytest.mark.parametrize("name", MP_NAMES)
def test_motion_planning_costs_match_reference(mp, name):
    g, S = mp
    vars_, values, cost = _mp_costs(g, S)[name]
    out, spec = _eval(vars_, values, cost)
    _check(g, name, out, len(vars_))
    assert nls.cost_dim(spec, spec["costs"][0]) == g[f"c_{name}_we"].shape[1]


@pytest.mark.parametrize("name", TC_NAMES)
def test_tactile_costs_match_reference(tc, name):
    g, S = tc
    vars_, values, cost = _tc_costs(S)[name]
    out, spec = _eval(vars_, values, cost)
    _check(g, name, out, len(vars_))


def test_fixture_edges_are_present(mp, tc):
    """The edge cases the comparisons above rely on are really in the fixtures."""
    g, S = mp
    x = S["xy"]
    dist, _, _, _ = embodied.sdf_lookup(x[:, 0], x[:, 1], S["origin"], S["sdf"], S["cell"])
    assert dist[2] == 0 and np.array_equal(dist[3:4], g["eps_at_dist"][3]), "out of the grid / dist == eps"
    assert np.isinf(S["h_down"]).any() and np.isinf(S["h_up"]).any()
    g, S = tc
    d, _, _, _ = embodied.sdf_lookup(S["eff"][:, 0], S["eff"][:, 1], S["origin"], S["sdf"], S["cell"])
    assert d[2] == S["radius"][2, 0] and (d[5:9] == 0).all()
    assert (S["c2"][3] == 0).all() and np.array_equal(S["e2"][2, :2], S["o2"][2, :2])


def test_linearize_sparse_on_a_mixed_objective(mp):
    """linearize_sparse / error_metric over several of these kinds sharing variables: each cost function's row block equals its own
    evaluation, the columns follow the variables, and the error is 0.5 |b|^2."""
    g, S = mp
    spec = dict(dtype=np.dtype(np.float64), vars=[V("SE2", 3), V("Vector", 3), V("SE2", 3), V("Vector", 3)], costs=[
        dict(kind="nonholonomic", vars=(2, 3), weight=("scale", np.array([[2.0]]))),
        dict(kind="double_integrator", vars=(0, 1, 2, 3), aux=dict(dt=S["dt_b"]), weight=("gp", S["qc3_b"], S["dt_b"])),
        dict(kind="collision", vars=(2,), aux=dict(origin=S["origin"], sdf=S["sdf"], cell=S["cell"], eps=S["eps"]), weight=("scale", np.array([[3.0]]))),
        dict(kind="hinge", vars=(1,), aux=dict(down=S["h_down"], up=S["h_up"], threshold=S["h_thr"]), weight=("diag", S["diag_w"][:, :3])),
    ])
    values = [S["s1"], S["w1"], S["s2"], S["w2"]]
    st = nls.sparse_structure(spec)
    A_val, b = nls.linearize_sparse(spec, values, st)
    A = nls.csr_to_dense(st, A_val)
    row = 0
    for f, c in enumerate(spec["costs"]):
        jacs, e = nls.eval_costs(dict(spec, costs=[c]), values)[0]
        d = e.shape[1]
        np.testing.assert_array_equal(b[:, row:row + d], -e)
        for k, v in enumerate(c["vars"]):
            np.testing.assert_array_equal(A[:, row:row + d, 3 * v:3 * v + 3], jacs[k])
        row += d
    assert row == st["num_rows"] == 1 + 6 + 1 + 3
    np.testing.assert_allclose(nls.error_metric(spec, values), 0.5 * (b ** 2).sum(1), rtol=1e-14)


def test_gp_weight_follows_the_lower_triangle_of_the_transpose():
    """For a non-symmetric Qc_inv the reference factors the symmetric matrix built from the lower triangle of W^T, which is not
    chol(S)^T (x) chol(Q)^T of either triangle of Q."""
    dt = 0.1
    Q = np.array([[[1.5, 0.31], [0.29, 0.8]]])
    L = embodied.gp_weight(Q, np.array([[dt]]))[0]
    S = np.array([[12 / dt ** 3, -6 / dt ** 2], [-6 / dt ** 2, 4 / dt]])
    Wt = np.block([[12 / dt ** 3 * Q[0].T, -6 / dt ** 2 * Q[0].T], [-6 / dt ** 2 * Q[0].T, 4 / dt * Q[0].T]])
    M = np.tril(Wt) + np.tril(Wt, -1).T
    np.testing.assert_allclose(L.T @ L, M, rtol=1e-13)
    assert np.allclose(np.triu(L), L)
    kron = np.kron(np.linalg.cholesky(S).T, np.linalg.cholesky(np.tril(Q[0]) + np.tril(Q[0], -1).T).T)
    assert np.abs(L - kron).max() > 1e-3 * np.abs(L).max()
    Qs = np.array([[[1.5, 0.3], [0.3, 0.8]]])
    np.testing.assert_allclose(embodied.gp_weight(Qs, np.array([[dt]]))[0], np.kron(np.linalg.cholesky(S).T, np.linalg.cholesky(Qs[0]).T),
                               rtol=1e-13, atol=1e-13 * 1e4)
