"""The kernels every LM iteration runs around the linear solver, each compared directly with a float64 restatement:
  1. the fused linearize / error kernels of the core cost kinds (Between / Local on SE3, SO3, SE2, Vector Difference, Reprojection,
     with Huber / Welsch), against oracle/nls.py + oracle/lie.py, at the batch / cost counts where the warp-staged A_val store and the
     8-cost error chunks change shape, and on both sides of every branch threshold of the Lie logarithms;
  2. the Gram kernels (thb_gram_f64 / _f32: every gram_block_kernel<DI, DJ> instance, the split 6x6 path and the entry-per-thread
     gram_kernel; dense mirrored output and a block-by-block factor layout) against float64 A^T A of the same A_val;
  3. lm_control (thb_lm_control_f64 / _f32) against a numpy restatement of its accept / reject decision;
  4. retract / commit on SE3, SO3, SE2, SO2 and Vector variables.

fp64 kernels are compared with the oracle in float64.  fp32 kernels are compared with the oracle evaluated in float64 arithmetic but with
the float32 eps tables (fixture `oracle_eps`): the reference takes the same branches as the kernel and adds no rounding of its own; the
inputs are the fp32-rounded values, so only the kernel's own rounding is measured.

Tolerances are componentwise, of the form C u kappa scale with u the unit roundoff of the kernel's dtype; each check says where its
bound comes from.  Dry run on the CPU:  THB_SIMT_EMULATION=1 python -m pytest tests/test_gpu_cost_kernels.py -m gpu"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import theseus_b200 as th
from oracle import lie, nls
from theseus_b200 import _lib
from theseus_b200.structure import build_gram_plan, build_structure, lower_blocks

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EMU = os.environ.get("THB_SIMT_EMULATION") == "1"      # host emulation: one OS thread per CUDA thread, so the large cases shrink
U = {torch.float64: 2.0 ** -53, torch.float32: 2.0 ** -24}
NP = {torch.float64: np.float64, torch.float32: np.float32}
SFX = {torch.float64: "f64", torch.float32: "f32"}
DTYPES = [torch.float64, torch.float32]
RATIOS = {}     # section -> largest |error| / bound seen (printed at the end of the module with -s)


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for k in sorted(RATIOS):
        print(f"max error/bound {k}: {RATIOS[k]:.3g}")


@pytest.fixture
def oracle_eps(monkeypatch):
    """use(dtype): evaluate the float64 oracle with `dtype`'s eps tables (torchlie global_params / theseus global_params)."""
    def use(dtype):
        if dtype == torch.float32:
            f32, f64 = np.dtype("float32"), np.dtype("float64")
            monkeypatch.setitem(lie._EPS, f64, dict(lie._EPS[f32]))
            monkeypatch.setitem(lie._EPS_TH, f64, dict(lie._EPS_TH[f32]))
    return use


def _within(section, got, ref, tol, what):
    """|got - ref| <= tol componentwise; entries where the reference is not finite must be non-finite in the same places (and equal)."""
    got, ref, tol = np.asarray(got, np.float64), np.asarray(ref, np.float64), np.broadcast_to(np.asarray(tol, np.float64), np.shape(ref))
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), (what, "NaN pattern", np.argwhere(np.isnan(got) != np.isnan(ref))[:5])
    assert np.array_equal(got[~fin & ~np.isnan(ref)], ref[~fin & ~np.isnan(ref)]), (what, "inf pattern")
    err = np.abs(got[fin] - ref[fin])
    bad = err > tol[fin]
    if err.size:
        ratio = float(np.max(np.where(tol[fin] > 0, err / np.where(tol[fin] > 0, tol[fin], 1.0), np.where(err > 0, np.inf, 0.0))))
        RATIOS[section] = max(RATIOS.get(section, 0.0), ratio)
    if bad.any():
        i = np.argwhere(fin)[np.flatnonzero(bad)[0]]
        raise AssertionError(f"{what}: {int(bad.sum())} entries out of bound, first at {tuple(i)}: got {got[tuple(i)]!r} "
                             f"ref {ref[tuple(i)]!r} bound {tol[tuple(i)]!r}")


# ====================================================================================================================================
# 1. fused linearization and error
# ------------------------------------------------------------------------------------------------------------------------------------
CLS = {"SE3": th.SE3, "SO3": th.SO3, "SE2": th.SE2}
GDIM = {"SE3": 6, "SO3": 3, "SE2": 3}


def _unit(rng, B):
    a = rng.standard_normal((B, 3))
    return a / np.linalg.norm(a, axis=1, keepdims=True)


def _rot(rng, B, lo=0.0, hi=np.pi):
    return lie.so3_exp(_unit(rng, B) * rng.uniform(lo, hi, (B, 1)))


def _elem(group, rng, B):
    if group == "SO3":
        return _rot(rng, B)
    if group == "SE3":
        return np.concatenate([_rot(rng, B), rng.uniform(-2, 2, (B, 3, 1))], axis=-1)
    a = rng.uniform(-np.pi, np.pi, B)
    return np.stack([rng.uniform(-2, 2, B), rng.uniform(-2, 2, B), np.cos(a), np.sin(a)], axis=-1)


class _Problem:
    """An objective built through the public API and its oracle description (oracle/nls.py spec) over the same fp-rounded values."""

    def __init__(self, dtype):
        self.dtype, self.np = dtype, NP[dtype]
        self.objective = th.Objective(dtype=dtype)
        self.vars, self.values, self.costs = [], [], []      # values: float64 copies of the dtype-rounded tensors

    def r(self, a):
        return np.asarray(a, np.float64).astype(self.np).astype(np.float64)

    def t(self, a):
        return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float64).astype(self.np)))

    nan_items = ()      # batch items whose per-item aux tensors are NaN in the objective (the oracle keeps the finite values)

    def at(self, a):
        t = self.t(a)
        if t.shape[0] > 1 and len(self.nan_items):
            t[list(self.nan_items)] = float("nan")
        return t

    def var(self, cls, value, kind, dof):
        value = self.r(value)
        v = cls(tensor=self.t(value)) if issubclass(cls, th.Vector) else cls(tensor=self.t(value), disable_checks=True)
        self.vars.append(dict(obj=v, kind=kind, dof=dof))
        self.values.append(value)
        return len(self.vars) - 1

    def weight(self, wkind, Bw, dim, rng, zero=()):
        w = self.r(rng.uniform(0.5, 2.0, (Bw, 1 if wkind == "scale" else dim)))
        w[list(zero)] = 0.0
        tw = th.Variable(self.t(w))
        return (th.ScaleCostWeight(tw) if wkind == "scale" else th.DiagonalCostWeight(tw)), (wkind, w)

    def add(self, cf, spec, robust=None, rng=None, Br=1):
        if robust is not None:
            lr = self.r(rng.uniform(np.log(0.05), np.log(5.0), (Br, 1)))
            cf = th.RobustCostFunction(cf, dict(huber=th.HuberLoss, welsch=th.WelschLoss)[robust], th.Vector(tensor=self.t(lr)))
            spec["robust"] = (robust, lr)
        self.objective.add(cf)
        self.costs.append(spec)

    def build(self):
        self.objective.to(DEV)
        eng = self.objective.engine()
        assert not eng.generic, "every cost function of these tests has a fused kernel"
        # the oracle's variables in the engine's column order
        pos = {v["obj"].name: i for i, v in enumerate(self.vars)}
        order = [pos[v.name] for v in eng.ordering]
        remap = {old: new for new, old in enumerate(order)}
        self.spec = dict(dtype=np.dtype(np.float64), vars=[dict(kind=self.vars[i]["kind"], dof=self.vars[i]["dof"]) for i in order],
                         costs=[dict(c, vars=tuple(remap[v] for v in c["vars"])) for c in self.costs])
        self.ovalues = [self.values[i] for i in order]
        self.eng = eng
        return self


def _exact_elem(group, rng, B):
    """Elements whose rotation is a signed permutation (SE2: a quarter turn): composing with them only moves and negates entries, so
    Z^-1 X0^-1 X1 reproduces a placed relative rotation exactly."""
    if group == "SE2":
        q = rng.integers(0, 4, B)
        cs = np.array([[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]])[q]
        return np.concatenate([rng.uniform(-2, 2, (B, 2)), cs], -1)
    R = np.stack([np.eye(3)[rng.permutation(3)] * rng.choice([-1.0, 1.0], (3, 1)) for _ in range(B)])
    R[np.linalg.det(R) < 0, 0] *= -1
    return R if group == "SO3" else np.concatenate([R, rng.uniform(-2, 2, (B, 3, 1))], -1)


def _group_problem(kind, B, K, dtype, rng, wkind="diag", w_b1=False, aux_b1=False, robust=None, zero=(), rel=None, nan_items=()):
    """K Between / Local cost functions on SE3 / SO3 / SE2 over N shared variables.  rel: [B] relative elements E = Z^-1 X0^-1 X1
    (Between) or T^-1 X (Local) to place over exact variables (_exact_elem), or None: random variables and measurements."""
    mode, group = kind.split("_")
    P = _Problem(dtype)
    P.nan_items = nan_items
    nv = 2 if mode == "between" else 1
    N = max(nv, min(K + 1, (K + 3) // 2))
    ids = [P.var(CLS[group], (_elem if rel is None else _exact_elem)(group, rng, B), group, GDIM[group]) for _ in range(N)]
    G = nls._GROUP[group]
    for k in range(K):
        i = k % N
        j = (i + 1 + k // N) % N
        j = j if j != i else (i + 1) % N
        Bz = 1 if aux_b1 else B
        Z = _elem(group, rng, Bz)
        if rel is not None:
            D = G["compose"](G["inverse"](P.values[ids[i]]), P.values[ids[j]]) if mode == "between" else P.values[ids[i]]
            Z = G["compose"](D[:Bz], G["inverse"](rel))         # Z^-1 D = E
        Z = P.r(Z)
        zv = CLS[group](tensor=P.at(Z), disable_checks=True)
        wt, ws = P.weight(wkind, 1 if w_b1 else B, GDIM[group], rng, zero=() if w_b1 else zero)
        cf = th.Between(P.vars[ids[i]]["obj"], P.vars[ids[j]]["obj"], zv, wt) if mode == "between" else th.Difference(P.vars[ids[i]]["obj"], zv, wt)
        P.add(cf, dict(kind=mode, group=group, vars=(ids[i], ids[j]) if mode == "between" else (ids[i],), aux=Z, weight=ws),
              robust=robust, rng=rng, Br=1 if aux_b1 else B)
    return P.build()


def _vector_problem(d, B, K, dtype, rng, wkind="diag", w_b1=False, aux_b1=False, zero=(), nan_items=()):
    P = _Problem(dtype)
    P.nan_items = nan_items
    N = max(1, (K + 1) // 2)
    ids = [P.var(th.Vector, rng.uniform(-3, 3, (B, d)), "Vector", d) for _ in range(N)]
    for k in range(K):
        tg = P.r(rng.uniform(-3, 3, (1 if aux_b1 else B, d)))
        wt, ws = P.weight(wkind, 1 if w_b1 else B, d, rng, zero=() if w_b1 else zero)
        cf = th.Difference(P.vars[ids[k % N]]["obj"], th.Vector(tensor=P.at(tg)), wt)
        P.add(cf, dict(kind="local", group="Vector", vars=(ids[k % N],), aux=tg, weight=ws))
    return P.build()


def _reproj_problem(B, K, dtype, rng, wkind="diag", w_b1=False, aux_b1=False, robust=None, zero=(), nan_items=()):
    """Cameras near the identity looking down -z at points 4-6 units away: q_z stays well away from 0."""
    P = _Problem(dtype)
    P.nan_items = nan_items
    Nc, Np = max(1, (K + 2) // 3), max(1, (K + 1) // 2)
    cams = [P.var(th.SE3, np.concatenate([_rot(rng, B, 0.0, 0.3), rng.uniform(-0.5, 0.5, (B, 3, 1))], -1), "SE3", 6) for _ in range(Nc)]
    pts = [P.var(th.Point3, np.concatenate([rng.uniform(-2, 2, (B, 2)), rng.uniform(-6, -4, (B, 1))], -1), "Vector", 3) for _ in range(Np)]
    for k in range(K):
        Ba = 1 if aux_b1 else B
        f, z = P.r(rng.uniform(0.5, 1.5, (Ba, 1))), P.r(rng.uniform(-1, 1, (Ba, 2)))
        k1, k2 = P.r(rng.uniform(-0.1, 0.1, (Ba, 1))), P.r(rng.uniform(-0.05, 0.05, (Ba, 1)))
        wt, ws = P.weight(wkind, 1 if w_b1 else B, 2, rng, zero=() if w_b1 else zero)
        c, p = cams[k % Nc], pts[k % Np]
        cf = th.eb.Reprojection(camera_pose=P.vars[c]["obj"], world_point=P.vars[p]["obj"], focal_length=th.Vector(tensor=P.at(f)),
                                calib_k1=th.Vector(tensor=P.t(k1)), calib_k2=th.Vector(tensor=P.t(k2)),
                                image_feature_point=th.Point2(tensor=P.at(z)), weight=wt)
        P.add(cf, dict(kind="reproj", vars=(c, p), aux=dict(f=f, z=z, k1=k1, k2=k2), weight=ws), robust=robust, rng=rng, Br=Ba)
    return P.build()


def _make(kind, B, K, dtype, rng, **kw):
    if kind.startswith("vector"):
        return _vector_problem(int(kind.split("_")[1]), B, K, dtype, rng, **{k: v for k, v in kw.items() if k != "robust"})
    if kind == "reproj":
        return _reproj_problem(B, K, dtype, rng, **kw)
    return _group_problem(kind, B, K, dtype, rng, **kw)


def _kappa(P, dtype):
    """[B, F] condition factor of each (item, cost function), from the formulas the kernel evaluates:
    - above the near-zero branch of the SE3 log and the d_near_zero branch of the SO3 jlog, the coefficients divide by 2 cos(theta) - 2,
      which has lost a relative 2 / theta^2 to cancellation (in fp32, 2e4 just above near_zero = 1e-2); the SE2 jlog's
      0.5 sin / (1 - cos) term (~1/theta) carries the same loss into a 1/theta coefficient: 2 / |theta|^3 above its d_near_zero;
    - above d_near_zero the SE3 jlog's c coefficient divides 2 (2 cos - 2) + theta sin + theta^2, which cancels to theta^6 / 360, by
      theta^6: the absolute error ~u of cos becomes 8 u / theta^6 in c, and c enters the Jacobian times (w . lin) w w^T ~ |lin| theta^3,
      so 8 / theta^3 (7e6 just above the fp64 threshold 1e-2; the kernel reproduces the reference formula, conditioning included);
    - outside the near-pi branch the rotation log reads the axis from the antisymmetric part scaled by theta / sin(theta) (~ 1/(pi - theta));
      the Jacobian and the translation part then use w up to quadratically (b w w^T, b w (w . t) with b |w|^2 <= 1, and |w| <= pi in
      the adjoint products), which multiplies that error by a small constant: 6 theta / sin(theta).  Inside the near-pi branch the axis
      comes from the symmetric part and is well conditioned.  SE2 has no near-pi branch: its (1 + cos) theta / sin term grows the same way;
    - a Welsch rescale exp(-x / r) has relative condition x / r in x = |w e|^2."""
    B = P.ovalues[0].shape[0]
    kap = np.ones((B, len(P.spec["costs"])))
    for f, c in enumerate(P.spec["costs"]):
        if c["kind"] in ("between", "local") and c["group"] != "Vector":
            G = nls._GROUP[c["group"]]
            x0 = P.ovalues[c["vars"][0]]
            D = G["compose"](G["inverse"](x0), P.ovalues[c["vars"][1]]) if c["kind"] == "between" else x0
            E = G["compose"](G["inverse"](np.broadcast_to(c["aux"], D.shape)), D)
            with np.errstate(divide="ignore", invalid="ignore"):
                if c["group"] == "SE2":
                    theta, sine = np.abs(np.arctan2(E[:, 3], E[:, 2])), np.abs(E[:, 3])
                    cancel = np.where(theta >= lie._EPS_TH[np.dtype(np.float64)]["se2_d_near_zero"], 2 / theta ** 3, 0.0)
                    npi = np.zeros(B, bool)
                else:
                    _, (theta, sine, cosine) = lie.so3_log_helper(E[..., :3])
                    npi = 1 + cosine <= lie.eps("near_pi", np.float64)
                    th0 = lie.eps("near_zero" if c["group"] == "SE3" else "d_near_zero", np.float64)
                    cancel = np.where(theta >= th0, 2 / theta ** 2, 0.0)
                    if c["group"] == "SE3":
                        cancel = np.maximum(cancel, np.where(theta >= lie.eps("d_near_zero", np.float64), 8 / theta ** 3, 0.0))
                k = (1 + cancel) * np.where(npi | (theta < 1.0), 1.0, 6 * theta / sine)
            kap[:, f] = np.where(np.isfinite(k), k, 1.0)
        if c.get("robust") is not None and c["robust"][0] == "welsch":
            _, e = nls.eval_costs(dict(P.spec, costs=[dict(c, robust=None)]), P.ovalues, want_jac=False)[0]
            kap[:, f] *= 1.0 + (e ** 2).sum(1) / np.exp(np.broadcast_to(c["robust"][1], (B, 1))[:, 0])
    return kap


# Every entry of A and e is a sum of a few dozen products whose factors are bounded by the magnitudes in the cost function's own row of the
# reference (the Jacobian entries and the residual: rotation entries are <= 1, the translation / reprojection terms appear in both).  Its
# rounding error is then at most gamma_k (k ~ 40 operations along the longest chain: compose, log, jlog, adjoint product, weight, robust
# rescale) times kappa times that row scale.
C_LIN = 48


def _lin_bounds(P, A_ref, b_ref, dtype):
    S = P.eng.structure
    B = A_ref.shape[0]
    rows = np.repeat(np.arange(S.num_rows), np.diff(S.A_row_ptr))
    rowmax = np.zeros((B, S.num_rows))
    nz = np.diff(S.A_row_ptr) > 0
    rowmax[:, nz] = np.maximum.reduceat(np.nan_to_num(np.abs(A_ref), nan=0.0), S.A_row_ptr[:-1][nz], axis=1)
    scale = np.maximum(rowmax, np.nan_to_num(np.abs(b_ref), nan=0.0))
    row_cost = np.repeat(np.arange(len(S.cost_dims)), S.cost_dims)
    tol_row = C_LIN * U[dtype] * _kappa(P, dtype)[:, row_cost] * scale
    return tol_row[:, rows], tol_row


def _linearize(P):
    eng, B = P.eng, P.eng.batch_size
    guard = 256                                  # NaN entries after A_val and b: a store past the end shows up instead of corrupting memory
    A_buf = torch.full((B * eng.nnz + guard,), float("nan"), dtype=P.dtype, device=eng.device)   # an entry the kernel does not write stays NaN
    b_buf = torch.full((B * eng.m + guard,), float("nan"), dtype=P.dtype, device=eng.device)
    A, b = A_buf[:B * eng.nnz].view(B, eng.nnz), b_buf[:B * eng.m].view(B, eng.m)
    eng.linearize_sparse(A, b)
    assert torch.isnan(A_buf[B * eng.nnz:]).all() and torch.isnan(b_buf[B * eng.m:]).all(), "store past the end of A_val / b"
    return A.cpu().double().numpy(), b.cpu().double().numpy()


def _check_problem(P, dtype, section, check_error=True):
    S, ref_struct = P.eng.structure, nls.sparse_structure(P.spec)
    assert np.array_equal(S.A_row_ptr, ref_struct["A_row_ptr"]) and np.array_equal(S.A_col_ind, ref_struct["A_col_ind"])
    A, b = _linearize(P)
    with np.errstate(divide="ignore", invalid="ignore"):      # SE2 at theta = +-pi: the reference's own 0 * inf
        A_ref, b_ref = nls.linearize_sparse(P.spec, P.ovalues, ref_struct)
    tol_A, tol_b = _lin_bounds(P, A_ref, b_ref, dtype)
    _within(section, A, A_ref, tol_A, "A_val")
    _within(section, b, b_ref, tol_b, "b")
    if not check_error:
        return A, b
    em = P.objective.error_metric().cpu().double().numpy()
    with np.errstate(divide="ignore", invalid="ignore"):
        em_ref = nls.error_metric(P.spec, P.ovalues)
    # 0.5 sum e^2: a perturbation |de| <= tol_b of every residual moves it by at most sum(|e| tol_b + tol_b^2 / 2); the chunked sum of
    # m squares adds gamma_(m+2) of the (non-negative) total
    m = b.shape[1]
    gam = (m + 2) * U[dtype]
    tol_em = (np.abs(b_ref) * tol_b + 0.5 * tol_b ** 2).sum(1) + gam * em_ref
    _within(section + " error", em, em_ref, tol_em, "error_metric vs oracle")
    if not any(c.get("robust") for c in P.spec["costs"]):
        # the error path (WITH_J = false) and the linearize path evaluate the same residuals: 0.5 |b|^2 of the kernel's own b, in float64
        _within(section + " error", em, 0.5 * (b ** 2).sum(1), 2 * tol_em, "error_metric vs 0.5 |b|^2")
    return A, b


KINDS = ["between_SE3", "local_SE3", "between_SO3", "local_SO3", "between_SE2", "local_SE2", "vector_1", "vector_2", "vector_3",
         "vector_6", "vector_7", "reproj"]
SHAPES = [(B, K) for B in (1, 5, 32, 33, 129) for K in (1, 7, 8, 9, 33)]
WEIGHTS = [("diag", False, False), ("scale", False, True), ("diag", True, True), ("scale", True, False)]   # (kind, weight [1,..], aux [1,..])


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("kind", KINDS)
def test_linearize_and_error_shapes(kind, dtype, oracle_eps):
    """Every (B, K) of SHAPES: one warp spans several cost functions when B < 32, K B is not a multiple of 32, the last error chunk is
    short when K % 8 != 0.  Weights and aux tensors alternate between per-item and broadcast [1, ...]; items 1 and 3 have zero weight."""
    oracle_eps(dtype)
    for s, (B, K) in enumerate(SHAPES):
        rng = np.random.default_rng(1000 * s + len(kind))
        wkind, w_b1, aux_b1 = WEIGHTS[s % len(WEIGHTS)]
        P = _make(kind, B, K, dtype, rng, wkind=wkind, w_b1=w_b1, aux_b1=aux_b1, zero=[q for q in (1, 3) if q < B])
        _check_problem(P, dtype, f"1 linearize {SFX[dtype]}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("robust", ["huber", "welsch"])
@pytest.mark.parametrize("kind", ["between_SE3", "local_SE3", "between_SO3", "local_SO3", "between_SE2", "local_SE2", "reproj"])
def test_robust_fused_kinds(kind, robust, dtype, oracle_eps):
    """The fused robust rescale: radii on both sides of |w e|^2, per item and broadcast."""
    oracle_eps(dtype)
    for s, (B, K) in enumerate([(5, 9), (33, 8), (1, 7)]):
        rng = np.random.default_rng(77 + s)
        P = _make(kind, B, K, dtype, rng, wkind=("diag", "scale")[s % 2], aux_b1=s == 1, robust=robust)
        _check_problem(P, dtype, f"1 robust {SFX[dtype]}")


def _branch_angles(group, dtype):
    """Relative rotation angles around every branch threshold of the dtype's table, at a relative margin of 5 % (far above the rounding
    of the angle the kernel recomputes: ~1e-7 relative in fp32, ~1e-15 in fp64): theta = 0 exactly, one margin below and above near_zero
    and d_near_zero, 1 + cos one margin inside and outside near_pi, theta = pi exactly, and one generic angle.  SE2 uses its own table
    and both signs."""
    m, npd = 0.05, NP[dtype]
    if group == "SE2":
        e = lie._EPS_TH[np.dtype(npd)]
        nz, dnz = e["se2_near_zero"], e["se2_d_near_zero"]
        a = [0.0, nz * (1 - m), nz * (1 + m), dnz * (1 - m), dnz * (1 + m), 1.0, np.pi - 0.1]
        return a + [-x for x in a[1:]]
    e = lie._EPS[np.dtype(npd)]
    nz, dnz, npi = e["near_zero"], e["d_near_zero"], e["near_pi"]
    return [0.0, nz * (1 - m), nz * (1 + m), dnz * (1 - m), dnz * (1 + m), 1.0, np.arccos(npi * (1 - m) - 1), np.arccos(npi * (1 + m) - 1),
            np.pi]


def _rel_elements(group, angles, rng, nonortho=0.0):
    """[B] relative elements with the given rotation angles.  Rotations by 0 and pi are the exact matrices I and diag(1, -1, -1);
    nonortho > 0 adds a symmetric traceless perturbation of that size to the rotation block (the reference never re-projects a rotation,
    so which part of a slightly non-orthogonal matrix the logarithm reads depends on the branch it takes)."""
    B = len(angles)
    ang = np.asarray(angles, np.float64)
    if group == "SE2":
        E = np.stack([rng.uniform(-1, 1, B), rng.uniform(-1, 1, B), np.cos(ang), np.sin(ang)], -1)
        E[ang == 0, 2:] = (1.0, 0.0)
        return E
    R = lie.so3_exp(_unit(rng, B) * ang[:, None])
    R[ang == 0] = np.eye(3)
    R[ang == np.pi] = np.diag([1.0, -1.0, -1.0])
    if nonortho:
        Sm = np.array([[1.0, 0.5, 0.0], [0.5, -1.0, 0.25], [0.0, 0.25, 0.0]])
        R = R + nonortho * Sm
    return R if group == "SO3" else np.concatenate([R, rng.uniform(-1, 1, (B, 3, 1))], -1)


def _branch_angles(group, dtype):
    """Relative rotation angles around every branch threshold of the dtype's table, at a relative margin of 5 % (far above the rounding
    of the angle the kernel recomputes: ~1e-7 relative in fp32, ~1e-15 in fp64): theta = 0 exactly, one margin below and above near_zero
    and d_near_zero, 1 + cos one margin inside and outside near_pi, theta = pi exactly, and one generic angle.  SE2 uses its own table,
    both signs, and theta = +-pi exactly."""
    m, npd = 0.05, np.dtype(NP[dtype])
    if group == "SE2":
        e = lie._EPS_TH[npd]
        nz, dnz = e["se2_near_zero"], e["se2_d_near_zero"]
        a = [nz * (1 - m), nz * (1 + m), dnz * (1 - m), dnz * (1 + m), 1.0, np.pi - 0.1, np.pi]
        return [0.0] + a + [-x for x in a]
    e = lie._EPS[npd]
    nz, dnz, npi = e["near_zero"], e["d_near_zero"], e["near_pi"]
    return [0.0, nz * (1 - m), nz * (1 + m), dnz * (1 - m), dnz * (1 + m), 1.0, np.arccos(npi * (1 - m) - 1), np.arccos(npi * (1 + m) - 1),
            np.pi]


def _rel_elements(group, angles, rng, nonortho=0.0):
    """[B] relative elements with the given rotation angles.  Rotations by 0 and pi are the exact matrices I and diag(1, -1, -1) (SE2:
    cos / sin exactly (1, 0) and (-1, +-0)).  nonortho > 0 adds a symmetric traceless perturbation of that size to the rotation block: the
    reference never re-projects a rotation, and which part of a slightly non-orthogonal matrix the logarithm reads (antisymmetric part,
    or the symmetric part in the near-pi branch) depends on the branch it takes."""
    B = len(angles)
    ang = np.asarray(angles, np.float64)
    if group == "SE2":
        E = np.stack([rng.uniform(-1, 1, B), rng.uniform(-1, 1, B), np.cos(ang), np.sin(ang)], -1)
        E[ang == 0, 2:] = (1.0, 0.0)
        E[np.abs(ang) == np.pi, 2] = -1.0
        E[np.abs(ang) == np.pi, 3] = np.copysign(0.0, ang[np.abs(ang) == np.pi])
        return E
    R = lie.so3_exp(_unit(rng, B) * ang[:, None])
    R[ang == 0] = np.eye(3)
    R[ang == np.pi] = np.diag([1.0, -1.0, -1.0])
    R = R + nonortho * np.array([[1.0, 0.5, 0.0], [0.5, -1.0, 0.25], [0.0, 0.25, 0.0]])
    return R if group == "SO3" else np.concatenate([R, rng.uniform(-1, 1, (B, 3, 1))], -1)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("kind", ["between_SE3", "local_SE3", "between_SO3", "local_SO3", "between_SE2", "local_SE2"])
def test_log_branch_thresholds(kind, dtype, oracle_eps):
    """Relative rotations on both sides of near_zero, d_near_zero and near_pi of the kernel dtype's table, over exact variables (signed
    permutations / quarter turns) so that the kernel's E = Z^-1 X0^-1 X1 is the placed element.  SE2 at theta = +-pi exactly: the
    reference's (1 + cos) theta / sin is 0 * inf there, and the kernel must give the same NaN entries, not a value of its own."""
    oracle_eps(dtype)
    group = kind.split("_")[1]
    angles = _branch_angles(group, dtype)
    for nonortho in ([0.0] if group == "SE2" else [0.0, 1e-4 if dtype == torch.float32 else 1e-6]):
        rng = np.random.default_rng(5)
        rels = _rel_elements(group, angles, rng, nonortho)
        P = _group_problem(kind, len(angles), 3, dtype, rng, rel=rels)
        _check_problem(P, dtype, f"1 branches {SFX[dtype]}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("kind", KINDS)
def test_zero_weight_masks_items_with_nan_aux(kind, dtype, oracle_eps):
    """A cost function whose weights are all zero for an item is masked (theseus cost_function.py: its rows are zero and it adds nothing
    to the error), whatever its aux tensors hold: items 1 and 4 have zero weight and NaN aux.  Every kind must give exactly-zero finite
    rows there, and the other items must be unaffected."""
    oracle_eps(dtype)
    B, K = 6, 9
    for s, wkind in enumerate(("diag", "scale")):
        P = _make(kind, B, K, dtype, np.random.default_rng(40 + s), wkind=wkind, zero=[1, 4], nan_items=[1, 4])
        A, b = _check_problem(P, dtype, f"1 masking {SFX[dtype]}")
        assert np.all(A[[1, 4]] == 0) and np.all(b[[1, 4]] == 0)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_large_batch_against_oracle(dtype, oracle_eps):
    """A few hundred thousand (cost, item) pairs in one launch: 129 SE3 Local cost functions at batch 2048."""
    oracle_eps(dtype)
    B = 64 if EMU else 2048
    P = _group_problem("local_SE3", B, 129, dtype, np.random.default_rng(9), wkind="diag", zero=[q for q in (7, 1000) if q < B])
    _check_problem(P, dtype, f"1 large {SFX[dtype]}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_items_at_scale_bitwise_equal_alone(dtype):
    """B ~ 2048 items x 600 SE3 Between cost functions: the A_val row, b and error of a few chosen items are bitwise those of the same
    item run alone (batch 1), which pins the item / cost indexing of every kernel at a scale a full oracle comparison would not reach."""
    B, K, N = (96, 600, 200) if EMU else (2048, 600, 200)
    rng = np.random.default_rng(11)
    X = [_elem("SE3", rng, B) for _ in range(N)]
    pairs = [(k % N, (k % N + 1 + k // N) % N) for k in range(K)]
    Z = [_elem("SE3", rng, B) for _ in range(K)]
    W = [rng.uniform(0.5, 2.0, (B, 6)) for _ in range(K)]

    def run(sel):
        P = _Problem(dtype)
        ids = [P.var(th.SE3, x[sel], "SE3", 6) for x in X]
        for k, (i, j) in enumerate(pairs):
            wt = th.DiagonalCostWeight(th.Variable(P.t(W[k][sel])))
            P.objective.add(th.Between(P.vars[ids[i]]["obj"], P.vars[ids[j]]["obj"], th.SE3(tensor=P.t(Z[k][sel]), disable_checks=True), wt))
        P.build()
        A, b = _linearize(P)
        return A, b, P.objective.error_metric().cpu().double().numpy()

    A, b, em = run(slice(None))
    assert np.isfinite(A).all() and np.isfinite(b).all()
    for q in ([0, 31, 32, 95] if EMU else [0, 31, 32, 1000, 2047]):
        a1, b1, e1 = run(slice(q, q + 1))
        assert np.array_equal(A[q], a1[0]) and np.array_equal(b[q], b1[0]) and np.array_equal(em[q], e1[0]), q


# ====================================================================================================================================
# 2. Gram kernels
# ------------------------------------------------------------------------------------------------------------------------------------
def _gram_structure(sizes, rng):
    """Every pair of variables shares one cost function (its off-diagonal block has ONE contribution, listed in either variable order),
    one pair shares five more (many contributions), and each variable has a cost function of its own; rows 1-7."""
    N = len(sizes)
    costs = []
    for i in range(N):
        for j in range(i + 1, N):
            costs.append((int(rng.integers(1, 8)), [i, j] if rng.random() < 0.5 else [j, i]))
    costs += [(int(rng.integers(1, 8)), [N - 1, 3]) for _ in range(5)]
    costs += [(int(rng.integers(1, 8)), [v]) for v in range(N)]
    return build_structure(sizes, costs)


def _run_gram(S, B, dtype, rng, out_offsets=None, out_size=None):
    np_dt = NP[dtype]
    arrs = build_gram_plan(S, out_offsets=out_offsets)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in arrs.items() if isinstance(v, np.ndarray)}
    plan = _lib.make_gram_plan(arrs, dev)
    A = rng.standard_normal((B, S.nnz)).astype(np_dt)
    bv = rng.standard_normal((B, S.num_rows)).astype(np_dt)
    n = S.num_cols
    size = n * n if out_offsets is None else out_size
    out = torch.full((B, size), float("nan"), dtype=dtype, device=DEV)
    Atb = torch.full((B, n), float("nan"), dtype=dtype, device=DEV)
    diag = torch.full((B, n), float("nan"), dtype=dtype, device=DEV)
    At, bt = torch.from_numpy(A).to(DEV), torch.from_numpy(bv).to(DEV)
    lib = _lib.load()
    _lib.check(getattr(lib, f"thb_gram_{SFX[dtype]}")(C.byref(plan), B, _lib.ptr(At), S.nnz, _lib.ptr(bt), S.num_rows, _lib.ptr(out), size,
                                                      _lib.ptr(Atb), _lib.ptr(diag), _lib.stream_ptr()), "gram")
    torch.cuda.synchronize()
    return arrs, A.astype(np.float64), bv.astype(np.float64), out.cpu().double().numpy(), Atb.cpu().double().numpy(), diag.cpu().double().numpy()


def _dense_of(S, A_val):
    B = A_val.shape[0]
    A = np.zeros((B, S.num_rows, S.num_cols))
    rows = np.repeat(np.arange(S.num_rows), np.diff(S.A_row_ptr))
    A[:, rows, S.A_col_ind] = A_val
    return A


def _gamma(k, u):
    return k * u / (1 - k * u)


def _dot_bound(k, dtype):
    """|fl(a^T b) - a^T b| <= gamma_k(u) |a|^T |b| for the kernel's k-term sum, plus the same bound at float64 for the reference's own
    evaluation (numpy einsum in float64: the comparison is between two rounded sums)."""
    return _gamma(k, U[dtype]) + _gamma(k, U[torch.float64])


def _check_gram_common(section, S, A_val, bv, Atb, diag, dtype):
    """Atb and diag against float64 A^T b / sum a^2 of the same A_val: |fl(a^T b) - a^T b| <= gamma_k |a|^T |b| with k the number of
    rows in the column (the kernel's sum has k products and k - 1 additions)."""
    A = _dense_of(S, A_val)
    k = (_dense_of(S, np.ones((1, S.nnz)))[0] != 0).sum(0)[None]
    _within(section, Atb, np.einsum("bri,br->bi", A, bv), _dot_bound(k, dtype) * np.einsum("bri,br->bi", np.abs(A), np.abs(bv)), "Atb")
    sq = np.einsum("bri,bri->bi", A, A)
    _within(section, diag, sq, _dot_bound(k, dtype) * sq, "diag")
    return A


GRAM_CASES = [([1, 2, 3, 6, 1, 2, 3, 6], 1), ([1, 2, 3, 6, 1, 2, 3, 6], 33), ([6, 6, 3, 6, 2], 5)]


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("sizes,B", GRAM_CASES)
def test_gram_blocks_dense_mirrored(sizes, B, dtype):
    """Variable sizes 1, 2, 3, 6 on both sides of every off-diagonal block: all 16 gram_block_kernel<DI, DJ> instances run, and the 6 x 6
    blocks take the split path (two threads per block, rows [0, 3) and [3, 6)).  Dense output: every pattern block and its mirror is
    written (the rest of the NaN-filled output stays NaN), the result is exactly symmetric, and within gamma_k |A|^T |A| of float64 A^T A
    (k = rows shared by the two columns).  diag equals the diagonal of A^T A within the same bound."""
    S = _gram_structure(sizes, np.random.default_rng(len(sizes) + B))
    arrs, A_val, bv, out, Atb, diag = _run_gram(S, B, dtype, np.random.default_rng(B))
    shapes = {(int(a), int(b)) for a, b in zip(arrs["blk_rows"], arrs["blk_cols"])}
    if len(sizes) == 8:
        assert shapes == {(a, b) for a in (1, 2, 3, 6) for b in (1, 2, 3, 6)} and len(arrs["segments"]) == 16
    n = S.num_cols
    out = out.reshape(B, n, n)
    A = _check_gram_common(f"2 gram {SFX[dtype]}", S, A_val, bv, Atb, diag, dtype)
    P = (np.abs(_dense_of(S, np.ones((1, S.nnz))))[0] > 0).astype(np.float64)
    pattern = (P.T @ P) > 0
    assert np.isfinite(out[:, pattern]).all() and np.isnan(out[:, ~pattern]).all()
    assert np.array_equal(out, np.swapaxes(out, 1, 2), equal_nan=True)
    k = (P.T @ P)[None]
    ata = np.einsum("bri,brj->bij", A, A)
    bound = _dot_bound(k, dtype) * np.einsum("bri,brj->bij", np.abs(A), np.abs(A))
    _within(f"2 gram {SFX[dtype]}", np.where(pattern, out, 0.0), ata, bound, "AtA")
    idx = np.arange(n)
    _within(f"2 gram {SFX[dtype]}", diag, out[:, idx, idx], 2 * bound[:, idx, idx], "diag vs diag(AtA)")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("sizes", [[1, 2, 3, 6, 1, 2, 3, 6], [2, 4, 1, 6, 3]])
def test_gram_factor_layout(sizes, dtype):
    """A non-mirrored block layout (one row-major block per lower pattern block, ld = its width, three NaN guard entries between blocks),
    read back block by block.  With a size-4 variable no block-per-thread kernel exists for some shapes, so every block goes through the
    entry-per-thread gram_kernel."""
    S = _gram_structure(sizes, np.random.default_rng(3))
    blocks, _ = lower_blocks(S)
    offs, pos = {}, 0
    for (i, j) in blocks:
        offs[(i, j)] = pos
        pos += int(S.var_dims[i]) * int(S.var_dims[j]) + 3
    B = 7
    arrs, A_val, bv, out, Atb, diag = _run_gram(S, B, dtype, np.random.default_rng(4), out_offsets=lambda i, j: (offs[(i, j)], int(S.var_dims[j]), -1),
                                                out_size=pos)
    assert (len(arrs["segments"]) == 0) == (4 in sizes)
    A = _check_gram_common(f"2 gram {SFX[dtype]}", S, A_val, bv, Atb, diag, dtype)
    P = (np.abs(_dense_of(S, np.ones((1, S.nnz))))[0] > 0).astype(np.float64)
    written = np.zeros(pos, bool)
    c0 = S.var_start_cols
    for (i, j) in blocks:
        di, dj = int(S.var_dims[i]), int(S.var_dims[j])
        o = offs[(i, j)]
        got = out[:, o:o + di * dj].reshape(B, di, dj)
        Ai, Aj = A[:, :, c0[i]:c0[i] + di], A[:, :, c0[j]:c0[j] + dj]
        k = (P[:, c0[i]:c0[i] + di].T @ P[:, c0[j]:c0[j] + dj])[None]
        _within(f"2 gram {SFX[dtype]}", got, np.einsum("bri,brj->bij", Ai, Aj),
                _dot_bound(k, dtype) * np.einsum("bri,brj->bij", np.abs(Ai), np.abs(Aj)), f"block {(i, j)}")
        written[o:o + di * dj] = True
    assert np.isfinite(out[:, written]).all() and np.isnan(out[:, ~written]).all()


# ====================================================================================================================================
# 3. lm_control
# ------------------------------------------------------------------------------------------------------------------------------------
ACCEPT, DOWN, UP = 0.25, 9.0, 11.0


def _lm_restated(delta, Atb, diag, step, ep, en, lam, ellipsoidal, dt):
    """lm_control_kernel in numpy: den = sum_j d (lam_e d + Atb) / 2 with d = delta step; rho = (err_prev - err_new) / den; reject iff
    rho <= accept (NaN accepts); lam *= up or /= down in the kernel's dtype, clamped to [1e-7, 1e7]; err_out = the error kept.  den is
    formed in float64: the cases below keep rho away from `accept` except where the data make every sum exact."""
    d = (delta * dt(step)).astype(np.float64)
    le = (lam[:, None] * diag).astype(np.float64) if ellipsoidal else lam.astype(np.float64)[:, None]
    den = (d * (le * d + Atb.astype(np.float64))).sum(1) / 2
    with np.errstate(divide="ignore", invalid="ignore"):
        rho = (ep.astype(np.float64) - en.astype(np.float64)) / den
    rej = rho <= ACCEPT
    nl = np.where(rej, lam * dt(UP), lam / dt(DOWN)).astype(dt)
    nl = np.where(nl < dt(1e-7), dt(1e-7), np.where(nl > dt(1e7), dt(1e7), nl)).astype(dt)
    return nl, rej, np.where(rej, ep, en).astype(dt), den


LM_SIZES = [(n, B) for n in (1, 6, 255, 256, 257, 15000) for B in (1, 33, 2048) if not (EMU and B * max(n, 256) > 33 * 15000)]


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("ellipsoidal", [1, 0])
@pytest.mark.parametrize("n,B", LM_SIZES)
def test_lm_control(n, B, ellipsoidal, dtype):
    """Items cycle through: a clear accept / reject (rho placed away from `accept`); delta = 0 (den = 0: rho = +inf, -inf or NaN); equal
    errors (rho = 0: reject); rho exactly equal to `accept` from power-of-two data (every sum exact: the tie must reject); lam driven into
    the 1e-7 and 1e7 clamps.  lam, reject and err_out must be bitwise those of the restatement, stats[0] the number of rejects."""
    dt, rng, step = NP[dtype], np.random.default_rng(n + B), 0.5
    delta = rng.standard_normal((B, n)).astype(dt)
    Atb = (np.abs(rng.standard_normal((B, n))) * np.sign(delta)).astype(dt)      # every term of den positive: den well conditioned
    diag = rng.uniform(0.5, 2.0, (B, n)).astype(dt)
    lam = (10.0 ** rng.uniform(-3, 3, B)).astype(dt)
    ep = rng.uniform(1.0, 10.0, B).astype(dt)
    en = np.zeros(B, dt)
    cat = np.arange(B) % 7
    for b in range(B):
        c = cat[b]
        if c == 1:                                  # delta = 0
            delta[b] = 0
            en[b] = ep[b] * dt((0.5, 2.0, 1.0)[b % 3])
        elif c == 3:                                # exact tie: d = 0.5, lam_e d + Atb = 1.25, den = n 0.3125, err_prev - err_new = accept den
            delta[b], Atb[b], diag[b], lam[b] = 1.0, 1.0, 1.0, 0.5
            en[b] = 1.0
            ep[b] = dt(1.0 + ACCEPT * n * 0.3125)
    _, _, _, den = _lm_restated(delta, Atb, diag, step, ep, ep, lam, ellipsoidal, dt)
    for b in range(B):
        c = cat[b]
        if c in (0, 4, 5, 6):                       # rho well away from accept; 5 / 6 push lam into the clamps
            rho_t = {0: (-0.5, 0.05, 0.6, 3.0)[b % 4], 4: 0.9, 5: 0.9, 6: 0.01}[c]
            if c == 5:
                lam[b] = dt(5e-7)
            if c == 6:
                lam[b] = dt(5e6)
            _, _, _, den_b = _lm_restated(delta[b:b + 1], Atb[b:b + 1], diag[b:b + 1], step, ep[b:b + 1], ep[b:b + 1], lam[b:b + 1], ellipsoidal, dt)
            en[b] = dt(ep[b] - rho_t * den_b[0])
        elif c == 2:                                # equal errors
            en[b] = ep[b]
    want_l, want_r, want_e, _ = _lm_restated(delta, Atb, diag, step, ep, en, lam, ellipsoidal, dt)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    d_delta, d_atb, d_diag, d_ep, d_en, d_lam = T(delta), T(Atb), T(diag), T(ep), T(en), T(lam.copy())
    reject = torch.full((B,), 7, dtype=torch.uint8, device=DEV)
    err_out = torch.full((B,), float("nan"), dtype=dtype, device=DEV)
    stats = torch.full((4,), -1, dtype=torch.int32, device=DEV)
    lib = _lib.load()
    _lib.check(getattr(lib, f"thb_lm_control_{SFX[dtype]}")(_lib.ptr(d_delta), _lib.ptr(d_atb), _lib.ptr(d_diag), B, n, step, _lib.ptr(d_ep),
                                                           _lib.ptr(d_en), _lib.ptr(d_lam), ellipsoidal, ACCEPT, DOWN, UP, _lib.ptr(reject),
                                                           _lib.ptr(err_out), _lib.ptr(stats), _lib.stream_ptr()), "lm_control")
    torch.cuda.synchronize()
    if B > 3:
        assert want_r[cat == 3].all() and want_r[cat == 2].all() and (want_l[cat == 5] == dt(1e-7)).all() and (want_l[cat == 6] == dt(1e7)).all()
    assert np.array_equal(reject.cpu().numpy(), want_r.astype(np.uint8))
    assert np.array_equal(d_lam.cpu().numpy(), want_l)
    assert np.array_equal(err_out.cpu().numpy(), want_e)
    assert int(stats[0]) == int(want_r.sum())


# ====================================================================================================================================
# 4. retract / commit
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("B", [1, 37])
def test_retract_and_commit(B, dtype, oracle_eps):
    """X <- X exp(step delta) on SE3, SO3, SE2, SO2 and Vector variables with step != 1, tangent steps on both sides of the exp near-zero
    branch, and an ignore mask; then commit with a different keep_old mask.  Retracted values are within C u (1 + |X| + |xi|) of
    lie.*_retract at xi = fl(step delta) (the exp is a few dozen operations on entries bounded by |xi|, composed with entries bounded by
    |X|); ignored and kept items are bitwise unchanged and committed items bitwise equal to the retracted ones."""
    oracle_eps(dtype)
    rng = np.random.default_rng(B)
    dt = NP[dtype]
    P = _Problem(dtype)
    specs = [("SE3", th.SE3, _elem("SE3", rng, B), 6), ("SO3", th.SO3, _elem("SO3", rng, B), 3), ("SE2", th.SE2, _elem("SE2", rng, B), 3)]
    a = rng.uniform(-np.pi, np.pi, B)
    specs += [("SO2", th.SO2, np.stack([np.cos(a), np.sin(a)], -1), 1), ("Vector", th.Vector, rng.uniform(-3, 3, (B, 4)), 4)]
    for kind, cls, val, dof in specs:
        i = P.var(cls, val, kind, dof)
        v = P.vars[i]["obj"]
        P.objective.add(th.Difference(v, cls(tensor=P.t(val), disable_checks=True) if cls is not th.Vector else th.Vector(tensor=P.t(val)),
                                      th.ScaleCostWeight(th.Variable(P.t(np.ones((1, 1)))))))
    P.objective.to(DEV)
    eng = P.objective.engine()
    eng.adopt_optim_vars()
    n = eng.n
    delta = rng.standard_normal((B, n)) * 0.8
    delta[::2] *= 1e-3                                   # small tangent steps: the near-zero branches of so3 / se3 / se2 exp
    delta = delta.astype(dt)
    step = 0.7
    ignore = np.zeros(B, bool)
    ignore[1::3] = True
    before = [v.tensor.cpu().numpy().copy() for v in eng.ordering]
    outs = [v.copy() for v in eng.ordering]
    eng.retract_into(torch.from_numpy(delta).to(DEV), outs, step, torch.from_numpy(ignore).to(DEV))
    got = [t.cpu().numpy().copy() for t in eng.tmp_views]
    xi = (delta * dt(step)).astype(np.float64)
    S = eng.structure
    for q, v in enumerate(eng.ordering):
        kind = type(v).__name__ if type(v).__name__ in ("SE3", "SO3", "SE2", "SO2") else "Vector"
        X = before[q].astype(np.float64)
        d = xi[:, S.var_start_cols[q]:S.var_start_cols[q] + S.var_dims[q]]
        ref = dict(SE3=lie.se3_retract, SO3=lie.so3_retract, SE2=lie.se2_retract, SO2=lie.so2_retract).get(kind, lambda x, dd: x + dd)(X, d)
        mag = 1 + np.abs(X).reshape(B, -1).max(1) + np.abs(d).max(1)
        tol = 32 * U[dtype] * mag.reshape((B,) + (1,) * (X.ndim - 1))
        _within(f"4 retract {SFX[dtype]}", got[q][~ignore], ref[~ignore], tol[~ignore], f"retract {kind}")
        assert np.array_equal(got[q][ignore], before[q][ignore]), kind
    keep = np.zeros(B, bool)
    keep[::2] = True
    eng.commit(torch.from_numpy(keep).to(DEV))
    for q, v in enumerate(eng.ordering):
        now = v.tensor.cpu().numpy()
        assert np.array_equal(now[keep], before[q][keep]) and np.array_equal(now[~keep], got[q][~keep]), type(v).__name__
