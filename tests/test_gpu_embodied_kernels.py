"""The fused motion-planning and planar-pushing kernels (linearize_kernel / error_kernel over MpCost: Collision2D on Point2 / SE2,
DoubleIntegrator on Vector (D = 1, 2, 3) / SE2 with Scale, Diagonal or GP weights, HingeCost (D = 1, 2, 3), Nonholonomic on SE2 / Vector,
QuasiStaticPushingPlanar, EffectorObjectContactPlanar) compared entry by entry with the float64 restatement of oracle/embodied.py, through
the public API (th.eb.*) and the engine's linearize_sparse / error_metric:
  - every kind at the (B, K) where the warp-staged A_val store and the 8-cost error chunks change shape, over variables shared in chains
    so that the block pointers, A_val offsets and first rows differ per cost function;
  - an objective mixing the kinds over shared variables; zero-weight items whose inputs are NaN;
  - GP weights at D = 1, 2, 3 and dt from 0.01 to 2, a weight dt different from the cost's dt, symmetric and non-symmetric Qc_inv;
  - both sides of every switch, placed exactly: grid nodes, cell lines, the last row and column and just outside each side of the grid,
    dist == eps (Collision2D) and dist == radius (EffectorObjectContactPlanar) on a dyadic grid, crossing and infinite hinge limits,
    relative angles across +-pi with p = 0 and c^2 = 0, DoubleIntegrator-SE2 relative angles around the SE2 log's branch thresholds.
fp32 kernels are compared with the oracle evaluated in float64 on the fp32-rounded inputs, with the switch decisions (SDF cell and
out-of-grid test, dist > eps, dist < radius, the hinge tests, the +-pi wrap) taken in float32 as the kernel takes them (spec
"switch_dtype") and the float32 SE2 branch tables (fixture oracle_eps).  Bounds are componentwise, C u kappa scale per row of each cost
function (see _kappa_scale / _weight_rows).  Dry run on the CPU:  THB_SIMT_EMULATION=1 python -m pytest tests/test_gpu_embodied_kernels.py -m gpu"""
import numpy as np
import pytest
import torch

import test_gpu_cost_kernels as tgc
import theseus_b200 as th
from oracle import embodied, lie, nls
from test_gpu_cost_kernels import DTYPES, EMU, NP, SFX, U, _elem, _linearize, _Problem, _within, oracle_eps  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for k in sorted(k for k in tgc.RATIOS if k.startswith("mp ")):
        print(f"max error/bound {k}: {tgc.RATIOS[k]:.3g}")


# ====================================================================================================================================
# bounds
# ------------------------------------------------------------------------------------------------------------------------------------
# Every entry is a short chain (<= ~30 operations) of products and sums whose terms are bounded by the per-kind scale below; C covers
# gamma_k of that chain.
C_MP = 64


def _se2_kappa(D):
    """The SE2 log / jlog of DoubleIntegrator-SE2's local(pose1, pose2): above d_near_zero its 0.5 sin / (1 - cos) coefficient has lost
    2 / theta^2 to cancellation and multiplies a 1/theta term (2 / |theta|^3); (1 + cos) theta / sin grows like theta / sin (as in
    tests/test_gpu_cost_kernels._kappa)."""
    theta, sine = np.abs(np.arctan2(D[:, 3], D[:, 2])), np.abs(D[:, 3])
    with np.errstate(divide="ignore", invalid="ignore"):
        cancel = np.where(theta >= lie._EPS_TH[np.dtype(np.float64)]["se2_d_near_zero"], 2 / theta ** 3, 0.0)
        k = (1 + cancel) * np.where(theta < 1.0, 1.0, 6 * theta / sine)
    return np.where(np.isfinite(k), k, 1.0)


def _kappa_scale(spec, c, B):
    """kappa * scale of one cost function's unweighted error ([B]) and of each column of its Jacobian blocks ([B, dof] per variable,
    in the cost function's variable order).
    - Collision2D / EOC: the point's cell coordinate (p - origin) / cell carries an absolute error of u (|p - origin| / cell + 2) cells
      (EOC: + (|t_eff| + |t_obj|) / cell from the rotation into the object frame); it moves the interpolation weights, so the distance
      is off by that many cells times the grid values' magnitude G, and the gradient columns by G / cell times as much (the 1 / cell of
      the gradient).  EOC's object theta column is the gradient times p: |p| more.  SE2 Collision2D's and EOC's effector theta columns
      are exactly zero.  Every other kind uses one scale for its error and all its columns:
    - DoubleIntegrator: the terms |p1| + |p2| + (1 + dt)(1 + |v1| + |v2|); SE2: times the log's conditioning (_se2_kappa).
    - Hinge: |x| + |down| + |up| + |threshold| (finite parts): e = (down + thr) - x cancels.
    - Nonholonomic: |v0| + |v1|, times 1 + |theta| for the rounding of sin / cos of the Vector pose's angle.
    - QSP: the products of p, v and w: (1 + |p|)(1 + |v| + |vp|)(1 + pi) + c^2 (1 + pi), with |p| <= |t_e2| + |t_o2| etc. (the
      differences of positions cancel)."""
    x = [np.asarray(spec["_values"][i], np.float64) for i in c["vars"]]
    aux = {k: embodied._b(v, B) for k, v in c.get("aux", {}).items()}
    k = c["kind"]
    n1 = lambda a: np.abs(np.nan_to_num(a, posinf=0.0, neginf=0.0)).reshape(B, -1).sum(1)
    if k in ("collision", "eoc"):
        cell, o = aux["cell"].reshape(B), aux["origin"]
        G = np.abs(aux["sdf"]).reshape(B, -1).max(1)
        if k == "collision":
            p, extra, lim = x[0][:, :2], 0.0, aux["eps"]
        else:
            ob, ef = x
            d = ef[:, :2] - ob[:, :2]
            p = np.stack([ob[:, 2] * d[:, 0] + ob[:, 3] * d[:, 1], -ob[:, 3] * d[:, 0] + ob[:, 2] * d[:, 1]], 1)
            extra, lim = (n1(ef[:, :2]) + n1(ob[:, :2])) / cell, aux["radius"]
        pc = n1(p - o) / cell + extra + 2
        sg, z = G * (1 + pc) / cell, np.zeros(B)
        if k == "collision":
            cols = [np.stack([sg, sg] + ([z] if x[0].shape[1] == 4 else []), 1)]
        else:
            cols = [np.stack([sg, sg, sg * (1 + n1(p))], 1), np.stack([sg, sg, z], 1)]
        return G * (1 + pc) + n1(lim), cols
    s = _kappa_scale_one(spec, c, x, aux, B, n1)
    return s, [np.broadcast_to(s[:, None], (B, v.shape[1] if v.shape[1] != 4 else 3)) for v in x]


def _kappa_scale_one(spec, c, x, aux, B, n1):
    k = c["kind"]
    if k == "double_integrator":
        p1, v1, p2, v2 = x
        dt = aux["dt"].reshape(B)
        se2 = spec["vars"][c["vars"][0]]["kind"] == "SE2"
        s = (n1(p1[:, :2]) + n1(p2[:, :2]) if se2 else n1(p1) + n1(p2)) + (1 + dt) * (1 + n1(v1) + n1(v2))
        return s * (_se2_kappa(lie.se2_compose(lie.se2_inverse(p1), p2)) if se2 else 1.0)
    if k == "hinge":
        return 1 + n1(x[0]) + n1(aux["down"]) + n1(aux["up"]) + n1(aux["threshold"])
    if k == "nonholonomic":
        pose, vel = x
        return 1 + (np.abs(vel[:, 0]) + np.abs(vel[:, 1])) * (1 + (0 if pose.shape[1] == 4 else np.abs(pose[:, 2])))
    if k == "qsp":
        o1, o2, e1, e2 = x
        xy = lambda T: n1(T[:, :2])
        c2 = np.abs(aux["c_square"].reshape(B))
        return (1 + xy(e2) + xy(o2)) * (1 + xy(o2) + xy(o1) + xy(e2) + xy(e1)) * (1 + np.pi) + c2 * (1 + np.pi)
    raise NotImplementedError(k)


def _weight_rows(weight, B, d):
    """[B, d] magnitude of each weighted row's weight.  Scale / Diagonal: |w| (exact products).  GP: max_j |W_rj| times 4 cond(Q): the
    factor's last block c = sqrt(4/dt - (6/dt^2)^2 / (12/dt^3)) = sqrt(1/dt) cancels by a factor of about 4, and the Cholesky of the
    2D x 2D matrix carries Q's conditioning into the entries of W."""
    kind, w = weight[0], weight[1]
    w = embodied._b(w, B)
    if kind == "scale":
        return np.broadcast_to(np.abs(w.reshape(B, 1)), (B, d))
    if kind == "diag":
        return np.abs(w)
    W = embodied.gp_weight(w, embodied._b(weight[2], B))
    Qs = np.triu(w) + np.swapaxes(np.triu(w, 1), 1, 2)
    return np.abs(W).max(2) * 4 * np.linalg.cond(Qs)[:, None]


def _tols(P, dtype, st):
    """Componentwise bounds (tol_A [B, nnz], tol_b [B, m]) in the layout of the oracle's sparse structure `st`: C u times the weighted
    row's weight magnitude times the unweighted error's / column's kappa * scale."""
    B = P.ovalues[0].shape[0]
    spec = dict(P.spec, _values=P.ovalues)
    tol_A, tol_b = np.zeros((B, len(st["A_col_ind"]))), []
    for f, c in enumerate(P.spec["costs"]):
        d = nls.cost_dim(P.spec, c)
        wr = C_MP * U[dtype] * _weight_rows(c["weight"], B, d)
        s_e, cols = _kappa_scale(spec, c, B)
        tol_b.append(wr * s_e[:, None])
        blk = tol_A[:, st["row_block_starts"][f]:st["row_block_starts"][f] + d * st["stride"][f]].reshape(B, d, st["stride"][f])
        for q, sc in enumerate(cols):
            bp = st["block_pointers"][f][q]
            blk[:, :, bp:bp + sc.shape[1]] = wr[:, :, None] * sc[:, None, :]
    return tol_A, np.concatenate(tol_b, 1)


def _check(P, dtype, section):
    """A_val, b and error_metric of the engine against the oracle (NaN-guarded: an entry the kernel does not write, or a store past the
    end, fails)."""
    P.spec["switch_dtype"] = NP[dtype] if dtype == torch.float32 else None
    S, ref_struct = P.eng.structure, nls.sparse_structure(P.spec)
    assert np.array_equal(S.A_row_ptr, ref_struct["A_row_ptr"]) and np.array_equal(S.A_col_ind, ref_struct["A_col_ind"])
    A, b = _linearize(P)
    A_ref, b_ref = nls.linearize_sparse(P.spec, P.ovalues, ref_struct)
    tol_A, tol_b = _tols(P, dtype, ref_struct)
    _within(section, A, A_ref, tol_A, "A_val")
    _within(section, b, b_ref, tol_b, "b")
    em = P.objective.error_metric().cpu().double().numpy()
    em_ref = nls.error_metric(P.spec, P.ovalues)
    gam = (b.shape[1] + 2) * U[dtype]
    tol_em = (np.abs(b_ref) * tol_b + 0.5 * tol_b ** 2).sum(1) + gam * em_ref
    _within(section + " error", em, em_ref, tol_em, "error_metric vs oracle")
    _within(section + " error", em, 0.5 * (b ** 2).sum(1), 2 * tol_em, "error_metric vs 0.5 |b|^2")
    return A, b


# ====================================================================================================================================
# problems
# ------------------------------------------------------------------------------------------------------------------------------------
ROWS, COLS = 12, 16
NPOOL = 5      # variables per pool (prime: the slots (k + j step) % NPOOL of one cost function are distinct for step in 1..4)
KINDS = ["coll_point2", "coll_se2", "di_vec1", "di_vec2", "di_vec3", "di_se2", "hinge1", "hinge2", "hinge3", "nh_se2", "nh_vec", "qsp", "eoc"]
SLOTS = {   # kind -> pool of each optimisation variable (pose1, vel1, pose2, vel2 of a DoubleIntegrator: pools "p" and "v")
    "coll": "p", "di": "pvpv", "hinge": "v", "nh": "pv", "qsp": "pppp", "eoc": "pp"}


def _family(kind):
    return kind.split("_")[0].rstrip("0123456789")


def _dof(kind):
    if kind.startswith(("di_vec", "hinge")):
        return int(kind[-1])
    return 2 if kind == "coll_point2" else 3


def _grid(P, rng, Bs):
    """Dyadic SDF grids (exact in both dtypes): a cone around the middle plus noise, multiples of 1/256 in about [-1, 1]; cell 1/8 or
    1/16, origin a multiple of 1/16."""
    yy, xx = np.meshgrid(np.arange(ROWS), np.arange(COLS), indexing="ij")
    base = np.sqrt((xx - 7.5) ** 2 + (yy - 5.5) ** 2) / 6.0 - 0.5
    sdf = np.round((base[None] + 0.2 * rng.standard_normal((Bs, ROWS, COLS))) * 256) / 256
    cell = rng.choice([0.125, 0.0625], (Bs, 1))
    origin = rng.integers(-24, 8, (Bs, 2)) / 16.0
    return sdf, origin, cell


class _Builder:
    """K cost functions of one kind over pools of NPOOL variables; cost function k takes slot j of a pool from variable
    (k + j step_k) % NPOOL, step_k = 1 + k % 4, so consecutive cost functions share variables and list them in different column orders."""

    def __init__(self, kind, B, dtype, rng, wkind="diag", w_b1=False, aux_b1=False, zero=(), nan_items=(), gp=None, problem=None):
        """problem: an existing _Problem to add the cost functions to (several kinds in one objective), else a new one."""
        self.kind, self.fam, self.D = kind, _family(kind), _dof(kind)
        self.B, self.rng, self.wkind, self.w_b1, self.aux_b1, self.zero, self.gp = B, rng, wkind, w_b1, aux_b1, zero, gp
        self.P = problem if problem is not None else _Problem(dtype)
        self.P.nan_items = nan_items
        self.pools = {}

    def pool(self, name, make):
        if name not in self.pools:
            self.pools[name] = [make() for _ in range(NPOOL)]
        return self.pools[name]

    def new_var(self, what, value=None):
        P, B, rng = self.P, self.B, self.rng
        if what == "se2":
            return P.var(th.SE2, _elem("SE2", rng, B) if value is None else value, "SE2", 3)
        cls = {1: th.Vector, 2: th.Point2, 3: th.Point3}[value.shape[1] if value is not None else self.D]
        v = rng.uniform(-2, 2, (B, self.D)) if value is None else value
        return P.var(cls, v, "Vector", v.shape[1])

    def obj(self, i):
        return self.P.vars[i]["obj"]

    def weight(self, dim):
        if self.gp is not None:
            return self.gp(self)
        return self.P.weight(self.wkind, 1 if self.w_b1 else self.B, dim, self.rng, zero=() if self.w_b1 else self.zero)

    def aux(self, a):
        return self.P.at(self.P.r(a))

    def ab(self):
        return 1 if self.aux_b1 else self.B

    def add(self, k, ids=None, **kw):
        """Cost function k (ids: its variables, or the chain choice of the class docstring); kw: aux values (defaults at random)."""
        P, rng, fam, Ba = self.P, self.rng, self.fam, self.ab()
        if ids is None:
            step = 1 + k % 4
            se2 = self.kind in ("coll_se2", "di_se2", "nh_se2", "qsp", "eoc")
            mk = {"p": (lambda: self.new_var("se2")) if se2 else (lambda: self.new_var("vec", rng.uniform(-2, 2, (self.B, 3)) if fam == "nh" else None)),
                  "v": (lambda: self.new_var("vec", rng.uniform(-2, 2, (self.B, 3)) if fam == "nh" else None))}
            used = {}
            ids = []
            for s in SLOTS[fam]:
                j = used.get(s, 0)
                used[s] = j + 1
                ids.append(self.pool(s, mk[s])[(k + j * step) % NPOOL])
        o = [self.obj(i) for i in ids]
        if fam in ("coll", "eoc"):
            sdf, origin, cell = kw.get("grid") or _grid(P, rng, Ba)
            sdf, origin, cell = P.r(sdf), P.r(origin), P.r(cell)
            lim = P.r(kw["lim"] if "lim" in kw else (rng.uniform(0.2, 0.8, (Ba, 1)) if fam == "coll" else rng.uniform(0.02, 0.5, (Ba, 1))))
            wt, ws = self.weight(1)
            if fam == "coll":
                cf = th.eb.Collision2D(o[0], self.aux(origin), self.aux(sdf), th.Variable(self.aux(cell)), th.Variable(self.aux(lim)), wt)
                aux = dict(origin=origin, sdf=sdf, cell=cell, eps=lim)
            else:
                cf = th.eb.EffectorObjectContactPlanar(o[0], o[1], self.aux(origin), self.aux(sdf), th.Variable(self.aux(cell)), self.aux(lim), wt)
                aux = dict(origin=origin, sdf=sdf, cell=cell, radius=lim)
            P.add(cf, dict(kind="collision" if fam == "coll" else "eoc", vars=tuple(ids), aux=aux, weight=ws))
        elif fam == "di":
            dt = P.r(kw["dt"] if "dt" in kw else rng.uniform(0.05, 1.0, (Ba, 1)))
            wt, ws = self.weight(2 * self.D)
            cls = th.eb.GPMotionModel if ws[0] == "gp" else th.eb.DoubleIntegrator
            P.add(cls(o[0], o[1], o[2], o[3], th.Variable(self.aux(dt)), wt), dict(kind="double_integrator", vars=tuple(ids), aux=dict(dt=dt), weight=ws))
        elif fam == "hinge":
            D = self.D
            down = P.r(kw["down"] if "down" in kw else rng.uniform(-1.5, 0.0, (Ba, D)))
            up = P.r(kw["up"] if "up" in kw else rng.uniform(0.0, 1.5, (Ba, D)))
            thr = P.r(kw["thr"] if "thr" in kw else rng.uniform(0.0, 0.4, (Ba, D)))
            if "down" not in kw:
                down[rng.random((Ba, D)) < 0.15] = -np.inf
                up[rng.random((Ba, D)) < 0.15] = np.inf
            wt, ws = self.weight(D)
            # (the constructor checks down <= up, so only the threshold of a masked item can be NaN)
            cf = th.eb.HingeCost(o[0], th.Variable(P.t(down)), th.Variable(P.t(up)), th.Variable(self.aux(thr)), wt)
            P.add(cf, dict(kind="hinge", vars=tuple(ids), aux=dict(down=down, up=up, threshold=thr), weight=ws))
        elif fam == "nh":
            wt, ws = self.weight(1)
            P.add(th.eb.Nonholonomic(o[0], o[1], wt), dict(kind="nonholonomic", vars=tuple(ids), weight=ws))
        elif fam == "qsp":
            c2 = P.r(kw["c2"] if "c2" in kw else rng.uniform(0.1, 1.0, (Ba, 1)))
            wt, ws = self.weight(3)
            P.add(th.eb.QuasiStaticPushingPlanar(o[0], o[1], o[2], o[3], th.Variable(self.aux(c2)), wt),
                  dict(kind="qsp", vars=tuple(ids), aux=dict(c_square=c2), weight=ws))
        else:
            raise NotImplementedError(self.kind)
        return ids

    def build(self):
        return self.P.build()


def _gp_weight(Q, dt):
    """A GP weight over fixed Qc_inv [Bq, D, D] and dt [Bd, 1]."""
    def make(bld):
        Qr, dtr = bld.P.r(Q), bld.P.r(dt)
        return th.eb.GPCostWeight(bld.P.t(Qr), th.Variable(bld.P.t(dtr))), ("gp", Qr, dtr)
    return make


def _spd(rng, Bq, D):
    A = rng.standard_normal((Bq, D, D))
    return A @ np.swapaxes(A, 1, 2) + 0.5 * np.eye(D)


def _random_gp(rng, D, per_item, B):
    Bq = B if per_item else 1
    return _gp_weight(_spd(rng, Bq, D), rng.uniform(0.05, 1.5, (Bq, 1)))


# ====================================================================================================================================
# tests
# ------------------------------------------------------------------------------------------------------------------------------------
SHAPES = [(B, K) for B in (1, 5, 32, 33, 129) for K in (1, 7, 8, 9, 33)]
if EMU:
    SHAPES = [(B, K) for B in (1, 5, 33) for K in (1, 8, 9)]
WEIGHTS = [("diag", False, False), ("scale", False, True), ("diag", True, True), ("scale", True, False)]   # (kind, weight [1,..], aux [1,..])


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("kind", KINDS)
def test_linearize_and_error_shapes(kind, dtype, oracle_eps):
    """Every (B, K) of SHAPES: one warp spans several cost functions when B < 32, K B is not a multiple of 32, the last error chunk is
    short when K % 8 != 0.  Weights and aux tensors alternate between per-item and broadcast [1, ...]; items 1 and 3 have zero weight;
    DoubleIntegrators take a GP weight on every third shape."""
    oracle_eps(dtype)
    for s, (B, K) in enumerate(SHAPES):
        rng = np.random.default_rng(3000 * s + len(kind))
        wkind, w_b1, aux_b1 = WEIGHTS[s % len(WEIGHTS)]
        gp = _random_gp(rng, _dof(kind), s % 2 == 0, B) if kind.startswith("di") and s % 3 == 0 else None
        bld = _Builder(kind, B, dtype, rng, wkind, w_b1, aux_b1, zero=[q for q in (1, 3) if q < B], gp=gp)
        for k in range(K):
            bld.add(k)
        _check(bld.build(), dtype, f"mp shapes {SFX[dtype]}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_mixed_objective(dtype, oracle_eps):
    """DoubleIntegrator-SE2 (GP), Collision2D-SE2, HingeCost on the velocities and Nonholonomic-SE2 over shared SE2 poses and velocity
    vectors, added in interleaved order: the groups' row blocks alternate and their column blocks interleave."""
    oracle_eps(dtype)
    for B in (5, 33):
        rng = np.random.default_rng(B)
        P = _Problem(dtype)
        T = 6
        poses = [P.var(th.SE2, _elem("SE2", rng, B), "SE2", 3) for _ in range(T)]
        vels = [P.var(th.Point3, rng.uniform(-2, 2, (B, 3)), "Vector", 3) for _ in range(T)]
        parts = {}
        for kind in ("di_se2", "coll_se2", "hinge3", "nh_se2"):
            parts[kind] = _Builder(kind, B, dtype, rng, "scale" if kind != "hinge3" else "diag",
                                   gp=_random_gp(rng, 3, True, B) if kind == "di_se2" else None, problem=P)
        for t in range(T - 1):
            parts["nh_se2"].add(t, ids=[poses[t + 1], vels[t + 1]])
            parts["di_se2"].add(t, ids=[poses[t], vels[t], poses[t + 1], vels[t + 1]])
            parts["coll_se2"].add(t, ids=[poses[T - 1 - t]])
            parts["hinge3"].add(t, ids=[vels[(3 * t) % T]])
        _check(P.build(), dtype, f"mp mixed {SFX[dtype]}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("kind", KINDS)
def test_zero_weight_masks_items_with_nan_inputs(kind, dtype, oracle_eps):
    """Items 1 and 4 have all-zero weights and NaN aux tensors (grids, origins, limits, dt, c^2): the kernel must not read them, their
    rows are exactly zero and finite, and the other items are unaffected."""
    oracle_eps(dtype)
    B, K = 6, 9
    for s, wkind in enumerate(("diag", "scale")):
        bld = _Builder(kind, B, dtype, np.random.default_rng(60 + s), wkind, zero=[1, 4], nan_items=[1, 4])
        for k in range(K):
            bld.add(k)
        P = bld.build()
        if kind not in ("nh_se2", "nh_vec"):
            assert any(torch.isnan(v.tensor).any() for cf in P.objective.cost_functions.values() for v in cf.aux_vars)
        A, b = _check(P, dtype, f"mp masking {SFX[dtype]}")
        assert np.all(A[[1, 4]] == 0) and np.all(b[[1, 4]] == 0)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("kind", ["di_vec1", "di_vec2", "di_vec3", "di_se2"])
def test_gp_weights(kind, dtype, oracle_eps):
    """GPMotionModel at dt from 0.01 to 2, with the weight's dt different from the cost function's dt (the kernel must read each from its
    own aux slot), symmetric positive definite Qc_inv per item and broadcast."""
    oracle_eps(dtype)
    D = _dof(kind)
    for s, (dt_w, dt_c) in enumerate([(0.01, 0.013), (0.1, 0.25), (0.7, 0.3), (2.0, 1.1)]):
        rng = np.random.default_rng(90 + s)
        B = 33
        per_item = s % 2 == 1
        Bq = B if per_item else 1
        dtw = np.full((Bq, 1), dt_w) * (rng.uniform(0.9, 1.1, (Bq, 1)) if per_item else 1.0)
        bld = _Builder(kind, B, dtype, rng, gp=_gp_weight(_spd(rng, Bq, D), dtw))
        for k in range(9):
            bld.add(k, dt=np.full((1, 1), dt_c))
        _check(bld.build(), dtype, f"mp gp {SFX[dtype]}")


def _nonsymmetric_qc_inv(rng, Bq, D):
    """Qc_inv = SPD + a non-symmetric part that the reference accepts and can weight with: cholesky(Qc_inv) (its constructor's check,
    which reads the lower triangle) and the factor of the 2D x 2D matrix (which needs Qu - 3/4 Q Qu^-1 Q^T > 0, Qu the symmetric matrix
    of Q's upper triangle) both exist."""
    Q = _spd(rng, Bq, D) + 0.3 * rng.uniform(-1, 1, (Bq, D, D)) * (1 - np.eye(D))
    for b in range(Bq):
        while True:
            try:
                np.linalg.cholesky(np.tril(Q[b]) + np.tril(Q[b], -1).T)
                embodied.gp_weight(Q[b:b + 1], np.ones((1, 1)))
                break
            except np.linalg.LinAlgError:
                Q[b] = _spd(rng, 1, D)[0] + 0.3 * rng.uniform(-1, 1, (D, D)) * (1 - np.eye(D))
    assert np.abs(Q - np.swapaxes(Q, 1, 2)).max() > 0.01
    return Q


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("kind", ["di_vec2", "di_vec3", "di_se2"])
def test_gp_weight_nonsymmetric_qc_inv(kind, dtype, oracle_eps):
    """The reference factors cholesky(W^T)^T of the full 2D x 2D matrix W = [[12/dt^3, -6/dt^2], [-6/dt^2, 4/dt]] (x) Qc_inv; for a
    non-symmetric Qc_inv that is not chol(S)^T (x) chol(Qc_inv)^T.  Q = [[1.5, 0.31], [0.29, 0.8]] at dt = 0.1 (the two factors differ
    by 1.3 % of the largest entry), and random per-item non-symmetric Qc_inv."""
    oracle_eps(dtype)
    D = _dof(kind)
    rng = np.random.default_rng(7)
    B = 33
    fixed = np.array([[[1.5, 0.31], [0.29, 0.8]]]) if D == 2 else _nonsymmetric_qc_inv(rng, 1, D)
    for Q, dt in ((fixed, np.full((1, 1), 0.1)), (_nonsymmetric_qc_inv(rng, B, D), rng.uniform(0.05, 1.5, (B, 1)))):
        bld = _Builder(kind, B, dtype, rng, gp=_gp_weight(Q, dt))
        for k in range(8):
            bld.add(k, dt=np.full((1, 1), 0.1))
        _check(bld.build(), dtype, f"mp gp {SFX[dtype]}")


def _edge_grid():
    """One dyadic grid (6 x 8, cell 1/4, origin (-1, -1/2)): values multiples of 1/64, so every placed point and every node value is
    exact in both dtypes."""
    R, C, cell = 6, 8, 0.25
    rng = np.random.default_rng(0)
    sdf = np.round(rng.uniform(-1, 1, (1, R, C)) * 64) / 64
    return sdf, np.array([[-1.0, -0.5]]), np.array([[cell]])


def _edge_points():
    """(points [n, 2], node (r, c) or None): grid nodes (corners, interior, last row / column), points on cell lines, on the last row and
    column between nodes, and 2^-10 outside each of the four sides."""
    sdf, o, cell = _edge_grid()
    R, C = sdf.shape[1:]
    h = 2.0 ** -10
    nodes = [(0, 0), (R - 1, C - 1), (R - 1, 0), (0, C - 1), (2, 3), (R - 1, 4), (3, C - 1)]
    pts = [(o[0, 0] + c * cell[0, 0], o[0, 1] + r * cell[0, 0]) for r, c in nodes]
    X = lambda c: o[0, 0] + c * cell[0, 0]
    Y = lambda r: o[0, 1] + r * cell[0, 0]
    pts += [(X(2.5), Y(3)), (X(3), Y(1.5)), (X(C - 1), Y(2.5)), (X(4.5), Y(R - 1)), (X(1.25), Y(0.75)),
            (X(0) - h, Y(2)), (X(C - 1) + h, Y(2)), (X(3), Y(0) - h), (X(3), Y(R - 1) + h), (X(C - 1) - h, Y(R - 1) - h)]
    return np.array(pts), nodes + [None] * 10


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("kind", ["coll_point2", "coll_se2", "eoc"])
def test_sdf_edges(kind, dtype, oracle_eps):
    """Points placed exactly on grid nodes, cell lines, the last row and column and just outside each side (SE2 poses and EOC objects
    turned by quarter turns, so the point in the grid's frame is exact); at each node the threshold (Collision2D's eps, EOC's radius)
    equals the node value (dist == threshold), is 2^-8 below it and 2^-8 above it: both sides of the switch, and the tie."""
    oracle_eps(dtype)
    sdf, origin, cell = _edge_grid()
    pts, nodes = _edge_points()
    n = len(pts)
    rng = np.random.default_rng(1)
    lim = rng.uniform(0.1, 0.6, (n, 1))
    items = []
    for q, (p, nd) in enumerate(zip(pts, nodes)):
        for dl in ((0.0, -2.0 ** -8, 2.0 ** -8) if nd is not None else (None,)):
            L = lim[q, 0] if nd is None else sdf[0, nd[0], nd[1]] + dl
            items.append((p, L))
    B = len(items)
    P_ = np.array([p for p, _ in items])
    L = np.array([[x] for _, x in items])
    turns = np.array([[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]])[np.arange(B) % 4]
    bld = _Builder(kind, B, dtype, rng, "scale")
    if kind == "coll_point2":
        ids = [bld.new_var("vec", P_)]
    elif kind == "coll_se2":
        ids = [bld.new_var("se2", np.concatenate([P_, turns], 1))]
    else:    # t_eff = t_obj + R_obj p with t_obj a multiple of 1/16
        t_obj = rng.integers(-16, 16, (B, 2)) / 16.0
        c, s = turns[:, 0], turns[:, 1]
        t_eff = t_obj + np.stack([c * P_[:, 0] - s * P_[:, 1], s * P_[:, 0] + c * P_[:, 1]], 1)
        ids = [bld.new_var("se2", np.concatenate([t_obj, turns], 1)), bld.new_var("se2", np.concatenate([t_eff, _elem("SE2", rng, B)[:, 2:]], 1))]
    bld.add(0, ids=ids, grid=(sdf, origin, cell), lim=L)
    bld.add(1, ids=ids, grid=(sdf, origin, cell), lim=L[::-1].copy())
    P = bld.build()
    A, b = _check(P, dtype, f"mp edges {SFX[dtype]}")
    # the placed ties really are ties in the kernel: e = 0 at dist == eps, |dist - r| = 0 at dist == radius
    tie = np.array([nd is not None and dl == 0.0 for (p, nd) in zip(pts, nodes) for dl in ((0.0, -1, 1) if nd is not None else (None,))])
    assert np.all(b[tie, 0] == 0)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_hinge_edges(dtype, oracle_eps):
    """x exactly on the tightened limits (no error either way), one 2^-8 inside and outside them, +-inf limits, and thresholds that make
    the tightened limits cross (down + thr > up - thr: above wins where both tests hold, and a point between them is both)."""
    oracle_eps(dtype)
    h = 2.0 ** -8
    arr = np.array([   # (x, down, up, thr) per item; the components of a D > 1 vector take rolled copies of this list
        (-0.75, -1.0, 1.0, 0.25), (0.75, -1.0, 1.0, 0.25), (-0.75 - h, -1.0, 1.0, 0.25), (0.75 + h, -1.0, 1.0, 0.25),
        (-0.75 + h, -1.0, 1.0, 0.25), (5.0, -np.inf, np.inf, 0.5), (-5.0, -np.inf, 1.0, 0.5), (5.0, -1.0, np.inf, 0.5),
        (0.0, -0.25, 0.25, 0.5), (-0.5, -0.25, 0.25, 0.5), (0.5, -0.25, 0.25, 0.5), (0.125, -0.25, 0.25, 0.5),
        (-1.0, -1.0, -1.0, 0.0), (0.25, 0.25, 0.25, 0.0)])
    n = B = len(arr)
    rng = np.random.default_rng(2)
    for D in (1, 2, 3):
        perm = [np.roll(np.arange(n), 5 * j) for j in range(D)]
        comp = lambda col: np.stack([arr[perm[j], col] for j in range(D)], 1)
        bld = _Builder(f"hinge{D}", B, dtype, rng, "diag")
        x = bld.new_var("vec", comp(0))
        bld.add(0, ids=[x], down=comp(1), up=comp(2), thr=comp(3))
        bld.add(1, ids=[x], down=comp(1)[::-1].copy(), up=comp(2)[::-1].copy(), thr=comp(3)[::-1].copy())
        _check(bld.build(), dtype, f"mp edges {SFX[dtype]}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_qsp_edges(dtype, oracle_eps):
    """theta2 - theta1 across +pi and -pi (the wrap of w = theta(obj1^-1 obj2)), the contact point at obj2's origin (p = 0) and c^2 = 0."""
    oracle_eps(dtype)
    rng = np.random.default_rng(3)
    pairs = [(np.pi - 0.1, -np.pi + 0.15), (-np.pi + 0.05, np.pi - 0.2), (3.0, -3.0), (-3.0, 3.0), (np.pi - 0.01, -np.pi + 0.01),
             (0.5, 0.5 + np.pi - 0.02), (0.5, 0.5 - np.pi + 0.02), (0.3, 0.2), (1.0, -1.0), (-2.0, 2.5)]
    B = len(pairs)
    t1, t2 = np.array(pairs).T
    se2 = lambda xy, t: np.concatenate([xy, np.stack([np.cos(t), np.sin(t)], 1)], 1)
    o1 = se2(rng.uniform(-1, 1, (B, 2)), t1)
    o2 = se2(o1[:, :2] + 0.1 * rng.standard_normal((B, 2)), t2)
    e1 = se2(o1[:, :2] + 0.2 * rng.standard_normal((B, 2)), rng.uniform(-3, 3, B))
    e2 = se2(e1[:, :2] + 0.1 * rng.standard_normal((B, 2)), rng.uniform(-3, 3, B))
    e2[[2, 5], :2] = o2[[2, 5], :2]                 # p = 0
    c2 = rng.uniform(0.1, 1.0, (B, 1))
    c2[[3, 5]] = 0.0
    bld = _Builder("qsp", B, dtype, rng, "diag")
    ids = [bld.new_var("se2", v) for v in (o1, o2, e1, e2)]
    bld.add(0, ids=ids, c2=c2)
    bld.add(1, ids=[ids[1], ids[0], ids[3], ids[2]], c2=c2[::-1].copy())
    _check(bld.build(), dtype, f"mp edges {SFX[dtype]}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_di_se2_branch_angles(dtype, oracle_eps):
    """DoubleIntegrator-SE2's local(pose1, pose2) at relative angles 0, 5 % below and above the dtype's se2 near_zero and d_near_zero, 1,
    pi - 0.1, both signs: pose1 a quarter turn, pose2 = pose1 (x) rel (a quarter turn composes exactly)."""
    oracle_eps(dtype)
    e = lie._EPS_TH[np.dtype(NP[dtype])]
    m = 0.05
    a = [e["se2_near_zero"] * (1 - m), e["se2_near_zero"] * (1 + m), e["se2_d_near_zero"] * (1 - m), e["se2_d_near_zero"] * (1 + m), 1.0, np.pi - 0.1]
    ang = np.array([0.0] + a + [-x for x in a])
    B = len(ang)
    rng = np.random.default_rng(4)
    turns = np.array([[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]])[np.arange(B) % 4]
    p1 = np.concatenate([rng.integers(-16, 16, (B, 2)) / 8.0, turns], 1)
    rel = np.stack([rng.uniform(-1, 1, B), rng.uniform(-1, 1, B), np.cos(ang), np.sin(ang)], 1)
    rel[ang == 0, 2:] = (1.0, 0.0)
    p2 = lie.se2_compose(p1, rel)
    for wk in ("scale", "gp"):
        bld = _Builder("di_se2", B, dtype, rng, "scale", gp=_random_gp(rng, 3, True, B) if wk == "gp" else None)
        ids = [bld.new_var("se2", p1), bld.new_var("vec", rng.uniform(-2, 2, (B, 3))), bld.new_var("se2", p2), bld.new_var("vec", rng.uniform(-2, 2, (B, 3)))]
        bld.add(0, ids=ids)
        _check(bld.build(), dtype, f"mp branches {SFX[dtype]}")
