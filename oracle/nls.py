"""Oracle: batched nonlinear least squares inner loop (numpy restatement; test infrastructure only).

Restates, for a flat problem description, what the reference does per LM / GN
iteration: cost-function Jacobians (theseus/embodied/...), linearization
(theseus/optimizer/{dense,sparse}_linearization.py), damping + dense Cholesky
(theseus/optimizer/linear/dense_solver.py), retract / error metric
(theseus/core/objective.py) and the LM accept/reject control
(theseus/optimizer/nonlinear/levenberg_marquardt.py).

Problem description ("spec"), batch-first like the reference:
    spec = {
      "dtype": np.float64 | np.float32,
      "vars":  [ {"kind": "SE3"|"SO3"|"SE2"|"Vector", "dof": int, "value": ndarray [B, ...]} , ...]   # in column order
      "costs": [ {"kind": "between"|"local", "group": "SE3"|..., "vars": (i, j) | (i,),
                  "aux": ndarray [B or 1, ...]   (measurement / target),
                  "weight": ("diag", ndarray [B or 1, dim]) | ("scale", ndarray [B or 1, 1])}, ...]  # objective order
    }
The motion-planning and planar-pushing kinds (collision, double_integrator, hinge, nonholonomic, qsp, eoc) and the GP weight
("gp", Qc_inv [B or 1, D, D], dt [B or 1, 1]) are described in oracle/embodied.py.
"""
import numpy as np

from . import embodied, lie

_GROUP = {
    "SE3": dict(dof=6, inverse=lie.se3_inverse, compose=lie.se3_compose, jlog=lie.se3_jlog,
                log=lie.se3_log, adjoint=lie.se3_adjoint, exp=lie.se3_exp),
    "SO3": dict(dof=3, inverse=lie.so3_inverse, compose=lie.so3_compose, jlog=lie.so3_jlog,
                log=lie.so3_log, adjoint=lie.so3_adjoint, exp=lie.so3_exp),
    "SE2": dict(dof=3, inverse=lie.se2_inverse, compose=lie.se2_compose, jlog=lie.se2_jlog,
                log=lie.se2_log, adjoint=lie.se2_adjoint, exp=lie.se2_exp),
    "SO2": dict(dof=1, inverse=lie.so2_inverse, compose=lie.so2_compose, jlog=lie.so2_jlog,
                log=lie.so2_log, adjoint=lie.so2_adjoint, exp=lie.so2_exp),
}


def _bcast(a, B):
    return np.broadcast_to(a, (B,) + a.shape[1:]) if a.shape[0] != B else a


# ----------------------------------------------------------------------------- cost functions
def between_error_jacobians(group, X0, X1, Z, want_jac=True):
    """theseus/embodied/measurements/between.py:34-45.

    D = X0^-1 X1 ; e = log(Z^-1 D) ; J1 = dlog ; J0 = -dlog @ Ad(D^-1).
    """
    g = _GROUP[group]
    D = g["compose"](g["inverse"](X0), X1)
    E = g["compose"](g["inverse"](Z), D)
    if not want_jac:
        return None, g["log"](E)
    dlog, e = g["jlog"](E)
    J0 = -dlog @ g["adjoint"](g["inverse"](D))
    return [J0, dlog], e


def local_error_jacobians(group, X, T, want_jac=True):
    """theseus/embodied/misc/local_cost_fn.py:40-61 + geometry/lie_group.py:180-195.

    e = log(T^-1 X); J = dlog(T^-1 X).
    """
    g = _GROUP[group]
    D = g["compose"](g["inverse"](T), X)
    if not want_jac:
        return None, g["log"](D)
    dlog, e = g["jlog"](D)
    return [dlog], e


def weight_jacobians_error(weight, jacs, err):
    """theseus/core/cost_weight.py:81-90 (Scale), :125-136 (Diagonal); GPCostWeight (embodied/motionmodel/double_integrator.py:154-170):
    W e and W J with W the factor of embodied.gp_weight."""
    kind, w = weight[0], weight[1]
    B = err.shape[0]
    if kind == "gp":
        W = embodied.gp_weight(_bcast(np.asarray(w, dtype=err.dtype), B), _bcast(np.asarray(weight[2], dtype=err.dtype), B))
        e = (W @ err[:, :, None])[:, :, 0]
        return (None if jacs is None else [W @ J for J in jacs]), e
    w = _bcast(np.asarray(w, dtype=err.dtype), B)
    if kind == "scale":
        w = w.reshape(B, 1)
    e = err * w
    if jacs is None:
        return None, e
    return [J * w[:, :, None] for J in jacs], e


def cost_weighted_jacobians_error(spec, cost, values, want_jac=True):
    """theseus/core/cost_function.py:107-122 (weighted_jacobians_error), un-masked path."""
    B = values[0].shape[0]
    aux = _bcast(np.asarray(cost["aux"], dtype=spec["dtype"]), B)
    if cost["kind"] == "between":
        jacs, e = between_error_jacobians(cost["group"], values[cost["vars"][0]], values[cost["vars"][1]], aux, want_jac)
    elif cost["kind"] == "local":
        jacs, e = local_error_jacobians(cost["group"], values[cost["vars"][0]], aux, want_jac)
    else:
        raise NotImplementedError(cost["kind"])
    return weight_jacobians_error(cost["weight"], jacs, e)


def reprojection_error_jacobians(X, p, f, z, k1, k2, want_jac=True):
    """theseus/embodied/measurements/reprojection.py:54-94 (+ torchlie se3_impl.py:757-777 for the transform Jacobians).
    X [...,3,4] camera pose, p [...,3] world point, f/k1/k2 [...,1], z [...,2]."""
    R, t = X[..., :3], X[..., 3]
    q = (R @ p[..., None])[..., 0] + t
    proj = -q[..., :2] / q[..., 2:3]
    n = (proj * proj).sum(axis=-1, keepdims=True)
    pf = f * (1.0 + n * (k1 + n * k2))
    err = proj * pf - z
    if not want_jac:
        return None, err
    J = np.concatenate([R, -R @ lie.hat3(p), R], axis=-1)                       # [...,3,9]
    dpf = f * (k1 + 2.0 * n * k2)
    num_dden_den = q[..., :2, None] * (J[..., 2, :] / q[..., 2:3])[..., None, :]
    proj_jac = (num_dden_den - J[..., 0:2, :]) / q[..., 2:3, None]
    proj_sqn_jac = 2.0 * proj[..., :, None] * (proj[..., None, :] @ proj_jac)
    Jp = proj_jac * pf[..., None] + proj_sqn_jac * dpf[..., None]
    return [Jp[..., :6], Jp[..., 6:]], err


def _robust_rho(kind, x, radius, mu):
    """rho(x) of robust_loss.py:33-118 (x = squared norm, radius = exp(log_radius), mu = GNC control value of Geman-McClure)."""
    if kind == "welsch":
        return radius - radius * np.exp(-x / (radius + 1e-20))
    if kind == "huber":
        return np.where(x > radius, 2 * np.sqrt(radius * np.maximum(x, radius) + 1e-20) - radius, x)
    if kind == "hinge":
        return np.where(x > radius, np.sqrt(x) - np.sqrt(radius), 1e-20)
    if kind == "geman":
        return mu * radius * x / (mu * radius + x + 1e-20)
    raise ValueError(kind)


def _robust_drho(kind, x, radius, mu):
    """rho'(x) as the reference's `linearize` gives it (same lines)."""
    if kind == "welsch":
        return np.exp(-x / (radius + 1e-20))
    if kind == "huber":
        return np.sqrt(radius / np.maximum(x, radius) + 1e-20)
    if kind == "hinge":
        return np.where(x > radius, 1.0 / (2 * np.sqrt(x) + 1e-20), 0.0)
    if kind == "geman":
        return (mu * radius) ** 2 / ((mu * radius + x) ** 2 + 1e-20)
    raise ValueError(kind)


def robust_apply(robust, jacs, e, flatten_dims=False):
    """theseus/core/robust_cost_function.py:87-135 with the losses of robust_loss.py:33-118.
    robust = (kind, log_radius [..,1]) or (kind, log_radius, mu); e weighted error [...,dim].  With jacs: linearisation rescale;
    without: the 'hacky' error whose squared norm equals rho(||e||^2).  flatten_dims: the loss per error dimension."""
    kind, log_radius = robust[0], robust[1]
    mu = robust[2] if len(robust) > 2 else None
    radius = np.exp(log_radius)
    x = e ** 2 if flatten_dims else (e ** 2).sum(axis=-1, keepdims=True)
    if jacs is not None:
        sc = np.sqrt(_robust_drho(kind, x, radius, mu) + 1e-20)
        return [sc[..., None] * J for J in jacs], sc * e
    val = _robust_rho(kind, x, radius, mu)
    if flatten_dims:
        return None, np.sqrt(val + 1e-20)
    return None, np.ones_like(e) * np.sqrt(val / e.shape[-1] + 1e-20)


def cost_dim(spec, cost):
    if cost["kind"] in embodied.KINDS:
        return embodied.cost_dim(spec, cost)
    if cost["kind"] == "reproj":
        return 2
    if cost.get("group") == "Vector":
        return spec["vars"][cost["vars"][0]]["dof"]
    return _GROUP[cost["group"]]["dof"]


def eval_costs(spec, values, want_jac=True):
    """All cost functions, batched by schema like theseus/core/vectorizer.py:222-332 (Vectorize): cost functions of
    the same (type, group, weight type) are stacked into one [K, B, ...] evaluation, then sliced back.
    Returns a list aligned with spec["costs"] of (jacobians or None, weighted error)."""
    B = values[0].shape[0]
    dt = spec["dtype"]
    groups = {}
    out = [None] * len(spec["costs"])
    for f, c in enumerate(spec["costs"]):
        if c["kind"] in embodied.KINDS:      # one cost function at a time (float64 throughout: no stacking order to follow)
            if c.get("robust") is not None:
                raise NotImplementedError(f"robust loss on a {c['kind']} cost function")
            jac_list, err = embodied.cost_jacobians_error(spec, c, values, want_jac)
            out[f] = weight_jacobians_error(c["weight"], jac_list, err.astype(dt))
            continue
        groups.setdefault((c["kind"], c.get("group", "-") + (str(spec["vars"][c["vars"][0]]["dof"]) if c.get("group") == "Vector" else ""),
                           c["weight"][0]), []).append(f)

    def put(f, jac_list, err):
        c = spec["costs"][f]
        if c.get("robust") is not None:
            rk, lr = c["robust"][0], c["robust"][1]
            extra = tuple(_bcast(np.asarray(m, dtype=dt), B) for m in c["robust"][2:])   # GNC control value (Geman-McClure)
            jac_list, err = robust_apply((rk, _bcast(np.asarray(lr, dtype=dt), B)) + extra, jac_list, err)
        out[f] = (jac_list, err)

    for (kind, grp, wkind), idx in groups.items():
        grp = "Vector" if grp.startswith("Vector") else grp
        cs = [spec["costs"][f] for f in idx]
        if kind == "reproj":
            st = lambda key: np.stack([_bcast(np.asarray(c["aux"][key], dtype=dt), B) for c in cs], 0)
            x0 = np.stack([values[c["vars"][0]] for c in cs], 0)
            x1 = np.stack([values[c["vars"][1]] for c in cs], 0)
            jacs, e = reprojection_error_jacobians(x0, x1, st("f"), st("z"), st("k1"), st("k2"), want_jac)
            w = np.stack([_bcast(np.asarray(c["weight"][1], dtype=dt), B) for c in cs], 0)
            if wkind == "scale":
                w = w.reshape(w.shape[0], B, 1)
            e = e * w
            if jacs is not None:
                jacs = [J * w[..., None] for J in jacs]
            for r, f in enumerate(idx):
                put(f, [J[r] for J in jacs] if jacs is not None else None, e[r])
            continue
        aux = np.stack([_bcast(np.asarray(c["aux"], dtype=dt), B) for c in cs], 0)          # [K,B,...]
        if grp == "Vector":  # Difference on Vector/Point: e = x - target, J = I (geometry/vector.py)
            x0 = np.stack([values[c["vars"][0]] for c in cs], 0)
            e = x0 - aux
            w = np.stack([_bcast(np.asarray(c["weight"][1], dtype=dt), B) for c in cs], 0)
            if wkind == "scale":
                w = w.reshape(w.shape[0], B, 1)
            e = e * w
            d = e.shape[-1]
            J = np.broadcast_to(np.eye(d, dtype=dt), e.shape[:-1] + (d, d)) * np.broadcast_to(w, e.shape)[..., None]
            for r, f in enumerate(idx):
                out[f] = ([J[r]] if want_jac else None, e[r])
            continue
        w = np.stack([_bcast(np.asarray(c["weight"][1], dtype=dt), B) for c in cs], 0)       # [K,B,dim or 1]
        x0 = np.stack([values[c["vars"][0]] for c in cs], 0)
        if kind == "between":
            x1 = np.stack([values[c["vars"][1]] for c in cs], 0)
            jacs, e = between_error_jacobians(grp, x0, x1, aux, want_jac)
        elif kind == "local":
            jacs, e = local_error_jacobians(grp, x0, aux, want_jac)
        else:
            raise NotImplementedError(kind)
        if wkind == "scale":
            w = w.reshape(w.shape[0], B, 1)
        e = e * w                                                                             # cost_weight.py:81-90,125-136
        if jacs is not None:
            jacs = [J * w[..., None] for J in jacs]
        for r, f in enumerate(idx):
            put(f, [J[r] for J in jacs] if jacs is not None else None, e[r])
    return out


# ----------------------------------------------------------------------------- structure
def var_layout(spec):
    """theseus/optimizer/linearization.py:30-41: var_dims, var_start_cols, num_cols."""
    dims = [v["dof"] for v in spec["vars"]]
    starts = np.concatenate([[0], np.cumsum(dims)[:-1]]).astype(np.int64)
    return dims, starts, int(np.sum(dims))


def sparse_structure(spec):
    """theseus/optimizer/sparse_linearization.py:34-84: batch-shared CSR of A.

    Returns dict(A_row_ptr, A_col_ind, block_pointers (list), row_block_starts, stride, num_rows, num_cols).
    """
    dims, starts, n = var_layout(spec)
    col_ind, row_ptr = [], [0]
    bptrs, rstarts, strides = [], [], []
    for cost in spec["costs"]:
        d = cost_dim(spec, cost)
        slices = sorted(((int(starts[v]), int(starts[v] + dims[v])), k) for k, v in enumerate(cost["vars"]))
        sizes = [s[1] - s[0] for s, _ in slices]
        sptr = np.cumsum([0] + sizes)[:-1]
        bp = np.zeros(len(slices), dtype=np.int64)
        bp[np.array([k for _, k in slices])] = sptr
        bptrs.append(bp)
        rstarts.append(len(col_ind))
        ci = [c for s, _ in slices for c in range(s[0], s[1])]
        strides.append(len(ci))
        for _ in range(d):
            col_ind += ci
            row_ptr.append(len(col_ind))
    return dict(A_row_ptr=np.array(row_ptr, dtype=np.int64), A_col_ind=np.array(col_ind, dtype=np.int64),
                block_pointers=bptrs, row_block_starts=np.array(rstarts, dtype=np.int64),
                stride=np.array(strides, dtype=np.int64), num_rows=len(row_ptr) - 1, num_cols=n)


def ata_block_structure(spec):
    """theseus/optimizer/linear/baspacho_sparse_solver.py:93-113: (param_size, block CSR of AtA, full symmetric)."""
    dims, _, _ = var_layout(spec)
    N = len(dims)
    nbr = [set([i]) for i in range(N)]
    for cost in spec["costs"]:
        for a in cost["vars"]:
            for b in cost["vars"]:
                nbr[a].add(b)
    ptrs = [0]
    inds = []
    for i in range(N):
        inds += sorted(nbr[i])
        ptrs.append(len(inds))
    return np.array(dims, dtype=np.int64), np.array(ptrs, dtype=np.int64), np.array(inds, dtype=np.int64)


# ----------------------------------------------------------------------------- linearization
def linearize_sparse(spec, values, struct=None):
    """sparse_linearization.py:102-140: A_val [B,nnz], b [B,m] (b = -weighted error)."""
    struct = struct or sparse_structure(spec)
    B = values[0].shape[0]
    dt = spec["dtype"]
    A_val = np.empty((B, len(struct["A_col_ind"])), dtype=dt)
    b = np.empty((B, struct["num_rows"]), dtype=dt)
    row = 0
    evaluated = eval_costs(spec, values)
    for f, cost in enumerate(spec["costs"]):
        jacs, e = evaluated[f]
        d = e.shape[1]
        st, stride = struct["row_block_starts"][f], struct["stride"][f]
        blk = A_val[:, st:st + stride * d].reshape(B, d, stride)
        for k, J in enumerate(jacs):
            p = struct["block_pointers"][f][k]
            blk[:, :, p:p + J.shape[2]] = J
        b[:, row:row + d] = -e
        row += d
    return A_val, b


def linearize_dense(spec, values):
    """dense_linearization.py:29-62: A [B,m,n], b [B,m], AtA = A^T A, Atb = A^T b ([B,n,1])."""
    dims, starts, n = var_layout(spec)
    B = values[0].shape[0]
    dt = spec["dtype"]
    m = sum(cost_dim(spec, c) for c in spec["costs"])
    A = np.zeros((B, m, n), dtype=dt)
    b = np.zeros((B, m), dtype=dt)
    row = 0
    evaluated = eval_costs(spec, values)
    for f, cost in enumerate(spec["costs"]):
        jacs, e = evaluated[f]
        d = e.shape[1]
        for k, J in enumerate(jacs):
            c0 = starts[cost["vars"][k]]
            A[:, row:row + d, c0:c0 + J.shape[2]] = J
        b[:, row:row + d] = -e
        row += d
    At = A.transpose(0, 2, 1)
    AtA = At @ A
    Atb = At @ b[:, :, None]
    return A, b, AtA, Atb


def csr_to_dense(struct, A_val):
    B = A_val.shape[0]
    A = np.zeros((B, struct["num_rows"], struct["num_cols"]), dtype=A_val.dtype)
    rp, ci = struct["A_row_ptr"], struct["A_col_ind"]
    for r in range(struct["num_rows"]):
        A[:, r, ci[rp[r]:rp[r + 1]]] = A_val[:, rp[r]:rp[r + 1]]
    return A


# ----------------------------------------------------------------------------- solve
def apply_damping(AtA, damping, ellipsoidal=True, eps=1e-8):
    """linear/dense_solver.py:38-64 (_apply_damping)."""
    B, n, _ = AtA.shape
    damping = np.asarray(damping, dtype=AtA.dtype)
    out = AtA.copy()
    idx = np.arange(n)
    if ellipsoidal:
        d = damping.reshape(-1, 1) * AtA[:, idx, idx] + eps
    else:
        d = np.broadcast_to(damping.reshape(-1, 1), (B, n)) if damping.ndim else np.full((B, n), damping, dtype=AtA.dtype)
    out[:, idx, idx] += d.astype(AtA.dtype)
    return out


def cholesky_solve(AtA, Atb):
    """linear/dense_solver.py:159-161: L = chol(AtA); x = cholesky_solve(Atb, L). Raises on non-PD."""
    import scipy.linalg as sla
    B, n, _ = AtA.shape
    x = np.empty((B, n), dtype=AtA.dtype)
    for i in range(B):
        c = sla.cho_factor(AtA[i], lower=True, check_finite=False)
        x[i] = sla.cho_solve(c, Atb[i, :, 0], check_finite=False)
    return x


def dense_solve(AtA, Atb, damping=None, ellipsoidal=True, eps=1e-8):
    """linear/dense_solver.py:66-78 (_apply_damping_and_solve)."""
    if damping is not None:
        AtA = apply_damping(AtA, damping, ellipsoidal, eps)
    return cholesky_solve(AtA, Atb)


# ----------------------------------------------------------------------------- retract / error
def _sparse_solve_item(args):
    row_ptr, col_ind, shape, a_val, b_i, alpha, beta = args
    import scipy.sparse as sp
    from scipy.sparse.linalg import splu
    A = sp.csr_matrix((a_val, col_ind, row_ptr), shape=shape)
    At = A.T.tocsr()
    AtA = (At @ A).tocsc()
    d = AtA.diagonal()
    AtA.setdiag(d * (1.0 + alpha) + beta)
    Atb = At @ b_i
    x = splu(AtA, permc_spec="MMD_AT_PLUS_A", diag_pivot_thresh=0.0).solve(Atb)
    return x, Atb, d


def sparse_solve(struct, A_val, b, damping=None, ellipsoidal=True, eps=1e-8, n_jobs=1):
    """BaspachoSolveFunction.forward (optimizer/autograd/baspacho_sparse_autograd.py:21-65: AtA = add_MtM, damp(alpha, beta), factor,
    Atb = tmat_vec, solve) and CholmodSolveFunction.forward (optimizer/autograd/cholmod_sparse_autograd.py:25-61: a Python loop over
    the batch, one sparse factorisation per item) on the CPU.  (alpha, beta) as linear/utils.py:14-33: ellipsoidal -> (damping, eps),
    else (0, damping).  SuperLU (scipy) stands in for CHOLMOD / BaSpaCho, neither of which is importable here.
    Returns (x [B,n], Atb [B,n], diag(AtA) [B,n]).  n_jobs > 1: items over a joblib process pool (the reference's loop is serial)."""
    B = A_val.shape[0]
    n = struct["num_cols"]
    if damping is None:
        alpha, beta = np.zeros(B), np.zeros(B)
    else:
        dv = np.broadcast_to(np.asarray(damping, dtype=np.float64), (B,))
        alpha, beta = (dv, np.full(B, eps)) if ellipsoidal else (np.zeros(B), dv)
    shape = (struct["num_rows"], n)
    jobs = [(struct["A_row_ptr"], struct["A_col_ind"], shape, np.asarray(A_val[i], dtype=np.float64), np.asarray(b[i], dtype=np.float64),
             float(alpha[i]), float(beta[i])) for i in range(B)]
    if n_jobs > 1 and B > 1:
        from joblib import Parallel, delayed
        res = Parallel(n_jobs=min(n_jobs, B))(delayed(_sparse_solve_item)(j) for j in jobs)
    else:
        res = [_sparse_solve_item(j) for j in jobs]
    x = np.stack([r[0] for r in res], 0)
    Atb = np.stack([r[1] for r in res], 0)
    diag = np.stack([r[2] for r in res], 0)
    return x.astype(A_val.dtype), Atb.astype(A_val.dtype), diag.astype(A_val.dtype)


def retract(spec, values, delta, ignore_mask=None):
    """core/objective.py:857-914 (retract_vars_sequence) + geometry/lie_group.py:197-198.

    ignore_mask [B] bool: those batch items keep their old value (variable.py:65-69).
    """
    dims, starts, _ = var_layout(spec)
    out = []
    for i, v in enumerate(spec["vars"]):
        d = delta[:, starts[i]:starts[i] + dims[i]]
        if v["kind"] == "SE3":
            new = lie.se3_retract(values[i], d)
        elif v["kind"] == "SO3":
            new = lie.so3_retract(values[i], d)
        elif v["kind"] == "SE2":
            new = lie.se2_retract(values[i], d)
        elif v["kind"] == "SO2":
            new = lie.so2_retract(values[i], d)
        elif v["kind"] == "Vector":
            new = values[i] + d
        else:
            raise NotImplementedError(v["kind"])
        if ignore_mask is not None and ignore_mask.any():
            m = ignore_mask.reshape((-1,) + (1,) * (new.ndim - 1))
            new = np.where(m, values[i], new)
        out.append(new.astype(spec["dtype"]))
    return out


def error_vector(spec, values):
    """core/objective.py:562-613: concatenated weighted errors, objective order."""
    return np.concatenate([e for _, e in eval_costs(spec, values, want_jac=False)], axis=1)


def error_metric(spec, values):
    """core/objective.py:37-38,615-641: 0.5 * sum(e^2)."""
    e = error_vector(spec, values)
    return (e**2).sum(axis=1) / 2


# ----------------------------------------------------------------------------- LM / GN loop
def check_convergence(err, last_err, abs_tol, rel_tol):
    """nonlinear/nonlinear_optimizer.py:109-119."""
    if np.abs(err).mean() < abs_tol:
        return np.ones_like(err, dtype=bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        chg = last_err - err
        return (np.abs(chg) < abs_tol) | (np.abs(chg / last_err) < rel_tol)


def optimize(spec, method="lm", max_iterations=20, step_size=1.0, abs_err_tolerance=1e-10, rel_err_tolerance=1e-8,
             damping=1e-3, adaptive_damping=False, ellipsoidal_damping=False, damping_eps=1e-8,
             down_damping_ratio=9.0, up_damping_ratio=11.0, damping_accept=0.1, sample_trace=True, solver="dense", n_jobs=1):
    """nonlinear/nonlinear_least_squares.py:100-215 (_optimize_loop) with
    levenberg_marquardt.py:90-201 (reset / compute_delta / _check_accept) or gauss_newton.py:46-47.

    Returns dict(values, err_history [B, it+1], trace=[per-iteration dict]).
    """
    dt = spec["dtype"]
    values = [np.array(v["value"], dtype=dt) for v in spec["vars"]]
    B = values[0].shape[0]
    lam = np.full(B, damping, dtype=dt) if adaptive_damping else damping
    last_err = error_metric(spec, values)
    hist = [last_err.copy()]
    converged = np.zeros(B, dtype=bool)
    trace = []
    it, all_reject_attempts = 0, 0
    while it < max_iterations:
        if solver == "sparse":   # SparseLinearization + per-item sparse direct solves (the reference's CPU sparse path)
            sstruct = sparse_structure(spec) if it == 0 and all_reject_attempts == 0 else sstruct
            A_val, b = linearize_sparse(spec, values, sstruct)
            delta, Atb2, AtA_diag = sparse_solve(sstruct, A_val, b, damping=lam if method == "lm" else None,
                                                 ellipsoidal=ellipsoidal_damping, eps=damping_eps, n_jobs=n_jobs)
            Atb, AtA = Atb2[:, :, None], None
        else:
            A, b, AtA, Atb = linearize_dense(spec, values)
            AtA_diag = AtA[:, np.arange(AtA.shape[1]), np.arange(AtA.shape[1])]
            if method == "lm":
                delta = dense_solve(AtA, Atb, damping=lam, ellipsoidal=ellipsoidal_damping, eps=damping_eps)
            else:
                delta = dense_solve(AtA, Atb)
        step = (delta * step_size).astype(dt)
        new_values = retract(spec, values, step, ignore_mask=converged)
        err = error_metric(spec, new_values)
        reject = None
        rec = dict(Atb=Atb[:, :, 0].copy(), delta=delta.copy(), lam=np.array(lam, dtype=dt, copy=True), new_err=err.copy())
        if sample_trace:
            rec["AtA_diag"] = AtA_diag.copy()
        if method == "lm" and adaptive_damping:
            dmp = lam.reshape(-1, 1)
            if ellipsoidal_damping:
                dmp = dmp * AtA_diag
            den = (step * (dmp * step + Atb[:, :, 0])).sum(axis=1) / 2
            with np.errstate(divide="ignore", invalid="ignore"):
                rho = (last_err - err) / den
            reject = rho <= damping_accept
            lam = np.where(reject, lam * up_damping_ratio, lam / down_damping_ratio)
            lam = np.clip(lam, 1e-7, 1e7).astype(dt)
            rec["rho"] = rho
            rec["reject"] = reject.copy()
        trace.append(rec)
        if reject is not None and reject.all():
            all_reject_attempts += 1
            if all_reject_attempts < 3:
                continue
            err = last_err  # _step returns previous_err (nonlinear_least_squares.py:358-359)
        else:
            if reject is not None and reject.any():
                m = reject
                values = [np.where(m.reshape((-1,) + (1,) * (v.ndim - 1)), v, nv) for v, nv in zip(values, new_values)]
                err = error_metric(spec, values)
            else:
                values = new_values
        all_reject_attempts = 0
        hist.append(err.copy())
        converged = check_convergence(err, last_err, abs_err_tolerance, rel_err_tolerance)
        if converged.all():
            break
        last_err = err
        it += 1
    return dict(values=values, err_history=np.stack(hist, axis=1), trace=trace, damping=lam)
