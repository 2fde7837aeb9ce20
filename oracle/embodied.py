"""Oracle: the motion-planning and planar-pushing cost functions (numpy restatement, written from the math; test infrastructure only).

Restates, in float64, what the reference evaluates for
  - the signed distance field lookup (theseus/embodied/collision/signed_distance_field.py:163-241),
  - Collision2D on Point2 / SE2 poses (embodied/collision/collision.py:44-73),
  - DoubleIntegrator on Vector / SE2 poses (embodied/motionmodel/double_integrator.py:45-80) and the GP cost weight (:131-152),
  - HingeCost (embodied/motionmodel/misc.py:62-84) and Nonholonomic on SE2 / Vector poses (misc.py:126-178),
  - QuasiStaticPushingPlanar (embodied/motionmodel/quasi_static_pushing_planar.py:47-276),
  - EffectorObjectContactPlanar without the Huber loss (embodied/collision/eff_obj_contact.py:55-104).

Cost dicts for oracle/nls.py (values in the column order of spec["vars"]; aux entries [B or 1, ...]):
    {"kind": "collision", "vars": (pose,), "aux": dict(origin, sdf, cell, eps)}          pose: Point2 ("Vector", dof 2) or SE2
    {"kind": "double_integrator", "vars": (pose1, vel1, pose2, vel2), "aux": dict(dt)}   poses: Vector (dof 1-3) or SE2
    {"kind": "hinge", "vars": (x,), "aux": dict(down, up, threshold)}
    {"kind": "nonholonomic", "vars": (pose, vel)}                                        pose: SE2 or a Vector (x, y, theta)
    {"kind": "qsp", "vars": (obj1, obj2, eff1, eff2), "aux": dict(c_square)}
    {"kind": "eoc", "vars": (obj, eff), "aux": dict(origin, sdf, cell, radius)}
with a "weight" of ("scale", w), ("diag", w) or ("gp", Qc_inv [B or 1, D, D], dt [B or 1, 1]).

Switch decisions (the SDF cell and the out-of-grid test, dist > eps, dist < radius, the hinge tests, the +-pi wrap of an angle) are
taken in spec["switch_dtype"] when it is given: a float32 kernel decides them in its own arithmetic, and the oracle then follows the same
branch while everything else stays float64."""
import numpy as np

from . import lie

KINDS = ("collision", "double_integrator", "hinge", "nonholonomic", "qsp", "eoc")


def _b(a, B):
    a = np.asarray(a, np.float64)
    return np.broadcast_to(a, (B,) + a.shape[1:]) if a.shape[0] != B else a


def _sd(x, sd):
    """x in the decision dtype (float64 when no switch dtype is given)."""
    return np.asarray(x, np.float64).astype(sd or np.float64)


# ----------------------------------------------------------------------------- signed distance field
def _bilinear(row, col, lr, lc, data, cell):
    """signed_distance_field.py:197-236: bilinear interpolation in the cell (lr, lc) and its gradient; indices clamped to the grid
    (lr.long().clamp(0, rows - 1), ...: the far edge reads its own row / column twice)."""
    B, R, C = data.shape
    hr, hc = lr + 1.0, lc + 1.0
    idx = lambda v, hi: np.clip(np.where(np.isfinite(v), v, 0), 0, hi).astype(np.int64)
    lri, lci, hri, hci = idx(lr, R - 1), idx(lc, C - 1), idx(hr, R - 1), idx(hc, C - 1)
    bi = np.arange(B)
    g00, g10, g01, g11 = data[bi, lri, lci], data[bi, hri, lci], data[bi, lri, hci], data[bi, hri, hci]
    hrd, hcd, lrd, lcd = hr - row, hc - col, row - lr, col - lc
    dist = hrd * hcd * g00 + lrd * hcd * g10 + hrd * lcd * g01 + lrd * lcd * g11
    jx = (hrd * (g01 - g00) + lrd * (g11 - g10)) / cell
    jy = (hcd * (g10 - g00) + lcd * (g11 - g01)) / cell
    return dist, jx, jy


def sdf_lookup(px, py, origin, data, cell, sd=None, p_sd=None):
    """Signed distance of the points (px, py) [B] in the grids data [B, R, C] whose node (r, c) lies at origin + (c, r) cell, and its
    gradient (d/dx, d/dy); distance and gradient 0 outside the grid (signed_distance_field.py:163-189 + 193-241).  The out-of-grid test
    and the cell (floor of (p - origin) / cell) are decided in `sd` on the points p_sd = (px, py) as the kernel computed them (default:
    the float64 points rounded to sd).  Returns (dist, jx, jy) in float64 and the distance as evaluated in `sd` (for the switches that
    compare it)."""
    B, R, C = data.shape
    ox, oy, cell = origin[:, 0], origin[:, 1], cell.reshape(B)
    pxs, pys = (_sd(px, sd), _sd(py, sd)) if p_sd is None else p_sd
    oxs, oys, cs, ds = _sd(ox, sd), _sd(oy, sd), _sd(cell, sd), _sd(data, sd)
    with np.errstate(invalid="ignore"):
        oob = (pxs < oxs) | (pxs > oxs + (C - 1.0) * cs) | (pys < oys) | (pys > oys + (R - 1.0) * cs)
        col_s, row_s = (pxs - oxs) / cs, (pys - oys) / cs
        lc, lr = np.floor(col_s), np.floor(row_s)
        dist_s, _, _ = _bilinear(row_s, col_s, lr, lc, ds, cs)
        dist, jx, jy = _bilinear((py - oy) / cell, (px - ox) / cell, lr.astype(np.float64), lc.astype(np.float64), data, cell)
    z = np.zeros(B)
    return np.where(oob, z, dist), np.where(oob, z, jx), np.where(oob, z, jy), np.where(oob, z.astype(dist_s.dtype), dist_s)


# ----------------------------------------------------------------------------- cost functions (unweighted)
def collision(x, is_se2, origin, data, cell, eps, sd=None):
    """collision.py:44-73: e = max(eps - sdf(xy), 0); J = -d sdf / d pose, zero where sdf > eps.  SE2: d xy / d tangent = [R | 0]."""
    dist, jx, jy, dist_s = sdf_lookup(x[:, 0], x[:, 1], origin, data, cell, sd)
    eps = eps.reshape(-1)
    e = np.maximum(eps - dist, 0.0)[:, None]
    far = dist_s > _sd(eps, sd)
    jx, jy = np.where(far, 0.0, jx), np.where(far, 0.0, jy)
    if not is_se2:
        return [-np.stack([jx, jy], -1)[:, None, :]], e
    c, s = x[:, 2], x[:, 3]
    J = -np.stack([jx * c + jy * s, -jx * s + jy * c, np.zeros_like(jx)], -1)
    return [J[:, None, :]], e


def double_integrator(p1, v1, p2, v2, dt, is_se2):
    """double_integrator.py:45-80: e = [local(pose1, pose2) - dt vel1, vel2 - vel1]; local's Jacobians those of log(pose1^-1 pose2)
    (a Between with an identity measurement: -dlog Ad(D^-1), dlog)."""
    B, D = v1.shape
    dt = dt.reshape(B, 1)
    if is_se2:
        D_ = lie.se2_compose(lie.se2_inverse(p1), p2)
        dlog, pd = lie.se2_jlog(D_)
        Jp1, Jp2 = -dlog @ lie.se2_adjoint(lie.se2_inverse(D_)), dlog
    else:
        pd = p2 - p1
        Jp1, Jp2 = np.broadcast_to(-np.eye(D), (B, D, D)), np.broadcast_to(np.eye(D), (B, D, D))
    e = np.concatenate([pd - dt * v1, v2 - v1], 1)
    I, Z = np.broadcast_to(np.eye(D), (B, D, D)), np.zeros((B, D, D))
    return [np.concatenate([Jp1, Z], 1), np.concatenate([-dt[:, :, None] * I, -I], 1), np.concatenate([Jp2, Z], 1),
            np.concatenate([Z, I], 1)], e


def gp_weight(Qc_inv, dt):
    """double_integrator.py:131-152: W = [[12/dt^3 Q, -6/dt^2 Q], [-6/dt^2 Q, 4/dt Q]] and its factor cholesky(W^T)^T.  The Cholesky
    reads only the lower triangle of W^T: for a non-symmetric Qc_inv the factored matrix is the symmetric one made from that triangle,
    which is not a Kronecker product.  Returns [B, 2D, 2D] (upper triangular)."""
    dt = dt.reshape(-1, 1, 1)
    Q = Qc_inv
    W = np.concatenate([np.concatenate([12.0 / dt ** 3 * Q, -6.0 / dt ** 2 * Q], 2), np.concatenate([-6.0 / dt ** 2 * Q, 4.0 / dt * Q], 2)], 1)
    Wt = np.swapaxes(W, 1, 2)
    M = np.tril(Wt) + np.swapaxes(np.tril(Wt, -1), 1, 2)
    return np.swapaxes(np.linalg.cholesky(M), 1, 2)


def hinge(x, down, up, thr, sd=None):
    """misc.py:62-84: limits tightened by the threshold; e = down - x below, x - up above, and above wins where both hold (tightened
    limits that cross); J = diag(-1 / +1 / 0)."""
    lo, hi = down + thr, up - thr
    with np.errstate(invalid="ignore"):
        below = _sd(x, sd) < _sd(down, sd) + _sd(thr, sd)
        above = _sd(x, sd) > _sd(up, sd) - _sd(thr, sd)
        e = np.where(above, x - hi, np.where(below, lo - x, 0.0))
    d = np.where(above, 1.0, np.where(below, -1.0, 0.0))
    return [d[:, :, None] * np.eye(x.shape[1])], e


def nonholonomic(pose, vel, is_se2):
    """misc.py:126-178: SE2 pose: e = vel[1], zero pose block; Vector pose (x, y, theta): e = vel[1] cos(theta) - vel[0] sin(theta)."""
    B = vel.shape[0]
    Jp, Jv = np.zeros((B, 1, 3)), np.zeros((B, 1, 3))
    if is_se2:
        Jv[:, 0, 1] = 1.0
        return [Jp, Jv], vel[:, 1:2]
    c, s = np.cos(pose[:, 2]), np.sin(pose[:, 2])
    Jp[:, 0, 2] = -(vel[:, 1] * s + vel[:, 0] * c)
    Jv[:, 0, 0], Jv[:, 0, 1] = -s, c
    return [Jp, Jv], (vel[:, 1] * c - vel[:, 0] * s)[:, None]


def _rel_angle(T1, T2, sd=None):
    """theta(T1^-1 T2) = atan2(c1 s2 - s1 c2, c1 c2 + s1 s2) (se2.py between + theta); on the branch cut +-pi the side is the one the
    sine's sign takes in `sd`."""
    sn = T1[:, 2] * T2[:, 3] - T1[:, 3] * T2[:, 2]
    cs = T1[:, 2] * T2[:, 2] + T1[:, 3] * T2[:, 3]
    w = np.arctan2(sn, cs)
    if sd is not None:
        a, b = _sd(T1, sd), _sd(T2, sd)
        ws = np.arctan2(a[:, 2] * b[:, 3] - a[:, 3] * b[:, 2], a[:, 2] * b[:, 2] + a[:, 3] * b[:, 3]).astype(np.float64)
        w = np.where(np.abs(ws - w) > np.pi, w + 2 * np.pi * np.sign(ws - w), w)
    return w


def qsp(o1, o2, e1, e2, c2, sd=None):
    """quasi_static_pushing_planar.py:47-276: with R2 obj2's rotation,
        p = R2^T (t_e2 - t_o2),  v = R2^T (t_o2 - t_o1),  vp = R2^T (t_e2 - t_e1),  w = theta(obj1^-1 obj2),
        e = D [v, w] - [vp, 0],  D = [[1, 0, -py], [0, 1, px], [-py, px, -c^2]].
    Jacobians by the chain rule along each variable's tangent (X exp(xi): dt = R du, dR = R hat(dtheta)): obj1 moves v by -R2^T R1 du
    and w by -dtheta; obj2 moves p by -du, v by +du and rotates p, v, vp by -dtheta (d q = (q_y, -q_x) dtheta), w by +dtheta; eff1 moves
    vp by -R2^T Re1 du; eff2 moves p and vp by R2^T Re2 du."""
    B = o1.shape[0]
    c2 = c2.reshape(B)
    c, s = o2[:, 2], o2[:, 3]
    unrot = lambda d: (c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1])
    px, py = unrot(e2[:, :2] - o2[:, :2])
    vx, vy = unrot(o2[:, :2] - o1[:, :2])
    vpx, vpy = unrot(e2[:, :2] - e1[:, :2])
    w = _rel_angle(o1, o2, sd)
    e = np.stack([vx - py * w - vpx, vy + px * w - vpy, -py * vx + px * vy - c2 * w], 1)

    def cols(dp, dv, dvp, dw):   # each [B, 2, 3] / [B, 3]: d(p, v, vp) and dw along the 3 tangent directions -> J [B, 3, 3]
        return np.stack([dv[:, 0] - w[:, None] * dp[:, 1] - py[:, None] * dw - dvp[:, 0],
                         dv[:, 1] + w[:, None] * dp[:, 0] + px[:, None] * dw - dvp[:, 1],
                         -vx[:, None] * dp[:, 1] - py[:, None] * dv[:, 0] + vy[:, None] * dp[:, 0] + px[:, None] * dv[:, 1] - c2[:, None] * dw], 1)

    def rel(x):   # R2^T R_x as [B, 2, 2]
        rc, rs = c * x[:, 2] + s * x[:, 3], c * x[:, 3] - s * x[:, 2]
        return np.stack([np.stack([rc, -rs], -1), np.stack([rs, rc], -1)], 1)

    Z2, Z = np.zeros((B, 2, 3)), np.zeros((B, 3))
    pad = lambda M: np.concatenate([M, np.zeros((B, 2, 1))], 2)             # [B,2,2] translation part -> [B,2,3]
    rot = lambda qx, qy: np.concatenate([np.zeros((B, 2, 2)), np.stack([qy, -qx], 1)[:, :, None]], 2)
    J1 = cols(Z2, -pad(rel(o1)), Z2, np.broadcast_to([0.0, 0.0, -1.0], (B, 3)))
    I2 = np.broadcast_to(np.eye(2), (B, 2, 2))
    J2 = cols(-pad(I2) + rot(px, py), pad(I2) + rot(vx, vy), rot(vpx, vpy), np.broadcast_to([0.0, 0.0, 1.0], (B, 3)))
    J3 = cols(Z2, Z2, -pad(rel(e1)), Z)
    Re2 = pad(rel(e2))
    J4 = cols(Re2, Z2, Re2, Z)
    return [J1, J2, J3, J4], e


def eoc(obj, eff, origin, data, cell, radius, sd=None):
    """eff_obj_contact.py:55-104: p = R_obj^T (t_eff - t_obj) (transform_to), e = |sdf(p) - r|, J = s d sdf/dp dp/d(obj, eff) with
    s = -1 where sdf < r and +1 otherwise; dp/d obj = [[-1, 0, py], [0, -1, -px]], dp/d eff = [R_obj^T R_eff | 0]."""
    B = obj.shape[0]
    r = radius.reshape(B)
    c, s = obj[:, 2], obj[:, 3]
    tp = lambda T: (T[:, 2] * (eff[:, 0] - T[:, 0]) + T[:, 3] * (eff[:, 1] - T[:, 1]), -T[:, 3] * (eff[:, 0] - T[:, 0]) + T[:, 2] * (eff[:, 1] - T[:, 1]))
    px, py = tp(obj)
    p_sd = None
    if sd is not None:
        o_s, ef_s = _sd(obj, sd), _sd(eff, sd)
        dx, dy = ef_s[:, 0] - o_s[:, 0], ef_s[:, 1] - o_s[:, 1]
        p_sd = (o_s[:, 2] * dx + o_s[:, 3] * dy, -o_s[:, 3] * dx + o_s[:, 2] * dy)
    dist, jx, jy, dist_s = sdf_lookup(px, py, origin, data, cell, sd, p_sd)
    e = np.abs(dist - r)[:, None]
    sg = np.where(dist_s < _sd(r, sd), -1.0, 1.0)
    gx, gy = sg * jx, sg * jy
    rc, rs = c * eff[:, 2] + s * eff[:, 3], c * eff[:, 3] - s * eff[:, 2]
    Jo = np.stack([-gx, -gy, gx * py - gy * px], -1)[:, None, :]
    Je = np.stack([gx * rc + gy * rs, -gx * rs + gy * rc, np.zeros(B)], -1)[:, None, :]
    return [Jo, Je], e


# ----------------------------------------------------------------------------- oracle/nls.py glue
def cost_dim(spec, cost):
    k = cost["kind"]
    if k in ("collision", "nonholonomic", "eoc"):
        return 1
    if k == "qsp":
        return 3
    d = spec["vars"][cost["vars"][0]]["dof"]
    return 2 * d if k == "double_integrator" else d


def cost_jacobians_error(spec, cost, values, want_jac=True):
    """Unweighted (jacobians, error) of one cost function of KINDS over `values` (one array [B, ...] per variable of spec["vars"])."""
    B = values[0].shape[0]
    sd = spec.get("switch_dtype")
    x = [np.asarray(values[i], np.float64) for i in cost["vars"]]
    se2 = spec["vars"][cost["vars"][0]]["kind"] == "SE2"
    aux = {k: _b(v, B) for k, v in cost.get("aux", {}).items()}
    k = cost["kind"]
    if k == "collision":
        jacs, e = collision(x[0], se2, aux["origin"], aux["sdf"], aux["cell"], aux["eps"], sd)
    elif k == "double_integrator":
        jacs, e = double_integrator(*x, aux["dt"], se2)
    elif k == "hinge":
        jacs, e = hinge(x[0], aux["down"], aux["up"], aux["threshold"], sd)
    elif k == "nonholonomic":
        jacs, e = nonholonomic(x[0], x[1], se2)
    elif k == "qsp":
        jacs, e = qsp(*x, aux["c_square"], sd)
    elif k == "eoc":
        jacs, e = eoc(x[0], x[1], aux["origin"], aux["sdf"], aux["cell"], aux["radius"], sd)
    else:
        raise NotImplementedError(k)
    return (jacs if want_jac else None), e
