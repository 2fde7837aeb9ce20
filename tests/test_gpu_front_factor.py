"""The multifrontal Cholesky factor (layout "front": theseus_b200/frontal.py, csrc/thb_front.cu, the partial mode of chol_col_kernel in
csrc/thb_chol_dense.cu) checked directly, per batch item: the factor L^ rebuilt from the panels against the damped AtA the kernels
read (componentwise backward error), on structures that each assert from the plan the kernel path they are there for; the solution per
item against numpy; no read of memory not written in the same call (NaN-poisoned buffers); bitwise batch independence and isolation of
failing items; the not-positive-definite pivot index; thb_potrf_partial_inplace_f64 and thb_potrf_f64 on their own; the tuning knobs.

Under the host emulation (THB_SIMT_EMULATION=1) the small-front parts run; the big-front, thb_potrf* parts skip: the emulation has no
DMMA dense kernel, and its dense stand-in reports info = 1."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import theseus_b200 as th
from theseus_b200 import _lib
from theseus_b200.frontal import SMALL_MAX_W, SMALL_SMEM_LIMIT, small_smem_bytes
from front_factor_cases import make_inputs, make_solver, panel_entries, var_columns
from test_gpu_sparse_solver import _dense_system

pytestmark = pytest.mark.gpu
EMU = os.environ.get("THB_SIMT_EMULATION") == "1"
needs_dmma = pytest.mark.skipif(EMU, reason="the host emulation has no DMMA dense kernel (its dense stand-in reports info = 1)")
U = 2.0 ** -53
EPS_DAMP = 1e-6


# ------------------------------------------------------------------------------------------------ the factor, rebuilt on the host
def _panel_index(plan):
    """For every stored entry of one item's factor on or below the diagonal: (row, column) in the permuted order and offset; plus the
    offsets of the entries above the diagonal of the pivot blocks (written as zeros)."""
    A = plan.arrays
    rows, cols, offs, upper = [], [], [], []
    for t in range(plan.S):
        w, b, f, po = (int(A[k][t]) for k in ("f_w", "f_b", "f_first", "f_panel_off"))
        grow = np.concatenate([f + np.arange(w), A["f_rows"][A["rows_ptr"][t]:A["rows_ptr"][t + 1]].astype(np.int64)])
        ii, jj = np.meshgrid(np.arange(w + b), np.arange(w), indexing="ij")
        e = po + ii * w + jj
        low = ii >= jj
        rows.append(grow[ii[low]]); cols.append(f + jj[low]); offs.append(e[low]); upper.append(e[~low])
    return [np.concatenate(v).astype(np.int64) for v in (rows, cols, offs, upper)]


def _inverted_blocks(plan):
    """(first pivot, size) of the diagonal blocks the kernels invert explicitly: 8 x 8 in small fronts, 64 x 64 in big ones."""
    A = plan.arrays
    out = []
    for t in range(plan.S):
        w, f = int(A["f_w"][t]), int(A["f_first"][t])
        bs = 64 if A["f_class"][t] == 3 else 8
        out += [(f + k, min(bs, w - k)) for k in range(0, w, bs)]
    return out


def _cond_inf(T):
    return np.linalg.norm(T, np.inf) * np.linalg.norm(np.linalg.inv(T), np.inf)


def _check_backward_error(L, M, kappa, what):
    """|L L^T - M| <= c u kappa |L||L^T| elementwise, c = 4 (largest row count of L + 2) (the check itself rounds in float64 too).
    Returns the largest ratio |L L^T - M| / (u kappa |L||L^T|)."""
    absL = np.abs(L)
    E = np.abs(L @ L.T - M)
    ref = U * kappa * (absL @ absL.T)
    c = 4.0 * (int((L != 0).sum(axis=1).max()) + 2)
    zero = ref == 0
    assert (E[zero] == 0).all(), what
    ratio = float((E[~zero] / ref[~zero]).max()) if (~zero).any() else 0.0
    assert ratio <= c, (what, ratio, c)
    return ratio


def _check_factor(solver, alpha, beta, items):
    """Per item: diag(L^) > 0, zeros above the pivot blocks, and the componentwise backward error of L^ against M_p = (AtA damped as the
    solve did)[perm][:, perm], where AtA is the compact block storage the factorisation read."""
    plan = solver._plan
    bufs = solver._dev["bufs"]
    F, ata = bufs["factor"].cpu().numpy(), bufs["ata"].cpu().numpy()
    rows, cols, offs, upper = _panel_index(plan)
    pm = plan.arrays["pmap"][offs]
    sel = pm >= 0
    n = plan.n
    idx = np.arange(n)
    blocks = _inverted_blocks(plan)
    worst = 0.0
    for k in items:
        assert (F[k, upper] == 0).all(), k
        L = np.zeros((n, n))
        L[rows, cols] = F[k, offs]
        assert (np.diagonal(L) > 0).all(), k
        M = np.zeros((n, n))
        M[rows[sel], cols[sel]] = ata[k, pm[sel]]
        if alpha is not None:
            d = M[idx, idx].copy()
            M[idx, idx] = d + (alpha[k] * d + beta[k])
        M = np.tril(M) + np.tril(M, -1).T
        kappa = max(_cond_inf(L[s:s + m, s:s + m]) for s, m in blocks)
        worst = max(worst, _check_backward_error(L, M, kappa, f"item {k}"))
    print(f"largest |L L^T - M| / (u kappa |L||L^T|): {worst:.3g}")
    return worst


def _check_solution(S, A, b, alpha, x):
    """Every item against numpy.linalg.solve, within that item's own condition number and scale."""
    AtA, Atb = _dense_system(S, torch.from_numpy(A), torch.from_numpy(b))
    idx = np.arange(S.num_cols)
    AtA[:, idx, idx] = AtA[:, idx, idx] * (1 + alpha[:, None]) + EPS_DAMP
    n = S.num_cols
    for k in range(A.shape[0]):
        xr = np.linalg.solve(AtA[k], Atb[k])
        err = np.abs(x[k] - xr).max()
        tol = 8 * n * U * _cond_inf(AtA[k]) * np.abs(xr).max()
        assert err <= tol, (k, err, tol)


def _solve(solver, S, A, b, alpha, damped=True):
    solver.linearization.A_val, solver.linearization.b = torch.from_numpy(A).cuda(), torch.from_numpy(b).cuda()
    if damped:
        return solver.solve(damping=torch.from_numpy(alpha).cuda(), ellipsoidal_damping=True, damping_eps=EPS_DAMP)
    return solver.solve()


# ------------------------------------------------------------------------------------------------ which paths a plan takes
def _class2_threads(smem):
    """Threads of front_small_kernel for a class-2 launch of `smem` bytes (thb_front_factor_f64, default knobs)."""
    return 256 if smem <= 56 * 1024 else (512 if smem <= 113 * 1024 else 1024)


def _assert_paths(name, plan):
    A = plan.arrays
    cls, w, b, par = A["f_class"], A["f_w"].astype(int), A["f_b"].astype(int), A["f_parent"]
    nch = np.diff(A["child_ptr"])
    small, big = cls < 3, cls == 3
    L = plan.launches
    if name == "small":
        assert {0, 1, 2} <= set(L[:, 1].tolist())
        assert {256, 512, 1024} <= {_class2_threads(int(s)) for s in L[L[:, 1] == 2][:, 4]}
        assert (small & (w % 8 != 0)).any()
        fronts_of = plan.front_of_pos
        odd = [t for t in range(plan.S) if small[t] and w[t] % 8]
        assert {1, 2, 3, 7} <= {int(plan.dims[p]) for p in range(plan.N) if fronts_of[p] in odd}
        for r in (0, 1, 15):
            assert (small & (b > 0) & (b % 16 == r)).any(), r
        assert (small & (b == 0)).any()                      # borderless root
        assert (small & (nch == 8)).any()                    # the most children the gather keeps
    elif name == "big":
        assert (big & (par >= 0) & big[np.maximum(par, 0)]).any()      # big child of a big parent
        assert (small & (par >= 0) & big[np.maximum(par, 0)]).any()    # small child of a big parent
        assert (big & (par >= 0) & small[np.maximum(par, 0)]).any()    # big child of a small parent
        assert (big & (w % 16 != 0)).any() and (big & (w % 16 == 0) & (w % 64 != 0)).any()
        assert (big & ((A["f_wpad"] + b) % 128 != 0)).any()
        assert (big & (b == 0) & (w % 64 != 0)).any()                  # borderless big root with pivot padding (config C5's root)
        assert (big & (nch == 8)).any() and (big & (nch == 9)).any()   # gather / scatter assembly
    elif name == "wide":
        for wt in (SMALL_MAX_W, SMALL_MAX_W + 1):
            t = int(np.nonzero(w == wt)[0][0])
            assert big[t], wt
            # (the shared-memory limit, not SMALL_MAX_W, is what sends these to the dense kernel: no shared-memory front is this wide)
            assert small_smem_bytes(wt, int(b[t]), int(nch[t])) > SMALL_SMEM_LIMIT
        assert (small & (nch > 0) & np.array([big[A["child_list"][A["child_ptr"][t]:A["child_ptr"][t + 1]]].any() for t in range(plan.S)])).any()


CASES = [("small", 1, None), ("small", 33, None), ("small", 130, 64),
         ("big", 1, None), ("big", 33, 16), ("big", 130, 64),
         ("wide", 1, None), ("wide", 33, 8)]


@pytest.mark.parametrize("name,B,chunk", CASES)
def test_factor_backward_error_per_item(name, B, chunk):
    if EMU and (name != "small" or B > 1):
        pytest.skip("host emulation: small fronts and small batches only")
    solver, S, first = make_solver(name, chunk=chunk)
    _assert_paths(name, solver._plan)
    if chunk is not None:
        assert chunk < B
    A, b, alpha = make_inputs(S, B, seed=B + len(name), small_var=first[-1] + 1)
    x = _solve(solver, S, A, b, alpha).cpu().numpy()
    _check_factor(solver, alpha, np.full(B, EPS_DAMP), range(B))
    _check_solution(S, A, b, alpha, x)


@needs_dmma
def test_c5_structure_at_a_small_batch():
    """Config C5's pose graph (n = 15 000, borderless 462-pivot root padded to 512) at batch 3 in chunks of 2: every item's normwise
    backward error, and each item bitwise equal to the same item solved alone."""
    import scipy.sparse as sp
    from helpers import load, pgo_objective
    objective, _ = pgo_objective(th, load("pgo_c5_lm"))
    S = th.BaspachoSparseSolver(objective).linearization.structure()
    solver = th.BaspachoSparseSolver.from_structure(S, layout="front", front_options=dict(chunk=2))
    one = th.BaspachoSparseSolver.from_structure(S, layout="front")
    one._plan, one._gram_arrays, one._ata_size = solver._plan, solver._gram_arrays, solver._ata_size   # the same plan, built once
    L = solver._plan.launches
    root = L[(L[:, 1] == 3) & (L[:, 11] == 0)]
    assert len(root) == 1 and root[0, 10] % 64 != 0 and root[0, 5] == 512
    B = 3
    A, b, alpha = make_inputs(S, B, seed=5)
    x = _solve(solver, S, A, b, alpha).cpu().numpy()
    for k in range(B):
        Am = sp.csr_matrix((A[k], S.A_col_ind, S.A_row_ptr), shape=(S.num_rows, S.num_cols))
        M = (Am.T @ Am).tocsr()
        d = M.diagonal()
        M = M + sp.diags(alpha[k] * d + EPS_DAMP)
        rhs = Am.T @ b[k]
        berr = np.abs(M @ x[k] - rhs).max() / (abs(M).sum(axis=1).max() * np.abs(x[k]).max() + np.abs(rhs).max())
        print(f"item {k}: normwise backward error {berr:.3g}")
        assert berr < 1e-13, (k, berr)
        xk = _solve(one, S, A[k:k + 1], b[k:k + 1], alpha[k:k + 1]).cpu().numpy()
        assert np.array_equal(xk[0], x[k]), k


# ------------------------------------------------------------------------------------------------ reads of memory not written in the call
@pytest.mark.parametrize("name", ["small", "big"])
def test_poisoned_buffers_give_bitwise_the_same_result(name):
    """Solve, fill every buffer the kernels write before they read (factor, update-matrix arena, border-vector arena, work, the W region
    of the dense workspace) with NaN, solve again: x and the factor must be bitwise equal.  The flag / counter / ticket words of the
    dense workspace are left alone (the entry point resets them on every call)."""
    if EMU and name != "small":
        pytest.skip("host emulation: no DMMA dense kernel")
    B, chunk = (33, 16) if not EMU else (5, 2)
    solver, S, first = make_solver(name, chunk=chunk)
    A, b, alpha = make_inputs(S, B, seed=3)
    x0 = _solve(solver, S, A, b, alpha).clone()
    bufs = solver._dev["bufs"]
    f0 = bufs["factor"].clone()
    for k in ("factor", "arena", "varena", "work"):
        bufs[k].fill_(float("nan"))
    max_np = solver._dev["max_np"]
    if max_np:
        nW = chunk * (max_np // 64) * 64 * 64
        bufs["ws"][:nW * 8].view(torch.float64).fill_(float("nan"))
    x1 = _solve(solver, S, A, b, alpha)
    assert torch.equal(x0, x1)
    used = torch.from_numpy(panel_entries(solver._plan)).to(f0.device)
    assert torch.equal(f0[:, used], bufs["factor"][:, used])


# ------------------------------------------------------------------------------------------------ batch independence and isolation
@pytest.mark.parametrize("name", ["small", "big"])
def test_items_are_bitwise_independent_of_the_batch_and_of_failing_items(name):
    """B = 37 in chunks of 16: every item bitwise equal to the same item solved alone; then two items made not positive definite: the
    healthy items' solutions and factors stay bitwise unchanged."""
    if EMU and name != "small":
        pytest.skip("host emulation: no DMMA dense kernel")
    B = 37 if not EMU else 5
    chunk = 16 if not EMU else 2
    solver, S, first = make_solver(name, chunk=chunk)
    A, b, alpha = make_inputs(S, B, seed=9)
    x = _solve(solver, S, A, b, alpha, damped=False).clone()
    used = torch.from_numpy(panel_entries(solver._plan)).to(x.device)
    fac = solver._dev["bufs"]["factor"][:, used].clone()
    one, _, _ = make_solver(name)
    for k in range(B):
        xk = _solve(one, S, A[k:k + 1], b[k:k + 1], alpha[k:k + 1], damped=False)
        assert torch.equal(xk[0], x[k]), k
        assert torch.equal(one._dev["bufs"]["factor"][0, used], fac[k]), k
    bad = [2, B - 3]
    A2 = A.copy()
    for k in bad:
        A2[k, var_columns(S, first[0])] = 0.0
    solver.defer_info_check = True
    x2 = _solve(solver, S, A2, b, alpha, damped=False)
    info = solver._last_info.cpu().numpy()
    assert (info[bad] > 0).all() and (np.delete(info, bad) == 0).all(), info
    ok = np.setdiff1d(np.arange(B), bad)
    assert torch.equal(x2[ok], x[ok])
    assert torch.equal(solver._dev["bufs"]["factor"][:, used][ok], fac[ok])


# ------------------------------------------------------------------------------------------------ the not-positive-definite report
PIVOT_CASES = [   # (structure, group, variable within the group): the group's front and where the variable's first scalar sits in it
    ("small", 3, 0),    # w 15 = 1 + 2 + 1 + 3 + 7 + 1: the front's first pivot (1-dof)
    ("small", 3, 2),    # a middle pivot (1-dof, position 3)
    ("small", 3, 5),    # the front's last pivot (1-dof, position 14 of a 15-pivot front: the padding pivot follows it)
    ("small", 8, 1),    # the root's second variable (shared-memory root with 8 children)
    ("big", 17, 0),     # first pivot of a big front (info_base + 0 * 64 + 1)
    ("big", 8, 9),      # pivot 72 of an 80-pivot big front: second 64-column block
]


@pytest.mark.parametrize("name,group,var", PIVOT_CASES)
def test_not_positive_definite_pivot_index(name, group, var):
    """Every A_val entry in the columns of variable v is zeroed in items 2 and 4 of 5 (no damping; the unary costs keep the rest positive
    definite): the pivot at v's first scalar is exactly 0.  info[k] - 1 must be v's first scalar in the plan's permuted order, the other
    items must report 0, and the error must name item 2."""
    if EMU and name != "small":
        pytest.skip("host emulation: no DMMA dense kernel")
    solver, S, first = make_solver(name, chunk=3)
    plan = solver._plan
    v = first[group] + var
    A, b, alpha = make_inputs(S, 5, seed=1)
    for k in (2, 4):
        A[k, var_columns(S, v)] = 0.0
    with pytest.raises(RuntimeError, match=r"batch element 2: matrix is not positive definite"):
        _solve(solver, S, A, b, alpha, damped=False)
    info = solver._last_info.cpu().numpy()
    col0 = int(np.sum(S.var_dims[:v]))
    assert (info[[0, 1, 3]] == 0).all(), info
    for k in (2, 4):
        assert info[k] > 0 and int(plan.perm[info[k] - 1]) == col0, (k, info[k])
    t = int(plan.front_of_pos[plan.pos[v]])
    assert (plan.arrays["f_class"][t] == 3) == (name == "big")


# ------------------------------------------------------------------------------------------------ the partial dense factorisation alone
def _read_region(n):
    R = np.arange(n)
    return R[None, :] < 128 * (R[:, None] // 128 + 1)   # row R: columns < 128 (R / 128 + 1) are read


def _partial_inputs(rng, npad, nb_piv, w_real, n_real, B):
    """Front matrices laid out as front_assemble_kernel writes them: real pivots [0, w_real), real border rows [64 nb_piv, n_real),
    identity padding, zeros above the diagonal inside the read region, NaN outside it.  Returns (F [B, npad, npad], symmetric M)."""
    wp = 64 * nb_piv
    real = np.r_[0:w_real, wp:n_real]
    m = real.shape[0]
    region = _read_region(npad)
    F = np.full((B, npad, npad), np.nan)
    Ms = np.zeros((B, npad, npad))
    for k in range(B):
        G = rng.standard_normal((m, m + 8))
        M = np.eye(npad)
        M[np.ix_(real, real)] = (G @ G.T / (m + 8) + 0.05 * np.eye(m)) * 10.0 ** (k - 2)
        Ms[k] = M
        F[k][region] = np.tril(M)[region]
    return F, Ms


def _run_partial(F, bstride, nb_piv, w_real, n_real, info_base, info0):
    lib = _lib.load()
    B, npad = F.shape[0], F.shape[1]
    buf = torch.full((B, bstride), float("nan"), dtype=torch.float64, device="cuda")
    buf[:, :npad * npad] = torch.from_numpy(F.reshape(B, -1)).cuda()
    ws = torch.empty(int(lib.thb_potrf_partial_workspace_bytes(B, npad)), dtype=torch.uint8, device="cuda")
    info = torch.from_numpy(np.asarray(info0, dtype=np.int32)).cuda()
    _lib.check(lib.thb_potrf_partial_inplace_f64(_lib.ptr(buf), bstride, npad, nb_piv, w_real, n_real, info_base, _lib.ptr(info), B,
                                                 _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "potrf_partial")
    out = buf.cpu().numpy()
    assert np.isnan(out[:, npad * npad:]).all()           # nothing written past the matrix inside the batch stride
    return out[:, :npad * npad].reshape(B, npad, npad), info.cpu().numpy()


def _partial_grid():
    out = []
    for npad in (128, 256, 384, 1024):
        nb = npad // 64
        for nb_piv in sorted({1, 2, 3, nb - 1, nb} & set(range(1, nb + 1))):
            for B in (1, 5):
                out.append((npad, nb_piv, B))
    return out


@needs_dmma
@pytest.mark.parametrize("npad,nb_piv,B", _partial_grid())
def test_potrf_partial_inplace(npad, nb_piv, B):
    """thb_potrf_partial_inplace_f64 on its own, batch stride > np^2: L11 and L21 by their componentwise backward error, the Schur
    complement against F22 - L21 L21^T from the kernel's own L21, the padding exactly identity / zero, nothing written outside the read
    region.  With B = 5: info preset in item 0 survives, a negative pivot only in the trailing block (item 1) is not reported, a negative
    pivot at the last real pivot column (item 4) is reported as info_base + 1 + column."""
    rng = np.random.default_rng(npad + 7 * nb_piv + B)
    nb, wp = npad // 64, 64 * nb_piv
    region = _read_region(npad)
    info_base = 1000
    worst = [0.0, 0.0]
    for w_real in (wp - 63, wp - 17, wp):
        for n_real in sorted({npad, npad - 1, wp + 1}):
            if n_real <= wp and nb_piv < nb or (nb_piv == nb and n_real != npad) or n_real > npad:
                continue
            F, M = _partial_inputs(rng, npad, nb_piv, w_real, n_real, B)
            info0 = np.zeros(B, dtype=np.int32)
            checked = range(B)
            if B == 5:
                info0[0] = 777
                if n_real > wp:
                    F[1, n_real - 1, n_real - 1] = M[1, n_real - 1, n_real - 1] = -1.0
                F[4, w_real - 1, w_real - 1] = M[4, w_real - 1, w_real - 1] = -1.0
                checked = range(4)
            out, info = _run_partial(F, npad * npad + 72, nb_piv, w_real, n_real, info_base, info0)
            what = (w_real, n_real)
            if B == 5:
                assert info[0] == 777 and info[1] == 0 and info[2] == 0 and info[3] == 0, (what, info)
                assert info[4] == info_base + w_real, (what, info)    # info_base + 1 + (w_real - 1)
            else:
                assert info[0] == 0, (what, info)
            for k in checked:
                O = out[k]
                assert np.isnan(O[~region]).all(), what
                up = np.triu(region, 1)
                up[wp:, wp:] = False     # (the trailing diagonal tiles also get the upper half of the Schur complement: never read)
                assert (O[up] == 0).all(), what
                # padding: identity pivots, zero L21 columns, zero L21 rows past n_real -- exactly
                pad = np.arange(w_real, wp)
                assert np.array_equal(O[np.ix_(pad, pad)], np.eye(pad.shape[0])), what
                assert (O[w_real:wp, :w_real] == 0).all() and (O[wp:, w_real:wp] == 0).all() and (O[n_real:, :wp] == 0).all(), what
                real = np.r_[0:w_real, wp:n_real]
                Lh = np.tril(np.where(region, O, 0.0))[:, :w_real][real]                           # real rows, real pivot columns
                L11 = Lh[:w_real]
                kappa = max(_cond_inf(L11[s:s + 64, s:s + 64]) for s in range(0, w_real, 64))
                absL = np.abs(Lh)
                E = np.abs(Lh @ L11.T - M[k][np.ix_(real, np.arange(w_real))])
                ref = U * kappa * (absL @ np.abs(L11).T)
                c = 4.0 * (w_real + 2)
                worst[0] = max(worst[0], float((E / ref).max()))
                assert (E <= c * ref).all(), (what, k, float((E / ref).max()))
                if n_real > wp:
                    L21 = O[wp:n_real, :w_real]
                    S = np.tril(O[wp:n_real, wp:n_real])
                    F22 = np.tril(M[k][wp:n_real, wp:n_real])
                    E2 = np.abs(S - np.tril(F22 - L21 @ L21.T))
                    ref2 = U * (np.abs(F22) + np.tril(np.abs(L21) @ np.abs(L21).T))
                    ok = ref2 > 0
                    assert (E2[~ok] == 0).all(), what
                    worst[1] = max(worst[1], float((E2[ok] / ref2[ok]).max()))
                    assert (E2[ok] <= 4.0 * (w_real + 2) * ref2[ok]).all(), (what, k)
                # the trailing rows / columns past n_real keep the assembled identity / zeros exactly
                tail = np.zeros((npad, npad), dtype=bool)
                tail[n_real:, wp:] = True
                tail[wp:, n_real:] = True
                tail &= region & (np.arange(npad)[:, None] >= np.arange(npad)[None, :])
                assert np.array_equal(O[tail], F[k][tail]), what
    print(f"largest ratios: L {worst[0]:.3g} (of u kappa |L||L^T|), Schur complement {worst[1]:.3g} (of u (|F22| + |L21||L21^T|))")


@needs_dmma
def test_potrf_reports_the_failing_column():
    """thb_potrf_f64 (n = 200, batch 3): a negative pivot at column c of item 1 only -> info = [0, c + 1, 0]."""
    lib = _lib.load()
    rng = np.random.default_rng(4)
    B, n = 3, 200
    G = rng.standard_normal((B, n, n + 8))
    M0 = G @ np.transpose(G, (0, 2, 1)) / (n + 8) + 0.05 * np.eye(n)
    ws = torch.empty(int(lib.thb_potrf_workspace_bytes(B, n)), dtype=torch.uint8, device="cuda")
    for c in (0, 7, 8, 31, 32, 63, 64, 65, 127, 128, n - 1):
        M = M0.copy()
        M[1, c, c] = -1.0
        Mt = torch.from_numpy(M).cuda()
        info = torch.full((B,), -5, dtype=torch.int32, device="cuda")
        _lib.check(lib.thb_potrf_f64(_lib.ptr(Mt), None, None, _lib.ptr(info), B, n, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "potrf")
        assert info.cpu().tolist() == [0, c + 1, 0], c


# ------------------------------------------------------------------------------------------------ tuning knobs, in child processes
KNOBS = [{"THB_SOLVE_STAGE": "5120"}, {"THB_FRONT_T0": "128"}, {"THB_FRONT_T0": "256"}, {"THB_FRONT_T1": "256"},
         {"THB_FRONT_PREFETCH": "0"}, {"THB_FRONT_PDL": "1"}]


def _run_cases(out_dir, env_extra):
    here = os.path.dirname(os.path.abspath(__file__))
    env = {k: v for k, v in os.environ.items() if not k.startswith(("THB_SOLVE_", "THB_FRONT_"))}
    env.update(env_extra)
    os.makedirs(out_dir)
    try:
        r = subprocess.run([sys.executable, os.path.join(here, "front_factor_cases.py"), out_dir], capture_output=True, text=True,
                           timeout=600, cwd=os.path.dirname(here), env=env)
    except subprocess.TimeoutExpired:
        pytest.fail(f"{env_extra}: child timed out after 600 s")   # subprocess.run has killed and reaped it
    assert r.returncode == 0, (env_extra, r.stderr[-2000:])
    return {f: np.load(os.path.join(out_dir, f)) for f in sorted(os.listdir(out_dir))}


@pytest.fixture(scope="module")
def default_knob_run(tmp_path_factory):
    return _run_cases(str(tmp_path_factory.mktemp("knobs") / "default"), {})


@pytest.mark.parametrize("knob", KNOBS, ids=lambda k: "-".join(f"{a}={b}" for a, b in k.items()))
def test_tuning_knobs_do_not_change_the_arithmetic(knob, default_knob_run, tmp_path):
    """Staging panels in shared memory (THB_SOLVE_STAGE), the thread counts of classes 0 / 1, the L2 prefetch and programmatic dependent
    launch change where data sits and who computes it, never the order of the arithmetic: x and the factor must be bitwise equal to the
    default run (one child process per setting: the knobs are read once per process)."""
    if EMU and ("THB_FRONT_PREFETCH" in knob or "THB_FRONT_PDL" in knob):
        pytest.skip("host emulation: no prefetch and no programmatic dependent launch")
    got = _run_cases(str(tmp_path / "run"), knob)
    assert sorted(got) == sorted(default_knob_run)
    for f, ref in default_knob_run.items():
        assert np.array_equal(got[f], ref, equal_nan=False), f
