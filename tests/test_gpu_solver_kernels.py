"""The dense Cholesky (csrc/thb_chol_dense.cu, full mode: thb_potrf_f64 / thb_potrs_f64 / thb_potrf_potrs_f64) and the block-sparse
Cholesky of the `item` (csrc/thb_sparse.cu) and plain `lane` (csrc/thb_sparse_lane.cu) layouts, checked directly, per batch item, against
float64 numpy / scipy: the factor and the explicitly inverted diagonal blocks read back from the kernels' buffers (componentwise backward
error against the damped matrix the kernels read), the solution against numpy, no read of memory not written in the same call
(NaN-poisoned buffers), bitwise batch independence and isolation of failing items, and the not-positive-definite pivot index.

Every bound has the form c u kappa scale of tests/test_gpu_front_factor.py: u = 2^-53, kappa the largest cond_inf of the diagonal blocks
the kernel inverts explicitly (64 x 64 dense, d x d block-sparse), c from the length of the inner products (the backward error of Cholesky
with inverted diagonal blocks, Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., Thm. 10.3 and Sec. 13.3).

Under the host emulation (THB_SIMT_EMULATION=1) the item / lane / front parts run at reduced sizes; the dense parts skip: the
emulation's dense stand-in is numpy."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.linalg
import scipy.sparse as sp
import torch

import theseus_b200 as th
from theseus_b200 import _lib
from theseus_b200.sparse import ITEM_MAX_DIM, LN_UH
from theseus_b200.structure import build_structure
from front_factor_cases import make_inputs, var_columns
from test_gpu_front_factor import _check_backward_error, _cond_inf
from test_gpu_sparse_solver import _clique_structure, _dense_system, _random_structure

pytestmark = pytest.mark.gpu
EMU = os.environ.get("THB_SIMT_EMULATION") == "1"
needs_dmma = pytest.mark.skipif(EMU, reason="the host emulation's dense Cholesky is a numpy stand-in")
U = 2.0 ** -53
TN, TM = 64, 128        # block-column width and row-tile height of chol_col_kernel


def _cuda(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _first_bad_pivot(M):
    """1-based index of the first non-positive pivot of a scalar (unblocked) Cholesky of M, 0 if there is none: the leading-minor
    rule of torch.linalg.cholesky / LAPACK potrf."""
    n = M.shape[0]
    L = np.zeros_like(M)
    for c in range(n):
        d = M[c, c] - L[c, :c] @ L[c, :c]
        if not d > 0:
            return c + 1
        L[c, c] = np.sqrt(d)
        L[c + 1:, c] = (M[c + 1:, c] - L[c + 1:, :c] @ L[c, :c]) / L[c, c]
    return 0


def _check_x(M, rhs, x, what):
    """x against numpy.linalg.solve within 8 n u kappa_inf(M) |x|_inf (normwise forward error of a backward-stable solve)."""
    xr = np.linalg.solve(M, rhs)
    err = np.abs(x - xr).max()
    tol = 8 * M.shape[0] * U * _cond_inf(M) * np.abs(xr).max()
    assert err <= tol, (what, err, tol)
    return err


# ================================================================================================ A. dense, full mode
def _dense_geometry(ws, B, n):
    """Mirror of geometry() in thb_chol_dense.cu: L [B, np, np] at offset 0 (np = n rounded up to 128), W_j = L_jj^-1 [B, nb, 64, 64]
    right after it."""
    npad = -(-n // TM) * TM
    nb = npad // TN
    f = ws.view(torch.float64)
    L = f[:B * npad * npad].view(B, npad, npad)
    W = f[B * npad * npad:B * npad * npad + B * nb * TN * TN].view(B, nb, TN, TN)
    return L, W


def _dense(M, rhs, alpha=None, beta=None, poison=False, split=False):
    """thb_potrf_potrs_f64 (split: thb_potrf_f64, then thb_potrs_f64) on [B, n, n] / [B, n]; returns L, W, x, info as numpy."""
    lib = _lib.load()
    B, n = rhs.shape
    ws = torch.empty(int(lib.thb_potrf_workspace_bytes(B, n)), dtype=torch.uint8, device="cuda")
    if poison:
        ws.fill_(0xFF)          # every double of the workspace is a NaN
    Mt, r, a, be = _cuda(M), _cuda(rhs), _cuda(alpha), _cuda(beta)
    x = torch.full((B, n), float("nan"), dtype=torch.float64, device="cuda")
    info = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    s = _lib.stream_ptr()
    if split:
        _lib.check(lib.thb_potrf_f64(_lib.ptr(Mt), _lib.ptr(a), _lib.ptr(be), _lib.ptr(info), B, n, _lib.ptr(ws), ws.numel(), s), "potrf")
        _lib.check(lib.thb_potrs_f64(_lib.ptr(r), _lib.ptr(x), B, n, _lib.ptr(ws), ws.numel(), s), "potrs")
    else:
        _lib.check(lib.thb_potrf_potrs_f64(_lib.ptr(Mt), _lib.ptr(r), _lib.ptr(a), _lib.ptr(be), _lib.ptr(x), _lib.ptr(info), B, n,
                                           _lib.ptr(ws), ws.numel(), s), "potrf_potrs")
    L, W = _dense_geometry(ws, B, n)
    return L.cpu().numpy(), W.cpu().numpy(), x.cpu().numpy(), info.cpu().numpy()


def _written(npad):
    """The part of L the kernel writes: every 64 x 64 block on or below the diagonal block."""
    R = np.arange(npad) // TN
    return R[:, None] >= R[None, :]


def _spd(rng, B, n):
    """Symmetric positive definite [B, n, n] in O(B n^2): a symmetric Gaussian matrix shifted past its spectral radius (cond ~ 5),
    item k scaled by 10^((k % 7) - 3)."""
    G = rng.standard_normal((B, n, n))
    M = (G + np.transpose(G, (0, 2, 1))) / 2 + 3 * np.sqrt(n) * np.eye(n)
    return M * (10.0 ** ((np.arange(B) % 7) - 3))[:, None, None]


def _damped_dense(M, alpha, beta):
    """diag <- d + (alpha d + beta), as chol_col_kernel applies it on its load of AtA."""
    if alpha is None:
        return M
    M = M.copy()
    idx = np.arange(M.shape[-1])
    d = M[:, idx, idx]
    M[:, idx, idx] = d + (alpha[:, None] * d + beta[:, None])
    return M


def _check_dense(M, rhs, L, W, x, items, what, check_x=True):
    """Per item: diag(L) > 0, exact zeros above the diagonal of every 64 x 64 diagonal block, exact identity in the padding, the
    componentwise backward error of L against the damped M the kernel read, W_j L_jj = I within 4 (64 + 2) u kappa(L_jj), x against
    numpy.  Returns the largest backward-error ratio."""
    B, n = rhs.shape
    npad, nb = L.shape[1], L.shape[1] // TN
    wr = _written(npad)
    pad = wr & ((np.arange(npad)[:, None] >= n) | (np.arange(npad)[None, :] >= n))
    eye = np.eye(npad)
    worst = 0.0
    for k in items:
        Lk = L[k]
        assert (np.diagonal(Lk)[:n] > 0).all(), (what, k)
        for j in range(nb):
            Ljj = Lk[j * TN:(j + 1) * TN, j * TN:(j + 1) * TN]
            assert (np.triu(Ljj, 1) == 0).all(), (what, k, j)
            # W_j L_jj = I: a triangular inverse has a residual of at most (d + 2) u |W||L| <= (d + 2) u kappa normwise
            res = np.linalg.norm(W[k, j] @ Ljj - np.eye(TN), np.inf)
            assert res <= 4 * (TN + 2) * U * _cond_inf(Ljj), (what, k, j, res)
        assert np.array_equal(Lk[pad], eye[pad]), (what, k)
        Ln = np.tril(Lk[:n, :n])
        kappa = max(_cond_inf(Ln[s:s + TN, s:s + TN]) for s in range(0, n, TN))
        worst = max(worst, _check_backward_error(Ln, M[k], kappa, f"{what} item {k}"))
        if check_x:
            _check_x(M[k], rhs[k], x[k], (what, k))
    return worst


DENSE_N = [1, 8, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 257, 383, 385, 640]
_dense_worst = {}


@needs_dmma
@pytest.mark.parametrize("B", [1, 3, 37])
@pytest.mark.parametrize("n", DENSE_N)
def test_dense_factor_per_item(n, B):
    """thb_potrf_potrs_f64 with no, spherical and ellipsoidal damping (per-item alpha and beta): the factor, the inverted diagonal blocks
    and x of every item."""
    rng = np.random.default_rng(100 * n + B)
    M0 = _spd(rng, B, n)
    rhs = rng.standard_normal((B, n))
    modes = {"none": (None, None), "spherical": (np.zeros(B), rng.random(B) * 0.1),
             "ellipsoidal": (rng.random(B) * 0.1, rng.random(B) * 1e-2)}
    for mode, (alpha, beta) in modes.items():
        L, W, x, info = _dense(M0, rhs, alpha, beta)
        assert (info == 0).all(), (mode, info)
        r = _check_dense(_damped_dense(M0, alpha, beta), rhs, L, W, x, range(B), (n, B, mode))
        _dense_worst["shapes"] = max(_dense_worst.get("shapes", 0.0), r)
    print(f"dense n {n} B {B}: largest |L L^T - M| / (u kappa |L||L^T|) so far {_dense_worst['shapes']:.3g}")


@needs_dmma
def test_dense_conditioning_sweep():
    """M = Q diag(sigma) Q^T with cond 1e2 .. 1e12 and a graded D M D (D spanning 1e-6 .. 1e6), n = 257: the same factor and solution
    bounds.  Prints the kernel's forward error over that of scipy.linalg.cho_solve (LAPACK) on the same system."""
    rng = np.random.default_rng(11)
    n = 257
    conds = [1e2, 1e4, 1e6, 1e8, 1e10, 1e12]
    Ms = []
    for c in conds:
        Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
        Ms.append((Q * np.logspace(0, -np.log10(c), n)) @ Q.T)
    D = np.logspace(-6, 6, n)[rng.permutation(n)]
    Ms.append(D[:, None] * _spd(rng, 1, n)[0] * 1e3 * D[None, :])
    M = np.stack([(m + m.T) / 2 for m in Ms])
    xt = rng.standard_normal((M.shape[0], n))
    rhs = np.einsum("bij,bj->bi", M, xt)
    L, W, x, info = _dense(M, rhs)
    assert (info == 0).all(), info
    worst = _check_dense(M, rhs, L, W, x, range(M.shape[0]), "conditioning")
    for k, name in enumerate([f"cond {c:.0e}" for c in conds] + ["graded 1e-6..1e6"]):
        ref = scipy.linalg.cho_solve(scipy.linalg.cho_factor(M[k], lower=True), rhs[k])
        e_ker, e_ref = np.abs(x[k] - xt[k]).max(), np.abs(ref - xt[k]).max()
        print(f"{name}: forward error kernel {e_ker:.3g}, scipy cho_solve {e_ref:.3g}, ratio {e_ker / max(e_ref, 1e-300):.3g}")
    print(f"conditioning sweep: largest |L L^T - M| / (u kappa |L||L^T|) {worst:.3g}")


@needs_dmma
@pytest.mark.parametrize("B,n", [(300, 256), (64, 1536)])
def test_dense_more_ctas_than_resident(B, n):
    """(B = 300, n = 256): 1 800 CTAs; (B = 64, n = 1536): about 10 000 -- far more than the 264 that are resident on an H100, so the
    tile queue and the per-tile flags order CTAs that start long after their dependencies.  Every item bitwise equal to the same item
    solved alone; the backward error of a sample of items."""
    rng = np.random.default_rng(B + n)
    M = _spd(rng, B, n)
    rhs = rng.standard_normal((B, n))
    alpha, beta = rng.random(B) * 0.1, rng.random(B) * 1e-2
    L, W, x, info = _dense(M, rhs, alpha, beta)
    assert (info == 0).all()
    wr = _written(L.shape[1])
    for k in range(B):
        L1, W1, x1, i1 = _dense(M[k:k + 1], rhs[k:k + 1], alpha[k:k + 1], beta[k:k + 1])
        assert np.array_equal(x1[0], x[k]) and np.array_equal(L1[0][wr], L[k][wr]) and np.array_equal(W1[0], W[k]), k
    sample = [0, 1, B // 2, B - 1]
    worst = _check_dense(_damped_dense(M, alpha, beta), rhs, L, W, x, sample, (B, n))
    print(f"B {B} n {n}: largest |L L^T - M| / (u kappa |L||L^T|) {worst:.3g}")


@needs_dmma
@pytest.mark.parametrize("n", [65, 385])
def test_dense_poisoned_workspace(n):
    """The whole workspace filled with NaN before the call: L (where written), W and x bitwise equal to a run on a zeroed workspace."""
    rng = np.random.default_rng(n)
    B = 3
    M, rhs = _spd(rng, B, n), rng.standard_normal((B, n))
    alpha, beta = rng.random(B) * 0.1, rng.random(B) * 1e-2
    L0, W0, x0, _ = _dense(M, rhs, alpha, beta)
    L1, W1, x1, info = _dense(M, rhs, alpha, beta, poison=True)
    wr = _written(L0.shape[1])
    assert (info == 0).all()
    assert np.array_equal(x0, x1) and np.array_equal(W0, W1) and np.array_equal(L0[:, wr], L1[:, wr])


@needs_dmma
@pytest.mark.parametrize("n", [130, 200, 256])
def test_dense_failing_items(n):
    """Item 1 not positive definite at column c (c = n - 1 included: for n not a multiple of 64 the last block is padded): info is exactly
    [0, c + 1, 0, 0], the healthy items' x and L stay bitwise unchanged; two failing columns in one item: the smaller one is reported."""
    rng = np.random.default_rng(n + 1)
    B = 4
    M, rhs = _spd(rng, B, n), rng.standard_normal((B, n))
    L0, _, x0, _ = _dense(M, rhs)
    wr = _written(L0.shape[1])
    ok = [0, 2, 3]
    for c in sorted({0, 63, 64, 100, n - 1}):
        M1 = M.copy()
        M1[1, c, c] = -1.0
        L, _, x, info = _dense(M1, rhs)
        assert info.tolist() == [0, c + 1, 0, 0], (c, info)
        assert np.array_equal(x[ok], x0[ok]) and np.array_equal(L[ok][:, wr], L0[ok][:, wr]), c
    for c1, c2 in ((3, 70), (64, 65), (10, n - 1)):
        M1 = M.copy()
        M1[2, c2, c2] = M1[2, c1, c1] = -1.0
        _, _, _, info = _dense(M1, rhs)
        assert info.tolist() == [0, 0, c1 + 1, 0], (c1, c2, info)


@needs_dmma
@pytest.mark.parametrize("n,B", [(5600, 1), (6000, 2)])
def test_dense_large_n_solve(n, B):
    """n > 5504: the solve needs more than 48 KB of shared memory ((np + 576) 8 bytes) and opts into it.  thb_potrf_f64 + thb_potrs_f64
    against numpy, the inverted diagonal blocks against the factor."""
    assert (-(-n // TM) * TM + TN + 8 * TN) * 8 > 48 * 1024
    rng = np.random.default_rng(n)
    M, rhs = _spd(rng, B, n), rng.standard_normal((B, n))
    L, W, x, info = _dense(M, rhs, split=True)
    assert (info == 0).all()
    for k in range(B):
        _check_x(M[k], rhs[k], x[k], (n, k))
        for j in (0, n // TN // 2, n // TN):
            Ljj = L[k, j * TN:(j + 1) * TN, j * TN:(j + 1) * TN]
            assert np.linalg.norm(W[k, j] @ Ljj - np.eye(TN), np.inf) <= 4 * (TN + 2) * U * _cond_inf(Ljj), (k, j)


# ================================================================================================ B / C. the item and lane layouts
def _vars_structure(sizes, pairs):
    """One 2-row cost on every pair of variables in `pairs`, one unary cost of d + 1 rows on every variable (positive definite AtA)."""
    return build_structure(sizes, [(2, [int(a), int(b)]) for a, b in pairs] + [(d + 1, [v]) for v, d in enumerate(sizes)])


def _structure(name):
    """(structure, ordering, what the structure is there for -- asserted from the plan by _assert_structure)."""
    rng = np.random.default_rng(len(name))
    if name == "mixed":
        return _random_structure(rng, 90 if not EMU else 40, [1, 2, 3, 6], 0.03, num_rows_blocks=3 * (90 if not EMU else 40)), "mindeg"
    if name == "generic":
        sizes = [int(d) for d in rng.permutation(list(range(4, ITEM_MAX_DIM + 1)) * 2)]
        N = len(sizes)
        pairs = {tuple(sorted(rng.choice(N, 2, replace=False))) for _ in range(2 * N)}
        return _vars_structure(sizes, sorted(pairs)), "mindeg"
    if name == "chain":
        N = 48 if not EMU else 16
        sizes = [int(d) for d in rng.choice([1, 2, 3, 6], N)]
        return _vars_structure(sizes, [(v, v + 1) for v in range(N - 1)]), "natural"
    if name == "star":
        # leaves first, then two hubs: 600 leaves on hub 0 and 301 on hub 1 -> 901 columns in level 0
        nl0, nl1 = 600, 301
        sizes = [1] * (nl0 + nl1) + [6, 3]
        hub0, hub1 = nl0 + nl1, nl0 + nl1 + 1
        return _vars_structure(sizes, [(v, hub0) for v in range(nl0)] + [(v, hub1) for v in range(nl0, nl0 + nl1)]), "natural"
    if name == "clique":
        return _clique_structure(rng, [6] * 10 + [3, 2, 1, 6] * 2), "mindeg"
    raise KeyError(name)


def _assert_structure(name, plan):
    dims = {int(d) for d in plan.dims}
    level = plan.level.astype(int)
    if name == "mixed":
        assert dims == {1, 2, 3, 6}
    elif name == "generic":
        assert set(range(4, ITEM_MAX_DIM + 1)) <= dims and max(dims) == ITEM_MAX_DIM     # all on potrf_inv_small<0>
    elif name == "chain":
        assert (np.bincount(level) == 1).all() and level.max() + 1 == plan.N              # one column per level
    elif name == "star":
        assert int((level == 0).sum()) > 512                                              # wider than SP_THREADS
        A = plan.arrays
        pairs = set()
        for j in np.nonzero(level == 1)[0]:
            e = np.nonzero(A["u_tgt"] == A["diag_off"][j])[0]
            assert len(e) == 1
            pairs.add(int(A["u_p1"][e[0]] - A["u_p0"][e[0]]) % 2)
        assert pairs == {0, 1}                                                            # an even and an odd number of update pairs
    elif name == "clique":
        assert (plan.lane["launches"][:, 0] == LN_UH).any()                               # heavy (split-K) update launches


class _Reader:
    """Rebuilds one item's L (permuted order, scipy.sparse) and the inverted / reciprocal diagonal blocks from the solver's buffers: the
    inverse of _factor_numpy in test_sparse_symbolic.py.  item: factor [B, data_size] holds every block of L (diagonal blocks with zeros
    above the diagonal), diag [B, winv_size] holds W_j = L_jj^-1 at winv_off[j].  lane: factor [data_size, Bp] holds the off-diagonal
    blocks, diag [winv_size, Bp] holds L_jj with the reciprocal of its diagonal on the diagonal."""

    def __init__(self, plan):
        self.plan = plan
        ps, dims = plan.pstart.astype(np.int64), plan.dims.astype(np.int64)
        o_r, o_c, o_e, d_r, d_c, d_e, d_w, d_up, w_up, on_diag = [], [], [], [], [], [], [], [], [], []
        for (i, j), t in plan.blk_index.items():
            di, dj, off = int(dims[i]), int(dims[j]), int(plan.blk_off[t])
            rr, cc = np.meshgrid(np.arange(di), np.arange(dj), indexing="ij")
            e = off + rr * dj + cc
            if i != j:
                o_r.append(ps[i] + rr.ravel()); o_c.append(ps[j] + cc.ravel()); o_e.append(e.ravel())
            else:
                low = rr >= cc
                w = int(plan.winv_off[j]) + rr * dj + cc
                d_r.append(ps[j] + rr[low]); d_c.append(ps[j] + cc[low]); d_e.append(e[low]); d_w.append(w[low])
                on_diag.append((rr == cc)[low]); d_up.append(e[~low]); w_up.append(w[~low])
        cat = lambda v: np.concatenate(v).astype(np.int64) if v else np.zeros(0, np.int64)   # noqa: E731
        self.o_r, self.o_c, self.o_e = cat(o_r), cat(o_c), cat(o_e)
        self.d_r, self.d_c, self.d_e, self.d_w, self.d_up, self.w_up = cat(d_r), cat(d_c), cat(d_e), cat(d_w), cat(d_up), cat(w_up)
        self.on_diag = np.concatenate(on_diag)
        self.perm = np.concatenate([np.arange(plan.col_start[j], plan.col_start[j] + dims[j]) for j in range(plan.N)]).astype(np.int64)

    def lower(self, F, Dg, lane):
        """L of one item (F: its factor storage, Dg: its diagonal storage)."""
        n = self.plan.n
        if lane:
            dv = Dg[self.d_w].copy()
            dv[self.on_diag] = 1.0 / dv[self.on_diag]
            assert (Dg[self.w_up] == 0).all()
        else:
            dv = F[self.d_e]
            assert (F[self.d_up] == 0).all()
        return sp.csr_matrix((np.concatenate([F[self.o_e], dv]), (np.concatenate([self.o_r, self.d_r]), np.concatenate([self.o_c, self.d_c]))),
                             shape=(n, n))

    def matrix(self, G, alpha, beta):
        """Symmetric permuted M from one item's Gram storage G (lower blocks at the factor offsets), diagonal damped as the damp kernels
        do it: d (1 + alpha) + beta."""
        n = self.plan.n
        dv = G[self.d_e].copy()
        if alpha is not None:
            dv[self.on_diag] = dv[self.on_diag] * (1.0 + alpha) + beta
        rows, cols = np.concatenate([self.o_r, self.d_r]), np.concatenate([self.o_c, self.d_c])
        Ml = sp.csr_matrix((np.concatenate([G[self.o_e], dv]), (rows, cols)), shape=(n, n))
        return (Ml + sp.triu(Ml.T, 1)).tocsr()


def _check_backward_error_sparse(L, M, kappa, what):
    """_check_backward_error of test_gpu_front_factor.py on scipy.sparse matrices: the same bound |L L^T - M| <= c u kappa |L||L^T|,
    c = 4 (largest row count of L + 2), without n x n products."""
    absL = abs(L)
    E = abs(L @ L.T - M).tocoo()
    R = ((U * kappa) * (absL @ absL.T)).tocsr()
    ref = np.asarray(R[E.row, E.col]).ravel()
    c = 4.0 * (int((L != 0).sum(axis=1).max()) + 2)
    zero = ref == 0
    assert (E.data[zero] == 0).all(), what
    ratio = float((E.data[~zero] / ref[~zero]).max()) if (~zero).any() else 0.0
    assert ratio <= c, (what, ratio, c)
    return ratio


def _solver(S, ordering, layout):
    solver = th.BaspachoSparseSolver.from_structure(S, ordering=ordering, layout=layout)
    return solver


def _solve(solver, A, b, alpha=None, beta=None):
    """add_MtM -> damp -> factor -> solve through the solver's own buffers, with per-item alpha / beta (None: no damping)."""
    A_t, b_t = _cuda(A), _cuda(b)
    solver.linearization.A_val, solver.linearization.b = A_t, b_t
    Atb = solver._numeric(A_t, b_t, _cuda(alpha), _cuda(beta))
    x = solver._substitute(Atb)
    return x.cpu().numpy(), solver._dev["bufs"]["info"].cpu().numpy().copy()


def _buffers(solver, B):
    """factor, diag as [B, ...] numpy arrays (lane: the padded lanes dropped)."""
    bufs = solver._dev["bufs"]
    f, d = bufs["factor"].cpu().numpy(), bufs["diag"].cpu().numpy()
    if bufs["key"][1] == "item":
        return f, d
    return f[:, :B].T.copy(), d[:, :B].T.copy()


def _gram(solver, A, b):
    """The AtA the factorisation read: the same deterministic Gram kernel of the layout, run again into a zeroed buffer ([B, data_size])."""
    d, P = solver._dev, solver._plan
    lib = _lib.load()
    B = A.shape[0]
    A_t, b_t = _cuda(A), _cuda(b)
    if d["bufs"]["key"][1] == "item":
        out = torch.zeros(B, P.data_size, dtype=torch.float64, device=A_t.device)
        atb = torch.empty(B, P.n, dtype=torch.float64, device=A_t.device)
        _lib.check(lib.thb_gram_f64(C.byref(d["gram"]), B, _lib.ptr(A_t), A.shape[1], _lib.ptr(b_t), b.shape[1], _lib.ptr(out), P.data_size,
                                    _lib.ptr(atb), None, _lib.stream_ptr()), "gram")
        return out.cpu().numpy()
    out = torch.zeros(P.data_size, int(lib.thb_sparse_lane_padded_batch(B)), dtype=torch.float64, device=A_t.device)
    _lib.check(lib.thb_sparse_lane_gram_f64(C.byref(d["gram"]), B, _lib.ptr(A_t), A.shape[1], _lib.ptr(out), _lib.stream_ptr()), "lane gram")
    return out.cpu().numpy()[:, :B].T.copy()


def _check_sparse(solver, A, b, alpha, beta, x, items, what):
    """Per item: diag(L) > 0, zeros above the diagonal of the diagonal blocks, W_j L_jj = I (item), the componentwise backward error of
    L against the damped permuted AtA the kernels read, x against numpy.  Returns the largest backward-error ratio."""
    plan = solver._plan
    lane = solver._dev["bufs"]["key"][1] != "item"
    rd = _Reader(plan)
    B = A.shape[0]
    F, Dg = _buffers(solver, B)
    G = _gram(solver, A, b)
    Atb = solver._dev["bufs"]["Atb"].cpu().numpy()
    ps, dims = plan.pstart, plan.dims
    worst = 0.0
    for k in items:
        L = rd.lower(F[k], Dg[k], lane)
        assert (L.diagonal() > 0).all(), (what, k)
        Ld = L.tolil()
        kappa = 0.0
        for j in range(plan.N):
            s, d = int(ps[j]), int(dims[j])
            Ljj = Ld[s:s + d, s:s + d].toarray()
            cj = _cond_inf(Ljj)
            kappa = max(kappa, cj)
            if not lane:
                Wj = Dg[k, int(plan.winv_off[j]):int(plan.winv_off[j]) + d * d].reshape(d, d)
                assert (np.triu(Wj, 1) == 0).all(), (what, k, j)
                res = np.linalg.norm(Wj @ Ljj - np.eye(d), np.inf)
                assert res <= 4 * (d + 2) * U * cj, (what, k, j, res)
        M = rd.matrix(G[k], None if alpha is None else alpha[k], None if beta is None else beta[k])
        worst = max(worst, _check_backward_error_sparse(L, M, kappa, f"{what} item {k}"))
        Mo = np.zeros((plan.n, plan.n))
        Mo[np.ix_(rd.perm, rd.perm)] = M.toarray()
        _check_x(Mo, Atb[k], x[k], (what, k))
    return worst


def _modes(rng, B):
    return {"none": (None, None), "spherical": (np.zeros(B), rng.random(B) * 0.1 + 1e-3),
            "ellipsoidal": (rng.random(B) * 0.1, rng.random(B) * 1e-2 + 1e-6)}


_sparse_worst = {}


def _factor_and_poison(name, layout, B):
    S, ordering = _structure(name)
    solver = _solver(S, ordering, layout)
    assert solver.layout_for(B) == layout
    _assert_structure(name, solver._plan)
    rng = np.random.default_rng(B + len(name))
    A, b, _ = make_inputs(S, B, seed=B)
    for mode, (alpha, beta) in _modes(rng, B).items():
        x, info = _solve(solver, A, b, alpha, beta)
        assert (info == 0).all(), (mode, info)
        r = _check_sparse(solver, A, b, alpha, beta, x, range(B), (name, layout, B, mode))
        _sparse_worst[layout] = max(_sparse_worst.get(layout, 0.0), r)
    print(f"{layout} {name} B {B}: largest |L L^T - M| / (u kappa |L||L^T|) so far {_sparse_worst[layout]:.3g}")
    # the buffers the kernels write before they read, NaN-poisoned: bitwise the same result (factor is zeroed by every call)
    F0, D0 = _buffers(solver, B)
    bufs = solver._dev["bufs"]
    for key in ("diag", "work"):
        bufs[key].fill_(float("nan"))
    x1, info1 = _solve(solver, A, b, alpha, beta)
    F1, D1 = _buffers(solver, B)
    assert (info1 == 0).all() and np.array_equal(x, x1) and np.array_equal(F0, F1) and np.array_equal(D0, D1)
    return solver, S, A, b


ITEM_NAMES = ["mixed", "generic", "chain", "star", "clique"]


@pytest.mark.parametrize("name", ITEM_NAMES)
def test_item_layout_factor_per_item(name):
    """layout='item' (sparse_damp / sparse_factor / sparse_solve kernels), three damping modes, every item; poisoned diag / work."""
    _factor_and_poison(name, "item", 3 if not EMU else 2)


LANE_CASES = [("mixed", 33), ("mixed", 64), ("mixed", 70), ("chain", 70), ("star", 33), ("clique", 64), ("clique", 70)]


@pytest.mark.parametrize("name,B", LANE_CASES)
def test_lane_layout_factor_per_item(name, B):
    """layout='lane' (gram, damp, update, split-K update, trsm, forward / backward kernels), three damping modes, every item (B = 33 and
    70: ragged padded lanes); poisoned diag / work."""
    if EMU and (B != 33 or name == "star"):
        pytest.skip("host emulation: one ragged batch, small structures")
    _factor_and_poison(name, "lane", B)


@pytest.mark.parametrize("layout,name", [("item", "mixed"), ("item", "generic"), ("lane", "mixed"), ("lane", "clique")])
def test_items_are_bitwise_independent_of_the_batch_and_of_failing_items(layout, name):
    """Every item bitwise equal (x, factor, diagonal blocks) to the same item solved alone; then every A_val entry in the columns of one
    variable zeroed in two items (no damping): info of those items is the leading-minor index of the permuted AtA, 0 elsewhere, and the
    healthy items stay bitwise unchanged."""
    B = (37 if layout == "item" else 70) if not EMU else (5 if layout == "item" else 33)
    S, ordering = _structure(name)
    solver = _solver(S, ordering, layout)
    A, b, _ = make_inputs(S, B, seed=3)
    x, info = _solve(solver, A, b)
    assert (info == 0).all()
    F, D = _buffers(solver, B)
    one = _solver(S, ordering, layout)
    for k in range(B) if not EMU else (0, B - 1):
        xk, _ = _solve(one, A[k:k + 1], b[k:k + 1])
        Fk, Dk = _buffers(one, 1)
        assert np.array_equal(xk[0], x[k]) and np.array_equal(Fk[0], F[k]) and np.array_equal(Dk[0], D[k]), k
    plan = solver._plan
    v = int(np.argmax(S.var_dims > 1) + len(S.var_dims) // 2) % len(S.var_dims)
    bad = [2, B - 3]
    A2 = A.copy()
    A2[np.ix_(bad, np.nonzero(var_columns(S, v))[0])] = 0.0
    x2, info2 = _solve(solver, A2, b)
    F2, D2 = _buffers(solver, B)
    AtA, _ = _dense_system(S, torch.from_numpy(A2[bad]), torch.from_numpy(b[bad]))
    perm = _Reader(plan).perm
    for q, k in enumerate(bad):
        assert info2[k] == _first_bad_pivot(AtA[q][np.ix_(perm, perm)]) > 0, (k, info2[k])
    ok = np.setdiff1d(np.arange(B), bad)
    assert (info2[ok] == 0).all(), info2
    assert np.array_equal(x2[ok], x[ok]) and np.array_equal(F2[ok], F[ok]) and np.array_equal(D2[ok], D[ok])


# ================================================================================================ D. the pivot rule
def _pivot_structure():
    """Leaves of dims 1, 2, 3, 6 (repeating) on two hubs, so that all leaves fall in one elimination level / one launch."""
    nl = 80 if not EMU else 24
    sizes = [[1, 6, 2, 3][v % 4] for v in range(nl)] + [6, 6]
    return _vars_structure(sizes, [(v, nl + v % 2) for v in range(nl)]), sizes, nl


def _pivot_pair(layout, sizes, nl, pos):
    """Two leaves (v_lo, v_hi), v_lo eliminated first.  item: v_lo a 1-dof leaf (generic potrf_inv_small<0>, the slow path), v_hi a 6-dof
    leaf (registers) -- the later column is done first; lane / front / dense: two 6-dof leaves (one trsm launch)."""
    leaves = np.arange(nl)
    by_pos = leaves[np.argsort(pos[leaves])]
    six = [int(v) for v in by_pos if sizes[v] == 6]
    if layout == "item":
        one = [int(v) for v in by_pos if sizes[v] == 1]
        return one[0], six[-1]
    return six[0], six[-1]


@pytest.mark.parametrize("ordering", ["natural", "mindeg"])
@pytest.mark.parametrize("layout", ["item", "lane", "front", "dense"])
def test_pivot_rule_two_failing_columns_in_one_launch(layout, ordering):
    """Two zeroed variables whose columns are factored by the same level / launch: info is the 1-based index of the first non-positive
    pivot of the permuted (undamped) AtA, the leading-minor rule of torch.linalg.cholesky, and it is the same in 5 runs."""
    if EMU and layout in ("dense", "front"):
        pytest.skip("host emulation: the dense Cholesky (and the front plan's borderless hub roots) need the DMMA kernel")
    S, sizes, nl = _pivot_structure()
    B = 3
    A, b, _ = make_inputs(S, B, seed=21)
    if layout == "dense":
        pos, perm = np.arange(len(sizes)), np.arange(S.num_cols)
    else:
        solver = th.BaspachoSparseSolver.from_structure(S, ordering=ordering, layout=layout,
                                                        front_options=dict(tau=-1.0, merge_flops=-1.0) if layout == "front" else None)
        plan = solver._plan
        pos = plan.pos
        perm = plan.perm if layout == "front" else _Reader(plan).perm
    v_lo, v_hi = _pivot_pair(layout, sizes, nl, pos)
    if layout in ("item", "lane"):
        assert plan.level[pos[v_lo]] == plan.level[pos[v_hi]] == 0
    elif layout == "front":
        t_lo, t_hi = int(plan.front_of_pos[pos[v_lo]]), int(plan.front_of_pos[pos[v_hi]])
        sched = plan.arrays["sched"]
        same = [r for r in plan.launches if r[1] < 3 and t_lo in sched[r[2]:r[2] + r[3]] and t_hi in sched[r[2]:r[2] + r[3]]]
        assert t_lo != t_hi and len(same) == 1
    A[1, var_columns(S, v_lo) | var_columns(S, v_hi)] = 0.0
    AtA, Atb = _dense_system(S, torch.from_numpy(A), torch.from_numpy(b))
    expect = _first_bad_pivot(AtA[1][np.ix_(perm, perm)])
    assert expect > 0
    got = []
    for _ in range(5):
        if layout == "dense":
            _, _, _, info = _dense(AtA, Atb)
        else:
            _, info = _solve(solver, A, b)
        got.append(info.tolist())
    assert all(g == [0, expect, 0] for g in got), (expect, got)


# ================================================================================================ E. blocks larger than 16 dofs
@pytest.mark.parametrize("B", [4, 40])
def test_default_layout_takes_blocks_larger_than_16(B):
    """A structure with a 20-dof block: the default layout solves it at any batch (the one-CTA-per-item kernels take blocks of at most
    16 dofs, so small batches go to the multifrontal layout too), every item against numpy; an explicit layout='item' is refused."""
    sizes = [6, 20, 3, 6, 1, 20, 2]
    S = _vars_structure(sizes, [(0, 1), (1, 2), (2, 3), (3, 5), (4, 5), (5, 6), (1, 5)])
    solver = th.BaspachoSparseSolver.from_structure(S)
    A, b, alpha = make_inputs(S, B, seed=B)
    solver.linearization.A_val, solver.linearization.b = _cuda(A), _cuda(b)
    x = solver.solve(damping=_cuda(alpha), ellipsoidal_damping=True, damping_eps=1e-6).cpu().numpy()
    assert solver.effective_layout == "front"
    AtA, Atb = _dense_system(S, torch.from_numpy(A), torch.from_numpy(b))
    idx = np.arange(S.num_cols)
    AtA[:, idx, idx] = AtA[:, idx, idx] * (1 + alpha[:, None]) + 1e-6
    for k in range(B):
        _check_x(AtA[k], Atb[k], x[k], k)
    item = th.BaspachoSparseSolver.from_structure(S, layout="item")
    item.linearization.A_val, item.linearization.b = _cuda(A), _cuda(b)
    with pytest.raises(ValueError, match="layout='item'"):
        item.solve()
