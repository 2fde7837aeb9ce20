"""Cases shared by the staged-Gram tests (tests/test_gpu_gram_staged.py on the device, tests/test_gram_staged_emulation.py on the host
emulation): structures, the four output layouts thb_gram_f64 / _f32 serve, one call of the library on a plan, and the float64 check."""
import ctypes as C

import numpy as np
import scipy.sparse as sp
import torch

import theseus_b200 as th
from theseus_b200 import _lib
from theseus_b200.structure import build_gram_plan, build_structure

NP = {torch.float64: np.float64, torch.float32: np.float32}
SFX = {torch.float64: "f64", torch.float32: "f32"}


def mixed_structure():
    """Block dims 1, 2, 3, 6 and 7; a chain of binary costs, long-range binary costs, a three-variable cost, a unary cost on every
    variable, and a 12-row cost over the 7- and 6-dim variables (168 staged scalars: more than one pass of a warp's copy loop)."""
    dims = [1, 2, 3, 6, 7, 6, 2, 3, 1, 6, 7, 3]
    rng = np.random.default_rng(7)
    N = len(dims)
    costs = [(int(rng.integers(1, 8)), [i, i + 1]) for i in range(N - 1)]
    costs += [(int(rng.integers(1, 8)), [j, i]) for i, j in ((0, 9), (2, 11), (4, 10), (1, 6))]
    costs += [(5, [3, 8, 10]), (12, [4, 3])]
    costs += [(int(dims[v]), [v]) for v in range(N)]
    return build_structure(dims, costs)


def c5_structure():
    """The bench's headline pose graph (2 500 SE3 poses on a sphere, 4 949 Between costs, a prior on pose 0)."""
    from bench import C5_PER_RING, C5_RINGS
    from theseus_b200.datasets import pose_graph_sphere
    E = np.asarray(pose_graph_sphere(C5_RINGS, C5_PER_RING, 1, seed=1000, device="cpu")["edges"])
    return build_structure([6] * (C5_RINGS * C5_PER_RING), [(6, [int(i), int(j)]) for i, j in E] + [(6, [0])])


def layouts(S, B, names=("dense", "front", "item", "atb")):
    """name -> (plan arrays, output scalars per item or None for Atb / diag only)."""
    out = {}
    for name in names:
        if name in ("dense", "atb"):
            out[name] = (build_gram_plan(S), S.num_cols ** 2 if name == "dense" else None)
        else:
            solver = th.BaspachoSparseSolver.from_structure(S, layout=name)
            solver.layout_for(B)
            out[name] = (solver._gram_arrays, solver._ata_size if name == "front" else solver._plan.data_size)
    return out


def fallback_of(arrs):
    """The same plan without groups or shape segments: thb_gram_* runs the entry-per-thread kernels (gram_kernel, atb_kernel) on it."""
    return dict(arrs, num_groups=0, segments=np.zeros((0, 4), dtype=np.int32))


def block_fallback_of(arrs):
    """The same plan without groups: thb_gram_* runs the block-per-thread kernels when the plan has shape segments."""
    return dict(arrs, num_groups=0)


def run_gram(fn, arrs, A, b, out_size, dtype, device):
    """One call of `fn` (thb_gram_f64 / _f32 of a library) on NaN-filled outputs; returns (out or None, Atb, diag) as numpy."""
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in arrs.items() if isinstance(v, np.ndarray)}
    plan = _lib.make_gram_plan(arrs, dev)
    B, n = A.shape[0], int(arrs["n"])
    At, bt = torch.from_numpy(A).to(device), torch.from_numpy(b).to(device)
    out = torch.full((B, out_size), float("nan"), dtype=dtype, device=device) if out_size is not None else None
    Atb = torch.full((B, n), float("nan"), dtype=dtype, device=device)
    diag = torch.full((B, n), float("nan"), dtype=dtype, device=device)
    _lib.check(fn(C.byref(plan), B, _lib.ptr(At), A.shape[1], _lib.ptr(bt), b.shape[1], _lib.ptr(out) if out is not None else None,
                  out_size or 0, _lib.ptr(Atb), _lib.ptr(diag), _lib.stream_ptr() if device != "cpu" else None), "gram")
    if device != "cpu":
        torch.cuda.synchronize()
    return tuple(None if x is None else x.cpu().numpy() for x in (out, Atb, diag))


def same_bits(x, y):
    return x is None and y is None or (x.shape == y.shape and x.tobytes() == y.tobytes())


def check_oracle(S, arrs, A_val, b, out, Atb, diag, rtol):
    """Every block of the plan, A^T b and diag(A^T A) against float64 scipy.sparse products of the same (rounded) inputs, item by
    item: |got - ref| <= rtol * (|A|^T |A|) componentwise (resp. |A|^T |b|, and A^T A's diagonal); mirrored blocks bitwise equal."""
    n = S.num_cols
    rows, cols, pos, mpos = [], [], [], []
    c0 = S.var_start_cols
    for k, (i, j) in enumerate(arrs["blocks"]):
        di, dj = int(S.var_dims[i]), int(S.var_dims[j])
        ld, off, mo = int(arrs["blk_ld"][k]), int(arrs["blk_out"][k]), int(arrs["blk_mirror"][k])
        p, q = np.meshgrid(np.arange(di), np.arange(dj), indexing="ij")
        rows.append((c0[i] + p).ravel()); cols.append((c0[j] + q).ravel()); pos.append((off + p * ld + q).ravel())
        mpos.append((mo + q * ld + p).ravel() if mo >= 0 else np.full(di * dj, -1))
    rows, cols, pos, mpos = (np.concatenate(x) if x else np.zeros(0, np.int64) for x in (rows, cols, pos, mpos))
    for bi in range(A_val.shape[0]):
        M = sp.csr_matrix((A_val[bi].astype(np.float64), S.A_col_ind, S.A_row_ptr), shape=(S.num_rows, n))
        Ma = abs(M)
        bb = b[bi].astype(np.float64)
        if out is not None:
            G, Ga = (M.T @ M).tocsr(), (Ma.T @ Ma).tocsr()
            ref, tol = np.asarray(G[rows, cols]).ravel(), np.asarray(Ga[rows, cols]).ravel()
            got = out[bi, pos].astype(np.float64)
            assert (np.abs(got - ref) <= rtol * tol).all(), (bi, np.abs(got - ref).max())
            m = mpos >= 0
            assert out[bi, mpos[m]].tobytes() == out[bi, pos[m]].tobytes()
        assert (np.abs(Atb[bi] - M.T @ bb) <= rtol * (Ma.T @ np.abs(bb))).all()
        sq = np.asarray(M.multiply(M).sum(0)).ravel()
        assert (np.abs(diag[bi] - sq) <= rtol * sq).all()
