"""front_small_kernel runs the forward substitution of a solve on its first warps while its other warps write the panel and form the
update-matrix tiles (taken from a shared counter).  Who computes what must not show: the fused solve is bitwise the two-pass path
(factor only, then the substitution kernels) on structures that put a front into every thread-count instance of the kernel --
among them a borderless front, fronts of fewer than 32 pivots (one elimination chunk), of more than 64 (three and more), and fronts
with more update-matrix tiles than warps -- also after every written buffer was filled with NaN, and with the fusion switched off."""
import numpy as np
import pytest
import torch

import theseus_b200 as th
from front_factor_cases import NO_MERGE, _group_structure, make_inputs, small_structure
from test_gpu_front_fused_forward import run_fused, run_two_pass, same_bits

pytestmark = pytest.mark.gpu
EPS_DAMP = 1e-6


def wide_border_structure():
    """Fronts whose update matrix has many more 16 x 16 tiles than the CTA has warps: borders of 162 rows (66 tiles) under a root of
    162 pivots, with 16, 48 and 72 pivots (one, two and three elimination chunks)."""
    root = [1, 1] + [8] * 20
    everything = list(range(len(root)))
    groups = [([8] * 2, 3, everything),    # w 16, b 162
              ([8] * 6, 3, everything),    # w 48, b 162
              ([8] * 9, 3, everything),    # w 72, b 162
              (root, -1, None)]
    return _group_structure(groups)


STRUCTURES = {"small": small_structure, "wide_border": wide_border_structure}


def make(name, chunk):
    S, _ = STRUCTURES[name]()
    opts = dict(NO_MERGE) if chunk is None else dict(NO_MERGE, chunk=chunk)
    solver = th.BaspachoSparseSolver.from_structure(S, layout="front", ordering="natural", front_options=opts)
    return solver, S


def cta_threads(plan):
    """Threads per CTA of every shared-memory front (front_factor's choice from the launch's class and shared-memory size)."""
    out = {}
    for depth, cls, s0, cnt, smem in plan.launches[:, :5]:
        if cls < 3:
            thr = 64 if cls == 0 else 128 if cls == 1 else 256 if smem <= 56 * 1024 else 512 if smem <= 113 * 1024 else 1024
            for t in plan.arrays["sched"][s0:s0 + cnt]:
                out[int(t)] = thr
    return out


def test_the_structures_reach_every_instance_and_shape():
    seen, shapes = set(), []
    for name in STRUCTURES:
        plan = make(name, None)[0]._plan
        thr = cta_threads(plan)
        seen |= set(thr.values())
        shapes += [(int(plan.arrays["f_w"][t]), int(plan.arrays["f_b"][t]), thr[t]) for t in thr]
    assert seen == {64, 128, 256, 512, 1024}, seen
    assert any(b == 0 for w, b, _ in shapes)
    assert any(w < 32 and b > 0 for w, b, _ in shapes) and any(w > 64 and b > 0 for w, b, _ in shapes)
    # more tiles than warps, with one, two and three elimination chunks
    for lo, hi in ((1, 32), (33, 64), (65, 96)):
        assert any(lo <= w <= hi and ((b + 15) // 16) * ((b + 15) // 16 + 1) // 2 > thr // 32 for w, b, thr in shapes), (lo, hi, shapes)


def inputs(S, B, seed):
    A, b, alpha = make_inputs(S, B, seed)
    return (torch.from_numpy(A).cuda(), torch.from_numpy(b).cuda(), torch.from_numpy(alpha).cuda(),
            torch.full((B,), EPS_DAMP, dtype=torch.float64, device="cuda"))


@pytest.mark.parametrize("name", sorted(STRUCTURES))
@pytest.mark.parametrize("B,chunk", [(1, None), (37, 16)])
def test_overlapped_phases_are_bitwise_the_two_pass_path(name, B, chunk):
    solver, S = make(name, chunk)
    args = inputs(S, B, seed=3 + B)
    fused = run_fused(solver, *args)
    two = run_two_pass(solver, *args)
    assert (fused[3] == 0).all()
    for what, u, v in zip(("factor", "y", "x", "info"), fused, two):
        assert torch.equal(u, v), what
    # and what they agree on is the solution: A^T A (1 + alpha) + beta on the diagonal, against a dense solve per item
    A, b, al, be = (v.cpu().numpy() for v in args)
    for k in range(0, B, 9):
        Ad = np.zeros((S.num_rows, S.num_cols))
        Ad[np.repeat(np.arange(S.num_rows), np.diff(S.A_row_ptr)), S.A_col_ind] = A[k]
        H = Ad.T @ Ad
        H[np.diag_indices_from(H)] += al[k] * np.diag(H) + be[k]
        x, g = fused[2][k].cpu().numpy(), Ad.T @ b[k]
        assert np.linalg.norm(H @ x - g) <= 1e-10 * (np.linalg.norm(H, 2) * np.linalg.norm(x) + np.linalg.norm(g))


@pytest.mark.parametrize("name", sorted(STRUCTURES))
def test_overlapped_phases_write_everything_they_own(name):
    """Fused solve, every buffer the kernels write filled with NaN, fused solve again: bitwise the same, no NaN left in what is read."""
    B, chunk = 37, 16
    solver, S = make(name, chunk)
    args = inputs(S, B, seed=17)
    r0 = run_fused(solver, *args)
    bufs = solver._dev["bufs"]
    for k in ("factor", "arena", "varena", "work"):
        bufs[k].fill_(float("nan"))
    r1 = run_fused(solver, *args)
    two = run_two_pass(solver, *args)
    for what, u, v, z in zip(("factor", "y", "x", "info"), r0, r1, two):
        assert torch.equal(u, v) and torch.equal(u, z), what
    assert not torch.isnan(r1[2]).any()


def test_without_the_fusion_the_result_is_the_same(tmp_path):
    """THB_FRONT_FUSE_MAX=0 (read once per process, so in a child process): every front's forward substitution runs in the substitution
    kernel after the factor kernel; x and the factor are bitwise those of the default run."""
    from test_gpu_front_factor import _run_cases
    ref = _run_cases(str(tmp_path / "default"), {})
    got = _run_cases(str(tmp_path / "unfused"), {"THB_FRONT_FUSE_MAX": "0"})
    assert sorted(got) == sorted(ref) and len(ref) > 0
    for f, v in ref.items():
        assert same_bits(torch.from_numpy(got[f]), torch.from_numpy(v)), f
