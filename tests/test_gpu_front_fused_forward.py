"""The forward substitution fused into the multifrontal factorisation (thb_front_factor_forward_f64, then thb_front_backward_f64) against
the two-pass path (thb_front_factor_f64, then thb_front_forward_f64 / thb_front_solve_f64): bitwise the same factor panels, y, x and
info -- on the structures of tests/front_factor_cases.py (every kernel path of the factorisation) and config C5, with a failing item,
after the buffers were filled with NaN, and for _substitute() of another right-hand side after a fused solve.

Under the host emulation (THB_SIMT_EMULATION=1) the small structure runs; tests/test_front_fused_forward_emulation.py runs the same
comparison on the emulation as part of the CPU suite."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import theseus_b200 as th
from theseus_b200 import _lib
from front_factor_cases import make_inputs, make_solver, panel_entries, var_columns

pytestmark = pytest.mark.gpu
EMU = os.environ.get("THB_SIMT_EMULATION") == "1"
EPS_DAMP = 1e-6


def same_bits(a, b):
    """Bitwise equal, NaN payloads aside (a NaN matches any NaN: the failing items' x are NaN on both paths)."""
    a, b = a.detach().cpu(), b.detach().cpu()
    if a.dtype == torch.float64:
        return bool(((a.view(torch.int64) == b.view(torch.int64)) | (torch.isnan(a) & torch.isnan(b))).all())
    return torch.equal(a, b)


def _forward_only(solver, rhs):
    """y = L^-1 rhs with the factor of the last _numeric call (thb_front_forward_f64, chunk by chunk); returns work."""
    d, bufs, lib = solver._dev, solver._dev["bufs"], _lib.load()
    B, chunk = bufs["key"][0], bufs["chunk"]
    L = d["launches"]
    for c0 in range(0, B, chunk):
        nb = min(chunk, B - c0)
        _lib.check(lib.thb_front_forward_f64(C.byref(d["front"]), L.ctypes.data, L.shape[0], _lib.ptr(bufs["factor"][c0:]), _lib.ptr(rhs[c0:]),
                                             _lib.ptr(bufs["work"][c0:]), _lib.ptr(bufs["varena"]), nb, _lib.stream_ptr()), "front_forward")
    return bufs["work"]


def run_fused(solver, A, b, alpha, beta):
    """Gram + factor with the fused forward substitution of A^T b, then the backward pass: (factor panels, y, x, info)."""
    solver._numeric_front(A, b, alpha, beta, forward=True)
    bufs = solver._dev["bufs"]
    y = bufs["work"].clone()
    x = solver._backward_front()
    used = torch.from_numpy(panel_entries(solver._plan)).to(x.device)
    return bufs["factor"][:, used].clone(), y, x, bufs["info"].clone()


def run_two_pass(solver, A, b, alpha, beta):
    """Gram + factor only, then the forward pass alone (y) and thb_front_solve_f64 (both passes, x): (factor panels, y, x, info)."""
    Atb = solver._numeric_front(A, b, alpha, beta)
    bufs = solver._dev["bufs"]
    y = _forward_only(solver, Atb).clone()
    x = solver._substitute(Atb)
    used = torch.from_numpy(panel_entries(solver._plan)).to(x.device)
    return bufs["factor"][:, used].clone(), y, x, bufs["info"].clone()


def compare_paths(solver, S, B, seed, device, bad_var=None):
    """The fused and the two-pass path on the same inputs, damped; then undamped with item B // 2 made not positive definite
    (the columns of variable bad_var zeroed).  Returns the info of the undamped run."""
    A, b, alpha = make_inputs(S, B, seed)
    At, bt = torch.from_numpy(A).to(device), torch.from_numpy(b).to(device)
    al = torch.from_numpy(alpha).to(device)
    be = torch.full((B,), EPS_DAMP, dtype=torch.float64, device=device)
    info = None
    for damped in (True, False):
        if not damped and bad_var is not None:
            A2 = A.copy()
            A2[B // 2, var_columns(S, bad_var)] = 0.0
            At = torch.from_numpy(A2).to(device)
        args = (At, bt, al, be) if damped else (At, bt, None, None)
        fused = run_fused(solver, *args)
        two = run_two_pass(solver, *args)
        for what, u, v in zip(("factor", "y", "x", "info"), fused, two):
            assert same_bits(u, v), (what, damped)
        info = fused[3].cpu().numpy()
        if damped:
            assert (info == 0).all(), info
            # the public entry point takes the fused path: the same x
            solver.linearization.A_val, solver.linearization.b = At, bt
            xs = solver.solve(damping=al, ellipsoidal_damping=True, damping_eps=EPS_DAMP)
            x_ref = run_two_pass(solver, *solver._keep)[2]
            assert same_bits(xs, x_ref)
    return info


CASES = [("small", 1, None), ("small", 33, 16), ("small", 130, 64),
         ("big", 1, None), ("big", 33, 16), ("big", 130, 64),
         ("wide", 1, None), ("wide", 33, 16), ("wide", 130, 64)]


@pytest.mark.parametrize("name,B,chunk", CASES)
def test_fused_forward_is_bitwise_the_two_pass_path(name, B, chunk):
    if EMU and (name != "small" or B > 1):
        pytest.skip("host emulation: small fronts and small batches only")
    solver, S, first = make_solver(name, chunk=chunk)
    if chunk is not None:
        assert chunk < B
    info = compare_paths(solver, S, B, seed=B + 3 * len(name), device="cuda", bad_var=first[0])
    assert info[B // 2] > 0 and (np.delete(info, B // 2) == 0).all(), info


@pytest.mark.skipif(EMU, reason="the host emulation has no DMMA dense kernel")
def test_fused_forward_c5_at_a_small_batch():
    """Config C5's pose graph (borderless 462-pivot root on the dense path) at batch 3 in chunks of 2."""
    from helpers import load, pgo_objective
    objective, _ = pgo_objective(th, load("pgo_c5_lm"))
    S = th.BaspachoSparseSolver(objective).linearization.structure()
    solver = th.BaspachoSparseSolver.from_structure(S, layout="front", front_options=dict(chunk=2))
    assert (solver._plan.launches[:, 1] == 3).any()
    compare_paths(solver, S, 3, seed=5, device="cuda")


@pytest.mark.parametrize("name", ["small", "big"])
def test_fused_forward_with_poisoned_buffers(name):
    """Fused solve, every buffer the kernels write before they read filled with NaN, fused solve again: bitwise the same."""
    if EMU and name != "small":
        pytest.skip("host emulation: no DMMA dense kernel")
    B, chunk = (33, 16) if not EMU else (3, 2)
    solver, S, _ = make_solver(name, chunk=chunk)
    A, b, alpha = make_inputs(S, B, seed=11)
    args = (torch.from_numpy(A).cuda(), torch.from_numpy(b).cuda(), torch.from_numpy(alpha).cuda(),
            torch.full((B,), EPS_DAMP, dtype=torch.float64, device="cuda"))
    r0 = run_fused(solver, *args)
    bufs = solver._dev["bufs"]
    for k in ("factor", "arena", "varena", "work"):
        bufs[k].fill_(float("nan"))
    if solver._dev["max_np"]:
        bufs["ws"][:chunk * (solver._dev["max_np"] // 64) * 64 * 64 * 8].view(torch.float64).fill_(float("nan"))
    r1 = run_fused(solver, *args)
    for what, u, v in zip(("factor", "y", "x", "info"), r0, r1):
        assert torch.equal(u, v), what


@pytest.mark.parametrize("name", ["small", "big"])
def test_substitute_after_a_fused_solve(name):
    """After a fused solve, _substitute(other rhs) (both passes, what autograd's backward calls) is the two-pass answer."""
    if EMU and name != "small":
        pytest.skip("host emulation: no DMMA dense kernel")
    B, chunk = (33, 16) if not EMU else (3, 2)
    solver, S, _ = make_solver(name, chunk=chunk)
    A, b, alpha = make_inputs(S, B, seed=13)
    solver.linearization.A_val, solver.linearization.b = torch.from_numpy(A).cuda(), torch.from_numpy(b).cuda()
    solver.solve(damping=torch.from_numpy(alpha).cuda(), ellipsoidal_damping=True, damping_eps=EPS_DAMP)
    rhs = torch.from_numpy(np.random.default_rng(2).standard_normal((B, S.num_cols))).cuda()
    x1 = solver._substitute(rhs)
    A64, b64, al, be = solver._keep
    solver._numeric(A64, b64, al, be)
    x2 = solver._substitute(rhs)
    assert torch.equal(x1, x2)


@pytest.mark.skipif(EMU, reason="host emulation: no prefetch")
def test_update_matrix_prefetch_does_not_change_the_arithmetic(tmp_path):
    """The L2 prefetch of the children's update matrices is off by default; switched on (THB_FRONT_PREFETCH=1, read once per process,
    so in a child process) it only changes where data sits: x and the factor of the fused solve are bitwise those of the default run."""
    from test_gpu_front_factor import _run_cases
    ref = _run_cases(str(tmp_path / "default"), {})
    got = _run_cases(str(tmp_path / "prefetch"), {"THB_FRONT_PREFETCH": "1"})
    assert sorted(got) == sorted(ref)
    for f, v in ref.items():
        assert np.array_equal(got[f], v), f
