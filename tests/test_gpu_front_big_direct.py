"""Big fronts factored straight into their panel: the dense kernel gathers each tile of the front matrix from AtA and the children's update
matrices, stores the pivot columns' L in the front's panel and reads its operands back from there.  The reference is the assembled form
(THB_FRONT_BIG_DIRECT=0: front_assemble_kernel, the in-place partial factorisation, front_extract_kernel): the factor buffer, the solution
and the not-positive-definite report must be bitwise equal to it, for every ticket group size (THB_CHOL_GROUP), batch size and chunk size.

The "big" structure of front_factor_cases.py has every case: a borderless root with pivot padding (config C5's root), big fronts with a
border whose parent reads their update matrix, odd and non-multiple-of-64 pivot counts, a front with 9 children."""
import os

import numpy as np
import pytest
import torch

from front_factor_cases import make_inputs, make_solver, panel_entries, var_columns
from test_gpu_front_factor import EPS_DAMP, _check_factor, _check_solution

pytestmark = pytest.mark.gpu


def _env(**kv):
    """Set the given environment variables (None: unset); returns the previous values.  The library reads both knobs at every call."""
    old = {k: os.environ.get(k) for k in kv}
    for k, v in kv.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = str(v)
    return old


def _solve_with(solver, S, A, b, alpha, **env):
    old = _env(**env)
    try:
        solver.linearization.A_val, solver.linearization.b = torch.from_numpy(A).cuda(), torch.from_numpy(b).cuda()
        x = solver.solve(damping=torch.from_numpy(alpha).cuda(), ellipsoidal_damping=True, damping_eps=EPS_DAMP).clone()
        torch.cuda.synchronize()
        used = torch.from_numpy(panel_entries(solver._plan)).to(x.device)
        return x, solver._dev["bufs"]["factor"][:, used].clone()
    finally:
        _env(**old)


def _bits(t):
    return t.contiguous().view(torch.int64)


def test_the_big_structure_has_every_case():
    solver, _, _ = make_solver("big")
    A = solver._plan.arrays
    big, w, b = A["f_class"] == 3, A["f_w"].astype(int), A["f_b"].astype(int)
    nch, par = np.diff(A["child_ptr"]), A["f_parent"]
    assert (big & (b == 0) & (w % 64 != 0)).any()
    assert (big & (b > 0) & (par >= 0)).any()
    assert (big & (w % 2 == 1)).any()
    assert (big & (nch > 8)).any()


@pytest.mark.parametrize("group", [None, 1, 3, 16, 1 << 20])
def test_direct_is_bitwise_the_assembled_form(group):
    B, chunk = 37, 16
    solver, S, first = make_solver("big", chunk=chunk)
    A, b, alpha = make_inputs(S, B, seed=11, small_var=first[-1] + 1)
    x_ref, f_ref = _solve_with(solver, S, A, b, alpha, THB_FRONT_BIG_DIRECT=0, THB_CHOL_GROUP=group)
    x, f = _solve_with(solver, S, A, b, alpha, THB_FRONT_BIG_DIRECT=None, THB_CHOL_GROUP=group)
    assert torch.equal(_bits(f), _bits(f_ref))
    assert torch.equal(_bits(x), _bits(x_ref))
    _check_factor(solver, alpha, np.full(B, EPS_DAMP), range(B))
    _check_solution(S, A, b, alpha, x.cpu().numpy())


def test_direct_is_independent_of_the_batch_and_chunk_size():
    B = 21
    solver, S, first = make_solver("big", chunk=8)
    A, b, alpha = make_inputs(S, B, seed=4)
    x, f = _solve_with(solver, S, A, b, alpha, THB_CHOL_GROUP=3)
    one, _, _ = make_solver("big")
    for k in range(B):
        xk, fk = _solve_with(one, S, A[k:k + 1], b[k:k + 1], alpha[k:k + 1])
        assert torch.equal(_bits(xk[0]), _bits(x[k])), k
        assert torch.equal(_bits(fk[0]), _bits(f[k])), k


@pytest.mark.parametrize("group,var", [(17, 0), (8, 9), (18, 5)])
def test_not_positive_definite_pivot_is_the_assembled_forms(group, var):
    """A variable of a big front made singular in two items: the same items and the same pivot index as the assembled form."""
    B = 9
    solver, S, first = make_solver("big", chunk=4)
    A, b, alpha = make_inputs(S, B, seed=2)
    for k in (1, 6):
        A[k, var_columns(S, first[group] + var)] = 0.0
    alpha[:] = 0.0
    solver.defer_info_check = True
    infos = []
    for direct in (0, None):
        old = _env(THB_FRONT_BIG_DIRECT=direct)
        try:
            solver.linearization.A_val, solver.linearization.b = torch.from_numpy(A).cuda(), torch.from_numpy(b).cuda()
            solver.solve()
            infos.append(solver._last_info.cpu().numpy().copy())
        finally:
            _env(**old)
    assert (infos[0][[1, 6]] > 0).all() and (np.delete(infos[0], [1, 6]) == 0).all(), infos[0]
    assert np.array_equal(infos[0], infos[1]), infos
