"""NOT COLLECTED by the suite (no test_ prefix): the structures of tests/test_gpu_front_factor.py, and -- run as a script -- one solve of
two of them whose solution and factor are saved as .npy files:

    python tests/front_factor_cases.py OUT_DIR

test_gpu_front_factor.py runs the script in child processes, once per environment of the multifrontal kernels' tuning knobs
(THB_SOLVE_STAGE, THB_FRONT_T0 / _T1 / _PREFETCH / _PDL are read once per process).  With THB_SIMT_EMULATION=1 it runs on the host
emulation and solves the small-front structure only (the emulation has no DMMA dense kernel)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# no relaxed amalgamation: with natural ordering every group of _group_structure becomes exactly one front
NO_MERGE = dict(tau=-1.0, merge_flops=-1.0)


def _group_structure(groups):
    """groups: (variable dims, parent group or -1, indices of the parent's variables the group is coupled to), children before parents.
    Each group is one dense cost over its variables, a second dense cost couples it to the chosen variables of its parent, and every
    variable has a unary cost (so AtA is positive definite).  With natural ordering and NO_MERGE every group is one front: w = its dofs,
    border = the chosen parent variables.  Every coupled set holds the parent's variable 0, so that the parent stays one supernode.
    Returns (structure, first variable of every group)."""
    from theseus_b200.structure import build_structure
    var_dims, first = [], []
    for dims, _, _ in groups:
        first.append(len(var_dims))
        var_dims += list(dims)
    costs = []
    for g, (dims, parent, coupled) in enumerate(groups):
        vs = list(range(first[g], first[g] + len(dims)))
        if len(vs) > 1:
            costs.append((3, vs))
        if parent >= 0:
            assert coupled[0] == 0
            costs.append((2, vs + [first[parent] + c for c in coupled]))
    costs += [(d + 2, [v]) for v, d in enumerate(var_dims)]
    return build_structure(var_dims, costs), first


def small_structure():
    """Shared-memory fronts only.  Root: 104 pivots, borderless, exactly 8 children (gather).  Its children: class 2 fronts whose shared
    memory falls in each thread-count band (24 x 80, 64 x 48, 96 x 80), a 15-pivot front of 1-, 2-, 3- and 7-dof variables with b = 1,
    fronts with b = 15, 16, 33 and 50 (class 1)."""
    root = [1, 1, 7, 7] + [8] * 11
    R = 8
    groups = [
        ([6] * 4, R, [0, 2] + list(range(4, 13))),    # w 24, b 80
        ([8] * 8, R, [0, 2] + list(range(4, 9))),     # w 64, b 48
        ([6] * 16, R, [0, 2] + list(range(4, 13))),   # w 96, b 80
        ([1, 2, 1, 3, 7, 1], R, [0]),                 # w 15, b 1
        ([7], R, [0, 2, 3]),                          # w 7, b 15
        ([3], R, [0, 1, 2, 3]),                       # w 3, b 16
        ([2], R, [0, 4, 5, 6, 7]),                    # w 2, b 33
        ([1, 2], R, [0, 1] + list(range(4, 10))),     # w 3, b 50
        (root, -1, None),
    ]
    return _group_structure(groups)


def big_structure():
    """Run with small_limit=60: big fronts (assembled in global memory, factored by the DMMA kernel in partial mode).  Borderless big root
    of 70 pivots (padded to 128, like config C5's root) with 8 children; a big child with 9 children (scatter assembly) of which one is
    big (80 pivots: np = 256); a small child whose own child is big."""
    Q, P1, BR = 7, 17, 18
    groups = [([5] * 10, Q, [0, 1, 2, 3])]                     # 0: w 50, b 20: big child of a small parent
    groups += [([2], BR, [0, k]) for k in range(1, 7)]         # 1-6: small leaves of the root
    groups += [([5] * 4, BR, [0, 1, 2, 3, 4])]                 # 7 (Q): w 20, b 25: small child of a big parent
    groups += [([8] * 10, P1, list(range(7)))]                 # 8: w 80, b 25: big child of a big parent
    groups += [([3], P1, [0, k]) for k in range(1, 9)]         # 9-16: small children of P1
    groups += [([1] + [4] * 11, BR, list(range(7)))]           # 17 (P1): w 45, b 37, 9 children
    groups += [([1] + [6] * 11 + [3], -1, None)]               # 18 (BR): w 70, b 0, 8 children
    return _group_structure(groups)


def wide_structure():
    """Run with split_wide=False: fronts of SMALL_MAX_W and SMALL_MAX_W + 1 pivots under a small parent."""
    groups = [([6] * 32, 3, [0, 1, 2]),          # w 192
              ([6] * 32 + [1], 3, [0, 3]),       # w 193
              ([6] * 4, 3, [0, 1]),
              ([6] * 5, -1, None)]
    return _group_structure(groups)


CASES = {   # name -> (structure builder, front_options without chunk)
    "small": (small_structure, dict(NO_MERGE)),
    "big": (big_structure, dict(NO_MERGE, small_limit=60)),
    "wide": (wide_structure, dict(NO_MERGE, split_wide=False)),
}


def make_solver(name, chunk=None):
    import theseus_b200 as th
    build, opts = CASES[name]
    S, first = build()
    if chunk is not None:
        opts = dict(opts, chunk=chunk)
    return th.BaspachoSparseSolver.from_structure(S, layout="front", ordering="natural", front_options=opts), S, first


def make_inputs(S, B, seed, small_var=None):
    """A_val, b, alpha (numpy): item k scaled by 10^((k % 7) - 3), the columns of variable `small_var` by a further 1e-4."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((B, S.nnz)) * (10.0 ** ((np.arange(B) % 7) - 3))[:, None]
    if small_var is not None:
        A[:, var_columns(S, small_var)] *= 1e-4
    return A, rng.standard_normal((B, S.num_rows)), rng.random(B) * 0.1


def var_columns(S, v):
    """Mask of the A_val entries in the columns of variable v."""
    c0 = int(np.sum(S.var_dims[:v]))
    return (S.A_col_ind >= c0) & (S.A_col_ind < c0 + int(S.var_dims[v]))


def panel_entries(plan):
    """Offsets of the entries of one item's factor that belong to a panel (the alignment gaps between panels are never written)."""
    A = plan.arrays
    return np.concatenate([int(A["f_panel_off"][t]) + np.arange(int(A["f_w"][t]) * (int(A["f_w"][t]) + int(A["f_b"][t])))
                           for t in range(plan.S)])


def main(out_dir):
    if os.environ.get("THB_SIMT_EMULATION") == "1":
        import importlib.util
        spec = importlib.util.spec_from_file_location("emulation_mode", os.path.join(HERE, "simt", "emulation_mode.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.enable()
    import torch
    emu = os.environ.get("THB_SIMT_EMULATION") == "1"
    B, chunk = (3, 2) if emu else (33, 16)
    for name in (["small"] if emu else ["small", "big"]):
        solver, S, _ = make_solver(name, chunk=chunk)
        A, b, alpha = make_inputs(S, B, 7)
        solver.linearization.A_val, solver.linearization.b = torch.from_numpy(A).cuda(), torch.from_numpy(b).cuda()
        x = solver.solve(damping=torch.from_numpy(alpha).cuda(), ellipsoidal_damping=True, damping_eps=1e-6)
        np.save(os.path.join(out_dir, f"{name}_x.npy"), x.cpu().numpy())
        np.save(os.path.join(out_dir, f"{name}_factor.npy"), solver._dev["bufs"]["factor"].cpu().numpy()[:, panel_entries(solver._plan)])


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, HERE)
    main(sys.argv[1])
