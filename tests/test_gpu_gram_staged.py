"""The staged Gram kernel (theseus_b200/csrc/thb_gram.cu: gram_staged_kernel) on the device, on every output layout thb_gram_f64 /
_f32 serves: the multifrontal solver's compact AtA, the dense n x n AtA with mirrored blocks, the item layout's factor storage, and
Atb / diag alone.  Each output -- blocks, Atb, diag -- must be bitwise what the entry-per-thread kernels (gram_kernel, atb_kernel)
give on the same plan, and within 1e-12 (fp64) of float64 scipy.  Plans whose groups do not fit the shared-memory budget take the
block-per-thread or the entry-per-thread kernels, with the same bits."""
import numpy as np
import pytest
import torch

from theseus_b200 import _lib
from theseus_b200.structure import build_gram_plan, build_structure

from gram_staged_cases import (NP, SFX, block_fallback_of, c5_structure, check_oracle, fallback_of, layouts, mixed_structure, run_gram,
                               same_bits)

DEV = "cuda:0"
DTYPES = [torch.float64, torch.float32]


def _compare(S, arrs, size, B, dtype, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((B, S.nnz)).astype(NP[dtype])
    b = rng.standard_normal((B, S.num_rows)).astype(NP[dtype])
    fn = getattr(_lib.load(), f"thb_gram_{SFX[dtype]}")
    got = run_gram(fn, arrs, A, b, size, dtype, DEV)
    ref = run_gram(fn, fallback_of(arrs), A, b, size, dtype, DEV)
    for name, g, r in zip(("AtA", "Atb", "diag"), got, ref):
        assert same_bits(g, r), name
    check_oracle(S, arrs, A, b, *got, rtol=1e-12 if dtype == torch.float64 else 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("layout", ["dense", "front", "item", "atb"])
@pytest.mark.parametrize("B", [1, 33])
def test_staged_gram_mixed(layout, B, dtype):
    S = mixed_structure()
    arrs, size = layouts(S, B, (layout,))[layout]
    assert arrs["num_groups"] >= 1
    _compare(S, arrs, size, B, dtype, seed=B)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("budget", [600, 900])
def test_staged_gram_mixed_several_groups(budget, dtype):
    S = mixed_structure()
    arrs = build_gram_plan(S, stage_budget=budget)
    assert arrs["num_groups"] >= 2
    _compare(S, arrs, S.num_cols ** 2, 5, dtype, seed=budget)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("layout", ["front", "item", "atb"])
def test_staged_gram_c5(layout, dtype):
    """The bench's pose graph at batch 3 (its dense n x n AtA would be 1.8 GB per item); the block-per-thread kernels that serve the
    same plan without groups give the same bits too."""
    S = c5_structure()
    arrs, size = layouts(S, 3, (layout,))[layout]
    assert arrs["num_groups"] > 100 and len(arrs["segments"]) == 1
    _compare(S, arrs, size, 3, dtype, seed=5)
    rng = np.random.default_rng(6)
    A = rng.standard_normal((3, S.nnz)).astype(NP[dtype])
    b = rng.standard_normal((3, S.num_rows)).astype(NP[dtype])
    fn = getattr(_lib.load(), f"thb_gram_{SFX[dtype]}")
    for g, r in zip(run_gram(fn, block_fallback_of(arrs), A, b, size, dtype, DEV), run_gram(fn, arrs, A, b, size, dtype, DEV)):
        assert same_bits(g, r)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_gram_star_over_budget_takes_block_kernels(dtype):
    """A hub pose with 70 Between-like costs (70 x 6 x 13 = 5 460 staged scalars) does not fit the budget: the plan has no groups,
    its block shapes are all 6 x 6 / 1 x 6 / 1 x 1, so thb_gram runs the block-per-thread kernels -- bitwise what the entry-per-thread
    kernel gives, and the float64 AtA."""
    S = build_structure([6] * 71 + [1], [(6, [0, k]) for k in range(1, 71)] + [(6, [0]), (2, [5, 71]), (1, [71])])
    arrs = build_gram_plan(S)
    assert arrs["num_groups"] == 0 and len(arrs["segments"]) > 0
    rng = np.random.default_rng(9)
    B = 5
    A = rng.standard_normal((B, S.nnz)).astype(NP[dtype])
    b = rng.standard_normal((B, S.num_rows)).astype(NP[dtype])
    fn = getattr(_lib.load(), f"thb_gram_{SFX[dtype]}")
    got = run_gram(fn, arrs, A, b, S.num_cols ** 2, dtype, DEV)
    for g, r in zip(got, run_gram(fn, fallback_of(arrs), A, b, S.num_cols ** 2, dtype, DEV)):
        assert same_bits(g, r)
    check_oracle(S, arrs, A, b, *got, rtol=1e-12 if dtype == torch.float64 else 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_gram_over_budget_falls_back(dtype):
    """A 70-dim variable whose 80-row cost (5 680 staged scalars) exceeds the budget: the plan has no groups, thb_gram runs the
    entry-per-thread kernels, and the result is the float64 AtA."""
    S = build_structure([6, 70, 3], [(6, [0, 2]), (80, [1]), (4, [1, 2]), (3, [2])])
    arrs = build_gram_plan(S)
    assert arrs["num_groups"] == 0
    rng = np.random.default_rng(3)
    B = 4
    A = rng.standard_normal((B, S.nnz)).astype(NP[dtype])
    b = rng.standard_normal((B, S.num_rows)).astype(NP[dtype])
    got = run_gram(getattr(_lib.load(), f"thb_gram_{SFX[dtype]}"), arrs, A, b, S.num_cols ** 2, dtype, DEV)
    check_oracle(S, arrs, A, b, *got, rtol=1e-12 if dtype == torch.float64 else 1e-4)
