"""The staged Gram kernel (theseus_b200/csrc/thb_gram.cu: gram_staged_kernel) executed on the CPU through the host emulation of
tests/simt (the same source, one OS thread per CUDA thread): its staging, task and column indexing on the dense, multifrontal, item and
Atb-only layouts, bitwise against the entry-per-thread kernels on the same plan and against float64 numpy."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

from theseus_b200 import _lib
from theseus_b200.structure import build_gram_plan

from gram_staged_cases import (NP, SFX, check_oracle, fallback_of, layouts, mixed_structure, run_gram, same_bits)

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu():
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "simt", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lib = C.CDLL(mod.build())
    for name in ("thb_gram_f64", "thb_gram_f32"):
        res, args = _lib.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("layout", ["dense", "front", "item", "atb"])
def test_staged_gram_emulated(emu, layout, dtype):
    S = mixed_structure()
    B = 2
    arrs, size = layouts(S, B, (layout,))[layout]
    assert arrs["num_groups"] >= 1
    rng = np.random.default_rng(11)
    A = rng.standard_normal((B, S.nnz)).astype(NP[dtype])
    b = rng.standard_normal((B, S.num_rows)).astype(NP[dtype])
    fn = getattr(emu, f"thb_gram_{SFX[dtype]}")
    got = run_gram(fn, arrs, A, b, size, dtype, "cpu")
    ref = run_gram(fn, fallback_of(arrs), A, b, size, dtype, "cpu")
    for g, r in zip(got, ref):
        assert same_bits(g, r)
    check_oracle(S, arrs, A, b, *got, rtol=1e-12 if dtype == torch.float64 else 1e-5)


def test_staged_gram_emulated_many_groups(emu):
    """A budget of 600 scalars cuts the twelve variables into four groups: cost functions staged by two CTAs, columns and blocks
    owned by each group."""
    S = mixed_structure()
    arrs = build_gram_plan(S, stage_budget=600)
    assert arrs["num_groups"] == 4 and arrs["stage_elems"] <= 600
    rng = np.random.default_rng(12)
    A, b = rng.standard_normal((2, S.nnz)), rng.standard_normal((2, S.num_rows))
    got = run_gram(emu.thb_gram_f64, arrs, A, b, S.num_cols ** 2, torch.float64, "cpu")
    ref = run_gram(emu.thb_gram_f64, fallback_of(arrs), A, b, S.num_cols ** 2, torch.float64, "cpu")
    for g, r in zip(got, ref):
        assert same_bits(g, r)
    check_oracle(S, arrs, A, b, *got, rtol=1e-12)
