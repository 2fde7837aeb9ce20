"""The fused forward substitution of the multifrontal factor kernel against the two-pass path on the host emulation of the kernels
(tests/simt; shared-memory fronts only, the DMMA dense kernel is not emulated): bitwise the same factor panels, y, x and info, with a
failing item, at a batch larger than the chunk.  tests/test_gpu_front_fused_forward.py makes the same comparison on the GPU."""
import os

import numpy as np
import pytest

from theseus_b200 import _lib
from front_factor_cases import make_solver
from test_gpu_front_fused_forward import compare_paths


@pytest.fixture(scope="module")
def emulated():
    import importlib.util
    here = os.path.dirname(os.path.abspath(__file__))
    spec = importlib.util.spec_from_file_location("emulation_mode", os.path.join(here, "simt", "emulation_mode.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.load_emulated_lib()


def test_fused_forward_is_bitwise_the_two_pass_path_on_the_host_emulation(monkeypatch, emulated):
    monkeypatch.setattr(_lib, "load", lambda: emulated)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: None)
    solver, S, first = make_solver("small", chunk=2)
    assert (solver._plan.arrays["f_class"] < 3).all()
    B = 3
    info = compare_paths(solver, S, B, seed=4, device="cpu", bad_var=first[0])
    assert info[B // 2] > 0 and (np.delete(info, B // 2) == 0).all(), info
