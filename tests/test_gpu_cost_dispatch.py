"""Return codes of the fused cost entry points (thb_linearize_group_f64 / _f32, thb_error_group_f64 / _f32).  They are decided by the one
cost-kind dispatch of thb_costs.cu before any kernel is launched:
  - THB_OK (0) for an empty group (K == 0 or B == 0), whatever its kind and fields;
  - THB_ERR_UNSUPPORTED (-2) for a kind without a fused kernel;
  - THB_ERR_BAD_ARG (-1) for a group that lacks a field its kind reads, or whose pose dof has no motion-planning kernel.
No kernel runs in these cases, so the pointer fields are only tested for NULL, never read.
Dry run on the CPU:  THB_SIMT_EMULATION=1 python -m pytest tests/test_gpu_cost_dispatch.py -m gpu"""
import ctypes as C

import numpy as np
import pytest

import theseus_b200 as th  # noqa: F401  (torch before the library)
from theseus_b200 import _lib, core

pytestmark = pytest.mark.gpu
OK, BAD_ARG, UNSUPPORTED = 0, -1, -2
_HOST = np.zeros(64)
P = _HOST.ctypes.data       # a non-NULL address for the fields the checks test for NULL


def _group(kind, K=4, dim=6, **fields):
    g = _lib.CostGroup(kind=kind, weight_kind=0, K=K, dim=dim, x0=P, x1=P, aux=P, w=P, bstride=P, a_off=P, a_stride=P, bp=P, row0=P,
                       log_radius=P, bstride_lr=P)
    for name, value in fields.items():
        setattr(g, name, value)
    return g


def _codes(g, B=3):
    """The return code of each of the four entry points for the group g and batch size B."""
    lib = _lib.load()
    return [getattr(lib, f"thb_linearize_group_{sfx}")(C.byref(g), B, P, 64, P, 64, None) for sfx in ("f64", "f32")] + \
           [getattr(lib, f"thb_error_group_{sfx}")(C.byref(g), B, P, None) for sfx in ("f64", "f32")]


@pytest.mark.parametrize("kind", [17, 99, -1])
def test_unknown_kind_is_unsupported(kind):
    assert _codes(_group(kind)) == [UNSUPPORTED] * 4


@pytest.mark.parametrize("missing", ["aux2", "aux3", "aux4", "bstride2"])
def test_reprojection_without_its_aux_fields_is_a_bad_argument(missing):
    full = dict(aux2=P, aux3=P, aux4=P, bstride2=P)
    assert _codes(_group(core.COST_REPROJECTION, dim=2, **{**full, missing: None})) == [BAD_ARG] * 4


@pytest.mark.parametrize("dim", [1, 3, 5, 8])
def test_double_integrator_with_an_odd_dim_or_a_dof_above_3_is_a_bad_argument(dim):
    g = _group(core.COST_DOUBLE_INTEGRATOR_VECTOR, dim=dim, x2=P, x3=P, bstride3=P)
    assert _codes(g) == [BAD_ARG] * 4


@pytest.mark.parametrize("kind, fields", [(17, {}), (core.COST_REPROJECTION, {}), (core.COST_DOUBLE_INTEGRATOR_VECTOR, dict(dim=5)),
                                          (core.COST_BETWEEN_SE3, {})])
def test_an_empty_group_or_batch_is_ok_whatever_its_kind(kind, fields):
    assert _codes(_group(kind, K=0, **fields)) == [OK] * 4
    assert _codes(_group(kind, **fields), B=0) == [OK] * 4
