"""Shared by tests/test_tactile_costs.py (CPU: torch restatements, host emulation of the kernels) and tests/test_gpu_tactile_costs.py:
the planar-pushing cost functions of tests/golden/make_golden_tactile.py built from the states stored in tactile_costs_kat.npz."""
import importlib.util
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_tactile", os.path.join(HERE, "golden", "make_golden_tactile.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def cost_states(g, device="cpu", dtype=torch.float64):
    return {k[2:]: torch.from_numpy(g[k].copy()).to(device=device, dtype=dtype) for k in g.files if k.startswith("S_")}


def cost_functions(th, g, device="cpu", dtype=torch.float64):
    """name -> the fixture's cost functions built with `th` (on `device`, in `dtype`)."""
    return golden_module().tactile_cost_functions(th, torch, cost_states(g, device, dtype))


def torch_route(cf):
    """Re-class `cf` into a test-local subclass without a CUDA schema: the engine evaluates it on the torch route."""
    cls = type(cf)
    cf.__class__ = type("TorchRoute" + cls.__name__, (cls,), {"schema": lambda self: (None, cls.schema(self)[1])})
    return cf
