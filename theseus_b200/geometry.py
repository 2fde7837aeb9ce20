"""Variables and Lie groups: the host-side mirror of theseus.core.Variable / theseus.geometry.* for the
types on the hot path (SE3, SO3, Vector, Point3).

Same names, storage layouts and argument meaning as the reference:
  Variable            theseus/core/variable.py:17-120     (tensor, name, update(data, batch_ignore_mask), copy)
  Manifold / LieGroup theseus/geometry/manifold.py:31-195, theseus/geometry/lie_group.py:24-203
  SE3 [B,3,4], SO3 [B,3,3], Vector/Point3 [B,k]            theseus/geometry/{se3,so3,vector,point_types}.py
The group arithmetic runs in the CUDA library (theseus_b200/csrc/thb_lie.cuh through the C ABI); calling a
compute method on a CPU tensor raises -- there is no CPU implementation in the product.
"""
import itertools
import threading
import warnings
from contextlib import contextmanager
from typing import List, Optional

import torch

from . import _lib


def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f"theseus_b200.{what}: tensors must live on a CUDA device; the product has no CPU path")


# ---- consistency checks of group tensors at construction (theseus/geometry/lie_group_check.py:10-105, manifold.py:44-68,123-146) ----
class _LieGroupCheckContext:
    contexts = threading.local()

    @classmethod
    def get_context(cls):
        if not hasattr(cls.contexts, "check_lie_group"):
            cls.contexts.check_lie_group, cls.contexts.silent, cls.contexts.silence_internal_warnings = True, False, False
        return cls.contexts.check_lie_group, cls.contexts.silent, cls.contexts.silence_internal_warnings

    @classmethod
    def set_context(cls, check_lie_group: bool, silent: bool, silence_internal_warnings: bool):
        if not check_lie_group and not silent:
            print("Warnings for disabled Lie group checks can be turned off by passing silent=True.")
        cls.contexts.check_lie_group, cls.contexts.silent, cls.contexts.silence_internal_warnings = check_lie_group, silent, silence_internal_warnings


@contextmanager
def set_lie_group_check_enabled(mode: bool, silent: bool = False, silence_internal_warnings: bool = False):
    """lie_group_check.py:39-54: whether group tensors are checked (and, if invalid and not strict, normalised) at construction."""
    prev = _LieGroupCheckContext.get_context()
    _LieGroupCheckContext.set_context(mode, silent, silence_internal_warnings)
    try:
        yield
    finally:
        _LieGroupCheckContext.set_context(*prev)


@contextmanager
def enable_lie_group_check(silent: bool = False, silence_internal_warnings: bool = False):
    with set_lie_group_check_enabled(True, silent, silence_internal_warnings):
        yield


@contextmanager
def no_lie_group_check(silent: bool = False, silence_internal_warnings: bool = False):
    with set_lie_group_check_enabled(False, silent, silence_internal_warnings):
        yield


# eps of the checks: torchlie/global_params.py:44-58 (so3 matrix), theseus/global_params.py:46-59 (so2 matrix / norm)
_SO3_MATRIX_EPS = {torch.float32: 4e-4, torch.float64: 1e-6}
_SO2_MATRIX_EPS = {torch.float32: 1e-5, torch.float64: 4e-7}
_SO2_NORM_EPS = {torch.float32: 1e-12, torch.float64: 1e-12}


class enable_checks:
    """torchlie/functional/check_contexts.py:12-36: the SO3 / SE3 matrix checks live in torchlie and are OFF unless this context is
    active (thread-local) -- with the reference's defaults a rotation block is therefore never validated or normalised at construction,
    while the SE2 / SO2 checks (theseus' own, so2.py:132-146) always run.  Mirrored as is."""
    _ctx = threading.local()

    @classmethod
    def active(cls) -> bool:
        return getattr(cls._ctx, "on", False)

    def __enter__(self) -> None:
        self.prev = enable_checks.active()
        enable_checks._ctx.on = True

    def __exit__(self, typ, value, traceback) -> None:
        enable_checks._ctx.on = self.prev


def _so3_valid(R: torch.Tensor) -> bool:
    """so3_impl.py:30-48 under check_contexts.checks_base: max |R R^T - I| < eps and max |det R - 1| < eps, evaluated in fp64."""
    if not enable_checks.active():
        return True
    eps = _SO3_MATRIX_EPS[R.dtype]
    with torch.no_grad():
        R = R.double()
        ortho = (R @ R.transpose(-1, -2) - torch.eye(3, dtype=R.dtype, device=R.device)).abs().max()
        det = (R[..., 0] * torch.linalg.cross(R[..., 1], R[..., 2], dim=-1)).sum(-1)
        return bool(((ortho < eps) & ((det - 1).abs().max() < eps)).item())


def _so3_normalize(R: torch.Tensor) -> torch.Tensor:
    """so3_impl.py:1133-1141: nearest rotation by SVD, U diag(1, 1, det(U V^T)) V^T."""
    u, _, vh = torch.linalg.svd(R)
    v = vh.transpose(-1, -2)
    sign = torch.linalg.det(u @ v).view(-1, 1, 1)
    vt = torch.cat((v[..., :2], torch.where(sign > 0, v[..., 2:], -v[..., 2:])), dim=-1).transpose(-1, -2)
    return u @ vt


def _so2_valid(cs: torch.Tensor) -> bool:
    """so2.py:132-146."""
    with torch.no_grad():
        return bool(((torch.linalg.norm(cs.double(), dim=1) - 1).abs().max() <= _SO2_MATRIX_EPS[cs.dtype]).item())


def _so2_normalize(cs: torch.Tensor) -> torch.Tensor:
    """so2.py:188-204."""
    norm = torch.norm(cs, dim=1, keepdim=True)
    near_zero = norm < _SO2_NORM_EPS[cs.dtype]
    default = torch.tensor([1, 0], dtype=cs.dtype, device=cs.device).expand(cs.shape[0], 2)
    return torch.where(near_zero, default, cs / torch.where(near_zero, torch.ones_like(norm), norm))


class Variable:
    """theseus/core/variable.py:17-120."""
    _ids = itertools.count(0)
    _global_updates = 0  # bumped on every (re)binding of any variable's tensor; lets engines detect stale pointer tables in O(1)

    def __init__(self, tensor: torch.Tensor, name: Optional[str] = None):
        self._id = next(Variable._ids)
        self._num_updates = 0
        self.name = name if name else f"{self.__class__.__name__}__{self._id}"
        self._tensor = None
        self.tensor = tensor

    @property
    def tensor(self) -> torch.Tensor:
        return self._tensor

    @tensor.setter
    def tensor(self, t: torch.Tensor):
        self._tensor = t
        Variable._global_updates += 1

    def copy(self, new_name: Optional[str] = None) -> "Variable":
        if not new_name:
            new_name = f"{self.name}_copy"
        return self.__class__(tensor=self.tensor.clone(), name=new_name) if type(self) is not Variable \
            else Variable(self.tensor.clone(), name=new_name)

    def update(self, data, batch_ignore_mask: Optional[torch.Tensor] = None):
        tensor = data.tensor if isinstance(data, Variable) else data
        if len(tensor.shape) != len(self.tensor.shape) or tensor.shape[1:] != self.tensor.shape[1:]:
            raise ValueError(
                f"Tried to update tensor {self.name} with data incompatible with original tensor shape. "
                f"Given {tensor.shape[1:]}. Expected: {self.tensor.shape[1:]}")
        if tensor.dtype != self.dtype:
            raise ValueError(f"Tried to update used tensor of dtype {tensor.dtype} but Variable {self.name} has dtype {self.dtype}.")
        if batch_ignore_mask is not None and batch_ignore_mask.any():
            mask_shape = (-1,) + (1,) * (tensor.ndim - 1)
            self.tensor = torch.where(batch_ignore_mask.view(mask_shape), self.tensor, tensor)
        else:
            self.tensor = tensor
        self._num_updates += 1

    def to(self, *args, **kwargs):
        self.tensor = self.tensor.to(*args, **kwargs)

    @property
    def shape(self):
        return self.tensor.shape

    @property
    def device(self):
        return self.tensor.device

    @property
    def dtype(self):
        return self.tensor.dtype

    @property
    def ndim(self):
        return self.tensor.ndim

    def __getitem__(self, item):
        return self.tensor[item]

    def __repr__(self):
        return f"{self.__class__.__name__}(tensor={self.tensor}, name={self.name})"


def as_variable(value, device=None, dtype=None, name: Optional[str] = None) -> Variable:
    """theseus/core/variable.py:123-160 (as_variable)."""
    if isinstance(value, Variable):
        return value
    t = torch.as_tensor(value)
    if not t.is_floating_point():
        t = t.to(torch.get_default_dtype())
    t = t.to(device=device, dtype=dtype)
    if t.ndim == 0:
        t = t.view(1, 1)
    elif t.ndim == 1:
        t = t.view(1, -1)
    return Variable(t, name=name)


class Manifold(Variable):
    """theseus/geometry/manifold.py:31-195 (dof, retract, local)."""
    KIND = -1

    def dof(self) -> int:
        raise NotImplementedError

    def numel(self) -> int:
        return self.tensor[0].numel()

    def copy(self, new_name: Optional[str] = None):
        if not new_name:
            new_name = f"{self.name}_copy"
        with no_lie_group_check(silent=True):       # a copy of a checked tensor
            return self.__class__(tensor=self.tensor.clone(), name=new_name)

    # ---- construction-time checks (manifold.py:44-68, 123-146) ----
    @staticmethod
    def _check_tensor_impl(tensor: torch.Tensor) -> bool:
        return True

    @staticmethod
    def normalize(tensor: torch.Tensor) -> torch.Tensor:
        return tensor

    @classmethod
    def _check_tensor(cls, tensor: torch.Tensor, strict: bool = True, silent_normalization: bool = False) -> torch.Tensor:
        if not cls._check_tensor_impl(tensor):
            if strict:
                raise ValueError(f"The input tensor is not valid for {cls.__name__}.")
            tensor = cls.normalize(tensor)
            if not silent_normalization:
                warnings.warn(f"The input tensor is not valid for {cls.__name__} and has been normalized.")
        return tensor

    @classmethod
    def _checked(cls, tensor: torch.Tensor, strict_checks: bool, disable_checks: bool) -> torch.Tensor:
        """What Manifold.__init__ does with a user-given tensor: check it (strict: raise; else normalise with a warning) unless checks
        are disabled by the argument or by the thread's check context.  Inside torch.func transforms (a user's err_fn building group
        objects under vmap / jacrev) there is nothing to read back: the reference turns the checks off around those calls
        (cost_function.py:343-393), here the wrapped tensor itself says so."""
        if disable_checks or torch._C._functorch.is_batchedtensor(tensor) or torch._C._functorch.is_gradtrackingtensor(tensor):
            return tensor
        enabled, silent, silence_internal = _LieGroupCheckContext.get_context()
        if enabled:
            return cls._check_tensor(tensor, strict_checks, silent_normalization=silence_internal)
        if not silent:
            warnings.warn(f"Manifold consistency checks are disabled for {cls.__name__}.", RuntimeWarning)
        return tensor

    @staticmethod
    def project_tensor(group: torch.Tensor, euclidean_grad: torch.Tensor) -> torch.Tensor:
        """Euclidean Jacobian [B, dim, *group_shape] (derivative w.r.t. the group's storage entries, what vmap(jacrev) gives)
        -> tangent-space Jacobian [B, dim, dof]: `Manifold.project(., is_sparse=True)` of the reference, plain torch ops."""
        raise NotImplementedError


def _vee_skew_part(T: torch.Tensor) -> torch.Tensor:
    """(T32 - T23, T13 - T31, T21 - T12) of the leading 3x3 of T [..., 3, >=3] (so3_impl.py:977-986)."""
    return torch.stack((T[..., 2, 1] - T[..., 1, 2], T[..., 0, 2] - T[..., 2, 0], T[..., 1, 0] - T[..., 0, 1]), dim=-1)


class Vector(Manifold):
    """theseus/geometry/vector.py (Vector): x [+] d = x + d; local(a, b) = b - a."""
    KIND = 2  # THB_VAR_VECTOR

    def __init__(self, dof: Optional[int] = None, tensor: Optional[torch.Tensor] = None, name: Optional[str] = None,
                 dtype: Optional[torch.dtype] = None):
        if tensor is None:
            if dof is None:
                raise ValueError("Either dof or tensor must be given")
            tensor = torch.zeros(1, dof, dtype=dtype or torch.get_default_dtype())
        if tensor.ndim == 1:
            tensor = tensor.view(1, -1)
        if tensor.ndim != 2:
            raise ValueError("Vector tensors must have shape [batch, dof]")
        super().__init__(tensor, name=name)

    def dof(self) -> int:
        return self.tensor.shape[1]

    def retract(self, delta: torch.Tensor) -> "Vector":
        return self.__class__(tensor=self.tensor + delta)

    @staticmethod
    def project_tensor(group: torch.Tensor, euclidean_grad: torch.Tensor) -> torch.Tensor:
        return euclidean_grad  # geometry/vector.py:199-203

    def local(self, other: "Vector") -> torch.Tensor:
        return other.tensor - self.tensor


class Point3(Vector):
    """theseus/geometry/point_types.py (Point3)."""

    def __init__(self, tensor: Optional[torch.Tensor] = None, name: Optional[str] = None, dtype: Optional[torch.dtype] = None):
        if tensor is not None and tensor.shape[-1] != 3:
            raise ValueError("Point3 tensors must have shape [batch, 3]")
        super().__init__(dof=3, tensor=tensor, name=name, dtype=dtype)


class Point2(Vector):
    def __init__(self, tensor: Optional[torch.Tensor] = None, name: Optional[str] = None, dtype: Optional[torch.dtype] = None):
        if tensor is not None and tensor.shape[-1] != 2:
            raise ValueError("Point2 tensors must have shape [batch, 2]")
        super().__init__(dof=2, tensor=tensor, name=name, dtype=dtype)


def _sfx(t: torch.Tensor) -> str:
    if t.dtype == torch.float64:
        return "f64"
    if t.dtype == torch.float32:
        return "f32"
    raise ValueError(f"unsupported dtype {t.dtype}")


class LieGroup(Manifold):
    """theseus/geometry/lie_group.py:24-203."""

    def retract(self, delta: torch.Tensor) -> "LieGroup":
        return self.compose(self.exp_map(delta))

    def local(self, other: "LieGroup", jacobians: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
        return self.between(other).log_map(jacobians)

    def between(self, other: "LieGroup") -> "LieGroup":
        return self.inverse().compose(other)


def _group_ops(cls, prefix: str, dof: int, jshape):
    """Attach exp_map / log_map / adjoint / inverse / compose backed by the stand-alone kernels thb_<prefix>_* (csrc/thb_lie_ops.cu)."""
    def _shape(t):
        return tuple(t.shape[1:])

    def exp_map(tangent_vector: torch.Tensor):
        _require_cuda(tangent_vector, f"{cls.__name__}.exp_map")
        t = tangent_vector.contiguous()
        out = torch.empty((t.shape[0],) + cls._GROUP_SHAPE, dtype=t.dtype, device=t.device)
        _lib.check(getattr(_lib.load(), f"thb_{prefix}_exp_{_sfx(t)}")(_lib.ptr(t), _lib.ptr(out), t.shape[0], _lib.stream_ptr()), f"{prefix}_exp")
        return cls(tensor=out, disable_checks=True)

    def log_map(self, jacobians: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
        g = self.tensor.contiguous()
        _require_cuda(g, f"{cls.__name__}.log_map")
        out = torch.empty(g.shape[0], dof, dtype=g.dtype, device=g.device)
        jl = torch.empty((g.shape[0],) + jshape, dtype=g.dtype, device=g.device) if jacobians is not None else None
        _lib.check(getattr(_lib.load(), f"thb_{prefix}_log_{_sfx(g)}")(_lib.ptr(g), _lib.ptr(out), _lib.ptr(jl), g.shape[0], _lib.stream_ptr()), f"{prefix}_log")
        if jacobians is not None:
            jacobians.append(jl)
        return out

    def adjoint(self) -> torch.Tensor:
        g = self.tensor.contiguous()
        _require_cuda(g, f"{cls.__name__}.adjoint")
        out = torch.empty((g.shape[0],) + jshape, dtype=g.dtype, device=g.device)
        _lib.check(getattr(_lib.load(), f"thb_{prefix}_adjoint_{_sfx(g)}")(_lib.ptr(g), _lib.ptr(out), g.shape[0], _lib.stream_ptr()), f"{prefix}_adjoint")
        return out

    def inverse(self):
        g = self.tensor.contiguous()
        _require_cuda(g, f"{cls.__name__}.inverse")
        out = torch.empty_like(g)
        _lib.check(getattr(_lib.load(), f"thb_{prefix}_inverse_{_sfx(g)}")(_lib.ptr(g), _lib.ptr(out), g.shape[0], _lib.stream_ptr()), f"{prefix}_inverse")
        return cls(tensor=out, disable_checks=True)

    def compose(self, other):
        a, b = self.tensor.contiguous(), other.tensor.contiguous()
        _require_cuda(a, f"{cls.__name__}.compose")
        if a.shape[0] != b.shape[0]:
            B = max(a.shape[0], b.shape[0])
            a, b = a.expand((B,) + _shape(a)).contiguous(), b.expand((B,) + _shape(b)).contiguous()
        out = torch.empty_like(a)
        _lib.check(getattr(_lib.load(), f"thb_{prefix}_compose_{_sfx(a)}")(_lib.ptr(a), _lib.ptr(b), _lib.ptr(out), a.shape[0], _lib.stream_ptr()), f"{prefix}_compose")
        return cls(tensor=out, disable_checks=True)

    cls.exp_map = staticmethod(exp_map)
    cls.log_map, cls.adjoint, cls.inverse, cls.compose = log_map, adjoint, inverse, compose


class SE3(LieGroup):
    """theseus/geometry/se3.py:20 -- storage [B,3,4] = [R|t], tangent [v, w]."""
    KIND = 0  # THB_VAR_SE3

    def __init__(self, tensor: Optional[torch.Tensor] = None, name: Optional[str] = None,
                 dtype: Optional[torch.dtype] = None, strict_checks: bool = False, disable_checks: bool = False):
        given = tensor
        if tensor is None:
            tensor = torch.eye(3, 4, dtype=dtype or torch.get_default_dtype()).view(1, 3, 4)
        if tensor.ndim != 3 or tensor.shape[1:] != (3, 4):
            raise ValueError("SE3 data tensors can only be 3x4 matrices.")  # geometry/se3.py:117-125
        super().__init__(tensor if given is None else self._checked(tensor, strict_checks, disable_checks), name=name)

    @staticmethod
    def _check_tensor_impl(tensor: torch.Tensor) -> bool:
        return _so3_valid(tensor[..., :3])          # se3_impl.py check_group_tensor: the rotation block

    @staticmethod
    def normalize(tensor: torch.Tensor) -> torch.Tensor:
        return torch.cat((_so3_normalize(tensor[..., :3]), tensor[..., 3:]), dim=-1)

    def dof(self) -> int:
        return 6

    @staticmethod
    def project_tensor(group: torch.Tensor, euclidean_grad: torch.Tensor) -> torch.Tensor:
        # left_project (torchlie lie_group.py:36-48): project(R^T G), project = [last column, vee of the skew part] (se3_impl.py:911-923)
        T = group[:, None, :, :3].transpose(-1, -2) @ euclidean_grad
        return torch.cat((T[..., 3], _vee_skew_part(T)), dim=-1)

    # ---- group arithmetic on the GPU (torchlie.functional.SE3 equivalents) ----
    @staticmethod
    def exp_map(tangent_vector: torch.Tensor) -> "SE3":
        _require_cuda(tangent_vector, "SE3.exp_map")
        lib = _lib.load()
        t = tangent_vector.contiguous()
        out = torch.empty(t.shape[0], 3, 4, dtype=t.dtype, device=t.device)
        _lib.check(getattr(lib, f"thb_se3_exp_{_sfx(t)}")(_lib.ptr(t), _lib.ptr(out), t.shape[0], _lib.stream_ptr()), "se3_exp")
        return SE3(tensor=out, disable_checks=True)

    def log_map(self, jacobians: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
        g = self.tensor.contiguous()
        _require_cuda(g, "SE3.log_map")
        lib = _lib.load()
        out = torch.empty(g.shape[0], 6, dtype=g.dtype, device=g.device)
        jl = torch.empty(g.shape[0], 6, 6, dtype=g.dtype, device=g.device) if jacobians is not None else None
        _lib.check(getattr(lib, f"thb_se3_log_{_sfx(g)}")(_lib.ptr(g), _lib.ptr(out), _lib.ptr(jl), g.shape[0], _lib.stream_ptr()), "se3_log")
        if jacobians is not None:
            jacobians.append(jl)
        return out

    def adjoint(self) -> torch.Tensor:
        g = self.tensor.contiguous()
        _require_cuda(g, "SE3.adjoint")
        lib = _lib.load()
        out = torch.empty(g.shape[0], 6, 6, dtype=g.dtype, device=g.device)
        _lib.check(getattr(lib, f"thb_se3_adjoint_{_sfx(g)}")(_lib.ptr(g), _lib.ptr(out), g.shape[0], _lib.stream_ptr()), "se3_adjoint")
        return out

    def inverse(self) -> "SE3":
        g = self.tensor.contiguous()
        _require_cuda(g, "SE3.inverse")
        lib = _lib.load()
        out = torch.empty_like(g)
        _lib.check(getattr(lib, f"thb_se3_inverse_{_sfx(g)}")(_lib.ptr(g), _lib.ptr(out), g.shape[0], _lib.stream_ptr()), "se3_inverse")
        return SE3(tensor=out, disable_checks=True)

    def compose(self, other: "SE3") -> "SE3":
        a, b = self.tensor.contiguous(), other.tensor.contiguous()
        _require_cuda(a, "SE3.compose")
        if a.shape[0] != b.shape[0]:
            B = max(a.shape[0], b.shape[0])
            a, b = a.expand(B, 3, 4).contiguous(), b.expand(B, 3, 4).contiguous()
        lib = _lib.load()
        out = torch.empty_like(a)
        _lib.check(getattr(lib, f"thb_se3_compose_{_sfx(a)}")(_lib.ptr(a), _lib.ptr(b), _lib.ptr(out), a.shape[0], _lib.stream_ptr()), "se3_compose")
        return SE3(tensor=out, disable_checks=True)


class SO3(LieGroup):
    """theseus/geometry/so3.py:20 -- storage [B,3,3]."""
    KIND = 1  # THB_VAR_SO3

    def __init__(self, tensor: Optional[torch.Tensor] = None, name: Optional[str] = None,
                 dtype: Optional[torch.dtype] = None, strict_checks: bool = False, disable_checks: bool = False):
        given = tensor
        if tensor is None:
            tensor = torch.eye(3, dtype=dtype or torch.get_default_dtype()).view(1, 3, 3)
        if tensor.ndim != 3 or tensor.shape[1:] != (3, 3):
            raise ValueError("SO3 data tensors can only be 3x3 matrices.")
        super().__init__(tensor if given is None else self._checked(tensor, strict_checks, disable_checks), name=name)

    @staticmethod
    def _check_tensor_impl(tensor: torch.Tensor) -> bool:
        return _so3_valid(tensor)

    @staticmethod
    def normalize(tensor: torch.Tensor) -> torch.Tensor:
        return _so3_normalize(tensor)

    def dof(self) -> int:
        return 3

    @staticmethod
    def project_tensor(group: torch.Tensor, euclidean_grad: torch.Tensor) -> torch.Tensor:
        return _vee_skew_part(group[:, None].transpose(-1, -2) @ euclidean_grad)  # so3_impl.py:977-986 after the left action


class SE2(LieGroup):
    """theseus/geometry/se2.py:21 -- storage [B,4] = [x, y, cos, sin], tangent [ux, uy, theta]."""
    KIND = 3  # THB_VAR_SE2

    def __init__(self, x_y_theta: Optional[torch.Tensor] = None, tensor: Optional[torch.Tensor] = None, name: Optional[str] = None,
                 dtype: Optional[torch.dtype] = None, strict_checks: bool = False, disable_checks: bool = False):
        if x_y_theta is not None and tensor is not None:
            raise ValueError("Please provide only one of x_y_theta or tensor.")
        given = tensor          # only a user-given storage tensor is checked (cos / sin of an angle are valid by construction)
        if x_y_theta is not None:
            tensor = torch.cat([x_y_theta[:, :2], x_y_theta[:, 2:3].cos(), x_y_theta[:, 2:3].sin()], dim=1)
        if tensor is None:
            tensor = torch.tensor([[0.0, 0.0, 1.0, 0.0]], dtype=dtype or torch.get_default_dtype())
        if tensor.ndim != 2 or tensor.shape[1] != 4:
            raise ValueError("SE2 data tensors can only be 4D vectors.")  # geometry/se2.py:219-224
        super().__init__(tensor if given is None else self._checked(tensor, strict_checks, disable_checks), name=name)

    @staticmethod
    def _check_tensor_impl(tensor: torch.Tensor) -> bool:
        return _so2_valid(tensor[:, 2:])            # se2.py:231-236

    @staticmethod
    def normalize(tensor: torch.Tensor) -> torch.Tensor:
        return torch.cat([tensor[:, :2], _so2_normalize(tensor[:, 2:])], dim=1)   # se2.py:303-307

    def dof(self) -> int:
        return 3

    @staticmethod
    def project_tensor(group: torch.Tensor, euclidean_grad: torch.Tensor) -> torch.Tensor:
        # geometry/se2.py:341-358 (is_sparse branch): storage [x, y, cos, sin]
        cs = group[:, None, 2:]                                   # (cos, sin)
        perp = torch.stack((-group[:, 3], group[:, 2]), dim=1)[:, None]  # (-sin, cos)
        g_xy, g_cs = euclidean_grad[..., :2], euclidean_grad[..., 2:]
        return torch.stack(((g_xy * cs).sum(-1), (g_xy * perp).sum(-1), (g_cs * perp).sum(-1)), dim=-1)


class SO2(LieGroup):
    """theseus/geometry/so2.py:19-340 -- storage [B,2] = [cos, sin], tangent [theta].  Retraction inside the optimizer: the fused retract
    kernel (thb_retract, kind THB_VAR_SO2); cost functions on SO2 variables take the engine's generic (torch.func) route.  The group
    arithmetic below is two-element torch arithmetic on whatever device the tensor lives on, as in the reference."""
    KIND = 4  # THB_VAR_SO2

    def __init__(self, theta: Optional[torch.Tensor] = None, tensor: Optional[torch.Tensor] = None, name: Optional[str] = None,
                 dtype: Optional[torch.dtype] = None, strict_checks: bool = False, disable_checks: bool = False):
        if theta is not None and tensor is not None:
            raise ValueError("Please provide only one of theta or tensor.")
        given = tensor
        if theta is not None:
            if theta.ndim == 1:
                theta = theta.unsqueeze(1)
            if theta.ndim != 2 or theta.shape[1] != 1:
                raise ValueError("Argument theta must be have ndim = 1, or ndim=2 and shape[1] = 1.")   # so2.py:33-37
            tensor = torch.cat([theta.cos(), theta.sin()], dim=1)
        if tensor is None:
            tensor = torch.tensor([[1.0, 0.0]], dtype=dtype or torch.get_default_dtype())
        if tensor.ndim != 2 or tensor.shape[1] != 2:
            raise ValueError("SO2 data tensors can only be 2D vectors.")   # so2.py:189-190
        super().__init__(tensor if given is None else self._checked(tensor, strict_checks, disable_checks), name=name)

    @staticmethod
    def _check_tensor_impl(tensor: torch.Tensor) -> bool:
        return _so2_valid(tensor)

    @staticmethod
    def normalize(tensor: torch.Tensor) -> torch.Tensor:
        return _so2_normalize(tensor)

    def dof(self) -> int:
        return 1

    @staticmethod
    def project_tensor(group: torch.Tensor, euclidean_grad: torch.Tensor) -> torch.Tensor:
        perp = torch.stack((-group[:, 1], group[:, 0]), dim=1)[:, None]     # so2.py:119-129 (is_sparse branch)
        return (euclidean_grad * perp).sum(-1, keepdim=True)

    @staticmethod
    def exp_map(tangent_vector: torch.Tensor) -> "SO2":
        from . import lie_torch
        return SO2(tensor=lie_torch.so2_exp(tangent_vector), disable_checks=True)

    def log_map(self, jacobians: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
        from . import lie_torch
        if jacobians is not None:
            jacobians.append(torch.ones(self.tensor.shape[0], 1, 1, dtype=self.tensor.dtype, device=self.tensor.device))  # so2.py:209-219
        return lie_torch.so2_log(self.tensor)

    def theta(self) -> torch.Tensor:
        return self.log_map()

    def adjoint(self) -> torch.Tensor:
        return torch.ones(self.tensor.shape[0], 1, 1, dtype=self.tensor.dtype, device=self.tensor.device)   # so2.py:116-117

    def inverse(self) -> "SO2":
        from . import lie_torch
        return SO2(tensor=lie_torch.so2_inverse(self.tensor), disable_checks=True)

    def compose(self, other: "SO2") -> "SO2":
        from . import lie_torch
        return SO2(tensor=lie_torch.so2_compose(self.tensor, other.tensor), disable_checks=True)

    def to_cos_sin(self):
        return self.tensor[:, 0], self.tensor[:, 1]

    def to_matrix(self) -> torch.Tensor:
        c, s = self.to_cos_sin()
        return torch.stack((torch.stack((c, -s), dim=1), torch.stack((s, c), dim=1)), dim=1)   # so2.py:311-318

    def rotate(self, point) -> "Point2":
        p = point.tensor if isinstance(point, Variable) else point
        c, s = self.to_cos_sin()
        return Point2(tensor=torch.stack((c * p[:, 0] - s * p[:, 1], s * p[:, 0] + c * p[:, 1]), dim=1))   # so2.py:257-291

    def unrotate(self, point) -> "Point2":
        p = point.tensor if isinstance(point, Variable) else point
        c, s = self.to_cos_sin()
        return Point2(tensor=torch.stack((c * p[:, 0] + s * p[:, 1], -s * p[:, 0] + c * p[:, 1]), dim=1))  # so2.py:293-306


SO3._GROUP_SHAPE, SE2._GROUP_SHAPE, SO2._GROUP_SHAPE = (3, 3), (4,), (2,)
_group_ops(SO3, "so3", 3, (3, 3))   # torchlie.functional.SO3: exp / log (+jlog) / adjoint / inv / compose
_group_ops(SE2, "se2", 3, (3, 3))   # theseus.geometry.SE2: exp_map / log_map (+Jacobian) / adjoint / inverse / compose
