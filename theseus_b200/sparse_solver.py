"""BaspachoSparseSolver (alias BlockSparseSolver): batched block-sparse Cholesky on the GPU.

Mirror of theseus/optimizer/linear/baspacho_sparse_solver.py:23-160 + BaspachoSolveFunction.forward
(optimizer/autograd/baspacho_sparse_autograd.py:21-65): reset() builds the block structure of AtA and the symbolic
decomposition once; solve() = add_MtM (thb_gram into the factor storage) -> damp(alpha, beta) -> factor -> Atb -> solve,
all in fp64 like the reference (baspacho_sparse_autograd.py:41,65), result cast back to the objective dtype.
It is also what CholmodSparseSolver / LUCudaSparseSolver map to (same linear system, SURVEY.md a33/a34).
"""
import ctypes as C
import os
from typing import Any, Dict, Optional, Type, Union

import numpy as np
import torch

from . import _lib
from .autograd import LinearSolveFunction, wants_grad
from .core import Objective
from .optimizer import (Linearization, LinearSolver, SparseLinearization, convert_to_alpha_beta_damping_tensors)
from .frontal import build_front_plan
from .sparse import ITEM_MAX_DIM, LANE_DIMS, analyze, gram_out_offsets, piece_solve_lists, root_lane_lists, root_split, tile_lane_lists
from .structure import ata_block_structure, build_gram_plan


_ROOT_LAYOUTS = ("lane_root", "lane_tiled_root")     # dense DMMA factorisation of the top chain of the elimination tree
_TILED_LAYOUTS = ("lane_tiled", "lane_tiled_root")   # supernodal tile kernel for the external updates of chain pieces


class BaspachoSparseSolver(LinearSolver):
    def __init__(self, objective: Objective, linearization_cls: Optional[Type[Linearization]] = None,
                 linearization_kwargs: Optional[Dict[str, Any]] = None, num_solver_contexts=1, batch_size: Optional[int] = None,
                 auto_reset: bool = True, dev: Optional[str] = None, ordering: str = "mindeg", layout: Optional[str] = None,
                 supernodal_solve: bool = False, front_options: Optional[Dict[str, Any]] = None, **kwargs):
        linearization_cls = linearization_cls or SparseLinearization
        if not linearization_cls == SparseLinearization:
            raise RuntimeError(
                "BaspachoSparseSolver only works with theseus.optimizer.SparseLinearization,"
                + f" got {type(self.linearization)}")
        super().__init__(objective, linearization_cls, linearization_kwargs, **kwargs)
        self.linearization: SparseLinearization = self.linearization
        self._ordering = ordering
        self._layout = layout
        self._supernodal_solve = bool(supernodal_solve)   # opt-in: chain-piece substitution kernels (lane layouts only; not yet run on a GPU)
        self._front_options = dict(front_options or {})   # layout="front": frontal.build_front_plan keywords (tau, small_limit, ...)
        self._plan = None
        self._dev = None
        self.param_size = None
        self.reset()

    @classmethod
    def from_structure(cls, structure, ordering: str = "mindeg", layout: Optional[str] = None,
                       supernodal_solve: bool = False, front_options: Optional[Dict[str, Any]] = None) -> "BaspachoSparseSolver":
        """Solver over a bare CSR structure with hand-filled `linearization.A_val / b` -- the pattern of the reference's own
        solver tests (void Objective + filled linearization, tests/theseus_tests/optimizer/linear/test_baspacho_sparse_solver.py:15-41)."""
        class _Lin:
            def __init__(self, S):
                self._S, self.A_val, self.b = S, None, None
                self.A_row_ptr, self.A_col_ind = S.A_row_ptr, S.A_col_ind
                self.num_rows, self.num_cols = S.num_rows, S.num_cols

            def structure(self):
                return self._S
        self = cls.__new__(cls)
        self.linearization = _Lin(structure)
        self._ordering, self._plan, self._dev, self._layout = ordering, None, None, layout
        self._supernodal_solve = bool(supernodal_solve)
        self._front_options = dict(front_options or {})
        self.param_size = None
        self.reset()
        return self

    # ---- symbolic phase (baspacho_sparse_solver.py:58-113) ----
    def reset(self, **kwargs):
        if self._plan is not None:
            return
        S = self.linearization.structure()
        if getattr(self, "param_size", None) is None:
            param_size, ptrs, inds = ata_block_structure(S)
            self.param_size, self.block_ptrs, self.block_inds = param_size, ptrs, inds  # the reference's SymbolicDecomposition inputs
        param_size, ptrs, inds = self.param_size, self.block_ptrs, self.block_inds
        if self._layout is None:
            return      # default layout: chosen at the first solve, when the batch size is known (layout_for); the plan is built then
        if self._layout == "front":
            # multifrontal layout: own ordering (nested dissection / minimum degree, whichever costs fewer flops) and fronts
            opts = {k: v for k, v in getattr(self, "_front_options", {}).items() if k != "chunk"}
            for env, key, cast in (("THB_FRONT_TAU", "tau", float), ("THB_FRONT_MERGE_FLOPS", "merge_flops", float),
                                   ("THB_FRONT_MERGE_MAX_R", "merge_max_r", int)):      # tuning knobs of the amalgamation (experiments)
                if env in os.environ and key not in opts:
                    opts[key] = cast(os.environ[env])
            self._plan = build_front_plan(param_size, ptrs, inds, ordering="auto" if self._ordering == "mindeg" else self._ordering, **opts)
            # AtA goes to a COMPACT block storage; the factorisation reads it through the plan's panel map (no zero fill of the panels,
            # no reads of their structural zeros)
            from .structure import lower_blocks
            blocks, _ = lower_blocks(S, self._plan.pos)
            dims_of = S.var_dims
            f, self._ata_size = self._plan.gram_compact_offsets([(a, b, int(dims_of[a]), int(dims_of[b])) for a, b in blocks])
            self._gram_arrays = build_gram_plan(S, out_offsets=f, pos=self._plan.pos)
            return
        self._plan = analyze(param_size, ptrs, inds, ordering=self._ordering)
        self._gram_arrays = build_gram_plan(S, out_offsets=gram_out_offsets(self._plan), pos=self._plan.pos)

    def layout_for(self, B: int) -> str:
        """'lane' (batch-interleaved factor, one warp = 32 batch items, thb_sparse_lane.cu) or 'item' (one CTA per batch item,
        thb_sparse.cu).  Default: lane whenever a warp can be filled and every block size is one the lane kernels are built for."""
        if self._layout is None:
            # default: the multifrontal layout for batches that fill the GPU and for blocks larger than the one-CTA-per-item kernels take
            # (it takes any block size); one CTA per item for the other small batches
            big = int(np.max(self.param_size, initial=0)) > ITEM_MAX_DIM
            self._layout = os.environ.get("THB_SPARSE_LAYOUT") or ("front" if B >= 32 or big else "item")
            self.reset()
        if self._layout == "front":
            return "front"
        lane_ok = all(int(d) in LANE_DIMS for d in self._plan.dims)
        if self._layout is not None:
            if self._layout not in ("lane", "item", "lane_root", "lane_tiled", "lane_tiled_root"):
                raise ValueError(f"layout must be 'lane', 'item', 'lane_root', 'lane_tiled' or 'lane_tiled_root', got {self._layout}")
            if self._layout != "item" and not lane_ok:
                raise ValueError(f"layout='{self._layout}' needs block sizes in {LANE_DIMS}")
            if self._layout == "item" and int(self._plan.dims.max(initial=0)) > ITEM_MAX_DIM:
                raise ValueError(f"layout='item' needs block sizes <= {ITEM_MAX_DIM} (layout='front' takes any block size)")
            if self._layout in _ROOT_LAYOUTS and self._root_split() is None:
                raise ValueError(f"layout='{self._layout}': this structure has no dense root (top chain too short)")
            return self._layout
        return "lane" if (lane_ok and B >= 32) else "item"

    def _root_split(self):
        """Dense-root split of the plan (sparse.root_split), computed on first use.  Opt-in layout 'lane_root': the lane kernels
        below the cut, the dense DMMA Cholesky for the root -- written at the end of round 1, not yet timed on a GPU."""
        if not hasattr(self, "_root"):
            sp = root_split(self._plan)
            self._root = None if sp is None else (sp,) + root_lane_lists(self._plan, sp)
        return self._root

    @property
    def symbolic_stats(self):
        if self._plan is None:      # default layout not resolved yet: report the multifrontal plan (what large batches get)
            self._layout = os.environ.get("THB_SPARSE_LAYOUT") or "front"
            self.reset()
        return dict(self._plan.stats)

    @property
    def effective_layout(self):
        return self._layout

    def _device_plan(self, device):
        if self._dev is not None and self._dev["device"] == device:
            return self._dev
        if self._layout == "front":
            return self._device_plan_front(device)
        P = self._plan
        dev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in P.arrays.items()}
        st = _lib.SparsePlanStruct(N=P.N, num_levels=int(P.stats["levels"]), max_dim=int(P.dims.max()) if P.N else 0, reserved=0,
                                   n=P.n, data_size=P.data_size, winv_size=P.winv_size,
                                   **{k: dev[k].data_ptr() for k in dev})
        g = self._gram_arrays
        gdev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in g.items() if isinstance(v, np.ndarray)}
        gst = _lib.make_gram_plan(g, gdev)
        # batch-lane plan: shares the batch-independent arrays above, adds the per-level / per-shape work lists
        ln = P.lane
        lst, ldev, launches = self._lane_struct(ln, dev, device)
        self._dev = dict(device=device, plan=st, keep=dev, gram=gst, gkeep=gdev, bufs={}, lane=lst, lkeep=(ldev, launches))
        if self._layout in _ROOT_LAYOUTS:
            sp, rl, rr = self._root_split()
            qdev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in rr.items() if isinstance(v, np.ndarray) and k != "segments"}
            segs = np.ascontiguousarray(rr["segments"], dtype=np.int32)
            qst = _lib.SparseLaneRootStruct(
                num_blocks=int(rr["rb_off"].shape[0]), num_cols=int(rr["root_cols"].shape[0]), nt=int(rr["nt"]), root_start=int(rr["root_start"]),
                num_segments=int(segs.shape[0]), segments=segs.ctypes.data, rb_off=qdev["rb_off"].data_ptr(), rb_row=qdev["rb_row"].data_ptr(),
                rb_col=qdev["rb_col"].data_ptr(), rb_di=qdev["rb_di"].data_ptr(), rb_dj=qdev["rb_dj"].data_ptr(), rf_p0=qdev["rf_p0"].data_ptr(),
                rf_p1=qdev["rf_p1"].data_ptr(), root_cols=qdev["root_cols"].data_ptr(), root_dims=qdev["root_dims"].data_ptr())
            self._dev.update(root=qst, qkeep=(qdev, segs), nt=int(rr["nt"]))
            if self._layout == "lane_root":
                rst, rdev, rlaunch = self._lane_struct(rl, dev, device)
                self._dev.update(lane_root=rst, rkeep=(rdev, rlaunch))
        if self._layout in _TILED_LAYOUTS:
            tl, tt = self._tile_lists()
            tst, tdev, tlaunch = self._lane_struct(tl, dev, device)
            ttdev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in tt.items()}
            tiles = _lib.SparseLaneTilesStruct(num_tiles=int(tt["tile_tgt"].shape[0]), num_steps=int(tt["step_src"].shape[0]),
                                               tile_tgt=ttdev["tile_tgt"].data_ptr(), step_ptr=ttdev["step_ptr"].data_ptr(),
                                               step_src=ttdev["step_src"].data_ptr())
            self._dev.update({self._layout: tst}, tiles=tiles, tkeep=(tdev, tlaunch, ttdev))
        if getattr(self, "_supernodal_solve", False) and all(int(d) in LANE_DIMS for d in P.dims):
            ps = piece_solve_lists(P, cut=self._root_split()[0]["cut"] if self._layout in _ROOT_LAYOUTS else None)
            pdev = {k: torch.from_numpy(np.ascontiguousarray(ps[k] if k != "width" else ps[k].astype(np.int32))).to(device)
                    for k in ("first", "width", "fr_ext_end", "bc_int_end", "order")}
            plaunch = np.ascontiguousarray(ps["launches"][:, 1:], dtype=np.int32)    # (block size, begin, end); the level is implicit in the order
            pst = _lib.SparseLanePiecesStruct(num_pieces=int(ps["first"].shape[0]), num_launches=int(plaunch.shape[0]), launches=plaunch.ctypes.data,
                                              **{k: pdev[k].data_ptr() for k in pdev})
            self._dev.update(pieces=pst, pkeep=(pdev, plaunch, ps))
        return self._dev

    def _device_plan_front(self, device):
        P = self._plan
        dev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in P.arrays.items()}
        st = _lib.FrontPlanStruct(S=P.S, n=P.n, data_size=P.data_size, arena_size=P.arena_size, varena_size=P.varena_size,
                                  **{k: dev[k].data_ptr() for k in ("f_w", "f_b", "f_first", "f_class", "f_wpad", "f_np", "f_cb_ld", "f_depth",
                                                                    "f_panel_off", "f_cb_off", "f_fr_off", "f_u_off", "child_ptr", "child_list",
                                                                    "rel_ptr", "f_rel", "rows_ptr", "f_rows", "sched", "perm", "c_jw", "c_sp_ptr", "c_sp", "c_inv_ptr", "c_inv", "fd", "pc", "pmap")})
        g = self._gram_arrays
        gdev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in g.items() if isinstance(v, np.ndarray)}
        launches = np.ascontiguousarray(P.launches, dtype=np.int64)
        big = launches[launches[:, 1] == 3]
        self._dev = dict(device=device, front=st, keep=dev, gram=_lib.make_gram_plan(g, gdev), gkeep=gdev, bufs={}, launches=launches,
                         max_np=int(big[:, 5].max()) if len(big) else 0)
        return self._dev

    def _numeric_front(self, A_val, b, alpha, beta, forward=False):
        """Gram + factor, chunk by chunk.  forward=True: the forward substitution of A^T b runs inside the factorisation (each
        front on its panel while the panel is in shared memory, thb_front_factor_forward_f64) and leaves y in bufs['work'];
        _backward_front() finishes the solve."""
        B, device = A_val.shape[0], A_val.device
        d = self._device_plan(device)
        P = self._plan
        lib = _lib.load()
        s = _lib.stream_ptr()
        # the factor of every item stays resident ([B, data_size]: the substitutions and the backward pass need it); the update-matrix
        # arena, the border-vector arena and the dense workspace are per CHUNK of the batch (C5: 21 MB of arena per item)
        chunk = int(min(B, self._front_options.get("chunk", int(os.environ.get("THB_FRONT_CHUNK", "1024")))))
        if d["bufs"].get("key") != (B, "front"):
            ws_bytes = int(lib.thb_potrf_partial_workspace_bytes(chunk, d["max_np"])) if d["max_np"] else 0
            d["bufs"] = dict(key=(B, "front"), chunk=chunk, factor=torch.empty(B, P.data_size, dtype=torch.float64, device=device),
                             ata=torch.empty(B, self._ata_size, dtype=torch.float64, device=device),
                             arena=torch.empty(2, chunk, P.arena_size, dtype=torch.float64, device=device),
                             varena=torch.empty(2, chunk, P.varena_size, dtype=torch.float64, device=device),
                             work=torch.empty(B, P.n, dtype=torch.float64, device=device),
                             ws=torch.empty(max(ws_bytes, 8), dtype=torch.uint8, device=device),
                             Atb=torch.empty(B, P.n, dtype=torch.float64, device=device),
                             AtA_diag=torch.empty(B, P.n, dtype=torch.float64, device=device),
                             info=torch.empty(B, dtype=torch.int32, device=device))
        bufs = d["bufs"]
        factor, Atb, info = bufs["factor"], bufs["Atb"], bufs["info"]
        lin = self.linearization
        if getattr(lin, "_Atb", None) is Atb:   # the buffers are about to be overwritten: the linearization must not keep them as its Atb / diag
            lin._Atb = lin._AtA_diag = None
        nnz, m = A_val.shape[1], b.shape[1]
        self._factor_stamp = getattr(self, "_factor_stamp", 0) + 1
        ata = bufs["ata"]
        _lib.check(lib.thb_gram_f64(C.byref(d["gram"]), B, _lib.ptr(A_val), nnz, _lib.ptr(b), m, _lib.ptr(ata), self._ata_size,
                                    _lib.ptr(Atb), _lib.ptr(bufs["AtA_diag"]), s), "gram(front)")
        L = d["launches"]
        for c0 in range(0, B, chunk):
            nb = min(chunk, B - c0)
            args = (C.byref(d["front"]), L.ctypes.data, L.shape[0], _lib.ptr(factor[c0:]), _lib.ptr(ata[c0:]), self._ata_size,
                    _lib.ptr(alpha[c0:]) if alpha is not None else None,
                    _lib.ptr(beta[c0:]) if beta is not None else None, _lib.ptr(bufs["arena"]), _lib.ptr(bufs["ws"]) if d["max_np"] else None,
                    bufs["ws"].numel(), _lib.ptr(info[c0:]))
            if forward:
                _lib.check(lib.thb_front_factor_forward_f64(*args, _lib.ptr(Atb[c0:]), _lib.ptr(bufs["work"][c0:]), _lib.ptr(bufs["varena"]), nb, s),
                           "front_factor_forward")
            else:
                _lib.check(lib.thb_front_factor_f64(*args, nb, s), "front_factor")
        self._keep = (A_val, b, alpha, beta)
        return Atb

    def _substitute_front(self, rhs):
        d, P = self._dev, self._plan
        bufs = d["bufs"]
        B, chunk = bufs["key"][0], bufs["chunk"]
        lib = _lib.load()
        rhs = rhs.contiguous()
        x = torch.empty(B, P.n, dtype=torch.float64, device=rhs.device)
        L = d["launches"]
        for c0 in range(0, B, chunk):
            nb = min(chunk, B - c0)
            _lib.check(lib.thb_front_solve_f64(C.byref(d["front"]), L.ctypes.data, L.shape[0], _lib.ptr(bufs["factor"][c0:]), _lib.ptr(rhs[c0:]),
                                               _lib.ptr(x[c0:]), _lib.ptr(bufs["work"][c0:]), _lib.ptr(bufs["varena"]), nb, _lib.stream_ptr()),
                       "front_solve")
        return x

    def _backward_front(self):
        """x = L^-T y, y left in bufs['work'] by _numeric_front(..., forward=True)."""
        d, P = self._dev, self._plan
        bufs = d["bufs"]
        B, chunk = bufs["key"][0], bufs["chunk"]
        lib = _lib.load()
        x = torch.empty(B, P.n, dtype=torch.float64, device=bufs["work"].device)
        L = d["launches"]
        for c0 in range(0, B, chunk):
            nb = min(chunk, B - c0)
            _lib.check(lib.thb_front_backward_f64(C.byref(d["front"]), L.ctypes.data, L.shape[0], _lib.ptr(bufs["factor"][c0:]), _lib.ptr(x[c0:]),
                                                  _lib.ptr(bufs["work"][c0:]), nb, _lib.stream_ptr()), "front_backward")
        return x

    def _lane_struct(self, ln, dev, device):
        """thb_sparse_lane_plan over the plan's batch-independent device arrays `dev` + the work lists `ln` (uploaded here).
        Returns (struct, device arrays, host launch list) -- the caller keeps the last two alive."""
        P = self._plan
        ldev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in ln.items() if k != "launches"}
        launches = np.ascontiguousarray(ln["launches"], dtype=np.int32)
        lst = _lib.SparseLanePlanStruct(
            N=P.N, n=P.n, data_size=P.data_size, diag_size=P.winv_size, num_launches=int(launches.shape[0]),
            launches=launches.ctypes.data, dims=dev["dims"].data_ptr(), col_start=dev["col_start"].data_ptr(),
            pstart=dev["pstart"].data_ptr(), dl_off=dev["winv_off"].data_ptr(), diag_off=dev["diag_off"].data_ptr(),
            up_a=dev["up_a"].data_ptr(), up_b=dev["up_b"].data_ptr(), up_k=dev["up_k"].data_ptr(),
            u_tgt=ldev["u_tgt"].data_ptr(), u_p0=ldev["u_p0"].data_ptr(), u_p1=ldev["u_p1"].data_ptr(),
            t_off=ldev["t_off"].data_ptr(), t_diag=ldev["t_diag"].data_ptr(), t_dl=ldev["t_dl"].data_ptr(),
            t_pstart=ldev["t_pstart"].data_ptr(), s_col=ldev["s_col"].data_ptr(),
            fr_ptr=dev["fr_ptr"].data_ptr(), fr_off=dev["fr_off"].data_ptr(), fr_p=ldev["fr_p"].data_ptr(), fr_d=ldev["fr_d"].data_ptr(),
            bc_ptr=dev["bc_ptr"].data_ptr(), bc_off=dev["bc_off"].data_ptr(), bc_p=ldev["bc_p"].data_ptr(), bc_d=ldev["bc_d"].data_ptr())
        return lst, ldev, launches

    def _tile_lists(self):
        """Work lists of the opt-in layouts 'lane_tiled' / 'lane_tiled_root' (sparse.tile_lane_lists), computed on first use."""
        if not hasattr(self, "_tiles"):
            self._tiles = tile_lane_lists(self._plan, self._root_split()[0] if self._layout in _ROOT_LAYOUTS else None)
        return self._tiles

    # ---- numeric phase (baspacho_sparse_autograd.py:21-65) ----
    def solve(self, damping: Optional[Union[float, torch.Tensor]] = None, ellipsoidal_damping: bool = True,
              damping_eps: float = 1e-8, **kwargs) -> torch.Tensor:
        lin = self.linearization
        A_val, b = lin.A_val, lin.b
        if A_val is None:
            raise RuntimeError("linearize() must be called before solve()")
        if wants_grad(A_val, b):
            detach = bool(getattr(lin, "detached_hessian", False))
            return LinearSolveFunction.apply(A_val, b, self, damping, ellipsoidal_damping, damping_eps, detach)
        x = self._solve_nograd(A_val, b, damping, ellipsoidal_damping, damping_eps)[0]
        bufs = self._dev["bufs"] if self._dev is not None else {}
        if "AtA_diag" in bufs and A_val.dtype == torch.float64 and A_val.is_contiguous() and b.is_contiguous() and getattr(lin, "_Atb", 0) is None:
            # A^T b and diag(A^T A) of THIS linearization came out of the Gram pass: the LM accept test (optimizer._check_accept) reads them
            # from the linearization instead of running the Atb kernel a second time
            lin._Atb, lin._AtA_diag = bufs["Atb"], bufs["AtA_diag"]
        return x

    def _solve_nograd(self, A_val, b, damping, ellipsoidal_damping, damping_eps):
        out_dtype = A_val.dtype
        A64, b64 = A_val.detach(), b.detach()
        if A64.dtype != torch.float64:
            A64, b64 = A64.double(), b64.double()  # the sparse path computes in fp64 like the reference (baspacho_sparse_autograd.py:41,65)
        A64, b64 = A64.contiguous(), b64.contiguous()
        alpha = beta = None
        if damping is not None:
            alpha, beta = convert_to_alpha_beta_damping_tensors(damping, damping_eps, ellipsoidal_damping, A64.shape[0], A64.device, torch.float64)
        if self.layout_for(A64.shape[0]) == "front":
            # the forward substitution of A^T b rides on the factorisation (no second read of L), then the backward pass
            self._numeric_front(A64, b64, alpha, beta, forward=True)
            x = self._backward_front()
        else:
            Atb = self._numeric(A64, b64, alpha, beta)
            x = self._substitute(Atb)
        self._last_info = self._dev["bufs"]["info"]
        if not getattr(self, "defer_info_check", False):  # CUDA-graph capture: no host sync here, check_info() after the replay
            self.check_info()
        return x.to(out_dtype), (A64, b64, x, alpha, beta)

    def check_info(self, x=None):
        self._raise_if_bad(self._last_info)
        return x

    @staticmethod
    def _raise_if_bad(info):
        bad = info.nonzero()
        if bad.numel() > 0:
            k = int(bad[0, 0])
            raise RuntimeError(f"block-sparse Cholesky: batch element {k}: matrix is not positive definite (pivot {int(info[k])})")

    def _numeric(self, A_val, b, alpha, beta):
        """add_MtM -> damp -> factor (+ Atb) on fp64 inputs; leaves the factor in the solver's buffers."""
        B, device = A_val.shape[0], A_val.device
        layout = self.layout_for(B)     # validates an explicit layout (e.g. no dense root for 'lane_root') before anything is built
        if layout == "front":
            return self._numeric_front(A_val, b, alpha, beta)
        d = self._device_plan(device)
        P = self._plan
        lib = _lib.load()
        s = _lib.stream_ptr()
        key = (B, layout)
        if d["bufs"].get("key") != key:
            Bp = int(lib.thb_sparse_lane_padded_batch(B))
            shape = (lambda k: (k, Bp)) if layout != "item" else (lambda k: (B, k))
            d["bufs"] = dict(key=key, factor=torch.empty(shape(P.data_size), dtype=torch.float64, device=device),
                             diag=torch.empty(shape(P.winv_size), dtype=torch.float64, device=device),   # W_j = L_jj^-1 (item) / L_jj with reciprocal diagonal (lane)
                             work=torch.empty(shape(P.n), dtype=torch.float64, device=device),
                             Atb=torch.empty(B, P.n, dtype=torch.float64, device=device),
                             info=torch.empty(B, dtype=torch.int32, device=device))
            if layout in _ROOT_LAYOUTS:
                nt = d["nt"]
                d["bufs"].update(S=torch.empty(B, nt, nt, dtype=torch.float64, device=device),
                                 ws=torch.empty(int(lib.thb_potrf_workspace_bytes(B, nt)), dtype=torch.uint8, device=device),
                                 rhs_root=torch.empty(B, nt, dtype=torch.float64, device=device),
                                 x_root=torch.empty(B, nt, dtype=torch.float64, device=device),
                                 info_root=torch.empty(B, dtype=torch.int32, device=device))
        bufs = d["bufs"]
        factor, diag, Atb, info = bufs["factor"], bufs["diag"], bufs["Atb"], bufs["info"]
        nnz, m = A_val.shape[1], b.shape[1]
        self._factor_stamp = getattr(self, "_factor_stamp", 0) + 1
        # every structurally non-zero block of L that is not in AtA (fill-in) must start at zero
        _lib.check(lib.thb_fill_zero(_lib.ptr(factor), factor.numel() * 8, s), "fill_zero")
        if layout != "item":
            lplan = d[layout]   # *_root: launch list = bottom columns + the root's assembly updates; lane_tiled*: + tile launches
            _lib.check(lib.thb_sparse_lane_gram_f64(C.byref(d["gram"]), B, _lib.ptr(A_val), nnz, _lib.ptr(factor), s), "gram(lane)")
            _lib.check(lib.thb_gram_f64(C.byref(d["gram"]), B, _lib.ptr(A_val), nnz, _lib.ptr(b), m, None, 0, _lib.ptr(Atb), None, s), "Atb")
            if alpha is not None:
                _lib.check(lib.thb_sparse_lane_damp_f64(C.byref(d["lane"]), _lib.ptr(factor), _lib.ptr(alpha), _lib.ptr(beta), B, s), "lane_damp")
            if layout in _TILED_LAYOUTS:
                _lib.check(lib.thb_sparse_lane_factor_tiled_f64(C.byref(lplan), C.byref(d["tiles"]), _lib.ptr(factor), _lib.ptr(diag), _lib.ptr(info),
                                                                B, s), "lane_factor_tiled")
            else:
                _lib.check(lib.thb_sparse_lane_factor_f64(C.byref(lplan), _lib.ptr(factor), _lib.ptr(diag), _lib.ptr(info), B, s), "lane_factor")
            if layout in _ROOT_LAYOUTS:   # dense root: copy the assembled Schur complement out and factor it on the DMMA kernel
                _lib.check(lib.thb_sparse_lane_root_gather_f64(C.byref(d["root"]), _lib.ptr(factor), _lib.ptr(bufs["S"]), B, s), "root_gather")
                _lib.check(lib.thb_potrf_f64(_lib.ptr(bufs["S"]), None, None, _lib.ptr(bufs["info_root"]), B, d["nt"], _lib.ptr(bufs["ws"]),
                                             bufs["ws"].numel(), s), "root_potrf")
                torch.maximum(info, torch.where(bufs["info_root"] > 0, bufs["info_root"] + int(self._root[2]["root_start"]), bufs["info_root"]),
                              out=info)
        else:
            _lib.check(lib.thb_gram_f64(C.byref(d["gram"]), B, _lib.ptr(A_val), nnz, _lib.ptr(b), m, _lib.ptr(factor), P.data_size,
                                        _lib.ptr(Atb), None, s), "gram(sparse)")
            if alpha is not None:
                _lib.check(lib.thb_sparse_damp_f64(C.byref(d["plan"]), _lib.ptr(factor), _lib.ptr(alpha), _lib.ptr(beta), B, s), "sparse_damp")
            _lib.check(lib.thb_sparse_factor_f64(C.byref(d["plan"]), _lib.ptr(factor), _lib.ptr(diag), _lib.ptr(info), B, s), "sparse_factor")
        self._keep = (A_val, b, alpha, beta)
        return Atb

    def _substitute(self, rhs: torch.Tensor) -> torch.Tensor:
        """x = (L L^T)^-1 rhs with the factor of the last _numeric call (NumericDecomposition.solve); rhs, x: [B,n] fp64."""
        d, P = self._dev, self._plan
        bufs = d["bufs"]
        B, layout = bufs["key"]
        if layout == "front":
            return self._substitute_front(rhs)
        lib = _lib.load()
        rhs = rhs.contiguous()
        x = torch.empty(B, P.n, dtype=torch.float64, device=rhs.device)
        pieces = C.byref(d["pieces"]) if (layout != "item" and "pieces" in d) else None
        if layout in ("lane", "lane_tiled") and pieces is not None:
            s = _lib.stream_ptr()
            lp, F, D, W = C.byref(d[layout]), _lib.ptr(bufs["factor"]), _lib.ptr(bufs["diag"]), _lib.ptr(bufs["work"])
            _lib.check(lib.thb_sparse_lane_piece_forward_f64(lp, pieces, F, D, _lib.ptr(rhs), W, B, s), "piece_forward")
            _lib.check(lib.thb_sparse_lane_piece_backward_f64(lp, pieces, F, D, W, _lib.ptr(x), B, s), "piece_backward")
        elif layout in ("lane", "lane_tiled"):
            _lib.check(lib.thb_sparse_lane_solve_f64(C.byref(d[layout]), _lib.ptr(bufs["factor"]), _lib.ptr(bufs["diag"]), _lib.ptr(rhs), _lib.ptr(x),
                                                     _lib.ptr(bufs["work"]), B, _lib.stream_ptr()), "lane_solve")
        elif layout in _ROOT_LAYOUTS:
            s = _lib.stream_ptr()
            lp, rt = C.byref(d[layout]), C.byref(d["root"])
            F, D, W = _lib.ptr(bufs["factor"]), _lib.ptr(bufs["diag"]), _lib.ptr(bufs["work"])
            if pieces is not None:
                _lib.check(lib.thb_sparse_lane_piece_forward_f64(lp, pieces, F, D, _lib.ptr(rhs), W, B, s), "piece_forward")
            else:
                _lib.check(lib.thb_sparse_lane_forward_f64(lp, F, D, _lib.ptr(rhs), W, B, s), "lane_forward")
            _lib.check(lib.thb_sparse_lane_root_rhs_f64(lp, rt, F, _lib.ptr(rhs), W, _lib.ptr(bufs["rhs_root"]), B, s), "root_rhs")
            _lib.check(lib.thb_potrs_f64(_lib.ptr(bufs["rhs_root"]), _lib.ptr(bufs["x_root"]), B, d["nt"], _lib.ptr(bufs["ws"]), bufs["ws"].numel(), s),
                       "root_potrs")
            _lib.check(lib.thb_sparse_lane_root_scatter_f64(lp, rt, _lib.ptr(bufs["x_root"]), W, _lib.ptr(x), B, s), "root_scatter")
            if pieces is not None:
                _lib.check(lib.thb_sparse_lane_piece_backward_f64(lp, pieces, F, D, W, _lib.ptr(x), B, s), "piece_backward")
            else:
                _lib.check(lib.thb_sparse_lane_backward_f64(lp, F, D, W, _lib.ptr(x), B, s), "lane_backward")
        else:
            _lib.check(lib.thb_sparse_solve_f64(C.byref(d["plan"]), _lib.ptr(bufs["factor"]), _lib.ptr(bufs["diag"]), _lib.ptr(rhs), _lib.ptr(x),
                                                _lib.ptr(bufs["work"]), B, _lib.stream_ptr()), "sparse_solve")
        return x


BlockSparseSolver = BaspachoSparseSolver
CholmodSparseSolver = BaspachoSparseSolver   # same linear system; the CPU per-item CHOLMOD loop has no place on the GPU path
LUCudaSparseSolver = BaspachoSparseSolver    # AtA + damping is SPD: the LU variant is served by the same Cholesky
