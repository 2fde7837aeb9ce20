"""Host-side (numpy) index structure of the linear system; batch independent, computed once per objective.

Mirrors, bit for bit, the integer structure the reference builds in Python:
  * column layout          -- theseus/optimizer/linearization.py:30-41 (var_dims, var_start_cols)
  * batched-CSR of A       -- theseus/optimizer/sparse_linearization.py:34-84
                              (A_row_ptr, A_col_ind, cost_function_block_pointers / _row_block_starts / _stride)
  * block structure of AtA -- theseus/optimizer/linear/baspacho_sparse_solver.py:93-113
and adds the gather plans used by the CUDA Gram kernels (no reference analogue: the reference forms
AtA with a dense bmm or with fp64 atomics).
"""
from dataclasses import dataclass, field
from typing import List, Sequence, Tuple

import numpy as np


@dataclass
class Structure:
    var_dims: np.ndarray          # [N] int64
    var_start_cols: np.ndarray    # [N] int64
    num_cols: int
    num_rows: int
    cost_dims: np.ndarray         # [F] int64
    cost_vars: List[Tuple[int, ...]]
    cost_row0: np.ndarray         # [F] int64 first row of each cost function
    A_row_ptr: np.ndarray         # [m+1] int64
    A_col_ind: np.ndarray         # [nnz] int64
    block_pointers: List[np.ndarray]      # per cost fn: column offset of each variable's block inside a row
    row_block_starts: np.ndarray  # [F] int64 offset in A_val of the cost function's first row
    stride: np.ndarray            # [F] int64 entries per row
    extra: dict = field(default_factory=dict)

    @property
    def nnz(self) -> int:
        return int(self.A_col_ind.shape[0])


def build_structure(var_dims: Sequence[int], costs: Sequence[Tuple[int, Sequence[int]]]) -> Structure:
    """costs: (dim, variable indices in column order) per cost function, in objective order."""
    var_dims = np.asarray(var_dims, dtype=np.int64)
    starts = np.zeros_like(var_dims)
    if len(var_dims) > 1:
        starts[1:] = np.cumsum(var_dims)[:-1]
    n = int(var_dims.sum())
    col_chunks, rp_chunks = [], [np.zeros(1, dtype=np.int64)]
    bptrs, rstarts, strides, dims, row0s, cvars = [], [], [], [], [], []
    nnz = 0
    row = 0
    for dim, vs in costs:
        vs = tuple(int(v) for v in vs)
        # sort the variables' column slices the way the reference does (sparse_linearization.py:62-63)
        order = sorted(range(len(vs)), key=lambda k: (int(starts[vs[k]]), int(starts[vs[k]] + var_dims[vs[k]]), k))
        sizes = [int(var_dims[vs[k]]) for k in order]
        sptr = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        bp = np.zeros(len(vs), dtype=np.int64)
        bp[np.array(order, dtype=np.int64)] = sptr
        ci = np.concatenate([np.arange(starts[vs[k]], starts[vs[k]] + var_dims[vs[k]], dtype=np.int64) for k in order]) \
            if vs else np.zeros(0, dtype=np.int64)
        st = int(ci.shape[0])
        bptrs.append(bp)
        rstarts.append(nnz)
        strides.append(st)
        dims.append(int(dim))
        row0s.append(row)
        cvars.append(vs)
        col_chunks.append(np.tile(ci, int(dim)))
        rp_chunks.append(nnz + st * np.arange(1, int(dim) + 1, dtype=np.int64))
        nnz += st * int(dim)
        row += int(dim)
    return Structure(
        var_dims=var_dims, var_start_cols=starts, num_cols=n, num_rows=row,
        cost_dims=np.array(dims, dtype=np.int64), cost_vars=cvars, cost_row0=np.array(row0s, dtype=np.int64),
        A_row_ptr=np.concatenate(rp_chunks) if rp_chunks else np.zeros(1, dtype=np.int64),
        A_col_ind=np.concatenate(col_chunks) if col_chunks else np.zeros(0, dtype=np.int64),
        block_pointers=bptrs, row_block_starts=np.array(rstarts, dtype=np.int64),
        stride=np.array(strides, dtype=np.int64))


def ata_block_structure(s: Structure):
    """(param_size, block_ptrs, block_inds) int64: full symmetric block pattern of AtA, sorted indices
    (what BaspachoSparseSolver.reset hands to SymbolicDecomposition, baspacho_sparse_solver.py:93-113)."""
    N = len(s.var_dims)
    nbr = [set([i]) for i in range(N)]
    for vs in s.cost_vars:
        for a in vs:
            for b in vs:
                nbr[a].add(b)
    ptrs = np.zeros(N + 1, dtype=np.int64)
    inds = []
    for i in range(N):
        row = sorted(nbr[i])
        inds.extend(row)
        ptrs[i + 1] = len(inds)
    return s.var_dims.copy(), ptrs, np.array(inds, dtype=np.int64)


def lower_blocks(s: Structure, pos=None):
    """Lower-triangular variable-pair blocks (i >= j, or pos[i] >= pos[j] when an elimination order is given) that are
    structurally non-zero in AtA, with the contributing (cost function, slot a, slot b) triples.
    Returns (blocks [(i,j)], contribs [list of lists])."""
    index = {}
    blocks, contribs = [], []
    rank = (lambda v: v) if pos is None else (lambda v: int(pos[v]))
    for f, vs in enumerate(s.cost_vars):
        for a, i in enumerate(vs):
            for b, j in enumerate(vs):
                if rank(i) < rank(j):
                    continue
                key = (i, j)
                k = index.get(key)
                if k is None:
                    k = len(blocks)
                    index[key] = k
                    blocks.append(key)
                    contribs.append([])
                contribs[k].append((f, a, b))
    return blocks, contribs


GRAM_STAGE_ELEMS = 5120     # shared-memory budget of one staged Gram CTA, in scalars (40 KB of fp64: five CTAs per SM)
GRAM_STAGE_COLS = 6         # columns of a block one thread of the staged kernel accumulates (thb_gram.cu: STAGE_COLS)


def _gram_groups(s: Structure, per_var, budget):
    """Consecutive variables (structure order) cut into groups whose cost functions' rows of A and b fit `budget` scalars.
    Returns (group of each variable, [staged cost functions of each group, ascending]), or None when one variable alone does not fit."""
    if budget <= 0:
        return None
    size = s.cost_dims * (s.stride + 1)
    group_of = np.zeros(len(s.var_dims), dtype=np.int64)
    groups, cur, used = [], set(), 0
    for v in range(len(s.var_dims)):
        new = {f for f, _ in per_var[v]} - cur
        add = int(sum(size[f] for f in new))
        if cur and used + add > budget:
            groups.append(sorted(cur))
            cur, used = set(), 0
            new = {f for f, _ in per_var[v]}
            add = int(sum(size[f] for f in new))
        if add > budget:
            return None
        cur |= new
        used += add
        group_of[v] = len(groups)
    if len(s.var_dims):
        groups.append(sorted(cur))
    return group_of, groups


def build_gram_plan(s: Structure, out_offsets=None, pos=None, stage_budget=GRAM_STAGE_ELEMS):
    """Arrays of the thb_gram_plan struct (include/thb200.h).

    out_offsets: None -> dense AtA [n,n] row-major (lower blocks + mirrored upper blocks);
                 or a callable (i, j) -> (offset, ld, mirror_offset) for block-sparse factor storage.
    stage_budget: scalars of A and b one CTA of the staged kernel may hold in shared memory.  The variables are cut into groups
                 whose cost functions fit it; a variable whose cost functions alone do not fit (or stage_budget=0) leaves the plan
                 without groups, and thb_gram_f64 then runs the block-per-thread kernels (every block shape in
                 {1,2,3,6} x {1,2,3,6}) or the entry-per-thread one.
    """
    blocks, contribs = lower_blocks(s, pos)
    n = s.num_cols
    ent_blk, ent_p, ent_q = [], [], []
    blk_out, blk_ld, blk_mirror, blk_cptr = [], [], [], [0]
    blk_rows, blk_cols = [], []
    c_off, c_stride, c_rows, c_bpa, c_bpb = [], [], [], [], []
    for k, (i, j) in enumerate(blocks):
        di, dj = int(s.var_dims[i]), int(s.var_dims[j])
        pp, qq = np.meshgrid(np.arange(di), np.arange(dj), indexing="ij")
        blk_rows.append(di)
        blk_cols.append(dj)
        ent_blk.append(np.full(di * dj, k, dtype=np.int32))
        ent_p.append(pp.reshape(-1).astype(np.int16))
        ent_q.append(qq.reshape(-1).astype(np.int16))
        if out_offsets is None:
            ci, cj = int(s.var_start_cols[i]), int(s.var_start_cols[j])
            blk_out.append(ci * n + cj)
            blk_ld.append(n)
            blk_mirror.append(cj * n + ci if i != j else -1)
        else:
            off, ld, mir = out_offsets(i, j)
            blk_out.append(off)
            blk_ld.append(ld)
            blk_mirror.append(mir)
        for (f, a, b) in contribs[k]:
            c_off.append(int(s.row_block_starts[f]))
            c_stride.append(int(s.stride[f]))
            c_rows.append(int(s.cost_dims[f]))
            c_bpa.append(int(s.block_pointers[f][a]))
            c_bpb.append(int(s.block_pointers[f][b]))
        blk_cptr.append(len(c_off))
    # Atb / diag plan: per column, the cost functions that touch its variable
    per_var = [[] for _ in range(len(s.var_dims))]
    for f, vs in enumerate(s.cost_vars):
        for a, i in enumerate(vs):
            per_var[i].append((f, a))
    col_cptr = [0]
    cc_off, cc_stride, cc_rows, cc_row0 = [], [], [], []
    for i in range(len(s.var_dims)):
        for pc in range(int(s.var_dims[i])):
            for (f, a) in per_var[i]:
                cc_off.append(int(s.row_block_starts[f] + s.block_pointers[f][a] + pc))
                cc_stride.append(int(s.stride[f]))
                cc_rows.append(int(s.cost_dims[f]))
                cc_row0.append(int(s.cost_row0[f]))
            col_cptr.append(len(cc_off))

    def cat(lst, dt):
        return np.concatenate(lst).astype(dt) if lst else np.zeros(0, dtype=dt)

    # staged kernel (thb_gram.cu: gram_staged_kernel): per group of variables, the cost functions whose rows it copies to shared
    # memory (A rows, then b rows, ascending cost function), the work items (one row of one owned block, up to GRAM_STAGE_COLS
    # columns) and its columns; every contribution's shared-memory offset.  A block belongs to the group of its row variable.
    grouping = _gram_groups(s, per_var, stage_budget)
    stage_ptr, st_off, st_len, st_row0, st_dim, st_soff = [0], [], [], [], [], []
    task_ptr, task_blk, task_pq, grp_col = [0], [], [], [0]
    c_soff, cc_soff, cc_sb = np.zeros(len(c_off), np.int32), np.zeros(len(cc_off), np.int32), np.zeros(len(cc_off), np.int32)
    stage_elems = 0
    if grouping is not None:
        group_of, groups = grouping
        soff = []
        for fs in groups:
            at, o = {}, 0
            for f in fs:
                at[f] = o
                st_off.append(int(s.row_block_starts[f]))
                st_len.append(int(s.cost_dims[f] * s.stride[f]))
                st_row0.append(int(s.cost_row0[f]))
                st_dim.append(int(s.cost_dims[f]))
                st_soff.append(o)
                o += int(s.cost_dims[f] * (s.stride[f] + 1))
            soff.append(at)
            stage_ptr.append(len(st_off))
            stage_elems = max(stage_elems, o)
        owned = [[] for _ in groups]
        for k, (i, j) in enumerate(blocks):
            g = int(group_of[i])
            owned[g].append(k)
            for c, (f, a, b) in zip(range(blk_cptr[k], blk_cptr[k + 1]), contribs[k]):
                c_soff[c] = soff[g][f]
        for g, ks in enumerate(owned):
            for k in ks:
                for p in range(blk_rows[k]):
                    for q0 in range(0, blk_cols[k], GRAM_STAGE_COLS):
                        task_blk.append(k)
                        task_pq.append((p << 16) | q0)
            task_ptr.append(len(task_blk))
        cc = 0
        for i in range(len(s.var_dims)):
            g = int(group_of[i])
            for pc in range(int(s.var_dims[i])):
                for (f, a) in per_var[i]:
                    cc_soff[cc] = soff[g][f] + int(s.block_pointers[f][a]) + pc
                    cc_sb[cc] = soff[g][f] + int(s.cost_dims[f] * s.stride[f])
                    cc += 1
            if i + 1 == len(s.var_dims) or group_of[i + 1] != g:
                grp_col.append(int(s.var_start_cols[i] + s.var_dims[i]))
    # blocks grouped by shape for the block-per-thread kernels that serve plans without groups (thb_gram.cu: gram_block_kernel<DI, DJ>)
    shapes = sorted(set(zip(blk_rows, blk_cols)))
    if all(di in (1, 2, 3, 6) and dj in (1, 2, 3, 6) for di, dj in shapes):
        order, segments = [], []
        for di, dj in shapes:
            ids = [k for k in range(len(blocks)) if blk_rows[k] == di and blk_cols[k] == dj]
            segments.append((di, dj, len(order), len(order) + len(ids)))
            order.extend(ids)
        blk_order = np.array(order, dtype=np.int32)
        segments = np.ascontiguousarray(np.array(segments, dtype=np.int32).reshape(-1, 4))
    else:
        blk_order, segments = np.zeros(1, dtype=np.int32), np.zeros((0, 4), dtype=np.int32)
    return dict(
        blk_order=blk_order, segments=segments,
        num_groups=len(stage_ptr) - 1, stage_elems=stage_elems,
        stage_ptr=np.array(stage_ptr, dtype=np.int32), st_off=np.array(st_off, dtype=np.int64), st_len=np.array(st_len, dtype=np.int32),
        st_row0=np.array(st_row0, dtype=np.int32), st_dim=np.array(st_dim, dtype=np.int32), st_soff=np.array(st_soff, dtype=np.int32),
        task_ptr=np.array(task_ptr, dtype=np.int32), task_blk=np.array(task_blk, dtype=np.int32), task_pq=np.array(task_pq, dtype=np.int32),
        grp_col=np.array(grp_col, dtype=np.int32), c_soff=c_soff, cc_soff=cc_soff, cc_sb=cc_sb,
        ent_blk=cat(ent_blk, np.int32), ent_p=cat(ent_p, np.int16), ent_q=cat(ent_q, np.int16),
        blk_out=np.array(blk_out, dtype=np.int64), blk_ld=np.array(blk_ld, dtype=np.int32),
        blk_mirror=np.array(blk_mirror, dtype=np.int64), blk_cptr=np.array(blk_cptr, dtype=np.int32),
        blk_rows=np.array(blk_rows, dtype=np.int32), blk_cols=np.array(blk_cols, dtype=np.int32),
        c_off=np.array(c_off, dtype=np.int64), c_stride=np.array(c_stride, dtype=np.int32),
        c_rows=np.array(c_rows, dtype=np.int32), c_bpa=np.array(c_bpa, dtype=np.int32),
        c_bpb=np.array(c_bpb, dtype=np.int32),
        n=n, col_cptr=np.array(col_cptr, dtype=np.int32), cc_off=np.array(cc_off, dtype=np.int64),
        cc_stride=np.array(cc_stride, dtype=np.int32), cc_rows=np.array(cc_rows, dtype=np.int32),
        cc_row0=np.array(cc_row0, dtype=np.int32), blocks=blocks)
