"""Symbolic analysis for the batched block-sparse Cholesky (host side, batch independent, once per structure).

Replaces what the reference delegates to third-party code: `BaSpaCho::createSolver` behind
`SymbolicDecomposition(param_size, block_ptrs, block_inds, device)` (theseus/extlib/baspacho_solver.cpp:259-319),
`cusolverSpXcsrsymamdHost` + `csrluAnalysisHost` (extlib/cusolver_lu_solver.cpp:95-196) and CHOLMOD's `analyze_AAt`
(optimizer/linear/cholmod_sparse_solver.py:38-54).  The input is exactly what the reference hands over:
`param_size [N]` and the CSR (`ptrs`, `inds`) of the symmetric block pattern of AtA
(optimizer/linear/baspacho_sparse_solver.py:93-113).  The permutation / factor layout are internal ("parity
unpinned" in the reference too: no reference test observes them); the un-permuted solution is what is checked.

Steps: (1) minimum-degree ordering of the block graph (deterministic tie-break), (2) symbolic factorisation by
elimination -> column structures, (3) elimination-tree levels (columns of one level are independent),
(4) factor layout: per column the diagonal block then the sub-diagonal blocks, row-major,
(5) left-looking update lists: for every block (i,j) of L the pairs (L_ik, L_jk), k < j, that update it,
(6) flat per-level work-item arrays for the CUDA kernels (thb_sparse.cu).
"""
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np


def minimum_degree_order(N: int, ptrs: np.ndarray, inds: np.ndarray, weights: np.ndarray) -> np.ndarray:
    """Greedy minimum (weighted external) degree on the elimination graph.  Returns `order` (order[k] = variable eliminated k-th)."""
    adj = [set(int(x) for x in inds[ptrs[i]:ptrs[i + 1]] if int(x) != i) for i in range(N)]
    import heapq
    deg = [int(sum(weights[a] for a in adj[i])) for i in range(N)]
    heap = [(deg[i], i) for i in range(N)]
    heapq.heapify(heap)
    done = [False] * N
    order = []
    while heap:
        d, v = heapq.heappop(heap)
        if done[v] or d != deg[v]:
            continue
        done[v] = True
        order.append(v)
        nb = sorted(adj[v])
        for a in nb:
            adj[a].discard(v)
        for ai, a in enumerate(nb):  # clique among the neighbours
            sa = adj[a]
            for b in nb[ai + 1:]:
                if b not in sa:
                    sa.add(b)
                    adj[b].add(a)
        for a in nb:
            nd = int(sum(weights[x] for x in adj[a]))
            if nd != deg[a]:
                deg[a] = nd
            heapq.heappush(heap, (deg[a], a))
        adj[v] = set()
    return np.array(order, dtype=np.int64)


@dataclass
class SparsePlan:
    N: int
    n: int                       # scalar dimension
    param_size: np.ndarray       # [N] original order
    order: np.ndarray            # [N] order[k] = original variable eliminated k-th
    pos: np.ndarray              # [N] pos[v] = elimination position of original variable v
    dims: np.ndarray             # [N] block size per elimination position
    col_start: np.ndarray        # [N] scalar start (original column layout) per elimination position
    pstart: np.ndarray           # [N] scalar start in the permuted vector
    struct: List[np.ndarray]     # per position j: sorted positions i > j with L_ij != 0
    level: np.ndarray            # [N] etree level (0 = leaves)
    blk_index: Dict[Tuple[int, int], int]
    blk_off: np.ndarray          # [nblk] offset of each block of L in one batch item's factor storage
    blk_rows: np.ndarray         # [nblk] di
    blk_cols: np.ndarray         # [nblk] dj
    data_size: int
    winv_off: np.ndarray         # [N] offset of W_j = L_jj^-1 in the inverse-diagonal storage
    winv_size: int
    arrays: Dict[str, np.ndarray]
    stats: Dict[str, float]
    lane: Dict[str, np.ndarray] = None   # work lists of the batch-lane kernels (thb_sparse_lane.cu), see _lane_lists
    chain_of: np.ndarray = None          # [N] fundamental-supernode ("chain") index of every column, see _chains
    chain_level: np.ndarray = None       # [num_chains] level of the chain in the chain tree


_PLAN_KEYS = ("dims", "col_start", "pstart", "winv_off", "diag_off", "up_a", "up_b", "up_k", "u_ptr", "u_tgt", "u_r", "u_c", "u_ld", "u_p0",
              "u_p1", "f_ptr", "f_off", "f_dim", "f_w", "f_col", "t_ptr", "t_off", "t_r", "t_dim", "t_w", "s_ptr", "s_col", "fr_ptr",
              "fr_off", "fr_k", "bc_ptr", "bc_off", "bc_i")
_LANE_KEYS = ("u_tgt", "u_p0", "u_p1", "t_off", "t_diag", "t_dl", "t_pstart", "s_col", "launches", "fr_p", "fr_d", "bc_p", "bc_d")
_NP_OF_BYTES = {2: np.int16, 4: np.int32, 8: np.int64}


def analyze(param_size: np.ndarray, ptrs: np.ndarray, inds: np.ndarray, ordering: str = "mindeg") -> SparsePlan:
    """Symbolic analysis by the native library (thb_symbolic_create, csrc/thb_symbolic.cu); `analyze_py` below is the same
    algorithm in Python -- the executable specification the tests compare against, array by array."""
    import ctypes as C
    from . import _lib
    if ordering not in ("mindeg", "natural"):
        raise ValueError(ordering)
    lib = _lib.load()
    ps = np.ascontiguousarray(param_size, dtype=np.int64)
    pt = np.ascontiguousarray(ptrs, dtype=np.int64)
    ix = np.ascontiguousarray(inds, dtype=np.int64)
    N = int(ps.shape[0])
    h = C.c_void_p()
    _lib.check(lib.thb_symbolic_create(ps.ctypes.data, N, pt.ctypes.data, ix.ctypes.data, 0 if ordering == "mindeg" else 1, C.byref(h)),
               "symbolic_create")
    try:
        def arr(name):
            cnt = int(lib.thb_symbolic_array_count(h, name.encode()))
            if cnt < 0:
                raise KeyError(name)
            out = np.empty(cnt, dtype=_NP_OF_BYTES[int(lib.thb_symbolic_array_elem_bytes(h, name.encode()))])
            _lib.check(lib.thb_symbolic_array_copy(h, name.encode(), out.ctypes.data, out.nbytes), f"symbolic array {name}")
            return out

        def stat(name):
            return float(lib.thb_symbolic_stat(h, name.encode()))
        arrays = {k: arr(k) for k in _PLAN_KEYS}
        lane = {k: arr("ln_" + k) for k in _LANE_KEYS}
        lane["launches"] = lane["launches"].reshape(-1, 5)
        order, pos, level = arr("order"), arr("pos"), arr("level")
        sp, si = arr("struct_ptr"), arr("struct_idx")
        blk_off, blk_i, blk_j = arr("blk_off"), arr("blk_i"), arr("blk_j")
        blk_rows, blk_cols = arr("blk_rows"), arr("blk_cols")
        stats = {k: stat(k) for k in ("nnz_L", "flops", "levels", "max_front", "num_updates", "num_chains", "chain_levels")}
        chain_of, chain_level = arr("chain_of"), arr("chain_level")
        n, data_size, winv_size = int(stat("n")), int(stat("data_size")), int(stat("winv_size"))
        dims, col_start, pstart = arr("dims64"), arr("col_start64"), arr("pstart64")
    finally:
        lib.thb_symbolic_destroy(h)
    struct = [si[sp[j]:sp[j + 1]] for j in range(N)]
    blk_index = {(int(i), int(j)): t for t, (i, j) in enumerate(zip(blk_i.tolist(), blk_j.tolist()))}
    return SparsePlan(N=N, n=n, param_size=ps, order=order, pos=pos, dims=dims, col_start=col_start, pstart=pstart, struct=struct, level=level,
                      blk_index=blk_index, blk_off=blk_off, blk_rows=blk_rows, blk_cols=blk_cols, data_size=data_size,
                      winv_off=arrays["winv_off"], winv_size=winv_size, arrays=arrays, stats=stats, lane=lane,
                      chain_of=chain_of, chain_level=chain_level)


def analyze_py(param_size: np.ndarray, ptrs: np.ndarray, inds: np.ndarray, ordering: str = "mindeg") -> SparsePlan:
    param_size = np.asarray(param_size, dtype=np.int64)
    N = int(param_size.shape[0])
    if ordering == "mindeg":
        order = minimum_degree_order(N, ptrs, inds, param_size)
    elif ordering == "natural":
        order = np.arange(N, dtype=np.int64)
    else:
        raise ValueError(ordering)
    pos = np.empty(N, dtype=np.int64)
    pos[order] = np.arange(N)
    dims = param_size[order]
    orig_start = np.concatenate([[0], np.cumsum(param_size)[:-1]]).astype(np.int64)
    col_start = orig_start[order]
    pstart = np.concatenate([[0], np.cumsum(dims)[:-1]]).astype(np.int64)
    n = int(param_size.sum())

    # ---- symbolic factorisation in elimination order ----
    adj = [set() for _ in range(N)]
    for v in range(N):
        pv = int(pos[v])
        for u in inds[ptrs[v]:ptrs[v + 1]]:
            pu = int(pos[int(u)])
            if pu != pv:
                adj[pv].add(pu)
    struct: List[np.ndarray] = []
    for j in range(N):
        s = sorted(x for x in adj[j] if x > j)
        struct.append(np.array(s, dtype=np.int64))
        if s:
            p = s[0]  # etree parent: the column structure is merged into the parent's
            adj[p].update(x for x in s if x != p)
    parent = np.array([int(s[0]) if len(s) else -1 for s in struct], dtype=np.int64)
    level = np.zeros(N, dtype=np.int64)
    for j in range(N):
        if parent[j] >= 0:
            level[parent[j]] = max(level[parent[j]], level[j] + 1)
    nlev = int(level.max()) + 1 if N else 0

    # ---- factor layout ----
    blk_index: Dict[Tuple[int, int], int] = {}
    blk_off, blk_rows, blk_cols = [], [], []
    off = 0
    for j in range(N):
        for i in [j] + list(struct[j]):
            blk_index[(int(i), j)] = len(blk_off)
            blk_off.append(off)
            blk_rows.append(int(dims[i]))
            blk_cols.append(int(dims[j]))
            off += int(dims[i]) * int(dims[j])
    data_size = off
    winv_off = np.concatenate([[0], np.cumsum(dims * dims)[:-1]]).astype(np.int64)
    winv_size = int((dims * dims).sum())
    blk_off = np.array(blk_off, dtype=np.int64)
    blk_rows = np.array(blk_rows, dtype=np.int32)
    blk_cols = np.array(blk_cols, dtype=np.int32)
    nblk = len(blk_off)

    # ---- left-looking update lists: target block (a,b), a >= b > k, gets (L_ak, L_bk) ----
    upd: List[List[Tuple[int, int]]] = [[] for _ in range(nblk)]
    flops = 0
    for k in range(N):
        s = struct[k]
        dk = int(dims[k])
        flops += dk ** 3 // 3
        ids = [blk_index[(int(i), k)] for i in s]
        for bi in range(len(s)):
            flops += int(dims[s[bi]]) * dk * dk  # trsm
            for ai in range(bi, len(s)):
                t = blk_index[(int(s[ai]), int(s[bi]))]
                upd[t].append((ids[ai], ids[bi]))
                flops += 2 * int(dims[s[ai]]) * int(dims[s[bi]]) * dk
    up_ptr = np.zeros(nblk + 1, dtype=np.int64)
    for t in range(nblk):
        up_ptr[t + 1] = up_ptr[t] + len(upd[t])
    up_a = np.zeros(int(up_ptr[-1]), dtype=np.int64)
    up_b = np.zeros(int(up_ptr[-1]), dtype=np.int64)
    up_k = np.zeros(int(up_ptr[-1]), dtype=np.int32)
    for t in range(nblk):
        for q, (ia, ib) in enumerate(upd[t]):
            up_a[up_ptr[t] + q] = blk_off[ia]
            up_b[up_ptr[t] + q] = blk_off[ib]
            up_k[up_ptr[t] + q] = blk_cols[ia]

    # ---- per-level work items ----
    cols_by_level = [[] for _ in range(nlev)]
    for j in range(N):
        cols_by_level[int(level[j])].append(j)
    # stage U: one item per updated block of the level's columns: (offset, rows, cols, is_diagonal, update-pair range)
    u_ptr = [0]
    u_tgt, u_r, u_c, u_ld, u_p0, u_p1 = [], [], [], [], [], []
    # stage F: one item per column (diag potrf + inverse)
    f_ptr = [0]
    f_off, f_dim, f_w, f_col = [], [], [], []
    # stage T: one item per row of every sub-diagonal block
    t_ptr = [0]
    t_off, t_r, t_dim, t_w = [], [], [], []
    # solve: per column row-structure (forward) and column-structure (backward)
    row_lists: List[List[Tuple[int, int]]] = [[] for _ in range(N)]  # for target j: (offset of L_jk, k)
    for k in range(N):
        for i in struct[k]:
            row_lists[int(i)].append((int(blk_off[blk_index[(int(i), k)]]), k))
    s_ptr = [0]
    s_col = []
    for lv in range(nlev):
        for j in cols_by_level[lv]:
            dj = int(dims[j])
            for i in [j] + list(struct[j]):
                t = blk_index[(int(i), j)]
                di = int(dims[i])
                if up_ptr[t + 1] > up_ptr[t]:  # blocks without updates (leaves) need no work item
                    # one item per BLOCK (the kernel spreads its di*dj scalars over threads): keeps the index stream tiny
                    u_tgt.append(int(blk_off[t])); u_r.append(di); u_c.append(dj); u_ld.append(1 if i == j else 0)
                    u_p0.append(int(up_ptr[t])); u_p1.append(int(up_ptr[t + 1]))
                if i != j:
                    for r in range(di):
                        t_off.append(int(blk_off[t])); t_r.append(r); t_dim.append(dj); t_w.append(int(winv_off[j]))
            f_off.append(int(blk_off[blk_index[(j, j)]])); f_dim.append(dj); f_w.append(int(winv_off[j])); f_col.append(j)
            s_col.append(j)
        u_ptr.append(len(u_tgt)); f_ptr.append(len(f_off)); t_ptr.append(len(t_off)); s_ptr.append(len(s_col))
    # solve lists
    fr_ptr = [0]
    fr_off, fr_k = [], []
    bc_ptr = [0]
    bc_off, bc_i = [], []
    for j in range(N):
        for (o, k) in row_lists[j]:
            fr_off.append(o); fr_k.append(k)
        fr_ptr.append(len(fr_off))
        for i in struct[j]:
            bc_off.append(int(blk_off[blk_index[(int(i), j)]])); bc_i.append(int(i))
        bc_ptr.append(len(bc_off))

    i32, i64 = np.int32, np.int64
    arrays = dict(
        dims=dims.astype(i32), col_start=col_start.astype(i32), pstart=pstart.astype(i32), winv_off=winv_off.astype(i64),
        diag_off=np.array([blk_off[blk_index[(j, j)]] for j in range(N)], dtype=i64),
        up_a=up_a, up_b=up_b, up_k=up_k,
        u_ptr=np.array(u_ptr, dtype=i64), u_tgt=np.array(u_tgt, dtype=i64), u_r=np.array(u_r, dtype=np.int16),
        u_c=np.array(u_c, dtype=np.int16), u_ld=np.array(u_ld, dtype=np.int16), u_p0=np.array(u_p0, dtype=i64),
        u_p1=np.array(u_p1, dtype=i64),
        f_ptr=np.array(f_ptr, dtype=i64), f_off=np.array(f_off, dtype=i64), f_dim=np.array(f_dim, dtype=i32),
        f_w=np.array(f_w, dtype=i64), f_col=np.array(f_col, dtype=i32),
        t_ptr=np.array(t_ptr, dtype=i64), t_off=np.array(t_off, dtype=i64), t_r=np.array(t_r, dtype=np.int16),
        t_dim=np.array(t_dim, dtype=np.int16), t_w=np.array(t_w, dtype=i64),
        s_ptr=np.array(s_ptr, dtype=i64), s_col=np.array(s_col, dtype=i32),
        fr_ptr=np.array(fr_ptr, dtype=i64), fr_off=np.array(fr_off, dtype=i64), fr_k=np.array(fr_k, dtype=i32),
        bc_ptr=np.array(bc_ptr, dtype=i64), bc_off=np.array(bc_off, dtype=i64), bc_i=np.array(bc_i, dtype=i32))
    chain_of, chain_level = _chains(N, struct, parent)
    lane = _lane_lists(N, nlev, cols_by_level, struct, dims, blk_index, blk_off, up_ptr, winv_off, pstart)
    fr_k_arr, bc_i_arr = np.array(fr_k, dtype=np.int64), np.array(bc_i, dtype=np.int64)
    lane.update(fr_p=pstart[fr_k_arr].astype(np.int32), fr_d=dims[fr_k_arr].astype(np.int32),
                bc_p=pstart[bc_i_arr].astype(np.int32), bc_d=dims[bc_i_arr].astype(np.int32))
    stats = dict(nnz_L=float(data_size), flops=float(flops), levels=float(nlev), max_front=float(max((len(s) + 1 for s in struct), default=0)),
                 num_updates=float(up_ptr[-1]), num_chains=float(len(chain_level)),
                 chain_levels=float(chain_level.max() + 1 if len(chain_level) else 0))
    return SparsePlan(N=N, n=n, param_size=param_size, order=order, pos=pos, dims=dims, col_start=col_start, pstart=pstart,
                      struct=struct, level=level, blk_index=blk_index, blk_off=blk_off, blk_rows=blk_rows, blk_cols=blk_cols,
                      data_size=data_size, winv_off=winv_off, winv_size=winv_size, arrays=arrays, stats=stats, lane=lane,
                      chain_of=chain_of, chain_level=chain_level)


def _chains(N, struct, parent):
    """Fundamental supernodes ("chains"): maximal runs j, j+1, ... with parent(j) = j+1, struct(j) = {j+1} + struct(j+1) and j the only
    child of j+1.  Returns (chain_of [N]: index of the column's chain, chain_level [num_chains]: level in the chain tree).  Not used by
    the round-1 kernels; it is the partition the round-2 numeric phase will run on."""
    nchild = np.zeros(N, dtype=np.int64)
    for j in range(N):
        if parent[j] >= 0:
            nchild[parent[j]] += 1
    chain_of = np.full(N, -1, dtype=np.int64)
    nchains = 0
    for j in range(N):
        if chain_of[j] >= 0:
            continue
        chain_of[j] = nchains
        k = j
        while True:
            p = int(parent[k])
            if p != k + 1 or nchild[p] != 1 or len(struct[k]) != len(struct[p]) + 1:
                break
            chain_of[p] = nchains   # struct(k) = {p} + struct(p) follows from the equal sizes (struct(k) minus {p} is a subset of struct(p))
            k = p
        nchains += 1
    chain_level = np.zeros(nchains, dtype=np.int64)
    for j in range(N):
        p = int(parent[j])
        if p >= 0 and chain_of[p] != chain_of[j]:
            chain_level[chain_of[p]] = max(chain_level[chain_of[p]], chain_level[chain_of[j]] + 1)
    return chain_of, chain_level


LANE_DIMS = (1, 2, 3, 6)   # block sizes the batch-lane kernels are instantiated for (thb_sparse_lane.cu)
ITEM_MAX_DIM = 16          # largest block size of the one-CTA-per-item kernels (SP_MAXD, thb_sparse.cu)
LANE_HEAVY = 8             # update pairs per target block from which the split-K variant of the update kernel is used
LN_U, LN_T, LN_S, LN_UH, LN_TU = 0, 1, 2, 3, 4
TILE_DIM, TILE_ROWS, TILE_COLS = 6, 4, 4   # the tiled update kernel is instantiated for 6x6 blocks in 4 x 4 tiles (thb_sparse_lane.cu)


def _lane_lists(N, nlev, cols_by_level, struct, dims, blk_index, blk_off, up_ptr, winv_off, pstart, u_start=None, pre_launches=None):
    """Work lists for the batch-lane kernels: per level, the target blocks grouped by (rows, cols) class, because those
    kernels keep a whole block in registers and are compiled per block shape.  `launches` is a HOST array of
    (kind, di, dj, begin, end) rows in execution order: kind U = left-looking update of blocks [begin,end) of u_*,
    UH = the same for blocks with many update pairs (split over 8 warps), T = diagonal factor + triangular solve of blocks
    [begin,end) of t_*, S = columns [begin,end) of s_col for the substitutions (forward: in order, backward: reversed).
    `u_start[t]` (optional) = first update pair of block t that is still to be done by a U launch (the earlier ones are covered by
    a tile launch, tile_lane_lists); `pre_launches[lv]` (optional) = launch rows that open level lv."""
    u_tgt, u_p0, u_p1 = [], [], []
    t_off, t_diag, t_dl, t_pstart = [], [], [], []
    s_col = []
    launches = []
    for lv in range(nlev):
        ucls: Dict[Tuple[int, int, int], list] = {}
        tcls: Dict[Tuple[int, int], list] = {}
        scls: Dict[int, list] = {}
        if pre_launches is not None:
            launches.extend(pre_launches[lv])
        for j in cols_by_level[lv]:
            dj = int(dims[j])
            scls.setdefault(dj, []).append(j)
            dg = int(blk_off[blk_index[(j, j)]])
            for i in [j] + [int(x) for x in struct[j]]:
                t = blk_index[(i, j)]
                di = int(dims[i])
                first = int(up_ptr[t]) if u_start is None else int(u_start[t])
                npairs = int(up_ptr[t + 1]) - first
                if npairs > 0:
                    ucls.setdefault((1 if npairs >= LANE_HEAVY else 0, di, dj), []).append(t)
                tcls.setdefault((di, dj), []).append((t, dg, j))
        for (heavy, di, dj) in sorted(ucls):
            b0 = len(u_tgt)
            for t in ucls[(heavy, di, dj)]:
                u_tgt.append(int(blk_off[t])); u_p0.append(int(up_ptr[t]) if u_start is None else int(u_start[t])); u_p1.append(int(up_ptr[t + 1]))
            launches.append((LN_UH if heavy else LN_U, di, dj, b0, len(u_tgt)))
        for (di, dj) in sorted(tcls):
            b0 = len(t_off)
            for (t, dg, j) in tcls[(di, dj)]:
                t_off.append(int(blk_off[t])); t_diag.append(dg); t_dl.append(int(winv_off[j])); t_pstart.append(int(pstart[j]))
            launches.append((LN_T, di, dj, b0, len(t_off)))
        for dj in sorted(scls):
            b0 = len(s_col)
            s_col.extend(scls[dj])
            launches.append((LN_S, dj, dj, b0, len(s_col)))
    i64 = np.int64
    return dict(u_tgt=np.array(u_tgt, dtype=i64), u_p0=np.array(u_p0, dtype=i64), u_p1=np.array(u_p1, dtype=i64),
                t_off=np.array(t_off, dtype=i64), t_diag=np.array(t_diag, dtype=i64), t_dl=np.array(t_dl, dtype=i64),
                t_pstart=np.array(t_pstart, dtype=np.int32), s_col=np.array(s_col, dtype=np.int32),
                launches=np.array(launches, dtype=np.int32).reshape(-1, 5))


def gram_out_offsets(plan: SparsePlan):
    """Callable for structure.build_gram_plan: where block (a, b) of AtA (original variable indices, pos[a] >= pos[b])
    lands in the factor storage.  Returns (offset, leading dimension, mirror=-1)."""
    def f(a: int, b: int):
        t = plan.blk_index[(int(plan.pos[a]), int(plan.pos[b]))]
        return int(plan.blk_off[t]), int(plan.blk_cols[t]), -1
    return f


def root_split(plan: SparsePlan, max_root_dof: int = 1024, min_root_cols: int = 8):
    """Round-2 building block (host side, CPU-tested; no kernel consumes it yet).

    The top of the elimination tree is a long chain whose columns form a DENSE trailing block (C5: the last 64 columns, 384 dof):
    ~200 serial one-column levels for the lane kernels, one small job for the dense DMMA Cholesky.  This splits a plan at `cut`:
      * bottom: columns < cut with the usual per-level lane work lists (their blocks in root ROWS are ordinary blocks of those columns),
      * root assembly: for every root block (i, j), i >= j >= cut, the update pairs that come from bottom columns (k < cut: a prefix
        of the block's pair list) -> S = A_root - sum_k L_ik L_jk^T, copied into a dense [B, nt, nt] matrix and factored there,
      * root substitution: per root column the blocks L_jk, k < cut, to fold the bottom part of y into the dense right-hand side.
    Returns None if the plan has no useful dense root, else a dict of arrays."""
    N, dims, pstart = plan.N, plan.dims, plan.pstart
    if N == 0:
        return None
    last = plan.chain_of[N - 1]
    cut = int(np.argmax(plan.chain_of == last))
    while int(dims[cut:].sum()) > max_root_dof:
        cut += 1
    if N - cut < min_root_cols:
        return None
    for j in range(cut, N):
        assert np.array_equal(plan.struct[j], np.arange(j + 1, N)), "the root must be a dense trailing block"
    A = plan.arrays
    nblk = len(plan.blk_off)
    blk_j = np.empty(nblk, dtype=np.int64)
    blk_i = np.empty(nblk, dtype=np.int64)
    for (i, j), t in plan.blk_index.items():
        blk_i[t], blk_j[t] = i, j
    # source column of every update pair (pairs of a block are stored in increasing k)
    up_ptr = np.zeros(nblk + 1, dtype=np.int64)
    # rebuild up_ptr from the U items of both back ends is awkward; recompute it from the structure instead
    counts = np.zeros(nblk, dtype=np.int64)
    for k in range(N):
        s_ = plan.struct[k]
        for bi in range(len(s_)):
            for ai in range(bi, len(s_)):
                counts[plan.blk_index[(int(s_[ai]), int(s_[bi]))]] += 1
    up_ptr[1:] = np.cumsum(counts)
    src_blk = np.searchsorted(plan.blk_off, A["up_a"], side="right") - 1
    pair_k = blk_j[src_blk]
    level_cut = int(plan.level[cut])
    assert all(int(plan.level[j]) < level_cut for j in range(cut)) and all(int(plan.level[j]) >= level_cut for j in range(cut, N))
    nlev_bottom = level_cut
    cols_by_level = [[] for _ in range(nlev_bottom)]
    for j in range(cut):
        cols_by_level[int(plan.level[j])].append(j)
    bottom = _lane_lists(N, nlev_bottom, cols_by_level, plan.struct, dims, plan.blk_index, plan.blk_off, up_ptr, plan.winv_off, pstart)
    # root assembly: (target offset, first pair, one-past-last pair with k < cut), dense placement of every root block
    ru_tgt, ru_p0, ru_p1, rb_off, rb_row, rb_col, rb_di, rb_dj = [], [], [], [], [], [], [], []
    root0 = int(pstart[cut])
    for j in range(cut, N):
        for i in range(j, N):
            t = plan.blk_index[(i, j)]
            p0, p1 = int(up_ptr[t]), int(up_ptr[t + 1])
            n_bottom = int(np.searchsorted(pair_k[p0:p1], cut, side="left"))
            assert (pair_k[p0:p0 + n_bottom] < cut).all() and (pair_k[p0 + n_bottom:p1] >= cut).all()
            if n_bottom > 0:
                ru_tgt.append(int(plan.blk_off[t])); ru_p0.append(p0); ru_p1.append(p0 + n_bottom)
            rb_off.append(int(plan.blk_off[t])); rb_row.append(int(pstart[i]) - root0); rb_col.append(int(pstart[j]) - root0)
            rb_di.append(int(dims[i])); rb_dj.append(int(dims[j]))
    # root substitution: per root column the prefix of its row list that lies in bottom columns
    rf_p0, rf_p1 = [], []
    for j in range(cut, N):
        p0, p1 = int(A["fr_ptr"][j]), int(A["fr_ptr"][j + 1])
        ks = A["fr_k"][p0:p1]
        n_bottom = int(np.searchsorted(ks, cut, side="left"))
        assert (ks[:n_bottom] < cut).all() and (ks[n_bottom:] >= cut).all()
        rf_p0.append(p0); rf_p1.append(p0 + n_bottom)
    i64 = np.int64
    return dict(cut=cut, root_dof=int(dims[cut:].sum()), root_start=root0, bottom=bottom, up_ptr=up_ptr, pair_k=pair_k,
                ru_tgt=np.array(ru_tgt, dtype=i64), ru_p0=np.array(ru_p0, dtype=i64), ru_p1=np.array(ru_p1, dtype=i64),
                rb_off=np.array(rb_off, dtype=i64), rb_row=np.array(rb_row, dtype=np.int32), rb_col=np.array(rb_col, dtype=np.int32),
                rb_di=np.array(rb_di, dtype=np.int32), rb_dj=np.array(rb_dj, dtype=np.int32),
                rf_p0=np.array(rf_p0, dtype=i64), rf_p1=np.array(rf_p1, dtype=i64))


def root_lane_lists(plan: SparsePlan, sp) -> Tuple[Dict[str, np.ndarray], Dict[str, np.ndarray]]:
    """Work lists of the opt-in `lane_root` layout from a root_split: (lane lists = the bottom columns' lists followed by the root's
    assembly updates, grouped by block shape like every U launch; root arrays for thb_sparse_lane_root)."""
    bottom = sp["bottom"]
    u_tgt, u_p0, u_p1 = list(bottom["u_tgt"]), list(bottom["u_p0"]), list(bottom["u_p1"])
    launches = [tuple(int(x) for x in row) for row in bottom["launches"]]
    shape_of = {int(o): (int(a), int(b)) for o, a, b in zip(sp["rb_off"], sp["rb_di"], sp["rb_dj"])}
    cls: Dict[Tuple[int, int, int], list] = {}
    for e in range(len(sp["ru_tgt"])):
        di, dj = shape_of[int(sp["ru_tgt"][e])]
        heavy = 1 if int(sp["ru_p1"][e] - sp["ru_p0"][e]) >= LANE_HEAVY else 0
        cls.setdefault((heavy, di, dj), []).append(e)
    for (heavy, di, dj) in sorted(cls):
        b0 = len(u_tgt)
        for e in cls[(heavy, di, dj)]:
            u_tgt.append(int(sp["ru_tgt"][e])); u_p0.append(int(sp["ru_p0"][e])); u_p1.append(int(sp["ru_p1"][e]))
        launches.append((LN_UH if heavy else LN_U, di, dj, b0, len(u_tgt)))
    i64 = np.int64
    lane = dict(bottom)
    lane.update(u_tgt=np.array(u_tgt, dtype=i64), u_p0=np.array(u_p0, dtype=i64), u_p1=np.array(u_p1, dtype=i64),
                launches=np.array(launches, dtype=np.int32).reshape(-1, 5),
                fr_p=plan.lane["fr_p"], fr_d=plan.lane["fr_d"], bc_p=plan.lane["bc_p"], bc_d=plan.lane["bc_d"])
    cut = sp["cut"]
    root_cols = np.arange(cut, plan.N, dtype=np.int32)
    order = np.argsort(plan.dims[cut:], kind="stable")          # root columns grouped by block size for the rhs kernel
    cols_sorted = root_cols[order]
    segs, b0 = [], 0
    ds = plan.dims[cut:][order]
    for q in range(1, len(ds) + 1):
        if q == len(ds) or ds[q] != ds[b0]:
            segs.append((int(ds[b0]), b0, q)); b0 = q
    root = dict(rb_off=sp["rb_off"], rb_row=sp["rb_row"], rb_col=sp["rb_col"], rb_di=sp["rb_di"], rb_dj=sp["rb_dj"],
                rf_p0=sp["rf_p0"][order], rf_p1=sp["rf_p1"][order], root_cols=cols_sorted.astype(np.int32), root_dims=ds.astype(np.int32),
                segments=np.array(segs, dtype=np.int32).reshape(-1, 3), nt=sp["root_dof"], root_start=sp["root_start"])
    return lane, root


def chain_tiles(plan: SparsePlan, max_width: int = 4, tile_rows: int = 4, breaks=()):
    """Round-2 building block (host side, specification level: Python lists, checked by a numpy interpreter in
    tests/test_sparse_symbolic.py; no kernel consumes it yet).  The schedule of the TILED update stage:

      * chains (fundamental supernodes) are cut into pieces of <= max_width consecutive columns;
      * the update pairs of every block (i, j) split into EXTERNAL ones (source column k before the first column j0 of j's piece;
        a prefix of the pair list) and INTERNAL ones (j0 <= k < j);
      * external updates run per TILE = (piece, tile_rows consecutive rows of the piece's row structure): the tile's targets are the
        blocks (i, j), i in the row tile, j in the piece, i >= j; for every source column k that updates any of them the tile needs at
        most tile_rows + max_width source blocks L_ik, L_jk -- staged once (shared memory on the GPU) and used by all targets of the
        tile that have both.  This is where the 1.96 -> 0.70 block loads per update come from;
      * a piece's tiles are due at the level of its first column (all external sources are descendants of j0, hence finished);
        internal updates and the diagonal/triangular stage stay per column and per level as today.

    Returns dict(piece_first [N], per_level: list over levels of dict(tiles=[...], u_int=[(block id, p0, p1)], cols=[...]), up_ptr,
    block_loads, updates) with tiles = dict(targets=[(row slot, col slot, block id)], steps=[(k, [row block id or -1]*tile_rows,
    [col block id or -1]*width)])."""
    N, dims = plan.N, plan.dims
    struct = [np.asarray(s_, dtype=np.int64) for s_ in plan.struct]
    nblk = len(plan.blk_off)
    counts = np.zeros(nblk, dtype=np.int64)
    pair_k: List[List[int]] = [[] for _ in range(nblk)]
    for k in range(N):
        s_ = struct[k]
        for bi in range(len(s_)):
            for ai in range(bi, len(s_)):
                t = plan.blk_index[(int(s_[ai]), int(s_[bi]))]
                counts[t] += 1
                pair_k[t].append(k)
    up_ptr = np.zeros(nblk + 1, dtype=np.int64)
    up_ptr[1:] = np.cumsum(counts)
    # pieces
    piece_first = np.zeros(N, dtype=np.int64)
    j = 0
    while j < N:
        c = plan.chain_of[j]
        e = j
        while e + 1 < N and plan.chain_of[e + 1] == c and e + 1 - j < max_width and (e + 1) not in breaks:   # breaks: forced piece starts
            e += 1
        piece_first[j:e + 1] = j
        j = e + 1
    rowset = [set() for _ in range(N)]  # rowset[x] = {k : L_xk != 0}
    for k in range(N):
        for i in struct[k]:
            rowset[int(i)].add(k)
    nlev = int(plan.level.max()) + 1 if N else 0
    per_level = [dict(tiles=[], u_int=[], cols=[]) for _ in range(nlev)]
    block_loads = updates = 0
    for j0 in sorted(set(piece_first.tolist())):
        cols = [j for j in range(j0, N) if piece_first[j] == j0]
        j1 = cols[-1]
        rows = cols + [int(x) for x in struct[j1]]
        lv0 = int(plan.level[j0])
        for r0 in range(0, len(rows), tile_rows):
            rt = rows[r0:r0 + tile_rows]
            targets = [(a, b, plan.blk_index[(i, jj)]) for a, i in enumerate(rt) for b, jj in enumerate(cols) if i >= jj]
            ks = sorted(set(k for (_, _, t) in targets for k in pair_k[t] if k < j0))
            steps = []
            for k in ks:
                ro = [plan.blk_index[(i, k)] if k in rowset[i] else -1 for i in rt] + [-1] * (tile_rows - len(rt))
                co = [plan.blk_index[(jj, k)] if k in rowset[jj] else -1 for jj in cols]
                steps.append((k, ro, co))
                block_loads += len(set(x for x in ro + co if x >= 0))
                updates += sum(1 for (a, b, t) in targets if ro[a] >= 0 and co[b] >= 0)
            if steps:
                per_level[lv0]["tiles"].append(dict(targets=targets, steps=steps, piece=(j0, j1)))
    for j in range(N):
        lv = int(plan.level[j])
        per_level[lv]["cols"].append(j)
        for i in [j] + [int(x) for x in struct[j]]:
            t = plan.blk_index[(i, j)]
            ks = pair_k[t]
            n_ext = int(np.searchsorted(np.asarray(ks, dtype=np.int64), piece_first[j], side="left"))
            if n_ext < len(ks):
                per_level[lv]["u_int"].append((t, int(up_ptr[t]) + n_ext, int(up_ptr[t + 1])))
    return dict(piece_first=piece_first, per_level=per_level, up_ptr=up_ptr, block_loads=block_loads, updates=updates)



def tile_lane_lists(plan: SparsePlan, sp=None) -> Tuple[Dict[str, np.ndarray], Dict[str, np.ndarray]]:
    """Work lists of the opt-in `lane_tiled` / `lane_tiled_root` layouts: the chain_tiles schedule flattened for
    thb_sparse_lane_factor_tiled_f64.

    Tiles whose targets and sources are all TILE_DIM x TILE_DIM blocks become rows of the tile arrays
      tile_tgt  [T, TILE_ROWS*TILE_COLS]  offset of target block (row slot a, column slot b) at a*TILE_COLS+b, -1 if absent
      step_ptr  [T+1]                      k steps of tile t = step_ptr[t] .. step_ptr[t+1]
      step_src  [S, TILE_ROWS+TILE_COLS]   offsets of the source blocks L_(row a),k (first TILE_ROWS entries) and L_(column b),k, -1 if zero
    and a launch row (LN_TU, 6, 6, first tile, one past last tile) opens the level of the piece's first column; the update pairs they
    cover (a prefix of each target's pair list) are dropped from the U / UH items.  Every other block keeps its full pair list.

    With a root split `sp` (root_split): the columns below the cut as above; the root's ASSEMBLY (update pairs with k < cut into root
    blocks: the Schur complement that the dense kernel factors) becomes ONE tile launch after the last bottom level -- every tile of a
    root piece with its steps restricted to k < cut, all independent of each other -- followed by the per-block items of the root blocks
    no tile covers.  (Without the split those tiles sit one piece per level at the top of the tree, a serial chain of long k loops.)
    Returns (lane lists, tile arrays)."""
    cut = plan.N
    if sp is not None:
        cut = int(sp["cut"])
    ct = chain_tiles(plan, max_width=TILE_COLS, tile_rows=TILE_ROWS, breaks=(cut,))
    N, dims = plan.N, plan.dims
    up_ptr = ct["up_ptr"]
    nblk = len(plan.blk_off)
    blk_shape = np.zeros((nblk, 2), dtype=np.int64)
    blk_col = np.zeros(nblk, dtype=np.int64)
    for (i, j), t in plan.blk_index.items():
        blk_shape[t] = (dims[i], dims[j])
        blk_col[t] = j
    nlev = len(ct["per_level"])
    level_cut = int(plan.level[cut]) if cut < N else nlev
    u_start = up_ptr[:-1].copy()
    tile_tgt, step_ptr, step_src = [], [0], []
    pre = [[] for _ in range(nlev)]
    # pairs of a block are stored in increasing source column k: the external ones (k < first column of the piece) are a prefix
    A = plan.arrays
    src_blk = np.searchsorted(plan.blk_off, A["up_a"], side="right") - 1
    pair_k = blk_col[src_blk]

    def emit(tile, steps, k_end):
        """Append one tile with the given steps; marks the pairs with k < k_end of its targets as done.  False if not all 6x6."""
        ids = [t for (_, _, t) in tile["targets"]] + [x for (_, ro, co) in steps for x in ro + co if x >= 0]
        if not steps or not all(blk_shape[t][0] == TILE_DIM and blk_shape[t][1] == TILE_DIM for t in ids):
            return False
        row = [-1] * (TILE_ROWS * TILE_COLS)
        for (a, b, t) in tile["targets"]:
            row[a * TILE_COLS + b] = int(plan.blk_off[t])
            p0, p1 = int(up_ptr[t]), int(up_ptr[t + 1])
            n_ext = int(np.searchsorted(pair_k[p0:p1], k_end, side="left"))
            assert (pair_k[p0:p0 + n_ext] < k_end).all() and (pair_k[p0 + n_ext:p1] >= k_end).all()
            u_start[t] = p0 + n_ext
        tile_tgt.append(row)
        for (_, ro, co) in steps:
            co = list(co) + [-1] * (TILE_COLS - len(co))
            step_src.append([int(plan.blk_off[x]) if x >= 0 else -1 for x in list(ro) + co])
        step_ptr.append(len(step_src))
        return True

    for lv in range(min(nlev, level_cut)):
        t0 = len(tile_tgt)
        for tile in ct["per_level"][lv]["tiles"]:
            assert tile["piece"][1] < cut
            emit(tile, tile["steps"], tile["piece"][0])
        if len(tile_tgt) > t0:
            pre[lv].append((LN_TU, TILE_DIM, TILE_DIM, t0, len(tile_tgt)))
    nlev_bottom = min(nlev, level_cut)
    cols_by_level = [[j for j in ct["per_level"][lv]["cols"]] for lv in range(nlev_bottom)]
    assert all(j < cut for L in cols_by_level for j in L)
    lane = _lane_lists(N, nlev_bottom, cols_by_level, plan.struct, dims, plan.blk_index, plan.blk_off, up_ptr, plan.winv_off, plan.pstart,
                       u_start=u_start, pre_launches=pre)
    if sp is not None:
        u_tgt, u_p0, u_p1 = list(lane["u_tgt"]), list(lane["u_p0"]), list(lane["u_p1"])
        launches = [tuple(int(x) for x in row) for row in lane["launches"]]
        t0 = len(tile_tgt)
        for lv in range(level_cut, nlev):
            for tile in ct["per_level"][lv]["tiles"]:
                assert tile["piece"][0] >= cut
                emit(tile, [st for st in tile["steps"] if st[0] < cut], cut)
        if len(tile_tgt) > t0:
            launches.append((LN_TU, TILE_DIM, TILE_DIM, t0, len(tile_tgt)))
        # root blocks no tile covers: their assembly pairs (k < cut) stay per block, grouped by shape like every U launch
        off_to_blk = {int(o): t for t, o in enumerate(plan.blk_off)}
        cls: Dict[Tuple[int, int, int], list] = {}
        for e in range(len(sp["ru_tgt"])):
            t = off_to_blk[int(sp["ru_tgt"][e])]
            assert int(sp["ru_p0"][e]) == int(up_ptr[t])
            first = int(u_start[t])
            if first < int(sp["ru_p1"][e]):
                assert first == int(sp["ru_p0"][e])   # a root block is covered by a tile entirely or not at all
                heavy = 1 if int(sp["ru_p1"][e]) - first >= LANE_HEAVY else 0
                cls.setdefault((heavy, int(blk_shape[t][0]), int(blk_shape[t][1])), []).append(e)
        for (heavy, di, dj) in sorted(cls):
            b0 = len(u_tgt)
            for e in cls[(heavy, di, dj)]:
                u_tgt.append(int(sp["ru_tgt"][e])); u_p0.append(int(sp["ru_p0"][e])); u_p1.append(int(sp["ru_p1"][e]))
            launches.append((LN_UH if heavy else LN_U, di, dj, b0, len(u_tgt)))
        i64 = np.int64
        lane.update(u_tgt=np.array(u_tgt, dtype=i64), u_p0=np.array(u_p0, dtype=i64), u_p1=np.array(u_p1, dtype=i64),
                    launches=np.array(launches, dtype=np.int32).reshape(-1, 5))
    lane.update(fr_p=plan.lane["fr_p"], fr_d=plan.lane["fr_d"], bc_p=plan.lane["bc_p"], bc_d=plan.lane["bc_d"])
    i64 = np.int64
    tiles = dict(tile_tgt=np.array(tile_tgt, dtype=i64).reshape(-1, TILE_ROWS * TILE_COLS), step_ptr=np.array(step_ptr, dtype=i64),
                 step_src=np.array(step_src, dtype=i64).reshape(-1, TILE_ROWS + TILE_COLS))
    return lane, tiles


def piece_solve_lists(plan: SparsePlan, max_width: int = 4, cut: Optional[int] = None):
    """Round-2 building block (host side, specification level; checked by a numpy interpreter in tests/test_sparse_symbolic.py; no kernel
    consumes it yet): the SUPERNODAL schedule of the substitutions.  Today every elimination-tree level is a launch and the top of the tree
    is one column per level (C5: 215 launches per pass, each a latency-bound list walk).  Consecutive columns of a chain (fundamental
    supernode) depend on each other only through a small dense triangle, so a PIECE of <= max_width chain columns (same pieces as
    chain_tiles; additionally cut where the block size changes) can be one work item:

      forward   per column j of the piece, in parallel: s_j = rhs_j - sum_{k < j0} L_jk y_k   (EXTERNAL part: a prefix of row j's list
                fr_*, because the list is sorted by k), then inside the work item, in order: s_j -= sum_{j0 <= k < j} L_jk y_k,
                y_j = L_jj^-1 s_j
      backward  the rows i > j1 below the piece are the SAME for all its columns (struct(j) = {j+1..j1} + struct(j1)): every x_i is
                loaded once and used by all columns: s_j = y_j - sum_{i > j1} L_ij^T x_i, then in reverse order
                s_j -= sum_{j < i <= j1} L_ij^T x_i, x_j = L_jj^-T s_j

    Pieces are levelled by their own dependency tree.  `cut`: only columns < cut (the bottom of a root split).
    Returns dict(first [P], width [P], dim [P], level [P], fr_ext_end [N] (index into fr_*: end of the external prefix of column j's row
    list), bc_int_end [N] (index into bc_*: end of the internal prefix of column j's column list), order [P] (pieces sorted by level,
    then block size), launches [(level, dim, begin, end)] into `order`)."""
    N, dims, A = plan.N, plan.dims, plan.arrays
    cut = N if cut is None else int(cut)
    first, width = [], []
    piece_of = np.full(N, -1, dtype=np.int64)
    j = 0
    while j < cut:
        e = j
        while (e + 1 < cut and plan.chain_of[e + 1] == plan.chain_of[j] and e + 1 - j < max_width and dims[e + 1] == dims[j]):
            e += 1
        piece_of[j:e + 1] = len(first)
        first.append(j); width.append(e + 1 - j)
        j = e + 1
    P = len(first)
    fr_ext_end = np.array(A["fr_ptr"][1:], dtype=np.int64).copy()
    bc_int_end = np.array(A["bc_ptr"][:-1], dtype=np.int64).copy()
    level = np.zeros(P, dtype=np.int64)
    for p in range(P):                      # pieces are numbered in elimination order: dependencies have smaller numbers
        j0, j1 = first[p], first[p] + width[p] - 1
        for jj in range(j0, j1 + 1):
            p0, p1 = int(A["fr_ptr"][jj]), int(A["fr_ptr"][jj + 1])
            ks = A["fr_k"][p0:p1]
            n_ext = int(np.searchsorted(ks, j0, side="left"))
            assert (ks[:n_ext] < j0).all() and (ks[n_ext:] >= j0).all() and n_ext + (jj - j0) == p1 - p0   # chain: all of j0..jj-1 are there
            fr_ext_end[jj] = p0 + n_ext
            if n_ext:
                level[p] = max(level[p], int(level[piece_of[ks[:n_ext]]].max()) + 1)
            q0, q1 = int(A["bc_ptr"][jj]), int(A["bc_ptr"][jj + 1])
            rows = A["bc_i"][q0:q1]
            assert np.array_equal(rows[:j1 - jj], np.arange(jj + 1, j1 + 1))
            bc_int_end[jj] = q0 + (j1 - jj)
        ext_rows = [A["bc_i"][bc_int_end[jj]:A["bc_ptr"][jj + 1]] for jj in range(j0, j1 + 1)]
        assert all(np.array_equal(r, ext_rows[0]) for r in ext_rows)    # shared external rows
    order = sorted(range(P), key=lambda p: (int(level[p]), int(dims[first[p]]), p))
    launches, b0 = [], 0
    for q in range(1, P + 1):
        if q == P or (level[order[q]], dims[first[order[q]]]) != (level[order[b0]], dims[first[order[b0]]]):
            launches.append((int(level[order[b0]]), int(dims[first[order[b0]]]), b0, q)); b0 = q
    return dict(first=np.array(first, dtype=np.int64), width=np.array(width, dtype=np.int64),
                dim=np.array([dims[f] for f in first], dtype=np.int64), level=level, fr_ext_end=fr_ext_end, bc_int_end=bc_int_end,
                order=np.array(order, dtype=np.int64), launches=np.array(launches, dtype=np.int64).reshape(-1, 4), cut=cut)
