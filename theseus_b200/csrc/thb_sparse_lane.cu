// Batched block-sparse Cholesky, "batch-lane" execution model, fp64.
//
// Same job and same symbolic plan as thb_sparse.cu (BaSpaCho NumericDecomposition::{add_MtM,damp,factor,solve},
// theseus/extlib/baspacho_solver.cpp:93-257, baspacho_solver_cuda.cu:96-293), different mapping onto the machine:
//
//   * every batch item has the SAME sparsity structure (one symbolic decomposition per objective, baspacho_sparse_solver.py:58-113),
//     so the factorisation is one fixed sequence of small block operations executed for B different sets of numbers.
//     Here a batch item is a LANE: the factor storage is interleaved, element e of item b at factor[e * Bp + b]
//     (Bp = B rounded up to 32), so a warp that executes one block operation for 32 batch items issues perfectly
//     coalesced 256-byte loads and stores and has no divergence; block indices are warp-uniform (broadcast loads);
//   * a thread keeps a whole di x dj block in registers (kernels are compiled per block shape, dims in {1,2,3,6}:
//     Vector/Point2/Point3/SO3/SE2/SE3), so the left-looking update of a block is a register-tiled rank-dk update chain:
//     (di+dj) loads per di*dj FMAs, the target is read and written once;
//   * elimination-tree levels are separate launches (the work lists are per level and per block shape, sparse.py:_lane_lists);
//     inside a launch all work items are independent, there are no atomics and the result is deterministic.
//
// Stages per level:  U  target(i,j) <- M_ij - sum_k L_ik L_jk^T            (one thread per (batch item, block))
//                    T  L_jj = chol(target(j,j)) in registers (recomputed by every block of the column: 56 FMAs, cheaper
//                       than a launch), L_ij = target(i,j) L_jj^-T; the diagonal factor goes to a separate store `diagl`
//                       with RECIPROCAL diagonal entries (the substitutions multiply instead of divide)
// Solve: per level forward (y_j = L_jj^-1 (rhs_j - sum_k L_jk y_k)), then per level backward, permutation folded into the
// first load / last store (K8 scramble/unscramble, baspacho_solver_cuda.cu:216-250).
#include "thb_common.cuh"

namespace thb {

constexpr int LN_WARPS = 4;  // warps per CTA; one warp = 32 batch lanes of one work item

// Compile-time fence: every element of x must be in a register here, i.e. all the loads that produce x are issued before any
// instruction that consumes the fenced values.  Without it the compiler sinks each load next to its FMA and recycles one
// register, which turns 36-72 independent loads into a chain of dependent memory latencies.
template <int N>
__device__ __forceinline__ void loads_issued(double (&x)[N]) {
#ifndef THB_SIMT_EMU  // (tests/simt: the same source compiled for the host, one OS thread per CUDA thread)
  constexpr int G = 12;
#pragma unroll
  for (int i = 0; i + G <= N; i += G)
    asm volatile("" : "+d"(x[i]), "+d"(x[i + 1]), "+d"(x[i + 2]), "+d"(x[i + 3]), "+d"(x[i + 4]), "+d"(x[i + 5]), "+d"(x[i + 6]),
                 "+d"(x[i + 7]), "+d"(x[i + 8]), "+d"(x[i + 9]), "+d"(x[i + 10]), "+d"(x[i + 11]));
#pragma unroll
  for (int i = N / G * G; i < N; i++) asm volatile("" : "+d"(x[i]));
#endif
}

// acc[r][c] -= sum_k A[r][k] B[c][k]   (A: di x DK at a_off, B: dj x DK at b_off, both row-major, lane-interleaved)
template <int DI, int DJ, int DK>
__device__ __forceinline__ void pair_update(double (&acc)[DI * DJ], const double* Fb, int64_t a_off, int64_t b_off, int64_t Bp) {
  constexpr int KS = (DK >= 3) ? 3 : DK;  // columns of the pair staged at once: KS*(DI+DJ) loads in flight
#pragma unroll
  for (int k0 = 0; k0 < DK; k0 += KS) {
    double v[KS * (DI + DJ)];
#pragma unroll
    for (int k = 0; k < KS; k++) {
#pragma unroll
      for (int r = 0; r < DI; r++) v[k * (DI + DJ) + r] = Fb[(a_off + r * DK + k0 + k) * Bp];
#pragma unroll
      for (int c = 0; c < DJ; c++) v[k * (DI + DJ) + DI + c] = Fb[(b_off + c * DK + k0 + k) * Bp];
    }
    loads_issued(v);
#pragma unroll
    for (int k = 0; k < KS; k++)
#pragma unroll
      for (int r = 0; r < DI; r++)
#pragma unroll
        for (int c = 0; c < DJ; c++) acc[r * DJ + c] -= v[k * (DI + DJ) + r] * v[k * (DI + DJ) + DI + c];
  }
}

template <int DI, int DJ>
__device__ __forceinline__ void pair_update_any(double (&acc)[DI * DJ], const double* Fb, int64_t a_off, int64_t b_off, int dk,
                                                int64_t Bp) {
  if (dk == 6) pair_update<DI, DJ, 6>(acc, Fb, a_off, b_off, Bp);
  else if (dk == 3) pair_update<DI, DJ, 3>(acc, Fb, a_off, b_off, Bp);
  else if (dk == 2) pair_update<DI, DJ, 2>(acc, Fb, a_off, b_off, Bp);
  else pair_update<DI, DJ, 1>(acc, Fb, a_off, b_off, Bp);
}

struct LaneArgs {
  const int64_t* up_a; const int64_t* up_b; const int32_t* up_k;
  const int64_t* u_tgt; const int64_t* u_p0; const int64_t* u_p1;
  const int64_t* t_off; const int64_t* t_diag; const int64_t* t_dl; const int32_t* t_pstart;
  int begin, end, nbx;
  int64_t B, Bp;
};

// ---- U: one warp = one target block x 32 batch items ----
template <int DI, int DJ>
__global__ void __launch_bounds__(32 * LN_WARPS) lane_update_kernel(LaneArgs p, double* __restrict__ F) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t b = (int64_t)(blockIdx.x % p.nbx) * 32 + lane;
  const int item = p.begin + (blockIdx.x / p.nbx) * LN_WARPS + warp;
  if (item >= p.end || b >= p.B) return;
  double* Fb = F + b;
  const int64_t tgt = p.u_tgt[item];
  double acc[DI * DJ];
#pragma unroll
  for (int e = 0; e < DI * DJ; e++) acc[e] = Fb[(tgt + e) * p.Bp];
  const int64_t q1 = p.u_p1[item];
  for (int64_t q = p.u_p0[item]; q < q1; q++) pair_update_any<DI, DJ>(acc, Fb, p.up_a[q], p.up_b[q], p.up_k[q], p.Bp);
#pragma unroll
  for (int e = 0; e < DI * DJ; e++) Fb[(tgt + e) * p.Bp] = acc[e];
}

// ---- U, heavy targets: the CTA's 8 warps split the update pairs of ONE target block; partial sums are combined through shared
// memory in a fixed order (deterministic).  Used for blocks with >= LANE_HEAVY pairs (sparse.py): a single thread walking a list
// of pairs is a chain of dependent memory latencies, and at the top of the elimination tree that chain is the critical path.
constexpr int LH_WARPS = 8;
template <int DI, int DJ>
__global__ void __launch_bounds__(32 * LH_WARPS, 1) lane_update_heavy_kernel(LaneArgs p, double* __restrict__ F) {
  __shared__ double red[(LH_WARPS / 2) * DI * DJ * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t b = (int64_t)(blockIdx.x % p.nbx) * 32 + lane;
  const int item = p.begin + (blockIdx.x / p.nbx);
  const bool live = b < p.B;
  const double* Fb = F + (live ? b : 0);
  double acc[DI * DJ];
#pragma unroll
  for (int e = 0; e < DI * DJ; e++) acc[e] = 0.0;
  const int64_t q1 = p.u_p1[item];
  if (live)
    for (int64_t q = p.u_p0[item] + warp; q < q1; q += LH_WARPS) pair_update_any<DI, DJ>(acc, Fb, p.up_a[q], p.up_b[q], p.up_k[q], p.Bp);
  // phase 1: warps 4..7 -> warps 0..3 ; phase 2: warps 1..3 -> warp 0
  if (warp >= LH_WARPS / 2) {
#pragma unroll
    for (int e = 0; e < DI * DJ; e++) red[((warp - LH_WARPS / 2) * DI * DJ + e) * 32 + lane] = acc[e];
  }
  __syncthreads();
  if (warp < LH_WARPS / 2) {
#pragma unroll
    for (int e = 0; e < DI * DJ; e++) acc[e] += red[(warp * DI * DJ + e) * 32 + lane];
  }
  __syncthreads();
  if (warp > 0 && warp < LH_WARPS / 2) {
#pragma unroll
    for (int e = 0; e < DI * DJ; e++) red[((warp - 1) * DI * DJ + e) * 32 + lane] = acc[e];
  }
  __syncthreads();
  if (warp == 0 && live) {
    const int64_t tgt = p.u_tgt[item];
    double* Fw = F + b;
#pragma unroll
    for (int e = 0; e < DI * DJ; e++) {
      double s = acc[e];
#pragma unroll
      for (int w = 0; w < LH_WARPS / 2 - 1; w++) s += red[(w * DI * DJ + e) * 32 + lane];
      Fw[(tgt + e) * p.Bp] += s;  // acc holds -(sum of products)
    }
  }
}

// ---- TU: tiled external updates of a chain piece (sparse.py:tile_lane_lists) ----
// One CTA = one tile (TR rows x TC columns of D x D target blocks) x 32 batch lanes; warp w owns target (w / TC, w % TC) in registers.
// Per k step the NS = TR + TC source blocks are copied ONCE into shared memory ([slot][element][lane]: every row is a coalesced
// 256-byte segment in global memory and conflict-free in shared memory), double buffered with cp.async so the copy of step s+1
// runs under the FP64 work of step s; a target takes part in a step iff both its row and its column source exist.
struct LaneTileArgs {
  const int64_t* tile_tgt; const int64_t* step_ptr; const int64_t* step_src;
  int begin; int64_t Bp;
};

#ifndef THB_SIMT_EMU
__device__ __forceinline__ void cp_async_8(double* smem_dst, const double* gmem_src) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
#else  // host emulation: the copy is synchronous, groups are no-ops (the barriers of the kernel still order buffer reuse)
inline void cp_async_8(double* smem_dst, const double* gmem_src) { *smem_dst = *gmem_src; }
inline void cp_async_commit() {}
template <int N> inline void cp_async_wait() {}
#endif

template <int D, int TR, int TC>
__global__ void __launch_bounds__(32 * TR * TC, 1) lane_tile_update_kernel(LaneTileArgs p, double* F) {
  constexpr int NS = TR + TC, E = D * D, NW = TR * TC, ROWS = NS * E;
  extern __shared__ double tile_sm[];  // [2][NS][E][32]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int tile = p.begin + (int)blockIdx.x;
  double* Fb = F + (int64_t)blockIdx.y * 32 + lane;   // padded lanes (b >= B) hold zeros / unused storage inside [*, Bp]: computed, harmless
  const int64_t tgt = p.tile_tgt[(int64_t)tile * NW + w];
  const int a = w / TC, b = w % TC;
  double acc[E];
  if (tgt >= 0) {
#pragma unroll
    for (int e = 0; e < E; e++) acc[e] = Fb[(tgt + e) * p.Bp];
  } else {
#pragma unroll
    for (int e = 0; e < E; e++) acc[e] = 0.0;
  }
  const int64_t s0 = p.step_ptr[tile], s1 = p.step_ptr[tile + 1];
  auto stage = [&](int64_t s, int buf) {
    const int64_t* src = p.step_src + s * NS;
    double* dst = tile_sm + (size_t)buf * ROWS * 32 + lane;
#pragma unroll 6
    for (int r = w; r < ROWS; r += NW) {
      const int slot = r / E, e = r - slot * E;
      const int64_t off = src[slot];
      if (off >= 0) cp_async_8(dst + r * 32, Fb + (off + e) * p.Bp);
    }
    cp_async_commit();
  };
  if (s0 < s1) stage(s0, 0);
  for (int64_t s = s0; s < s1; s++) {
    const int buf = (int)(s - s0) & 1;
    if (s + 1 < s1) { stage(s + 1, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();
    const int64_t ro = p.step_src[s * NS + a], co = p.step_src[s * NS + TR + b];
    if (tgt >= 0 && ro >= 0 && co >= 0) {
      const double* R = tile_sm + ((size_t)buf * ROWS + a * E) * 32 + lane;
      const double* Cc = tile_sm + ((size_t)buf * ROWS + (TR + b) * E) * 32 + lane;
#pragma unroll
      for (int q = 0; q < D; q++) {
        double rv[D], cv[D];
#pragma unroll
        for (int r = 0; r < D; r++) rv[r] = R[(r * D + q) * 32];
#pragma unroll
        for (int c = 0; c < D; c++) cv[c] = Cc[(c * D + q) * 32];
#pragma unroll
        for (int r = 0; r < D; r++)
#pragma unroll
          for (int c = 0; c < D; c++) acc[r * D + c] -= rv[r] * cv[c];
      }
    }
    __syncthreads();  // buffer `buf` is refilled by the stage() of the next iteration
  }
  if (tgt >= 0) {
#pragma unroll
    for (int e = 0; e < E; e++) Fb[(tgt + e) * p.Bp] = acc[e];
  }
}

// ---- T: Cholesky of the column's diagonal block (registers) + triangular solve of this block ----
template <int DI, int DJ>
__global__ void __launch_bounds__(32 * LN_WARPS) lane_trsm_kernel(LaneArgs p, double* __restrict__ F, double* __restrict__ DL,
                                                                  int32_t* __restrict__ info) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t b = (int64_t)(blockIdx.x % p.nbx) * 32 + lane;
  const int item = p.begin + (blockIdx.x / p.nbx) * LN_WARPS + warp;
  if (item >= p.end || b >= p.B) return;
  double* Fb = F + b;
  const int64_t off = p.t_off[item], dg = p.t_diag[item];
  double d[DJ * DJ], inv[DJ];
#pragma unroll
  for (int r = 0; r < DJ; r++)
#pragma unroll
    for (int c = 0; c <= r; c++) d[r * DJ + c] = Fb[(dg + r * DJ + c) * p.Bp];
  int fail = 0;
#pragma unroll
  for (int c = 0; c < DJ; c++) {
    double dd = d[c * DJ + c];
#pragma unroll
    for (int k = 0; k < c; k++) dd -= d[c * DJ + k] * d[c * DJ + k];
    if (!(dd > 0.0) && fail == 0) fail = c + 1;
    inv[c] = rsqrt(dd);
    d[c * DJ + c] = dd * inv[c];
#pragma unroll
    for (int r = c + 1; r < DJ; r++) {
      double s = d[r * DJ + c];
#pragma unroll
      for (int k = 0; k < c; k++) s -= d[r * DJ + k] * d[c * DJ + k];
      d[r * DJ + c] = s * inv[c];
    }
  }
  if (off == dg) {
    if constexpr (DI == DJ) {
      double* Dl = DL + p.t_dl[item] * p.Bp + b;
#pragma unroll
      for (int r = 0; r < DJ; r++)
#pragma unroll
        for (int c = 0; c < DJ; c++) Dl[(r * DJ + c) * p.Bp] = (c < r) ? d[r * DJ + c] : (c == r ? inv[c] : 0.0);
      if (fail != 0) atomicCAS(info + b, 0, p.t_pstart[item] + fail);
    }
    return;
  }
  double x[DI * DJ];
#pragma unroll
  for (int e = 0; e < DI * DJ; e++) x[e] = Fb[(off + e) * p.Bp];
#pragma unroll
  for (int c = 0; c < DJ; c++) {
#pragma unroll
    for (int r = 0; r < DI; r++) {
      double s = x[r * DJ + c];
#pragma unroll
      for (int k = 0; k < c; k++) s -= x[r * DJ + k] * d[c * DJ + k];
      x[r * DJ + c] = s * inv[c];
    }
  }
#pragma unroll
  for (int e = 0; e < DI * DJ; e++) Fb[(off + e) * p.Bp] = x[e];
}

struct LaneSolveArgs {
  const int32_t* s_col; const int32_t* pstart; const int32_t* col_start; const int64_t* dl_off;
  const int64_t* fr_ptr; const int64_t* fr_off; const int32_t* fr_p; const int32_t* fr_d;
  const int64_t* bc_ptr; const int64_t* bc_off; const int32_t* bc_p; const int32_t* bc_d;
  int begin, end, nbx;
  int64_t B, Bp, n;
};

constexpr int LS_WARPS = 16;  // substitution kernels: the CTA's warps split the block list of ONE column (x 32 batch items)

// s[r] -= sum_c L[r][c] v[c]  (L: DJ x DK row-major at off, v at Y[(pv + c)]).  All loads are issued before the first FMA:
// written as load-FMA pairs ptxas recycles one register and serialises the 42 loads.
template <int DJ, int DK>
__device__ __forceinline__ void blk_mv(double (&s)[DJ], const double* Fb, int64_t off, const double* Yb, int pv, int64_t Bp) {
  double v[DK], l[DJ * DK];
#pragma unroll
  for (int c = 0; c < DK; c++) v[c] = Yb[(int64_t)(pv + c) * Bp];
#pragma unroll
  for (int e = 0; e < DJ * DK; e++) l[e] = Fb[(off + e) * Bp];
  loads_issued(l);
#pragma unroll
  for (int r = 0; r < DJ; r++)
#pragma unroll
    for (int c = 0; c < DK; c++) s[r] -= l[r * DK + c] * v[c];
}
// s[c] -= sum_r L[r][c] v[r]  (L: DI x DJ row-major at off)
template <int DJ, int DI>
__device__ __forceinline__ void blk_tmv(double (&s)[DJ], const double* Fb, int64_t off, const double* Yb, int pv, int64_t Bp) {
  double v[DI], l[DI * DJ];
#pragma unroll
  for (int r = 0; r < DI; r++) v[r] = Yb[(int64_t)(pv + r) * Bp];
#pragma unroll
  for (int e = 0; e < DI * DJ; e++) l[e] = Fb[(off + e) * Bp];
  loads_issued(l);
#pragma unroll
  for (int r = 0; r < DI; r++)
#pragma unroll
    for (int c = 0; c < DJ; c++) s[c] -= l[r * DJ + c] * v[r];
}

// partial sums of warps 1.. -> shared memory -> warp 0 (fixed order: deterministic)
template <int DJ>
__device__ __forceinline__ void reduce_to_warp0(double (&s)[DJ], double* red, int warp, int lane) {
  if (warp > 0) {
#pragma unroll
    for (int r = 0; r < DJ; r++) red[((warp - 1) * DJ + r) * 32 + lane] = s[r];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int r = 0; r < DJ; r++)
      for (int w = 0; w < LS_WARPS - 1; w++) s[r] += red[(w * DJ + r) * 32 + lane];
  }
}

template <int DJ>
__global__ void __launch_bounds__(32 * LS_WARPS, 1) lane_forward_kernel(LaneSolveArgs p, const double* F, const double* __restrict__ DL,
                                                                     const double* __restrict__ rhs, double* Y) {
  __shared__ double red[(LS_WARPS - 1) * DJ * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t b = (int64_t)(blockIdx.x % p.nbx) * 32 + lane;
  const int item = p.begin + (blockIdx.x / p.nbx);
  const bool live = b < p.B;
  const int j = p.s_col[item];
  const double* Fb = F + (live ? b : 0);
  double* Yb = Y + (live ? b : 0);
  double s[DJ];
#pragma unroll
  for (int r = 0; r < DJ; r++) s[r] = 0.0;
  if (live) {
    const int64_t q1 = p.fr_ptr[j + 1];
    for (int64_t q = p.fr_ptr[j] + warp; q < q1; q += LS_WARPS) {
      const int dk = p.fr_d[q], pk = p.fr_p[q];
      const int64_t off = p.fr_off[q];
      if (dk == 6) blk_mv<DJ, 6>(s, Fb, off, Yb, pk, p.Bp);
      else if (dk == 3) blk_mv<DJ, 3>(s, Fb, off, Yb, pk, p.Bp);
      else if (dk == 2) blk_mv<DJ, 2>(s, Fb, off, Yb, pk, p.Bp);
      else blk_mv<DJ, 1>(s, Fb, off, Yb, pk, p.Bp);
    }
  }
  reduce_to_warp0<DJ>(s, red, warp, lane);
  if (warp != 0 || !live) return;
  double dl[DJ * DJ];
  const double* Dl = DL + p.dl_off[j] * p.Bp + b;
#pragma unroll
  for (int r = 0; r < DJ; r++)
#pragma unroll
    for (int c = 0; c <= r; c++) dl[r * DJ + c] = Dl[(r * DJ + c) * p.Bp];
  const int pj = p.pstart[j];
#pragma unroll
  for (int r = 0; r < DJ; r++) {
    double v = s[r] + rhs[b * p.n + p.col_start[j] + r];  // scramble on load
#pragma unroll
    for (int c = 0; c < r; c++) v -= dl[r * DJ + c] * s[c];
    s[r] = v * dl[r * DJ + r];
    Yb[(int64_t)(pj + r) * p.Bp] = s[r];
  }
}

template <int DJ>
__global__ void __launch_bounds__(32 * LS_WARPS, 1) lane_backward_kernel(LaneSolveArgs p, const double* F, const double* __restrict__ DL,
                                                                      double* Y, double* __restrict__ x) {
  __shared__ double red[(LS_WARPS - 1) * DJ * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t b = (int64_t)(blockIdx.x % p.nbx) * 32 + lane;
  const int item = p.begin + (blockIdx.x / p.nbx);
  const bool live = b < p.B;
  const int j = p.s_col[item];
  const double* Fb = F + (live ? b : 0);
  double* Yb = Y + (live ? b : 0);
  double s[DJ];
#pragma unroll
  for (int c = 0; c < DJ; c++) s[c] = 0.0;
  if (live) {
    const int64_t q1 = p.bc_ptr[j + 1];
    for (int64_t q = p.bc_ptr[j] + warp; q < q1; q += LS_WARPS) {
      const int di = p.bc_d[q], pi = p.bc_p[q];
      const int64_t off = p.bc_off[q];
      if (di == 6) blk_tmv<DJ, 6>(s, Fb, off, Yb, pi, p.Bp);
      else if (di == 3) blk_tmv<DJ, 3>(s, Fb, off, Yb, pi, p.Bp);
      else if (di == 2) blk_tmv<DJ, 2>(s, Fb, off, Yb, pi, p.Bp);
      else blk_tmv<DJ, 1>(s, Fb, off, Yb, pi, p.Bp);
    }
  }
  reduce_to_warp0<DJ>(s, red, warp, lane);
  if (warp != 0 || !live) return;
  const int pj = p.pstart[j];
  double dl[DJ * DJ];
  const double* Dl = DL + p.dl_off[j] * p.Bp + b;
#pragma unroll
  for (int r = 0; r < DJ; r++)
#pragma unroll
    for (int c = 0; c <= r; c++) dl[r * DJ + c] = Dl[(r * DJ + c) * p.Bp];
#pragma unroll
  for (int c = 0; c < DJ; c++) s[c] += Yb[(int64_t)(pj + c) * p.Bp];
#pragma unroll
  for (int c = DJ - 1; c >= 0; c--) {
    double v = s[c];
#pragma unroll
    for (int r = c + 1; r < DJ; r++) v -= dl[r * DJ + c] * s[r];
    s[c] = v * dl[c * DJ + c];
    Yb[(int64_t)(pj + c) * p.Bp] = s[c];
    x[b * p.n + p.col_start[j] + c] = s[c];  // unscramble on store
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Supernodal substitutions (sparse.py:piece_solve_lists): one work item = a PIECE of <= LP_MAXW consecutive chain columns of equal block
// size x 32 batch lanes.  Forward: the CTA's 16 warps split the EXTERNAL parts of the row lists of all columns of the piece (column
// c = warp % w), warp 0 then walks the piece's dense triangle in order.  Backward: the rows below the piece are the same for all its
// columns, so a warp loads x_i once and applies it to every column; warp 0 finishes the triangle in reverse order.  Launches: one per
// piece level and block size instead of one per elimination-tree level (C5 below the dense root: 39 instead of 119 per pass).
constexpr int LP_MAXW = 4;
struct LanePieceArgs {
  const int64_t* first; const int32_t* width; const int64_t* fr_ext_end; const int64_t* bc_int_end; const int64_t* order;
};

// s[r] -= sum_c l[r][c] v[c] with v in registers (L: DJ x DK row-major at off)
template <int DJ, int DK>
__device__ __forceinline__ void blk_mv_reg(double (&s)[DJ], const double* Fb, int64_t off, const double (&v)[DK], int64_t Bp) {
  double l[DJ * DK];
#pragma unroll
  for (int e = 0; e < DJ * DK; e++) l[e] = Fb[(off + e) * Bp];
  loads_issued(l);
#pragma unroll
  for (int r = 0; r < DJ; r++)
#pragma unroll
    for (int c = 0; c < DK; c++) s[r] -= l[r * DK + c] * v[c];
}
// s[c] -= sum_r l[r][c] v[r] with v in registers (L: DI x DJ row-major at off)
template <int DJ, int DI>
__device__ __forceinline__ void blk_tmv_reg(double (&s)[DJ], const double* Fb, int64_t off, const double (&v)[DI], int64_t Bp) {
  double l[DI * DJ];
#pragma unroll
  for (int e = 0; e < DI * DJ; e++) l[e] = Fb[(off + e) * Bp];
  loads_issued(l);
#pragma unroll
  for (int r = 0; r < DI; r++)
#pragma unroll
    for (int c = 0; c < DJ; c++) s[c] -= l[r * DJ + c] * v[r];
}

template <int DJ>
__global__ void __launch_bounds__(32 * LS_WARPS, 1) lane_piece_forward_kernel(LaneSolveArgs p, LanePieceArgs pc, const double* F,
                                                                           const double* __restrict__ DL, const double* __restrict__ rhs,
                                                                           double* Y) {
  __shared__ double red[LS_WARPS * DJ * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t b = (int64_t)(blockIdx.x % p.nbx) * 32 + lane;
  const int64_t piece = pc.order[p.begin + (blockIdx.x / p.nbx)];
  const bool live = b < p.B;
  const int64_t j0 = pc.first[piece];
  const int w = pc.width[piece];
  const double* Fb = F + (live ? b : 0);
  double* Yb = Y + (live ? b : 0);
  {  // external parts: warp -> column c = warp % w, every (LS_WARPS / w)-th entry of its list
    const int c = warp % w, sub = warp / w, nsub = (LS_WARPS - 1 - c) / w + 1;
    const int64_t j = j0 + c;
    double s[DJ];
#pragma unroll
    for (int r = 0; r < DJ; r++) s[r] = 0.0;
    if (live) {
      const int64_t q1 = pc.fr_ext_end[j];
      for (int64_t q = p.fr_ptr[j] + sub; q < q1; q += nsub) {
        const int dk = p.fr_d[q], pk = p.fr_p[q];
        const int64_t off = p.fr_off[q];
        if (dk == 6) blk_mv<DJ, 6>(s, Fb, off, Yb, pk, p.Bp);
        else if (dk == 3) blk_mv<DJ, 3>(s, Fb, off, Yb, pk, p.Bp);
        else if (dk == 2) blk_mv<DJ, 2>(s, Fb, off, Yb, pk, p.Bp);
        else blk_mv<DJ, 1>(s, Fb, off, Yb, pk, p.Bp);
      }
    }
#pragma unroll
    for (int r = 0; r < DJ; r++) red[(warp * DJ + r) * 32 + lane] = s[r];
  }
  __syncthreads();
  if (warp != 0 || !live) return;
  double y[LP_MAXW][DJ];
#pragma unroll
  for (int cc = 0; cc < LP_MAXW; cc++) {
    if (cc < w) {
      const int64_t jj = j0 + cc;
      double t[DJ];
#pragma unroll
      for (int r = 0; r < DJ; r++) {
        double v = rhs[b * p.n + p.col_start[jj] + r];  // scramble on load
        for (int ww = cc; ww < LS_WARPS; ww += w) v += red[(ww * DJ + r) * 32 + lane];  // fixed order: deterministic
        t[r] = v;
      }
      const int64_t qi = pc.fr_ext_end[jj];  // internal entries: k = j0 .. jj-1 in this order (the row list is sorted by k)
#pragma unroll
      for (int ci = 0; ci < LP_MAXW; ci++)
        if (ci < cc) blk_mv_reg<DJ, DJ>(t, Fb, p.fr_off[qi + ci], y[ci], p.Bp);
      double dl[DJ * DJ];
      const double* Dl = DL + p.dl_off[jj] * p.Bp + b;
#pragma unroll
      for (int r = 0; r < DJ; r++)
#pragma unroll
        for (int c = 0; c <= r; c++) dl[r * DJ + c] = Dl[(r * DJ + c) * p.Bp];
      const int pj = p.pstart[jj];
#pragma unroll
      for (int r = 0; r < DJ; r++) {
        double v = t[r];
#pragma unroll
        for (int c = 0; c < r; c++) v -= dl[r * DJ + c] * y[cc][c];
        y[cc][r] = v * dl[r * DJ + r];
        Yb[(int64_t)(pj + r) * p.Bp] = y[cc][r];
      }
    }
  }
}

template <int DJ, int DI>
__device__ __forceinline__ void piece_ext_row(double (&s)[LP_MAXW][DJ], int w, const double* Fb, const double* Yb, const LaneSolveArgs& p,
                                              const LanePieceArgs& pc, int64_t j0, int64_t e, int pi) {
  double v[DI];
#pragma unroll
  for (int r = 0; r < DI; r++) v[r] = Yb[(int64_t)(pi + r) * p.Bp];
#pragma unroll
  for (int cc = 0; cc < LP_MAXW; cc++)
    if (cc < w) blk_tmv_reg<DJ, DI>(s[cc], Fb, p.bc_off[pc.bc_int_end[j0 + cc] + e], v, p.Bp);
}

template <int DJ>
__global__ void __launch_bounds__(32 * LS_WARPS, 1) lane_piece_backward_kernel(LaneSolveArgs p, LanePieceArgs pc, const double* F,
                                                                            const double* __restrict__ DL, double* Y, double* __restrict__ x) {
  __shared__ double red[(LS_WARPS - 1) * DJ * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t b = (int64_t)(blockIdx.x % p.nbx) * 32 + lane;
  const int64_t piece = pc.order[p.begin + (blockIdx.x / p.nbx)];
  const bool live = b < p.B;
  const int64_t j0 = pc.first[piece];
  const int w = pc.width[piece];
  const int64_t j1 = j0 + w - 1;
  const double* Fb = F + (live ? b : 0);
  double* Yb = Y + (live ? b : 0);
  double s[LP_MAXW][DJ];
#pragma unroll
  for (int cc = 0; cc < LP_MAXW; cc++)
#pragma unroll
    for (int c = 0; c < DJ; c++) s[cc][c] = 0.0;
  if (live) {  // external rows i > j1: the same rows for every column of the piece; x_i is loaded once per row
    const int64_t qe = pc.bc_int_end[j1], n_ext = p.bc_ptr[j1 + 1] - qe;
    for (int64_t e = warp; e < n_ext; e += LS_WARPS) {
      const int di = p.bc_d[qe + e], pi = p.bc_p[qe + e];
      if (di == 6) piece_ext_row<DJ, 6>(s, w, Fb, Yb, p, pc, j0, e, pi);
      else if (di == 3) piece_ext_row<DJ, 3>(s, w, Fb, Yb, p, pc, j0, e, pi);
      else if (di == 2) piece_ext_row<DJ, 2>(s, w, Fb, Yb, p, pc, j0, e, pi);
      else piece_ext_row<DJ, 1>(s, w, Fb, Yb, p, pc, j0, e, pi);
    }
  }
#pragma unroll
  for (int cc = 0; cc < LP_MAXW; cc++) {  // one reduction round per column (the buffer is reused; w is uniform across the CTA)
    if (cc < w) {
      reduce_to_warp0<DJ>(s[cc], red, warp, lane);
      __syncthreads();
    }
  }
  if (warp != 0 || !live) return;
#pragma unroll
  for (int cc = LP_MAXW - 1; cc >= 0; cc--) {
    if (cc < w) {
      const int64_t jj = j0 + cc;
      const int pj = p.pstart[jj];
#pragma unroll
      for (int c = 0; c < DJ; c++) s[cc][c] += Yb[(int64_t)(pj + c) * p.Bp];
      const int64_t qi = p.bc_ptr[jj];  // internal entries: i = jj+1 .. j1 in this order
#pragma unroll
      for (int ci = 0; ci < LP_MAXW; ci++)
        if (ci > cc && ci < w) blk_tmv_reg<DJ, DJ>(s[cc], Fb, p.bc_off[qi + (ci - cc - 1)], s[ci], p.Bp);
      double dl[DJ * DJ];
      const double* Dl = DL + p.dl_off[jj] * p.Bp + b;
#pragma unroll
      for (int r = 0; r < DJ; r++)
#pragma unroll
        for (int c = 0; c <= r; c++) dl[r * DJ + c] = Dl[(r * DJ + c) * p.Bp];
#pragma unroll
      for (int c = DJ - 1; c >= 0; c--) {
        double v = s[cc][c];
#pragma unroll
        for (int r = c + 1; r < DJ; r++) v -= dl[r * DJ + c] * s[cc][r];
        s[cc][c] = v * dl[c * DJ + c];
        Yb[(int64_t)(pj + c) * p.Bp] = s[cc][c];
        x[b * p.n + p.col_start[jj] + c] = s[cc][c];  // unscramble on store
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Dense root (sparse.py:root_split): the top chain of the elimination tree is a dense trailing block; it is copied out of the
// lane-interleaved storage into a batch-major dense matrix, factored / solved by the dense DMMA kernels (thb_potrf_f64 /
// thb_potrs_f64), and its part of the solution copied back.
struct LaneRootArgs {
  const int64_t* rb_off; const int32_t* rb_row; const int32_t* rb_col; const int32_t* rb_di; const int32_t* rb_dj;  // root blocks
  int64_t num_blocks;
  const int64_t* rf_p0; const int64_t* rf_p1;       // per root column: range of its row-list entries that lie in bottom columns
  const int32_t* root_cols;                         // [num_cols] elimination positions of the root columns (grouped by block size)
  const int32_t* root_dims;                         // [num_cols] their block sizes
  int64_t num_cols, nt, root_start;
};

// S[b, r0+r, c0+c] = factor[(off + r*dj + c)*Bp + b]; one thread per (batch item, block element), lanes over b (coalesced reads)
__global__ void __launch_bounds__(256) lane_root_gather_kernel(LaneRootArgs r, const double* __restrict__ F, double* __restrict__ S, int64_t B,
                                                               int64_t Bp) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t q = t / Bp, b = t - q * Bp;  // q = blk * 36 + e  (blocks are at most 6x6)
  const int64_t blk = q / 36;
  const int e = (int)(q - blk * 36);
  if (blk >= r.num_blocks || b >= B) return;
  const int di = r.rb_di[blk], dj = r.rb_dj[blk];
  if (e >= di * dj) return;
  const int rr = e / dj, cc = e - rr * dj;
  S[b * r.nt * r.nt + (int64_t)(r.rb_row[blk] + rr) * r.nt + r.rb_col[blk] + cc] = F[(r.rb_off[blk] + e) * Bp + b];
}

// rhs_dense[b, pstart_j - root_start + r] = rhs[b, col_start_j + r] - sum over the bottom part of row j's list of L_jk y_k
template <int DJ>
__global__ void __launch_bounds__(32 * LS_WARPS, 1) lane_root_rhs_kernel(LaneSolveArgs p, LaneRootArgs r, const double* F, const double* __restrict__ rhs,
                                                                         const double* Y, double* __restrict__ rhs_dense) {
  __shared__ double red[(LS_WARPS - 1) * DJ * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t b = (int64_t)(blockIdx.x % p.nbx) * 32 + lane;
  const int item = p.begin + (blockIdx.x / p.nbx);
  const bool live = b < p.B;
  const int j = r.root_cols[item];
  const double* Fb = F + (live ? b : 0);
  const double* Yb = Y + (live ? b : 0);
  double s[DJ];
#pragma unroll
  for (int q = 0; q < DJ; q++) s[q] = 0.0;
  if (live) {
    const int64_t q1 = r.rf_p1[item];
    for (int64_t q = r.rf_p0[item] + warp; q < q1; q += LS_WARPS) {
      const int dk = p.fr_d[q], pk = p.fr_p[q];
      const int64_t off = p.fr_off[q];
      if (dk == 6) blk_mv<DJ, 6>(s, Fb, off, Yb, pk, p.Bp);
      else if (dk == 3) blk_mv<DJ, 3>(s, Fb, off, Yb, pk, p.Bp);
      else if (dk == 2) blk_mv<DJ, 2>(s, Fb, off, Yb, pk, p.Bp);
      else blk_mv<DJ, 1>(s, Fb, off, Yb, pk, p.Bp);
    }
  }
  reduce_to_warp0<DJ>(s, red, warp, lane);
  if (warp != 0 || !live) return;
  const int64_t e0 = p.pstart[j] - r.root_start;
#pragma unroll
  for (int q = 0; q < DJ; q++) rhs_dense[b * r.nt + e0 + q] = s[q] + rhs[b * p.n + p.col_start[j] + q];
}

// x of the root: dense [B, nt] -> permuted lane vector (for the bottom columns' backward substitution) and the caller's x (unscrambled)
__global__ void __launch_bounds__(256) lane_root_scatter_kernel(LaneSolveArgs p, LaneRootArgs r, const double* __restrict__ x_dense, double* __restrict__ Y,
                                                                double* __restrict__ x) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t q = t / p.Bp, b = t - q * p.Bp;  // q = column slot * 6 + component
  const int64_t c = q / 6;
  const int comp = (int)(q - c * 6);
  if (c >= r.num_cols || b >= p.B) return;
  const int j = r.root_cols[c];
  const int64_t e0 = p.pstart[j] - r.root_start;
  if (comp >= r.root_dims[c]) return;
  const double v = x_dense[b * r.nt + e0 + comp];
  Y[(int64_t)(p.pstart[j] + comp) * p.Bp + b] = v;
  x[b * p.n + p.col_start[j] + comp] = v;
}

__global__ void __launch_bounds__(256) lane_damp_kernel(thb_sparse_lane_plan p, double* __restrict__ F, const double* __restrict__ alpha,
                                                        const double* __restrict__ beta, int64_t B, int64_t Bp) {
  // diag <- diag * (1 + alpha_b) + beta_b   (extlib/baspacho_solver.cpp:181-183, baspacho_solver_cuda.cu:171-185)
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t e = t / Bp, b = t - e * Bp;
  if (e >= p.n || b >= B) return;
  int lo = 0, hi = (int)p.N;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (p.pstart[mid] <= e) lo = mid; else hi = mid;
  }
  const int d = p.dims[lo];
  const int r = (int)(e - p.pstart[lo]);
  double* D = F + (p.diag_off[lo] + (int64_t)r * d + r) * Bp + b;
  const double a = alpha != nullptr ? alpha[b] : 0.0, be = beta != nullptr ? beta[b] : 0.0;
  *D = *D * (1.0 + a) + be;
}

// add_MtM into the lane-interleaved factor storage (K6, baspacho_solver_cuda.cu:96-134; no atomics).  One thread per
// (batch item, block of AtA): for every cost function touching the variable pair it reads the two Jacobian blocks
// row by row (rows*(di+dj) loads, each row segment contiguous in A_val[b,:]) and accumulates the di x dj product in
// registers; the store is coalesced over the batch.  Block sizes <= 6 (the lane kernels' domain).
__global__ void __launch_bounds__(128) lane_gram_kernel(thb_gram_plan p, int64_t B, int64_t Bp, const double* __restrict__ A_val, int64_t nnz,
                                                        double* __restrict__ F) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t blk = t / Bp, b = t - blk * Bp;
  if (blk >= p.num_blocks || b >= B) return;
  const int di = p.blk_rows[blk], dj = p.blk_cols[blk];
  const double* A = A_val + b * nnz;
  double acc[36];
#pragma unroll
  for (int e = 0; e < 36; e++) acc[e] = 0.0;
  const int c1 = p.blk_cptr[blk + 1];
  for (int c = p.blk_cptr[blk]; c < c1; c++) {
    const double* base = A + p.c_off[c];
    const int stride = p.c_stride[c];
    const int rows = p.c_rows[c];
    const int oa = p.c_bpa[c], ob = p.c_bpb[c];
    for (int r = 0; r < rows; r++) {
      double ja[6], jb[6];
#pragma unroll
      for (int q = 0; q < 6; q++) ja[q] = q < di ? base[r * stride + oa + q] : 0.0;
#pragma unroll
      for (int q = 0; q < 6; q++) jb[q] = q < dj ? base[r * stride + ob + q] : 0.0;
#pragma unroll
      for (int pp = 0; pp < 6; pp++)
#pragma unroll
        for (int qq = 0; qq < 6; qq++) acc[pp * 6 + qq] += ja[pp] * jb[qq];
    }
  }
  double* o = F + p.blk_out[blk] * Bp + b;
  const int ld = p.blk_ld[blk];
#pragma unroll
  for (int pp = 0; pp < 6; pp++)
#pragma unroll
    for (int qq = 0; qq < 6; qq++)
      if (pp < di && qq < dj) o[(int64_t)(pp * ld + qq) * Bp] = acc[pp * 6 + qq];
}

}  // namespace thb

// ---------------------------------------------------------------------------------------------------------------------------------
#define LN_DIM_OK(d) ((d) == 1 || (d) == 2 || (d) == 3 || (d) == 6)
#define LN_SWITCH_DJ(DI, dj, CALL)                                                          \
  switch (dj) { case 1: { CALL(DI, 1); } break; case 2: { CALL(DI, 2); } break; case 3: { CALL(DI, 3); } break; case 6: { CALL(DI, 6); } break; default: return THB_ERR_UNSUPPORTED; }
#define LN_SWITCH(di, dj, CALL)                                                             \
  switch (di) { case 1: LN_SWITCH_DJ(1, dj, CALL) break; case 2: LN_SWITCH_DJ(2, dj, CALL) break; case 3: LN_SWITCH_DJ(3, dj, CALL) break; \
                case 6: LN_SWITCH_DJ(6, dj, CALL) break; default: return THB_ERR_UNSUPPORTED; }
#define LN_SWITCH1(dj, CALL)                                                                \
  switch (dj) { case 1: { CALL(1); } break; case 2: { CALL(2); } break; case 3: { CALL(3); } break; case 6: { CALL(6); } break; default: return THB_ERR_UNSUPPORTED; }

extern "C" {

int64_t thb_sparse_lane_padded_batch(int64_t B) { return (B + 31) / 32 * 32; }

int thb_sparse_lane_gram_f64(const thb_gram_plan* g, int64_t B, const double* A_val, int64_t nnz, double* factor, thb_stream_t s) {
  if (g == nullptr || A_val == nullptr || factor == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || g->num_blocks == 0) return THB_OK;
  const int64_t Bp = thb_sparse_lane_padded_batch(B);
  const int64_t total = g->num_blocks * Bp;
  thb::lane_gram_kernel<<<(unsigned)((total + 127) / 128), 128, 0, thb_cs(s)>>>(*g, B, Bp, A_val, nnz, factor);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

int thb_sparse_lane_damp_f64(const thb_sparse_lane_plan* p, double* factor, const double* alpha, const double* beta, int64_t B, thb_stream_t s) {
  if (p == nullptr || factor == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || p->n == 0) return THB_OK;
  const int64_t Bp = thb_sparse_lane_padded_batch(B);
  const int64_t total = p->n * Bp;
  thb::lane_damp_kernel<<<(unsigned)((total + 255) / 256), 256, 0, thb_cs(s)>>>(*p, factor, alpha, beta, B, Bp);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

static int lane_factor_impl(const thb_sparse_lane_plan* p, const thb_sparse_lane_tiles* tiles, double* factor, double* diagl, int32_t* info,
                            int64_t B, thb_stream_t s) {
  if (p == nullptr || factor == nullptr || diagl == nullptr || info == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || p->N == 0) return THB_OK;
  cudaStream_t cs = thb_cs(s);
  THB_CUDA(cudaMemsetAsync(info, 0, sizeof(int32_t) * B, cs));
  thb::LaneArgs a;
  a.up_a = p->up_a; a.up_b = p->up_b; a.up_k = p->up_k;
  a.u_tgt = p->u_tgt; a.u_p0 = p->u_p0; a.u_p1 = p->u_p1;
  a.t_off = p->t_off; a.t_diag = p->t_diag; a.t_dl = p->t_dl; a.t_pstart = p->t_pstart;
  a.B = B; a.Bp = thb_sparse_lane_padded_batch(B); a.nbx = (int)(a.Bp / 32);
  for (int64_t l = 0; l < p->num_launches; l++) {
    const int32_t* L = p->launches + 5 * l;
    const int kind = L[0], di = L[1], dj = L[2];
    a.begin = L[3]; a.end = L[4];
    const int items = a.end - a.begin;
    if (items <= 0 || kind == THB_LANE_S) continue;
    const unsigned grid_w = (unsigned)(((items + thb::LN_WARPS - 1) / thb::LN_WARPS) * a.nbx);
    if (kind == THB_LANE_U) {
#define CALL_U(DI, DJ) thb::lane_update_kernel<DI, DJ><<<grid_w, 32 * thb::LN_WARPS, 0, cs>>>(a, factor)
      LN_SWITCH(di, dj, CALL_U)
    } else if (kind == THB_LANE_UH) {
      const unsigned grid_h = (unsigned)(items * a.nbx);
#define CALL_UH(DI, DJ) thb::lane_update_heavy_kernel<DI, DJ><<<grid_h, 32 * thb::LH_WARPS, 0, cs>>>(a, factor)
      LN_SWITCH(di, dj, CALL_UH)
    } else if (kind == THB_LANE_T) {
#define CALL_T(DI, DJ) thb::lane_trsm_kernel<DI, DJ><<<grid_w, 32 * thb::LN_WARPS, 0, cs>>>(a, factor, diagl, info)
      LN_SWITCH(di, dj, CALL_T)
    } else if (kind == THB_LANE_TU) {
      if (tiles == nullptr || di != 6 || dj != 6 || a.end > tiles->num_tiles) return THB_ERR_BAD_ARG;
      constexpr int TR = THB_TILE_ROWS, TC = THB_TILE_COLS;
      constexpr int smem = 2 * (TR + TC) * 36 * 32 * (int)sizeof(double);
      auto kern = thb::lane_tile_update_kernel<6, TR, TC>;
      static bool smem_opted_in[64] = {};   // per device; idempotent, not a stream operation (legal under CUDA-graph capture)
      int dev = 0;
      THB_CUDA(cudaGetDevice(&dev));
      if (dev < 0 || dev >= 64 || !smem_opted_in[dev]) {
        THB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        if (dev >= 0 && dev < 64) smem_opted_in[dev] = true;
      }
      thb::LaneTileArgs ta;
      ta.tile_tgt = tiles->tile_tgt; ta.step_ptr = tiles->step_ptr; ta.step_src = tiles->step_src;
      ta.begin = a.begin; ta.Bp = a.Bp;
      kern<<<dim3((unsigned)items, (unsigned)a.nbx), 32 * TR * TC, smem, cs>>>(ta, factor);
    } else {
      return THB_ERR_BAD_ARG;
    }
    THB_CHECK_LAUNCH();
  }
  return THB_OK;
}

int thb_sparse_lane_factor_f64(const thb_sparse_lane_plan* p, double* factor, double* diagl, int32_t* info, int64_t B, thb_stream_t s) {
  return lane_factor_impl(p, nullptr, factor, diagl, info, B, s);
}

int thb_sparse_lane_factor_tiled_f64(const thb_sparse_lane_plan* p, const thb_sparse_lane_tiles* t, double* factor, double* diagl,
                                     int32_t* info, int64_t B, thb_stream_t s) {
  if (t == nullptr) return THB_ERR_BAD_ARG;
  return lane_factor_impl(p, t, factor, diagl, info, B, s);
}

static thb::LaneSolveArgs lane_solve_args(const thb_sparse_lane_plan* p, int64_t B) {
  thb::LaneSolveArgs a;
  a.s_col = p->s_col; a.pstart = p->pstart; a.col_start = p->col_start; a.dl_off = p->dl_off;
  a.fr_ptr = p->fr_ptr; a.fr_off = p->fr_off; a.fr_p = p->fr_p; a.fr_d = p->fr_d;
  a.bc_ptr = p->bc_ptr; a.bc_off = p->bc_off; a.bc_p = p->bc_p; a.bc_d = p->bc_d;
  a.begin = a.end = 0;
  a.B = B; a.Bp = thb_sparse_lane_padded_batch(B); a.nbx = (int)(a.Bp / 32); a.n = p->n;
  return a;
}

// passes: bit 0 = forward substitution, bit 1 = backward substitution (thb_sparse_lane_solve_f64 = both)
static int lane_solve_passes(const thb_sparse_lane_plan* p, const double* factor, const double* diagl, const double* rhs, double* x, double* work,
                             int64_t B, int passes, thb_stream_t s) {
  if (p == nullptr || factor == nullptr || diagl == nullptr || work == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (((passes & 1) && rhs == nullptr) || ((passes & 2) && x == nullptr)) return THB_ERR_BAD_ARG;
  if (B == 0 || p->N == 0) return THB_OK;
  cudaStream_t cs = thb_cs(s);
  thb::LaneSolveArgs a = lane_solve_args(p, B);
  for (int pass = 0; pass < 2; pass++) {
    if (!(passes & (1 << pass))) continue;
    for (int64_t q = 0; q < p->num_launches; q++) {
      const int64_t l = pass == 0 ? q : p->num_launches - 1 - q;
      const int32_t* L = p->launches + 5 * l;
      if (L[0] != THB_LANE_S) continue;
      const int dj = L[2];
      a.begin = L[3]; a.end = L[4];
      const int items = a.end - a.begin;
      if (items <= 0) continue;
      const unsigned grid_w = (unsigned)(items * a.nbx);
      if (pass == 0) {
#define CALL_F(DJ) thb::lane_forward_kernel<DJ><<<grid_w, 32 * thb::LS_WARPS, 0, cs>>>(a, factor, diagl, rhs, work)
        LN_SWITCH1(dj, CALL_F)
      } else {
#define CALL_B(DJ) thb::lane_backward_kernel<DJ><<<grid_w, 32 * thb::LS_WARPS, 0, cs>>>(a, factor, diagl, work, x)
        LN_SWITCH1(dj, CALL_B)
      }
      THB_CHECK_LAUNCH();
    }
  }
  return THB_OK;
}

int thb_sparse_lane_solve_f64(const thb_sparse_lane_plan* p, const double* factor, const double* diagl, const double* rhs, double* x,
                              double* work, int64_t B, thb_stream_t s) {
  return lane_solve_passes(p, factor, diagl, rhs, x, work, B, 3, s);
}
int thb_sparse_lane_forward_f64(const thb_sparse_lane_plan* p, const double* factor, const double* diagl, const double* rhs, double* work,
                                int64_t B, thb_stream_t s) {
  return lane_solve_passes(p, factor, diagl, rhs, nullptr, work, B, 1, s);
}
int thb_sparse_lane_backward_f64(const thb_sparse_lane_plan* p, const double* factor, const double* diagl, double* work, double* x, int64_t B,
                                 thb_stream_t s) {
  return lane_solve_passes(p, factor, diagl, nullptr, x, work, B, 2, s);
}

static int lane_piece_passes(const thb_sparse_lane_plan* p, const thb_sparse_lane_pieces* pc, const double* factor, const double* diagl,
                             const double* rhs, double* x, double* work, int64_t B, int passes, thb_stream_t s) {
  if (p == nullptr || pc == nullptr || factor == nullptr || diagl == nullptr || work == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (((passes & 1) && rhs == nullptr) || ((passes & 2) && x == nullptr)) return THB_ERR_BAD_ARG;
  if (B == 0 || pc->num_pieces == 0) return THB_OK;
  cudaStream_t cs = thb_cs(s);
  thb::LaneSolveArgs a = lane_solve_args(p, B);
  thb::LanePieceArgs g;
  g.first = pc->first; g.width = pc->width; g.fr_ext_end = pc->fr_ext_end; g.bc_int_end = pc->bc_int_end; g.order = pc->order;
  for (int pass = 0; pass < 2; pass++) {
    if (!(passes & (1 << pass))) continue;
    for (int64_t q = 0; q < pc->num_launches; q++) {
      const int64_t l = pass == 0 ? q : pc->num_launches - 1 - q;
      const int32_t* L = pc->launches + 3 * l;
      const int dj = L[0];
      a.begin = L[1]; a.end = L[2];
      const int items = a.end - a.begin;
      if (items <= 0) continue;
      const unsigned grid_w = (unsigned)(items * a.nbx);
      if (pass == 0) {
#define CALL_PF(DJ) thb::lane_piece_forward_kernel<DJ><<<grid_w, 32 * thb::LS_WARPS, 0, cs>>>(a, g, factor, diagl, rhs, work)
        LN_SWITCH1(dj, CALL_PF)
      } else {
#define CALL_PB(DJ) thb::lane_piece_backward_kernel<DJ><<<grid_w, 32 * thb::LS_WARPS, 0, cs>>>(a, g, factor, diagl, work, x)
        LN_SWITCH1(dj, CALL_PB)
      }
      THB_CHECK_LAUNCH();
    }
  }
  return THB_OK;
}

int thb_sparse_lane_piece_forward_f64(const thb_sparse_lane_plan* p, const thb_sparse_lane_pieces* pc, const double* factor, const double* diagl,
                                      const double* rhs, double* work, int64_t B, thb_stream_t s) {
  return lane_piece_passes(p, pc, factor, diagl, rhs, nullptr, work, B, 1, s);
}
int thb_sparse_lane_piece_backward_f64(const thb_sparse_lane_plan* p, const thb_sparse_lane_pieces* pc, const double* factor, const double* diagl,
                                       double* work, double* x, int64_t B, thb_stream_t s) {
  return lane_piece_passes(p, pc, factor, diagl, nullptr, x, work, B, 2, s);
}

static thb::LaneRootArgs lane_root_args(const thb_sparse_lane_root* r) {
  thb::LaneRootArgs a;
  a.rb_off = r->rb_off; a.rb_row = r->rb_row; a.rb_col = r->rb_col; a.rb_di = r->rb_di; a.rb_dj = r->rb_dj; a.num_blocks = r->num_blocks;
  a.rf_p0 = r->rf_p0; a.rf_p1 = r->rf_p1; a.root_cols = r->root_cols; a.root_dims = r->root_dims; a.num_cols = r->num_cols; a.nt = r->nt; a.root_start = r->root_start;
  return a;
}

int thb_sparse_lane_root_gather_f64(const thb_sparse_lane_root* r, const double* factor, double* S, int64_t B, thb_stream_t s) {
  if (r == nullptr || factor == nullptr || S == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || r->num_blocks == 0) return THB_OK;
  cudaStream_t cs = thb_cs(s);
  const int64_t Bp = thb_sparse_lane_padded_batch(B);
  THB_CUDA(cudaMemsetAsync(S, 0, sizeof(double) * (size_t)(B * r->nt * r->nt), cs));  // the strict upper triangle stays zero
  const int64_t total = r->num_blocks * 36 * Bp;
  thb::lane_root_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, cs>>>(lane_root_args(r), factor, S, B, Bp);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

int thb_sparse_lane_root_rhs_f64(const thb_sparse_lane_plan* p, const thb_sparse_lane_root* r, const double* factor, const double* rhs,
                                 const double* work, double* rhs_dense, int64_t B, thb_stream_t s) {
  if (p == nullptr || r == nullptr || factor == nullptr || rhs == nullptr || work == nullptr || rhs_dense == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || r->num_cols == 0) return THB_OK;
  cudaStream_t cs = thb_cs(s);
  thb::LaneSolveArgs a = lane_solve_args(p, B);
  const thb::LaneRootArgs ra = lane_root_args(r);
  // root columns grouped by block size on the host: seg [3*q] = dim, [3*q+1] = begin, [3*q+2] = end (indices into root_cols)
  for (int64_t q = 0; q < r->num_segments; q++) {
    const int dj = r->segments[3 * q];
    a.begin = r->segments[3 * q + 1]; a.end = r->segments[3 * q + 2];
    const int items = a.end - a.begin;
    if (items <= 0) continue;
    const unsigned grid_w = (unsigned)(items * a.nbx);
#define CALL_RR(DJ) thb::lane_root_rhs_kernel<DJ><<<grid_w, 32 * thb::LS_WARPS, 0, cs>>>(a, ra, factor, rhs, work, rhs_dense)
    LN_SWITCH1(dj, CALL_RR)
    THB_CHECK_LAUNCH();
  }
  return THB_OK;
}

int thb_sparse_lane_root_scatter_f64(const thb_sparse_lane_plan* p, const thb_sparse_lane_root* r, const double* x_dense, double* work, double* x,
                                     int64_t B, thb_stream_t s) {
  if (p == nullptr || r == nullptr || x_dense == nullptr || work == nullptr || x == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || r->num_cols == 0) return THB_OK;
  thb::LaneSolveArgs a = lane_solve_args(p, B);
  const int64_t total = r->num_cols * 6 * a.Bp;
  thb::lane_root_scatter_kernel<<<(unsigned)((total + 255) / 256), 256, 0, thb_cs(s)>>>(a, lane_root_args(r), x_dense, work, x);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

}  // extern "C"
