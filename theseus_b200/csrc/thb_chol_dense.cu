// Batched dense Cholesky factor + solve with fused LM damping, fp64, for sm_90a.
//
// Replaces torch.linalg.cholesky + torch.cholesky_solve + DenseSolver._apply_damping
// (theseus/optimizer/linear/dense_solver.py:38-64,159-161).
//
// Algorithm: left-looking blocked Cholesky over 64-wide block columns, 128x64 output tiles.  For block column j
// one launch runs a CTA per (matrix b, 128-row tile i at or below the diagonal block):
//   A. C = sum_{k<64j} L[rows,k] L[cols,k]^T   DMMA (mma.sync m8n8k4 f64) main loop, cp.async 3-stage pipeline,
//                                              operands staged in shared memory with a conflict-free padded stride
//   B. C = (AtA tile, LM damping fused on the diagonal) - C     (AtA is read exactly once and never modified)
//   C. the CTA holding the 64x64 diagonal block factors it (blocked 2x2: two 32x32 blocks are factored AND inverted
//      by one warp in registers with shuffles, the rest are DMMA block products), forms W = L_jj^-1, stores
//      L_jj and W and releases a per-(b,j) flag
//   D. every tile row below the diagonal block: acquire the flag, L[i,j] = C W^T as a second DMMA product
//      (triangular k-range skipped), so the TRSM also runs on the FP64 tensor pipe
// Two CTAs are resident per SM (<=128 registers, ~98 KB shared memory each): while one CTA is in its non-tensor
// phases (B: global loads, C: the serial 32x32 pivots, flag wait, stores) the other keeps the tensor pipe busy.
// The diagonal CTAs have the lowest block indices of their launch, so they are resident before (or together with)
// the CTAs that wait on them.  The left-looking order keeps every C tile in registers for its whole k-loop: L is
// written once and AtA read once (algorithmic bytes) instead of the read-modify-write sweeps of a right-looking update.
// Solve: x = M^-1 rhs with the stored W_j (triangular solves become mat-vecs), one CTA per matrix, HBM-bound.
//
// wgmma has no fp64 kind; the FP64 tensor pipe of sm_90a is reached with mma.sync DMMA (m8n8k4).
#include <stdlib.h>

#include "thb_common.cuh"

#ifndef THB_CHOL_GROUP_DEFAULT
#define THB_CHOL_GROUP_DEFAULT (1LL << 40)
#endif

namespace thb {

// *info <- the smallest failing position recorded so far (pos > 0; 0 = none yet).  Columns factored concurrently may fail in any order;
// the smallest failing position is the leading minor that torch.linalg.cholesky / LAPACK potrf name, whichever thread gets there first.
// (Defined in each kernel file rather than in thb_common.cuh: the host emulation of the kernels compiles the sources without that header.)
__device__ __forceinline__ void record_first_failure(int* info, int pos) {
  int old = 0;
  while (true) {
    const int prev = atomicCAS(info, old, pos);
    if (prev == old || (prev != 0 && prev <= pos)) return;
    old = prev;
  }
}

constexpr int TM = 128;        // tile rows
constexpr int TN = 64;         // tile cols = block-column width
#ifndef THB_CHOL_KB
#define THB_CHOL_KB 16
#endif
#ifndef THB_CHOL_STAGES
#define THB_CHOL_STAGES 3
#endif
constexpr int KB = THB_CHOL_KB;  // k-step of the pipelined product
constexpr int SA = KB + 4;     // smem row stride (doubles) of a [rows x KB] operand tile: 2*SA mod 32 == 8 -> conflict-free DMMA fragment loads
constexpr int KB_W = 16;       // k-step of the (short) TRSM product
constexpr int SW = KB_W + 4;
constexpr int SC = 68;         // smem row stride (doubles) of the 128x64 C tile (2*SC mod 32 == 8)
constexpr int SB32 = 36;       // row stride of the 32x32 inverse blocks
constexpr int STAGES = THB_CHOL_STAGES;
constexpr int WSTAGES = 3;
constexpr int CHOL_THREADS = 256;
constexpr int A_TILE = TM * SA;  // doubles
constexpr int B_TILE = TN * SA;
constexpr int W_TILE = TN * SW;
constexpr size_t SMEM_PHASE_A = (size_t)STAGES * (A_TILE + B_TILE) * 8;        // 92160 (KB=16, 3 stages)
constexpr size_t SMEM_PHASE_D = (size_t)(TM * SC + WSTAGES * W_TILE) * 8;      // 69632 + 30720 = 100352
constexpr size_t CHOL_SMEM = SMEM_PHASE_A > SMEM_PHASE_D ? SMEM_PHASE_A : SMEM_PHASE_D;
static_assert(2 * (CHOL_SMEM + 1024) <= 232448, "two CTAs per SM must fit in shared memory");

__device__ __forceinline__ void mma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
// with src_bytes < 16 (0 or 8) the rest of the 16 bytes is zero-filled
__device__ __forceinline__ void cp_async16_zfill(void* smem_dst, const void* gmem_src, int src_bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem_src), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async8_zfill(void* smem_dst, const void* gmem_src, int src_bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(s), "l"(gmem_src), "r"(src_bytes));
}
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// stage one [ROWS x KB] operand tile: ROWS consecutive rows of a row-major matrix (leading dimension ld), columns k0..k0+KB
template <int ROWS, int KBX>
__device__ __forceinline__ void load_oper_tile(double* dst, const double* __restrict__ src, int64_t ld, int k0, int tid) {
  constexpr int CPR = KBX / 2;  // 16-byte chunks per row
#pragma unroll
  for (int q = 0; q < (ROWS * CPR) / CHOL_THREADS; q++) {
    const int chunk = tid + q * CHOL_THREADS;
    const int row = chunk / CPR, cc = chunk % CPR;
    cp_async16(dst + row * (KBX + 4) + cc * 2, src + (int64_t)row * ld + k0 + cc * 2);
  }
}

// B operand given as rows of M:  B[k][n] = M[n][k]
__device__ __forceinline__ void tile_mma_rows(double& c0, double& c1, const double* __restrict__ A, int lda,
                                              const double* __restrict__ M, int ldm, int k4b, int k4e, int lr, int lc) {
  for (int k4 = k4b; k4 < k4e; k4++) mma884(c0, c1, A[lr * lda + 4 * k4 + lc], M[lr * ldm + 4 * k4 + lc]);
}
// B operand given as columns of M: B[k][n] = M[k][n]
__device__ __forceinline__ void tile_mma_cols(double& c0, double& c1, const double* __restrict__ A, int lda,
                                              const double* __restrict__ M, int ldm, int k4b, int k4e, int lr, int lc) {
  for (int k4 = k4b; k4 < k4e; k4++) mma884(c0, c1, A[lr * lda + 4 * k4 + lc], M[(4 * k4 + lc) * ldm + lr]);
}

#ifdef THB_CHOL_TIMING
__device__ long long thb_chol_timing[16 * 65536];
#define THB_TICK(slot) do { if (threadIdx.x == 0 && blockIdx.x < 65536) thb_chol_timing[blockIdx.x * 16 + (slot)] = clock64(); } while (0)
#else
#define THB_TICK(slot) do {} while (0)
#endif

// ------------------------------------------------------------------------------------------------
// One warp: Cholesky of the NxN block at T (lower part; row stride SC) and its inverse, in registers (one row / one column per
// lane, lanes >= N idle; pivots and multipliers exchanged with warp shuffles).
// L is written back to T (lower part), the inverse (full NxN, zeros above the diagonal) to Wout (row stride SB32).
// Returns 0 or 1 + index of the first non-positive pivot.
template <int N>
__device__ __noinline__ int warp_potrf_inv(double* __restrict__ T, double* __restrict__ Wout, int lane) {
  const int ln = lane < N ? lane : 0;  // idle lanes shadow lane 0 (their results are never stored)
  double row[N];
#pragma unroll
  for (int q = 0; q < N; q++) row[q] = T[ln * SC + q];
  int fail = 0;
  double invd = 0.0;  // 1 / L[lane][lane]
#pragma unroll
  for (int c = 0; c < N; c++) {
    const double d = __shfl_sync(0xffffffffu, row[c], c);
    if (!(d > 0.0) && fail == 0) fail = c + 1;
    // 1/sqrt(d) by the hardware seed + one Newton step (inline, no slow-path subroutine calls), sqrt(d) = d * rsqrt(d)
    double inv = rsqrt(d);
    inv = inv * (1.5 - 0.5 * d * inv * inv);
    const double sq = d * inv;
    if (lane == c) invd = inv;
    const double lrc = (lane == c) ? sq : row[c] * inv;
    row[c] = lrc;
#pragma unroll
    for (int q = c + 1; q < N; q++) {
      const double lqc = __shfl_sync(0xffffffffu, lrc, q);
      row[q] -= lrc * lqc;  // lanes < q update entries above the diagonal that are never read
    }
  }
  if (lane < N) {
#pragma unroll
    for (int q = 0; q < N; q++)
      if (q <= lane) T[lane * SC + q] = row[q];
  }
  // inverse: lane c owns column c of X = L^-1 (forward substitution, rows broadcast from their owner lane)
  double x[N];
#pragma unroll
  for (int r = 0; r < N; r++) {
    double s = (lane == r) ? 1.0 : 0.0;
#pragma unroll
    for (int k = 0; k < r; k++) {
      const double lrk = __shfl_sync(0xffffffffu, row[k], r);
      s -= lrk * x[k];
    }
    x[r] = s * __shfl_sync(0xffffffffu, invd, r);
  }
  if (lane < N) {
#pragma unroll
    for (int r = 0; r < N; r++) Wout[r * SB32 + lane] = (r >= lane) ? x[r] : 0.0;
  }
  return fail;
}

#ifndef THB_CHOL_LEAF
#define THB_CHOL_LEAF 8
#endif

// All 256 threads: Cholesky + inverse of the NxN block at T (row stride SC; L in place, lower part) -> Wb (row stride SB32; full
// block, zeros above the diagonal).  N == THB_CHOL_LEAF: one warp does it in registers.  Otherwise the same 2x2 recursion as one
// level up: factor+invert T00, L10 = T10 W00^T, T11 -= L10 L10^T, factor+invert T11, W10 = -W11 L10 W00 -- the products as DMMA on
// 8x8 tiles (one warp per tile).  Small leaves matter because the serial pivots are scalar FP64 instructions that compete for the
// FP64 pipe with the DMMA stream of the co-resident CTA: four 8x8 leaves + tile products cost a fraction of one 32x32 register
// leaf.  The return value is valid on warp 0.
template <int N>
__device__ __forceinline__ int block_factor_invert(double* __restrict__ T, double* __restrict__ Wb, int warp, int lane) {
  if constexpr (N <= THB_CHOL_LEAF) {
    int f = 0;
    if (warp == 0) f = warp_potrf_inv<N>(T, Wb, lane);
    __syncthreads();
    return f;
  } else {
    constexpr int H = N / 2, TPB = H / 8;  // half size, 8x8 tiles per side of a half block
    const int lr = lane >> 2, lc = lane & 3;
    const int rt = warp / TPB, ct = warp % TPB;
    const bool own = warp < TPB * TPB;
    double a0 = 0.0, a1 = 0.0;
    const int f0 = block_factor_invert<H>(T, Wb, warp, lane);
    // panel: L10 = T10 W00^T
    if (own) tile_mma_rows(a0, a1, T + (H + 8 * rt) * SC, SC, Wb + (8 * ct) * SB32, SB32, 0, 2 * ct + 2, lr, lc);
    __syncthreads();
    if (own) *reinterpret_cast<double2*>(&T[(H + 8 * rt + lr) * SC + 8 * ct + 2 * lc]) = make_double2(a0, a1);
    __syncthreads();
    // trailing: T11 -= L10 L10^T
    if (own) {
      a0 = a1 = 0.0;
      tile_mma_rows(a0, a1, T + (H + 8 * rt) * SC, SC, T + (H + 8 * ct) * SC, SC, 0, H / 4, lr, lc);
      double2* d = reinterpret_cast<double2*>(&T[(H + 8 * rt + lr) * SC + H + 8 * ct + 2 * lc]);
      double2 v = *d;
      v.x -= a0; v.y -= a1;
      *d = v;
    }
    __syncthreads();
    const int f1 = block_factor_invert<H>(T + H * SC + H, Wb + H * SB32 + H, warp, lane);
    // inverse: X = W11 L10 (W11 lower triangular) parked in the W01 corner, then W10 = -X W00, then W01 = 0
    if (own) {
      a0 = a1 = 0.0;
      tile_mma_cols(a0, a1, Wb + (H + 8 * rt) * SB32 + H, SB32, T + H * SC + 8 * ct, SC, 0, 2 * rt + 2, lr, lc);
      *reinterpret_cast<double2*>(&Wb[(8 * rt + lr) * SB32 + H + 8 * ct + 2 * lc]) = make_double2(a0, a1);
    }
    __syncthreads();
    if (own) {
      a0 = a1 = 0.0;
      tile_mma_cols(a0, a1, Wb + (8 * rt) * SB32 + H, SB32, Wb + 8 * ct, SB32, 2 * ct, H / 4, lr, lc);
      *reinterpret_cast<double2*>(&Wb[(H + 8 * rt + lr) * SB32 + 8 * ct + 2 * lc]) = make_double2(-a0, -a1);
    }
    __syncthreads();
    if (own) *reinterpret_cast<double2*>(&Wb[(8 * rt + lr) * SB32 + H + 8 * ct + 2 * lc]) = make_double2(0.0, 0.0);
    __syncthreads();
    return f0 != 0 ? f0 : (f1 != 0 ? H + f1 : 0);
  }
}

// All 256 threads.  T: the 64x64 diagonal block inside the C tile (row stride SC), Wd: scratch [2][32][SB32],
// Lg/ldl: where L_jj goes in global memory (its first lim rows and columns), Wg: where W = L_jj^-1 goes (row-major 64x64).
__device__ __noinline__ int diag64_factor_invert(double* __restrict__ T, double* __restrict__ Wd, double* __restrict__ Lg, int64_t ldl,
                                                 int lim, double* __restrict__ Wg) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int lr = lane >> 2, lc = lane & 3;
  __shared__ int s_fail;
  if (tid == 0) s_fail = 0;
  __syncthreads();
  // 16 tiles of 8x8 per 32x32 block: two per warp
  const int t0 = warp, t1 = warp + 8;
  const int rt0 = t0 >> 2, ct0 = t0 & 3, rt1 = t1 >> 2, ct1 = t1 & 3;
  double a0, a1, b0, b1;
  // ---- block column 0 ----
  {
    const int f = block_factor_invert<32>(T, Wd, warp, lane);
    if (tid == 0 && f != 0) s_fail = f;
  }
  __syncthreads();
  THB_TICK(8);
  // panel: L10 = T10 W00^T
  a0 = a1 = b0 = b1 = 0.0;
  tile_mma_rows(a0, a1, T + (32 + 8 * rt0) * SC, SC, Wd + (8 * ct0) * SB32, SB32, 0, 2 * ct0 + 2, lr, lc);
  tile_mma_rows(b0, b1, T + (32 + 8 * rt1) * SC, SC, Wd + (8 * ct1) * SB32, SB32, 0, 2 * ct1 + 2, lr, lc);
  __syncthreads();
  *reinterpret_cast<double2*>(&T[(32 + 8 * rt0 + lr) * SC + 8 * ct0 + 2 * lc]) = make_double2(a0, a1);
  *reinterpret_cast<double2*>(&T[(32 + 8 * rt1 + lr) * SC + 8 * ct1 + 2 * lc]) = make_double2(b0, b1);
  __syncthreads();
  // trailing: T11 -= L10 L10^T   (each 8x8 tile owned by one warp)
  a0 = a1 = b0 = b1 = 0.0;
  tile_mma_rows(a0, a1, T + (32 + 8 * rt0) * SC, SC, T + (32 + 8 * ct0) * SC, SC, 0, 8, lr, lc);
  tile_mma_rows(b0, b1, T + (32 + 8 * rt1) * SC, SC, T + (32 + 8 * ct1) * SC, SC, 0, 8, lr, lc);
  {
    double2* d0 = reinterpret_cast<double2*>(&T[(32 + 8 * rt0 + lr) * SC + 32 + 8 * ct0 + 2 * lc]);
    double2* d1 = reinterpret_cast<double2*>(&T[(32 + 8 * rt1 + lr) * SC + 32 + 8 * ct1 + 2 * lc]);
    double2 v0 = *d0, v1 = *d1;
    v0.x -= a0; v0.y -= a1; v1.x -= b0; v1.y -= b1;
    *d0 = v0;
    *d1 = v1;
  }
  __syncthreads();
  THB_TICK(9);
  // ---- block column 1 ----
  {
    const int f = block_factor_invert<32>(T + 32 * SC + 32, Wd + 32 * SB32, warp, lane);
    if (tid == 0 && f != 0 && s_fail == 0) s_fail = 32 + f;
  }
  __syncthreads();
  THB_TICK(10);
  // ---- store L_jj (lower part; zeros above) ----
  for (int e = tid; e < 64 * 64; e += CHOL_THREADS) {
    const int r = e >> 6, c = e & 63;
    if (r < lim && c < lim) Lg[(int64_t)r * ldl + c] = (c <= r) ? T[r * SC + c] : 0.0;
  }
  __syncthreads();
  // ---- inverse: diagonal blocks <- W_kk (explicit zeros above the diagonal), then W10 = -(W11 L10) W00 ----
  for (int e = tid; e < 2 * 32 * 32; e += CHOL_THREADS) {
    const int kb = e >> 10, r = (e >> 5) & 31, c = e & 31;
    T[(32 * kb + r) * SC + 32 * kb + c] = Wd[kb * 32 * SB32 + r * SB32 + c];
  }
  __syncthreads();
  a0 = a1 = b0 = b1 = 0.0;  // X = W11 L10 (W11 lower triangular)
  tile_mma_cols(a0, a1, T + (32 + 8 * rt0) * SC + 32, SC, T + 32 * SC + 8 * ct0, SC, 0, 2 * rt0 + 2, lr, lc);
  tile_mma_cols(b0, b1, T + (32 + 8 * rt1) * SC + 32, SC, T + 32 * SC + 8 * ct1, SC, 0, 2 * rt1 + 2, lr, lc);
  __syncthreads();
  *reinterpret_cast<double2*>(&T[(32 + 8 * rt0 + lr) * SC + 8 * ct0 + 2 * lc]) = make_double2(a0, a1);
  *reinterpret_cast<double2*>(&T[(32 + 8 * rt1 + lr) * SC + 8 * ct1 + 2 * lc]) = make_double2(b0, b1);
  __syncthreads();
  a0 = a1 = b0 = b1 = 0.0;  // W10 = -X W00 (W00 lower triangular)
  tile_mma_cols(a0, a1, T + (32 + 8 * rt0) * SC, SC, T + 8 * ct0, SC, 2 * ct0, 8, lr, lc);
  tile_mma_cols(b0, b1, T + (32 + 8 * rt1) * SC, SC, T + 8 * ct1, SC, 2 * ct1, 8, lr, lc);
  __syncthreads();
  *reinterpret_cast<double2*>(&T[(32 + 8 * rt0 + lr) * SC + 8 * ct0 + 2 * lc]) = make_double2(-a0, -a1);
  *reinterpret_cast<double2*>(&T[(32 + 8 * rt1 + lr) * SC + 8 * ct1 + 2 * lc]) = make_double2(-b0, -b1);
  __syncthreads();
  THB_TICK(11);
  for (int e = tid; e < 64 * 64; e += CHOL_THREADS) {
    const int r = e >> 6, c = e & 63;
    Wg[e] = (c <= r) ? T[r * SC + c] : 0.0;
  }
  return s_fail;
}

struct CholArgs {
  const double* AtA;   // [B,n,n]
  const double* alpha; // [B] or null
  const double* beta;  // [B] or null
  double* L;           // [B,np,np]   (np = n rounded up to a multiple of 128)
  double* W;           // [B,nb,64,64] (nb = np/64)
  int* flags;          // [B,nb]      W_j ready
  int* done;           // [B,ntr]     number of finished block columns of each 128-row tile
  int32_t* info;       // [B]
  int64_t B, n, np;
  int nb, ntr;
  int* ticket;         // tile queue: a CTA's position in the dependency order is the ticket it draws when it STARTS running
  int nb_piv;          // block columns that are factored; block columns >= nb_piv only receive the update of the pivot columns
                       // (partial factorisation of a frontal matrix: the trailing block becomes the Schur complement)
  int64_t a_bstride, l_bstride;  // batch strides (doubles) of AtA and L; AtA == L (in place) for frontal matrices
  int info_base;       // added to the reported pivot index (position of the front's first pivot in the permuted vector)
  int k_lim;           // partial mode: KB-steps of the k loop that hold real pivot columns (the identity padding of the last pivot
                       // block column contributes nothing to the rows below it); the full factorisation uses nb * TN / KB
  int n_real;          // partial mode: rows / columns >= n_real are padding (tiles that lie entirely there are skipped)
  int group;           // tickets go to groups of `group` matrices, one group after the other (B: one group)
  ThbCholDirect d;     // partial mode on a big front of the multifrontal factor (d.fd != null): the initial tiles are gathered from
                       // AtA and the children's update matrices, the pivot columns' L goes to the front's panel and is read from there
};

// Direct mode: front row (= row of its panel) of row fr of the padded front matrix, or -1 in the padding
__device__ __forceinline__ int direct_row(const ThbCholDirect& d, int fr) {
  return fr < d.w ? fr : ((fr >= d.wpad && fr - d.wpad < d.b) ? fr - d.wpad + d.w : -1);
}

// Direct mode: stage [ROWS x KB] of L from the panel (row-major, ld w): rows row0.. of the padded front matrix, columns k0..k0+KB.
// Padding rows and columns >= w are zero-filled.  Of the values the in-place form reads there (identity / zeros of the padding, L of
// the padding rows and of the columns between w and the next multiple of KB), the only ones that are not +0.0 multiply into rows or
// columns of the padding, which are never stored; a +0.0 product added to a real entry leaves it bitwise unchanged.
template <int ROWS>
__device__ __forceinline__ void load_panel_tile(double* dst, const double* __restrict__ Pn, const ThbCholDirect& d, int row0, int k0, int tid) {
  constexpr int CPR = KB / 2;
#pragma unroll
  for (int q = 0; q < (ROWS * CPR) / CHOL_THREADS; q++) {
    const int chunk = tid + q * CHOL_THREADS;
    const int row = chunk / CPR, cc = chunk % CPR;
    const int pr = direct_row(d, row0 + row), k = k0 + cc * 2;
    double* s = dst + row * SA + cc * 2;
    const double* g = Pn + (int64_t)(pr >= 0 ? pr : 0) * d.w + k;
    if ((d.w & 1) == 0) {   // every row 16-byte aligned (panels are)
      const bool ok = pr >= 0 && k < d.w;
      cp_async16_zfill(s, ok ? g : Pn, ok ? 16 : 0);
    } else {
      const bool ok0 = pr >= 0 && k < d.w, ok1 = pr >= 0 && k + 1 < d.w;
      cp_async8_zfill(s, ok0 ? g : Pn, ok0 ? 8 : 0);
      cp_async8_zfill(s + 1, ok1 ? g + 1 : Pn, ok1 ? 8 : 0);
    }
  }
}

__device__ __forceinline__ void wait_ge(const int* addr, int target) {
  int v;
  do {
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(addr) : "memory");
    if (v < target) __nanosleep(100);
  } while (v < target);
}

__global__ void __launch_bounds__(CHOL_THREADS, 2) chol_col_kernel(CholArgs p) {
  extern __shared__ __align__(16) double smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // Tile queue: the CTA draws a ticket when it starts RUNNING; ticket -> (group of matrices, block column j, row tile i, matrix b):
  // the matrices in groups of p.group, one group after the other; inside a group ordered by column, the diagonal tile of a column
  // first, the matrix index fastest.  A CTA only ever waits on tiles of its own matrix in earlier block columns, or on the diagonal
  // tile of its own column: all in its group, with a smaller ticket.  Every smaller ticket was drawn by a CTA that is already running
  // (or done): no deadlock whatever order the hardware dispatches blocks in (no reliance on in-order dispatch, MPS / preemption safe).
  // (A group keeps the operands its later columns read -- the L tiles its earlier columns wrote -- in L2; one group of all B matrices
  // sweeps the whole batch between a tile's write and its reads.)
  __shared__ int s_ticket;
  if (tid == 0) s_ticket = atomicAdd(p.ticket, 1);
  __syncthreads();
  const int64_t bid = s_ticket;
  // block column j of one matrix starts at tile cs1(j) = j ntr - floor((j-1)^2 / 4) of that matrix (column j owns ntr - j/2 tiles)
  auto cs1 = [&](int jj) -> int64_t { const int64_t m = jj > 0 ? jj - 1 : 0; return (int64_t)jj * p.ntr - (m * m) / 4; };
  const int64_t per_group = cs1(p.nb) * p.group;
  const int64_t g0 = (bid / per_group) * p.group;          // first matrix of the group
  const int64_t gs = min((int64_t)p.group, p.B - g0);      // matrices in the group (the last one may be smaller)
  const int64_t relg = bid - (g0 / p.group) * per_group;
  int j;
  {
    int lo = 0, hi = p.nb;  // largest j with cs1(j) gs <= relg
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (cs1(mid) * gs <= relg) lo = mid; else hi = mid;
    }
    j = lo;
  }
  const int64_t rel = relg - cs1(j) * gs;
  const int i0 = j >> 1;                     // 128-row tile that contains the diagonal block of column j
  const int64_t b = g0 + rel % gs;
  const int i = i0 + (int)(rel / gs);
  const bool direct = p.d.fd != nullptr;
  const bool is_diag = (i == i0);
  const int roff = (j & 1) * 64;             // row offset of the diagonal block inside its tile
  const int64_t np = p.np;
  if (j >= p.nb_piv && ((int64_t)j * TN >= p.n_real || (int64_t)i * TM >= p.n_real)) return;   // trailing tile entirely in the padding
  double* Lb = p.L + b * p.l_bstride;
  const int wm = warp >> 1, wn = warp & 1;   // 4 x 2 warps -> 32 x 32 warp tiles
  const int lr = lane >> 2, lc = lane & 3;

  // ---------------- phase A: acc = sum_k L[rows,k] L[cols,k]^T ----------------
  THB_TICK(0);
  // The accumulators start at -(AtA tile with the LM damping fused on the diagonal): the global loads are in flight
  // while the cp.async pipeline fills, and C = AtA - sum L L^T is simply -acc at the end (AtA is read exactly once).
  double acc[4][4][2];
  double* Pn = nullptr;   // direct mode: this matrix's panel
  if (direct) {
    // Direct mode: the tile of the front matrix that front_assemble_kernel would have written -- zeros above the diagonal, identity on the
    // padding, AtA (+ damping on the pivots' diagonal), then the children's update matrices added in list order -- gathered here: the same
    // per-entry sums in the same order, so every value is bitwise the one it reads from the assembled matrix
    const ThbCholDirect& d = p.d;
    const int64_t* FD = d.fd;
    Pn = d.factor + b * d.data_size + FD[4];
    const double al = d.alpha != nullptr ? d.alpha[b] : 0.0;
    const double be = d.beta != nullptr ? d.beta[b] : 0.0;
    int li[4], lj[4][2];
#pragma unroll
    for (int mi = 0; mi < 4; mi++) li[mi] = direct_row(d, i * TM + wm * 32 + mi * 8 + lr);
#pragma unroll
    for (int ni = 0; ni < 4; ni++)
#pragma unroll
      for (int u = 0; u < 2; u++) lj[ni][u] = direct_row(d, j * TN + wn * 32 + ni * 8 + lc * 2 + u);
    // AtA: the panel-map entries of the 32 elements, then their values
    int32_t m[4][4][2];
#pragma unroll
    for (int mi = 0; mi < 4; mi++)
#pragma unroll
      for (int ni = 0; ni < 4; ni++)
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const bool pan = li[mi] >= 0 && lj[ni][u] >= 0 && lj[ni][u] <= li[mi] && lj[ni][u] < d.w;
          const int e = li[mi] * d.w + lj[ni][u];
          m[mi][ni][u] = !pan ? -2 : (d.ata != nullptr ? __ldg(d.pmap + FD[4] + e) : e);
        }
#pragma unroll
    for (int mi = 0; mi < 4; mi++)
#pragma unroll
      for (int ni = 0; ni < 4; ni++)
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const int gr = i * TM + wm * 32 + mi * 8 + lr, gc = j * TN + wn * 32 + ni * 8 + lc * 2 + u;
          const int mm = m[mi][ni][u];
          double x;
          if (li[mi] < 0 || lj[ni][u] < 0) x = (gr == gc) ? 1.0 : 0.0;          // identity on the padding
          else if (lj[ni][u] > li[mi] || mm == -1 || mm == -2) x = 0.0;          // above the diagonal; fill-in; border x border
          else x = d.ata != nullptr ? __ldg(d.ata + b * d.ata_stride + mm) : Pn[mm];
          if (mm != -2 && li[mi] == lj[ni][u]) x = x + (al * x + be);            // linear/utils.py:14-33: diag <- diag (1 + alpha) + beta
          acc[mi][ni][u] = x;
        }
    // the children in list order, those whose rows reach the element; a child's inverse-map entries first, then its values
    const int c_begin = (int)(FD[7] & 0xffffffffLL), nch = (int)(FD[7] >> 32);
    for (int q = 0; q < nch; q++) {
      const int64_t* PC = d.pc + (int64_t)(c_begin + q) * 6;   // (cb_off, cb_ld | b << 32, lo, hi, inv_off, u_off)
      const double* src = d.arena_child + b * d.arena_size + PC[0];
      const int ldg = (int)(PC[1] & 0xffffffffLL), lo = (int)PC[2], hi = (int)PC[3];
      const int32_t* inv = d.c_inv + PC[4];
      int ci[4], cj[4][2];
#pragma unroll
      for (int mi = 0; mi < 4; mi++) ci[mi] = (li[mi] >= lo && li[mi] <= hi) ? __ldg(inv + li[mi]) : -1;
#pragma unroll
      for (int ni = 0; ni < 4; ni++)
#pragma unroll
        for (int u = 0; u < 2; u++) cj[ni][u] = (lj[ni][u] >= lo && lj[ni][u] <= hi) ? __ldg(inv + lj[ni][u]) : -1;
#pragma unroll
      for (int mi = 0; mi < 4; mi++) {
        double x[4][2];
#pragma unroll
        for (int ni = 0; ni < 4; ni++)
#pragma unroll
          for (int u = 0; u < 2; u++)
            x[ni][u] = (ci[mi] >= 0 && cj[ni][u] >= 0 && lj[ni][u] <= li[mi]) ? __ldg(src + (int64_t)ci[mi] * ldg + cj[ni][u]) : -0.0;
#pragma unroll
        for (int ni = 0; ni < 4; ni++)
#pragma unroll
          for (int u = 0; u < 2; u++) acc[mi][ni][u] = acc[mi][ni][u] + x[ni][u];
      }
    }
    // the in-place form's read of the assembled value (no damping there: alpha, beta null)
#pragma unroll
    for (int mi = 0; mi < 4; mi++)
#pragma unroll
      for (int ni = 0; ni < 4; ni++)
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const int gr = i * TM + wm * 32 + mi * 8 + lr, gc = j * TN + wn * 32 + ni * 8 + lc * 2 + u;
          double x = acc[mi][ni][u];
          if (gr == gc) x = x + (0.0 * x + 0.0);
          acc[mi][ni][u] = -x;
        }
  } else {
    const double* Ab = p.AtA + b * p.a_bstride;
    const double al = (p.alpha != nullptr) ? p.alpha[b] : 0.0;
    const double be = (p.beta != nullptr) ? p.beta[b] : 0.0;
#pragma unroll
    for (int mi = 0; mi < 4; mi++) {
      const int64_t gr = (int64_t)i * TM + wm * 32 + mi * 8 + lr;
#pragma unroll
      for (int ni = 0; ni < 4; ni++) {
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const int64_t gc = (int64_t)j * TN + wn * 32 + ni * 8 + lc * 2 + u;
          double x;
          if (gr < p.n && gc < p.n) {
            x = Ab[gr * p.n + gc];
            if (gr == gc) x = x + (al * x + be);  // dense_solver.py:38-64 ; linear/utils.py:14-33
          } else {
            x = (gr == gc) ? 1.0 : 0.0;  // identity padding
          }
          acc[mi][ni][u] = -x;
        }
      }
    }
  }
  // dependencies: all earlier block columns of this row tile and of the row tile holding block row j are finished
  const int jdep = j < p.nb_piv ? j : p.nb_piv;   // pivot block columns this tile depends on
  if (jdep > 0) {
    if (tid == 0) {
      wait_ge(p.done + b * p.ntr + i, jdep);
      if (i != i0) wait_ge(p.done + b * p.ntr + i0, jdep);
    }
    __syncthreads();
  }

  THB_TICK(1);
  const int nk = min(jdep * (TN / KB), p.k_lim);
  const bool skip_mma = is_diag && (wm * 32 < roff);  // odd block columns: the upper 64 rows of the diagonal tile lie above the diagonal
  const double* Arow = Lb + (int64_t)i * TM * np;
  const double* Brow = Lb + (int64_t)j * TN * np;
  auto load_stage = [&](int s, int k0) {
    double* st = smem + (size_t)s * (A_TILE + B_TILE);
    if (direct) {
      load_panel_tile<TM>(st, Pn, p.d, i * TM, k0, tid);
      if (!is_diag) load_panel_tile<TN>(st + A_TILE, Pn, p.d, j * TN, k0, tid);
    } else {
      load_oper_tile<TM, KB>(st, Arow, np, k0, tid);
      if (!is_diag) load_oper_tile<TN, KB>(st + A_TILE, Brow, np, k0, tid);
    }
  };
  if (nk > 0) {
#pragma unroll
    for (int s = 0; s < STAGES - 1; s++) {
      if (s < nk) load_stage(s, s * KB);
      cp_async_commit();
    }
    for (int ks = 0; ks < nk; ks++) {
      cp_async_wait<STAGES - 2>();
      __syncthreads();
      {
        const int nx = ks + STAGES - 1;
        if (nx < nk) load_stage(nx % STAGES, nx * KB);
        cp_async_commit();
      }
      const double* As = smem + (size_t)(ks % STAGES) * (A_TILE + B_TILE);
      const double* Bs = is_diag ? (As + roff * SA) : (As + A_TILE);  // diagonal tile: the column rows are a half of its own rows
      if (skip_mma) continue;  // rows above the diagonal block: nothing to compute (the warp still loads and syncs)
#pragma unroll
      for (int k4 = 0; k4 < KB / 4; k4++) {
        double a[4], bf[4];
#pragma unroll
        for (int mi = 0; mi < 4; mi++) a[mi] = As[(wm * 32 + mi * 8 + lr) * SA + k4 * 4 + lc];
#pragma unroll
        for (int ni = 0; ni < 4; ni++) bf[ni] = Bs[(wn * 32 + ni * 8 + lr) * SA + k4 * 4 + lc];
#pragma unroll
        for (int mi = 0; mi < 4; mi++)
#pragma unroll
          for (int ni = 0; ni < 4; ni++) mma884(acc[mi][ni][0], acc[mi][ni][1], a[mi], bf[ni]);
      }
    }
    cp_async_wait<0>();
    __syncthreads();
  }

  THB_TICK(2);
  if (j >= p.nb_piv) {
    // trailing block column of a partial factorisation: the tile of the Schur complement  S = F - L L^T  goes back in place
#pragma unroll
    for (int mi = 0; mi < 4; mi++) {
      double* dst = Lb + ((int64_t)i * TM + wm * 32 + mi * 8 + lr) * np + (int64_t)j * TN + wn * 32 + lc * 2;
#pragma unroll
      for (int ni = 0; ni < 4; ni++) *reinterpret_cast<double2*>(dst + ni * 8) = make_double2(-acc[mi][ni][0], -acc[mi][ni][1]);
    }
    return;
  }
  // ---------------- phase B: C = -acc, to shared memory ----------------
  double* Cs = smem;
#pragma unroll
  for (int mi = 0; mi < 4; mi++) {
    const int r = wm * 32 + mi * 8 + lr;
#pragma unroll
    for (int ni = 0; ni < 4; ni++) {
      const int c = wn * 32 + ni * 8 + lc * 2;
      *reinterpret_cast<double2*>(&Cs[r * SC + c]) = make_double2(-acc[mi][ni][0], -acc[mi][ni][1]);
    }
  }
  __syncthreads();

  THB_TICK(3);
  double* Wj = p.W + ((int64_t)b * p.nb + j) * TN * TN;
  int* flag = p.flags + b * p.nb + j;
  int row_lo = 0;  // first tile row that still needs the TRSM of phase D

  if (is_diag) {
    // ---------------- phase C: blocked potrf + triangular inverse of the 64x64 diagonal block ----------------
    int fail;
    if (direct) {
      // L_jj to the panel (its rows and columns below w), and the zeros of the panel above the diagonal in these rows
      const int lim = min(TN, p.d.w - j * TN), c0 = (j + 1) * TN, nz = p.d.w - c0;
      fail = diag64_factor_invert(Cs + roff * SC, smem + TM * SC, Pn + ((int64_t)j * TN) * p.d.w + (int64_t)j * TN, p.d.w, lim, Wj);
      for (int e = tid; nz > 0 && e < lim * nz; e += CHOL_THREADS) {
        const int rr = e / nz, c = e - rr * nz;
        Pn[(int64_t)(j * TN + rr) * p.d.w + c0 + c] = 0.0;
      }
    } else {
      fail = diag64_factor_invert(Cs + roff * SC, smem + TM * SC, Lb + ((int64_t)j * TN) * np + (int64_t)j * TN, np, TN, Wj);
    }
    if (tid == 0 && fail != 0) record_first_failure(p.info + b, p.info_base + j * TN + fail);
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      asm volatile("st.release.gpu.global.s32 [%0], %1;\n" ::"l"(flag), "r"(1) : "memory");
    }
    row_lo = roff + 64;         // rows of this tile below the diagonal block (none when the block is the lower half)
    if (row_lo >= TM) {
      if (tid == 0) asm volatile("red.release.gpu.global.add.s32 [%0], %1;\n" ::"l"(p.done + b * p.ntr + i), "r"(1) : "memory");
      return;
    }
  } else {
    if (tid == 0) wait_ge(flag, 1);
    __syncthreads();
  }

  THB_TICK(4);
  // ---------------- phase D: L[rows,j] = C W^T (DMMA, triangular k-range) ----------------
  double* Ws = smem + TM * SC;
  double acc2[2][8][2];
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int ni = 0; ni < 8; ni++) acc2[mi][ni][0] = acc2[mi][ni][1] = 0.0;
  constexpr int NKW = TN / KB_W;  // 4
  const bool active = (warp * 16 >= row_lo);
#pragma unroll
  for (int s = 0; s < WSTAGES - 1; s++) {
    load_oper_tile<TN, KB_W>(Ws + (size_t)s * W_TILE, Wj, TN, s * KB_W, tid);
    cp_async_commit();
  }
#pragma unroll
  for (int ks = 0; ks < NKW; ks++) {
    cp_async_wait<WSTAGES - 2>();
    __syncthreads();
    {
      const int nx = ks + WSTAGES - 1;
      if (nx < NKW) load_oper_tile<TN, KB_W>(Ws + (size_t)(nx % WSTAGES) * W_TILE, Wj, TN, nx * KB_W, tid);
      cp_async_commit();
    }
    const double* Wst = Ws + (size_t)(ks % WSTAGES) * W_TILE;
    if (active) {
#pragma unroll
      for (int k4 = 0; k4 < KB_W / 4; k4++) {
        const int kk = ks * KB_W + k4 * 4;
        double a[2];
#pragma unroll
        for (int mi = 0; mi < 2; mi++) a[mi] = Cs[(warp * 16 + mi * 8 + lr) * SC + kk + lc];
#pragma unroll
        for (int ni = 0; ni < 8; ni++) {
          if (ni * 8 + 7 >= kk) {  // W[c][k] == 0 for k > c: skip column blocks entirely above this k
            const double bfr = Wst[(ni * 8 + lr) * SW + k4 * 4 + lc];
            mma884(acc2[0][ni][0], acc2[0][ni][1], a[0], bfr);
            mma884(acc2[1][ni][0], acc2[1][ni][1], a[1], bfr);
          }
        }
      }
    }
  }
  cp_async_wait<0>();
  if (active && direct) {
#pragma unroll
    for (int mi = 0; mi < 2; mi++) {
      const int pr = direct_row(p.d, i * TM + warp * 16 + mi * 8 + lr);
      if (pr < 0) continue;
      double* dst = Pn + (int64_t)pr * p.d.w;
#pragma unroll
      for (int ni = 0; ni < 8; ni++)
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const int c = j * TN + ni * 8 + lc * 2 + u;
          if (c < p.d.w) dst[c] = acc2[mi][ni][u];
        }
    }
  } else if (active) {
#pragma unroll
    for (int mi = 0; mi < 2; mi++) {
      const int r = warp * 16 + mi * 8 + lr;
      double* dst = Lb + ((int64_t)i * TM + r) * np + (int64_t)j * TN;
#pragma unroll
      for (int ni = 0; ni < 8; ni++) {
        *reinterpret_cast<double2*>(dst + ni * 8 + lc * 2) = make_double2(acc2[mi][ni][0], acc2[mi][ni][1]);
      }
    }
  }
  THB_TICK(5);
  // publish: this row tile has one more finished block column
  __threadfence();
  __syncthreads();
  if (tid == 0) asm volatile("red.release.gpu.global.add.s32 [%0], %1;\n" ::"l"(p.done + b * p.ntr + i), "r"(1) : "memory");
  THB_TICK(6);
}

// ------------------------------------------------------------------------------------------------
// Solve with the stored factor: forward  y_j = W_j (rhs_j - sum_{k<j} L[j,k] y_k),
//                               backward x_j = W_j^T (y_j - sum_{k>j} L[k,j]^T x_k),   64-row blocks.
struct SolveArgs {
  const double* L;
  const double* W;
  const double* rhs;  // [B,n]
  double* x;          // [B,n]
  int64_t B, n, np;
  int nb;
};

constexpr int SOLVE_THREADS = 256;

__global__ void __launch_bounds__(SOLVE_THREADS, 2) chol_solve_kernel(SolveArgs p) {
  extern __shared__ __align__(16) double sm[];
  double* y = sm;               // [np]
  double* tmp = sm + p.np;      // [64]
  double* part = tmp + TN;      // [8][64]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t b = blockIdx.x;
  const int64_t np = p.np;
  const double* Lb = p.L + b * np * np;
  const double* Wb = p.W + b * p.nb * TN * TN;
  for (int64_t e = tid; e < np; e += SOLVE_THREADS) y[e] = (e < p.n) ? p.rhs[b * p.n + e] : 0.0;
  __syncthreads();
  // ---- forward ----
  for (int j = 0; j < p.nb; j++) {
    const int K = j * TN;
    // each warp: 8 rows, four at a time
    for (int rr = 0; rr < 8; rr += 4) {
      const int r0 = warp * 8 + rr;
      const double* row0 = Lb + ((int64_t)K + r0) * np;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      for (int k = lane * 2; k < K; k += 64) {
        const double2 yy = *reinterpret_cast<const double2*>(y + k);
        const double2 a0 = *reinterpret_cast<const double2*>(row0 + k);
        const double2 a1 = *reinterpret_cast<const double2*>(row0 + np + k);
        const double2 a2 = *reinterpret_cast<const double2*>(row0 + 2 * np + k);
        const double2 a3 = *reinterpret_cast<const double2*>(row0 + 3 * np + k);
        s0 += a0.x * yy.x + a0.y * yy.y;
        s1 += a1.x * yy.x + a1.y * yy.y;
        s2 += a2.x * yy.x + a2.y * yy.y;
        s3 += a3.x * yy.x + a3.y * yy.y;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        s3 += __shfl_xor_sync(0xffffffffu, s3, o);
      }
      if (lane == 0) {
        tmp[r0] = y[K + r0] - s0;
        tmp[r0 + 1] = y[K + r0 + 1] - s1;
        tmp[r0 + 2] = y[K + r0 + 2] - s2;
        tmp[r0 + 3] = y[K + r0 + 3] - s3;
      }
    }
    __syncthreads();
    const double* Wj = Wb + (int64_t)j * TN * TN;
    for (int rr = 0; rr < 8; rr++) {
      const int r = warp * 8 + rr;
      const double* wr = Wj + r * TN;
      double s = 0.0;
      for (int k = lane; k <= r; k += 32) s += wr[k] * tmp[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) y[K + r] = s;
    }
    __syncthreads();
  }
  // ---- backward ----
  for (int j = p.nb - 1; j >= 0; j--) {
    const int K = j * TN;
    // part[w][c] = sum over rows r (this warp's share) of L[r][K+c] * x[r], r in [K+64, np)
    double a0 = 0.0, a1 = 0.0;
    for (int64_t r = (int64_t)K + TN + warp; r < np; r += 8) {
      const double xr = y[r];
      const double2 v = *reinterpret_cast<const double2*>(Lb + r * np + K + lane * 2);
      a0 += v.x * xr;
      a1 += v.y * xr;
    }
    part[warp * TN + lane * 2 + 0] = a0;
    part[warp * TN + lane * 2 + 1] = a1;
    __syncthreads();
    if (tid < TN) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < 8; w++) s += part[w * TN + tid];
      tmp[tid] = y[K + tid] - s;
    }
    __syncthreads();
    // x_j[c] = sum_{r>=c} W[r][c] tmp[r]
    const double* Wj = Wb + (int64_t)j * TN * TN;
    a0 = a1 = 0.0;
    for (int r = warp; r < TN; r += 8) {
      const double tr = tmp[r];
      const double2 v = *reinterpret_cast<const double2*>(Wj + r * TN + lane * 2);
      a0 += v.x * tr;
      a1 += v.y * tr;
    }
    part[warp * TN + lane * 2 + 0] = a0;
    part[warp * TN + lane * 2 + 1] = a1;
    __syncthreads();
    if (tid < TN) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < 8; w++) s += part[w * TN + tid];
      y[K + tid] = s;
    }
    __syncthreads();
  }
  for (int64_t e = tid; e < p.n; e += SOLVE_THREADS) p.x[b * p.n + e] = y[e];
}

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

struct Geometry {
  int64_t np;
  int nb, ntr;
  double* L;
  double* W;
  int* flags;
  int* done;
  int* ticket;
};
static inline Geometry geometry(void* workspace, int64_t B, int64_t n) {
  Geometry g;
  g.np = align_up(n, TM);
  g.nb = (int)(g.np / TN);
  g.L = reinterpret_cast<double*>(workspace);
  g.W = g.L + B * g.np * g.np;
  g.ntr = (int)(g.np / TM);
  g.flags = reinterpret_cast<int*>(g.W + B * g.nb * TN * TN);
  g.done = g.flags + align_up(B * g.nb, 64);
  g.ticket = g.done + align_up(B * g.ntr, 64);
  return g;
}

// Partial mode: tickets in groups of this many matrices (THB_CHOL_GROUP, read at every call; 0 or unset: the default below, which is
// clamped to B)
static inline int64_t chol_partial_group(int64_t B) {
  const char* e = getenv("THB_CHOL_GROUP");
  int64_t g = e != nullptr ? atoll(e) : 0;
  if (g <= 0) g = THB_CHOL_GROUP_DEFAULT;
  return g < B ? g : B;
}

}  // namespace thb

extern "C" {

int64_t thb_potrf_workspace_bytes(int64_t B, int64_t n) {
  if (B <= 0 || n <= 0) return 0;
  const int64_t np = thb::align_up(n, thb::TM), nb = np / thb::TN;
  int64_t bytes = B * np * np * 8;                              // L
  bytes += B * nb * thb::TN * thb::TN * 8;                      // W
  bytes += thb::align_up(B * nb, 64) * 4;                       // flags (W_j ready)
  bytes += thb::align_up(B * (np / thb::TM), 64) * 4;           // finished-column counters per row tile
  bytes += 64 * 4;                                              // tile-queue ticket counter
  return thb::align_up(bytes, 256);
}

int thb_potrf_f64(const double* AtA, const double* alpha, const double* beta, int32_t* info, int64_t B, int64_t n, void* workspace,
                  int64_t workspace_bytes, thb_stream_t stream) {
  if (B < 0 || n < 0 || AtA == nullptr || info == nullptr || workspace == nullptr) return THB_ERR_BAD_ARG;
  if (B == 0 || n == 0) return THB_OK;
  if (workspace_bytes < thb_potrf_workspace_bytes(B, n)) return THB_ERR_BAD_ARG;
  cudaStream_t cs = thb_cs(stream);
  thb::Geometry g = thb::geometry(workspace, B, n);
  THB_CUDA(cudaMemsetAsync(g.flags, 0, (size_t)(thb::align_up(B * g.nb, 64) + thb::align_up(B * g.ntr, 64) + 64) * 4, cs));  // flags, done, ticket
  THB_CUDA(cudaMemsetAsync(info, 0, (size_t)B * 4, cs));
  // CTAs: column j owns (ntr - j/2) * B
  if (g.nb > 1024) return THB_ERR_UNSUPPORTED;
  int64_t total = 0;
  for (int j = 0; j < g.nb; j++) total += (int64_t)(g.ntr - (j >> 1)) * B;
  if (total > 2147483647LL) return THB_ERR_UNSUPPORTED;
  static bool attr_set = false;
  if (!attr_set) {
    THB_CUDA(cudaFuncSetAttribute(thb::chol_col_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)thb::CHOL_SMEM));
    attr_set = true;
  }
  thb::CholArgs a;
  a.AtA = AtA; a.alpha = alpha; a.beta = beta; a.L = g.L; a.W = g.W; a.flags = g.flags; a.done = g.done; a.info = info;
  a.B = B; a.n = n; a.np = g.np; a.nb = g.nb; a.ntr = g.ntr;
  a.ticket = g.ticket; a.nb_piv = g.nb; a.a_bstride = n * n; a.l_bstride = g.np * g.np; a.info_base = 0;
  a.k_lim = g.nb * (thb::TN / thb::KB); a.n_real = (int)g.np;
  a.group = (int)B; a.d = ThbCholDirect{};   // the whole batch is one group
  // ONE launch for the whole factorisation: block columns are chained through the per-tile counters, so there are
  // no per-column launch gaps and no per-column wave-quantisation tails.
  thb::chol_col_kernel<<<(unsigned)total, thb::CHOL_THREADS, thb::CHOL_SMEM, cs>>>(a);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

int thb_potrs_f64(const double* rhs, double* x, int64_t B, int64_t n, const void* workspace, int64_t workspace_bytes,
                  thb_stream_t stream) {
  if (B < 0 || n < 0 || rhs == nullptr || x == nullptr || workspace == nullptr) return THB_ERR_BAD_ARG;
  if (B == 0 || n == 0) return THB_OK;
  if (workspace_bytes < thb_potrf_workspace_bytes(B, n)) return THB_ERR_BAD_ARG;
  thb::Geometry g = thb::geometry(const_cast<void*>(workspace), B, n);
  thb::SolveArgs s;
  s.L = g.L; s.W = g.W; s.rhs = rhs; s.x = x; s.B = B; s.n = n; s.np = g.np; s.nb = g.nb;
  const size_t ssm = (size_t)(g.np + thb::TN + 8 * thb::TN) * 8;
  static size_t solve_smem_set = 0;
  if (ssm > 48 * 1024 && ssm > solve_smem_set) {
    THB_CUDA(cudaFuncSetAttribute(thb::chol_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssm));
    solve_smem_set = ssm;
  }
  thb::chol_solve_kernel<<<(unsigned)B, thb::SOLVE_THREADS, ssm, thb_cs(stream)>>>(s);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

/* Partial in-place factorisation of B frontal matrices (multifrontal block-sparse Cholesky, thb_front.cu): F_b = F + b * bstride is an
 * np x np row-major matrix (np a multiple of 128; lower part + diagonal tiles read).  The first nb_piv 64-wide block columns are
 * factored (L in place, zeros above the diagonal of the diagonal blocks), the trailing (np - 64 nb_piv)^2 block becomes the Schur
 * complement F22 - L21 L21^T in place.  w_real (> 0): number of real pivot columns -- the identity padding of the last pivot block column is
 * skipped by the k loops; n_real (> 0): rows / columns from n_real on are padding -- trailing tiles entirely there are skipped.
 * info[b] (NOT cleared here) receives info_base + 1 + index of the first non-positive pivot. */
int64_t thb_potrf_partial_workspace_bytes(int64_t B, int64_t np) {
  if (B <= 0 || np <= 0) return 0;
  const int64_t nb = np / thb::TN;
  int64_t bytes = B * nb * thb::TN * thb::TN * 8;               // W
  bytes += thb::align_up(B * nb, 64) * 4 + thb::align_up(B * (np / thb::TM), 64) * 4 + 64 * 4;
  return thb::align_up(bytes, 256);
}

static int potrf_partial(double* F, int64_t bstride, int64_t np, int32_t nb_piv, int32_t w_real, int32_t n_real, int32_t info_base,
                         int32_t* info, int64_t B, void* workspace, int64_t workspace_bytes, const ThbCholDirect* direct, thb_stream_t stream) {
  if (B < 0 || np <= 0 || np % thb::TM != 0 || F == nullptr || info == nullptr || workspace == nullptr) return THB_ERR_BAD_ARG;
  if (B == 0) return THB_OK;
  if (workspace_bytes < thb_potrf_partial_workspace_bytes(B, np)) return THB_ERR_BAD_ARG;
  const int nb = (int)(np / thb::TN), ntr = (int)(np / thb::TM);
  if (nb_piv < 0 || nb_piv > nb || nb > 1024) return THB_ERR_BAD_ARG;
  cudaStream_t cs = thb_cs(stream);
  double* W = reinterpret_cast<double*>(workspace);
  int* flags = reinterpret_cast<int*>(W + B * nb * thb::TN * thb::TN);
  int* done = flags + thb::align_up(B * nb, 64);
  int* ticket = done + thb::align_up(B * ntr, 64);
  THB_CUDA(cudaMemsetAsync(flags, 0, (size_t)(thb::align_up(B * nb, 64) + thb::align_up(B * ntr, 64) + 64) * 4, cs));
  int64_t total = 0;
  for (int j = 0; j < nb; j++) total += (int64_t)(ntr - (j >> 1)) * B;
  if (total > 2147483647LL) return THB_ERR_UNSUPPORTED;
  static bool attr_set = false;
  if (!attr_set) {
    THB_CUDA(cudaFuncSetAttribute(thb::chol_col_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)thb::CHOL_SMEM));
    attr_set = true;
  }
  thb::CholArgs a;
  a.AtA = F; a.alpha = nullptr; a.beta = nullptr; a.L = F; a.W = W; a.flags = flags; a.done = done; a.info = info;
  a.B = B; a.n = np; a.np = np; a.nb = nb; a.ntr = ntr;
  a.ticket = ticket; a.nb_piv = nb_piv; a.a_bstride = bstride; a.l_bstride = bstride; a.info_base = info_base;
  a.k_lim = (w_real > 0 && nb_piv < nb) ? (w_real + thb::KB - 1) / thb::KB : nb * (thb::TN / thb::KB);
  a.n_real = (n_real > 0 && n_real <= np) ? n_real : (int)np;
  a.group = (int)thb::chol_partial_group(B);
  a.d = direct != nullptr ? *direct : ThbCholDirect{};
  thb::chol_col_kernel<<<(unsigned)total, thb::CHOL_THREADS, thb::CHOL_SMEM, cs>>>(a);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

/* Partial in-place factorisation of B frontal matrices (multifrontal block-sparse Cholesky, thb_front.cu): F_b = F + b * bstride is an
 * np x np row-major matrix (np a multiple of 128; lower part + diagonal tiles read).  The first nb_piv 64-wide block columns are
 * factored (L in place, zeros above the diagonal of the diagonal blocks), the trailing (np - 64 nb_piv)^2 block becomes the Schur
 * complement F22 - L21 L21^T in place.  w_real (> 0): number of real pivot columns -- the identity padding of the last pivot block column is
 * skipped by the k loops; n_real (> 0): rows / columns from n_real on are padding -- trailing tiles entirely there are skipped.
 * info[b] (NOT cleared here) receives info_base + 1 + index of the first non-positive pivot. */
int thb_potrf_partial_inplace_f64(double* F, int64_t bstride, int64_t np, int32_t nb_piv, int32_t w_real, int32_t n_real, int32_t info_base,
                                  int32_t* info, int64_t B, void* workspace, int64_t workspace_bytes, thb_stream_t stream) {
  return potrf_partial(F, bstride, np, nb_piv, w_real, n_real, info_base, info, B, workspace, workspace_bytes, nullptr, stream);
}

/* The same factorisation of a big front of the multifrontal factor without the assembled matrix: its tiles are gathered from AtA and the
 * children's update matrices (direct->fd), the pivot columns' L goes to the front's panel (row-major (w + b) x w in the factor storage,
 * zeros above the diagonal) and is read back from there; only the trailing block -- the update matrix -- is written to F. */
int thb_potrf_partial_direct_f64(double* F, int64_t bstride, int64_t np, int32_t nb_piv, int32_t n_real, int32_t info_base, int32_t* info,
                                 int64_t B, void* workspace, int64_t workspace_bytes, const ThbCholDirect* direct, thb_stream_t stream) {
  if (direct == nullptr || direct->fd == nullptr || direct->w <= 0 || direct->wpad != nb_piv * thb::TN) return THB_ERR_BAD_ARG;
  return potrf_partial(F, bstride, np, nb_piv, direct->w, n_real, info_base, info, B, workspace, workspace_bytes, direct, stream);
}

#ifdef THB_CHOL_TIMING
int thb_debug_chol_timing(long long* host_out, int64_t count) {
  return (int)cudaMemcpyFromSymbol(host_out, thb::thb_chol_timing, sizeof(long long) * count);
}
#endif

int thb_potrf_potrs_f64(const double* AtA, const double* rhs, const double* alpha, const double* beta, double* x, int32_t* info,
                        int64_t B, int64_t n, void* workspace, int64_t workspace_bytes, thb_stream_t stream) {
  if (rhs == nullptr || x == nullptr) return THB_ERR_BAD_ARG;
  int rc = thb_potrf_f64(AtA, alpha, beta, info, B, n, workspace, workspace_bytes, stream);
  if (rc != THB_OK) return rc;
  return thb_potrs_f64(rhs, x, B, n, workspace, workspace_bytes, stream);
}

}  // extern "C"
