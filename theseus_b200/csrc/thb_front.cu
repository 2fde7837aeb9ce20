// Multifrontal (supernodal) batched block-sparse Cholesky, fp64, sm_90a -- numeric phase of layout "front".
//
// Replaces BaSpaCho's batched factor / solve behind NumericDecomposition::factor / solve
// (theseus/extlib/baspacho_solver_cuda.cu:203-214, 282-287) for B problems that share ONE structure.  Symbolic side:
// theseus_b200/frontal.py (fronts, depth schedule, relative maps); data layout: include/thb200.h (thb_front_plan).
//
// A front t is a dense symmetric matrix  F_t = [[D, .], [P, C]]  (w pivots, b border rows).  Per depth, deepest first:
//   assemble   F_t = panel of AtA entries (+ LM damping on the diagonal) + sum over children c of  extend-add(C_c)
//   factor     D = L L^T,  P <- P L^-T,  C <- C - P P^T       (C_t goes to the parent through the update-matrix arena)
// Small fronts (r <= 160): ONE CTA per (front, item), the whole front in shared memory: scatter-add of the children, scalar
//   right-looking pivots on the r x w panel, the rank-w update of C on the FP64 tensor pipe (mma.sync m8n8k4 DMMA, 16x16 macro
//   tiles per warp) -- every byte of a small front is read once and written once.
// Big fronts: the DMMA dense kernel of thb_chol_dense.cu in partial mode (left-looking tiles: the Schur complement is accumulated in
//   registers over all pivot columns and written once), each tile gathered from AtA and the children (in a fixed order), L stored
//   straight into the panel in the factor storage.
// Substitutions: per front one CTA per item, chunked by 32 pivot columns: a 32 x 32 triangular block is solved by one warp with
//   shuffles, the rest of the panel is a row-contiguous mat-vec; the forward pass hands border vectors to the parent through a
//   second ping-pong arena, the backward pass gathers the ancestors' solution.  The permutation is folded into the first load /
//   last store.  No atomics on data anywhere: bitwise reproducible, independent of B.
#include <stdlib.h>

#include "thb_common.cuh"

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

// Programmatic dependent launch (sm_90+): a kernel launched with the attribute may start while its predecessor in the stream drains;
// its CTAs run their prologue (plan descriptors, inverse maps, zero fill -- nothing the predecessor writes) and then wait for the
// predecessor's completion (griddepcontrol.wait, which also orders its memory) before the first dependent read or any global write.
// ~300 launches per linear solve of 10-200 us each: the launch gap, the tail of the last wave and the prologue are what this was meant to
// hide.  It made the substitutions slower (early CTAs sit on the SMs' thread slots while they wait), so the attribute is only set
// with THB_FRONT_PDL=1; without it the two instructions are no-ops.
#ifdef THB_SIMT_EMU
#define THB_PDL_TRIGGER() do { } while (0)
#define THB_PDL_WAIT() do { } while (0)
#define FRONT_LAUNCH(K, grid, block, smem, cs, arg) K<<<grid, block, smem, cs>>>(arg)
#else
#define THB_PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")
#define THB_PDL_WAIT() asm volatile("griddepcontrol.wait;" ::: "memory")
#define FRONT_LAUNCH(K, grid, block, smem, cs, arg) thb::front_launch_pdl(K, grid, block, smem, cs, arg)
static inline bool front_pdl_enabled() {
  static const bool on = [] { const char* e = getenv("THB_FRONT_PDL"); return e != nullptr && e[0] == '1'; }();   // opt-in: slower substitutions (see above)
  return on;
}
template <typename A>
static inline void front_launch_pdl(void (*kernel)(A), dim3 grid, dim3 block, size_t smem, cudaStream_t cs, const A& arg) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = cs;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = front_pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, arg);   // errors surface through THB_CHECK_LAUNCH (cudaGetLastError) at the call site
}
#endif

#ifdef THB_SIMT_EMU
// host emulation (tests/simt): the m8n8k4 fragment semantics with shuffles
__device__ inline void front_mma884(double& c0, double& c1, double a, double b) {
  const int lane = threadIdx.x & 31, lr = lane >> 2, lc = lane & 3;
  for (int k = 0; k < 4; k++) {
    const double av = __shfl_sync(0xffffffffu, a, lr * 4 + k);
    const double b0 = __shfl_sync(0xffffffffu, b, (2 * lc) * 4 + k);
    const double b1 = __shfl_sync(0xffffffffu, b, (2 * lc + 1) * 4 + k);
    c0 += av * b0;
    c1 += av * b1;
  }
}
#else
__device__ __forceinline__ void front_mma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
#endif

// smallest v >= x with v % 16 == 4: row stride (doubles) with conflict-free DMMA fragment loads / accumulator stores
__host__ __device__ __forceinline__ int front_pad_ld(int x) { return ((x + 11) / 16) * 16 + 4; }

struct FrontArgs {
  thb_front_plan p;
  int s0;                   // first entry of this launch in p.sched
  int64_t B;
  double* factor;           // [B, data_size]
  const double* alpha;      // [B] or null
  const double* beta;       // [B] or null
  double* arena_cur;        // [B, arena_size] of this depth's parity
  const double* arena_child;
  int32_t* info;
  int prefetch;             // ask L2 for the children's update matrices at kernel start (THB_FRONT_PREFETCH=1; off by default: slower on H100)
  const double* ata;        // [B, ata_stride] compact AtA blocks (thb_gram_f64 with the plan's compact offsets), or null: the panels
  int64_t ata_stride;       //   in `factor` already hold AtA (zero-filled + scattered by the caller: the extlib-style flow)
  const double* rhs;        // [B, n] original order, or null: factor only.  Else the forward substitution of every front runs on its
  double* work;             //   panel while it is still in shared memory: y of the pivots -> work [B, n] (permuted order),
  double* v_cur;            //   the border vector -> v_cur (this depth's parity of the border-vector arena),
  const double* v_child;    //   the children's border vectors <- v_child (the other parity)
};

// AtA entry of panel element e of the front whose panel starts at `poff`: through the plan's panel map when the compact block storage
// is given (pmap[poff + e] = offset in one item's `ata`, or -1 = fill-in), else from the pre-filled panel itself
__device__ __forceinline__ double front_panel_in(const FrontArgs& a, const double* Lg, int64_t poff, int64_t item, int64_t e) {
  if (a.ata == nullptr) return Lg[e];
  const int32_t m = a.p.pmap[poff + e];
  return m >= 0 ? a.ata[item * a.ata_stride + m] : 0.0;
}

// Load through the global read-only path.  The gathers read the children's update matrices (the other depth parity of the arena, only
// read during a launch), AtA and the plan's maps through pointers held in shared memory or computed per element; as generic loads each
// one was consumed before the next was issued.
template <typename T>
__device__ __forceinline__ T front_ldg(const T* p) {
#ifdef THB_SIMT_EMU
  return *p;
#else
  return __ldg(p);
#endif
}

// The gathers below issue the loads of several children before the first add: a child that does not reach an element contributes
// -0.0, which is the exact identity of the addition (v + -0.0 == v for every v, -0.0 included), so each sum is bitwise the one of
// adding only the children that reach the element, in list order.

// ------------------------------------------------------------------------------------------------ fronts in shared memory
// One CTA per (front, item).  Shared memory holds ONLY the panel: PN [w8 + b16 + 8][ldp] = pivot rows, identity padding up to w8 = w
// rounded to 8, the border rows from row w8 on (b16 = b rounded to 16, zero padding), and Wd [8][20] = the inverse of the current
// 8 x 8 diagonal block.  The update matrix never exists on chip.
//   1. panel <- AtA entries (+ damping) + GATHERED children: element (i, j) adds child c's update-matrix entry (inv_c[i], inv_c[j])
//      where inv_c maps this front's rows to the child's border rows (-1: none).  No scatter, no barrier between children, every
//      load independent (the latency of all of them overlaps); the children are added in list order: deterministic.
//   2. blocked LEFT-LOOKING factorisation over 8-column blocks: warp 0 forms the diagonal block (DMMA), factors and inverts it in
//      registers (shuffles); every warp then finishes 16-row tiles of that block column: X = A - sum_k L_ik L_jk^T, L_ij = X W^T,
//      both products on the FP64 tensor pipe -- pivot rows and border rows alike.
//   3. update matrix: per 16 x 16 tile of the lower triangle, -P_I P_J^T by DMMA straight from the panel, plus the gathered children,
//      written once from registers.
constexpr int FRONT_WD_LD = 20;
#ifndef FRONT_PL
#define FRONT_PL 4   // panel elements a thread gathers per pass (their global loads are in flight together)
#endif
constexpr int FRONT_MAX_CHILDREN = 8;   // fronts with more children are assembled by the scatter kernel of the dense path (frontal.py)

__host__ __device__ __forceinline__ int64_t front_smem_doubles(int w, int b, int nchildren) {
  const int b16 = (b + 15) & ~15, w8 = (w + 7) & ~7;
  return (int64_t)(w8 + b16 + 8) * front_pad_ld(w8) + 8 * FRONT_WD_LD + 3 * FRONT_MAX_CHILDREN     // + children descriptors
         + ((int64_t)nchildren * (w + b) + 1) / 2 + 2;                                           // + int32 inverse maps
}

// One warp: Cholesky of the 8 x 8 block at T (row stride ld; lower part read, L written in place) and its inverse (full 8 x 8, zeros
// above the diagonal) to Wd (row stride FRONT_WD_LD).  One row / one column per lane (lanes >= 8 shadow lane 0), pivots and
// multipliers exchanged with shuffles.  Returns 0 or 1 + index of the first non-positive pivot.
__device__ __forceinline__ int front_leaf8(double* __restrict__ T, int ld, double* __restrict__ Wd, int lane) {
  const int ln = lane < 8 ? lane : 0;
  double row[8];
#pragma unroll
  for (int q = 0; q < 8; q++) row[q] = T[ln * ld + q];
  int fail = 0;
  double invd = 0.0;
#pragma unroll
  for (int c = 0; c < 8; c++) {
    const double d = __shfl_sync(0xffffffffu, row[c], c);
    if (!(d > 0.0) && fail == 0) fail = c + 1;
    double inv = rsqrt(d);
    inv = inv * (1.5 - 0.5 * d * inv * inv);   // one Newton step on the hardware seed; sqrt(d) = d * rsqrt(d)
    const double sq = d * inv;
    if (lane == c) invd = inv;
    const double lrc = (lane == c) ? sq : row[c] * inv;
    row[c] = lrc;
#pragma unroll
    for (int q = c + 1; q < 8; q++) {
      const double lqc = __shfl_sync(0xffffffffu, lrc, q);
      row[q] -= lrc * lqc;
    }
  }
  if (lane < 8) {
#pragma unroll
    for (int q = 0; q < 8; q++)
      if (q <= lane) T[lane * ld + q] = row[q];
  }
  double x[8];
#pragma unroll
  for (int rr = 0; rr < 8; rr++) {
    double sacc = (lane == rr) ? 1.0 : 0.0;
#pragma unroll
    for (int k = 0; k < rr; k++) {
      const double lrk = __shfl_sync(0xffffffffu, row[k], rr);
      sacc -= lrk * x[k];
    }
    x[rr] = sacc * __shfl_sync(0xffffffffu, invd, rr);
  }
  if (lane < 8) {
#pragma unroll
    for (int rr = 0; rr < 8; rr++) Wd[rr * FRONT_WD_LD + lane] = (rr >= lane) ? x[rr] : 0.0;
  }
  return fail;
}

// Warp: the 8 x 8 diagonal block jb of the panel  D <- D - L_j L_j^T (DMMA over the columns already factored), then its Cholesky factor
// in place and its inverse to Wd (front_leaf8); a non-positive pivot inside the real columns is recorded once per item.
__device__ __forceinline__ void front_diag_block(double* PN, int ldp, int jb, double* Wd, int lane, int w, int first, int32_t* info) {
  const int lr = lane >> 2, lc = lane & 3;
  double c0 = 0.0, c1 = 0.0;
  const double* Arow = PN + (8 * jb + lr) * ldp + lc;
  for (int k = 0; k < 8 * jb; k += 4) {
    const double av = Arow[k];
    front_mma884(c0, c1, av, av);   // the column operand is the same 8 rows
  }
  double* d = PN + (8 * jb + lr) * ldp + 8 * jb + 2 * lc;
  d[0] -= c0;
  d[1] -= c1;
  __syncwarp();
  const int fail = front_leaf8(PN + (8 * jb) * ldp + 8 * jb, ldp, Wd, lane);
  if (lane == 0 && fail != 0 && 8 * jb + fail <= w) record_first_failure(info, first + 8 * jb + fail);
}

// Warp: block column jb of the row tiles rt0 (and rt0 + 1 when TWO):  X = A - sum_k L_tile,k L_jb,k^T,  L = X W_jb^T, in place.
template <bool TWO>
__device__ __forceinline__ void front_tile_column(double* PN, int ldp, int jb, int rt0, const double* Wd, int lane) {
  const int lr = lane >> 2, lc = lane & 3;
  double x00 = 0.0, x01 = 0.0, x10 = 0.0, x11 = 0.0;
  const double* A0 = PN + (8 * rt0 + lr) * ldp + lc;
  const double* Bj = PN + (8 * jb + lr) * ldp + lc;
  for (int k = 0; k < 8 * jb; k += 4) {
    const double bf = Bj[k];
    front_mma884(x00, x01, A0[k], bf);
    if (TWO) front_mma884(x10, x11, A0[8 * ldp + k], bf);
  }
  double* X0 = PN + (8 * rt0 + lr) * ldp + 8 * jb + 2 * lc;
  X0[0] -= x00; X0[1] -= x01;
  if (TWO) { X0[8 * ldp] -= x10; X0[8 * ldp + 1] -= x11; }
  __syncwarp();
  x00 = x01 = x10 = x11 = 0.0;
#pragma unroll
  for (int k = 0; k < 8; k += 4) {
    const double bf = Wd[lr * FRONT_WD_LD + k + lc];   // B[k][n] = Winv[n][k]
    front_mma884(x00, x01, A0[8 * jb + k], bf);
    if (TWO) front_mma884(x10, x11, A0[8 * ldp + 8 * jb + k], bf);
  }
  __syncwarp();
  X0[0] = x00; X0[1] = x01;
  if (TWO) { X0[8 * ldp] = x10; X0[8 * ldp + 1] = x11; }
}

struct FrontChild {       // one child of the front this CTA works on (shared memory, <= FRONT_MAX_CHILDREN)
  const double* src;      // its update matrix for this item
  int ldg, lo, hi, uoff;  // leading dimension; range [lo, hi] of this front's rows the child reaches; its border vector's offset (f_u_off)
};

// Panel assembly: children q and q + 1 (those below nch) at the FRONT_PL panel elements (ii[u], jj[u]) (ii[u] < 0: none) -> x[c][u],
// all loads issued before any is used
__device__ __forceinline__ void front_panel_gather2(const FrontChild* ch, const int32_t* INV, int r, int nch, int q, const int* ii,
                                                    const int* jj, double (&x)[2][FRONT_PL]) {
#pragma unroll
  for (int c = 0; c < 2; c++) {
    int lo = r, hi = -1, ldg = 0;   // lo = r: nothing passes the range test below
    const double* src = nullptr;
    if (q + c < nch) { lo = ch[q + c].lo; hi = ch[q + c].hi; ldg = ch[q + c].ldg; src = ch[q + c].src; }
    const int32_t* inv = INV + (q + c) * r;
#pragma unroll
    for (int u = 0; u < FRONT_PL; u++) {
      x[c][u] = -0.0;
      if (ii[u] >= lo && jj[u] <= hi) {
        const int ci = inv[ii[u]], cj = inv[jj[u]];
        if (ci >= 0 && cj >= 0) x[c][u] = front_ldg(src + (int64_t)ci * ldg + cj);
      }
    }
  }
}

// Index of the lowest set bit of mask (mask != 0), which is cleared
__device__ __forceinline__ int front_next_child(unsigned& mask) {
#ifdef THB_SIMT_EMU
  const int q = __builtin_ctz(mask);
#else
  const int q = __ffs(mask) - 1;
#endif
  mask &= mask - 1;
  return q;
}

// Update-matrix tile: this lane's entries (rows li0, li0 + 8 and columns lj0 + {0, 1, 8, 9}, front-local) of child c, whose inverse map
// is inv -> x, issued together
__device__ __forceinline__ void front_tile_gather(const FrontChild& c, const int32_t* inv, int r, int li0, int lj0, double (&x)[2][2][2]) {
  int ci[2], cj[2][2];
#pragma unroll
  for (int mi = 0; mi < 2; mi++) ci[mi] = (li0 + 8 * mi < r) ? inv[li0 + 8 * mi] : -1;
#pragma unroll
  for (int ni = 0; ni < 2; ni++)
#pragma unroll
    for (int u = 0; u < 2; u++) cj[ni][u] = (lj0 + 8 * ni + u < r) ? inv[lj0 + 8 * ni + u] : -1;
#pragma unroll
  for (int mi = 0; mi < 2; mi++)
#pragma unroll
    for (int ni = 0; ni < 2; ni++)
#pragma unroll
      for (int u = 0; u < 2; u++)
        x[mi][ni][u] = (ci[mi] >= 0 && cj[ni][u] >= 0 && cj[ni][u] <= ci[mi]) ? front_ldg(c.src + (int64_t)ci[mi] * c.ldg + cj[ni][u]) : -0.0;
}

// ------------------------------------------------------------------------------------------------ forward elimination of one front
// One warp: solve T y = u (lower triangular cw x cw, row stride ld) -- lane i owns u_i
__device__ __forceinline__ double front_warp_trsv_lower(const double* T, int ld, double ui, int cw, int lane) {
  const double rd = lane < cw ? 1.0 / T[lane * ld + lane] : 0.0;
  for (int k = 0; k < cw; k++) {
    const double yk = __shfl_sync(0xffffffffu, ui * rd, k);
    if (lane == k) ui = yk;
    else if (lane > k && lane < cw) ui -= T[lane * ld + k] * yk;
  }
  return ui;
}

// Rows of L as the substitution kernel reads them: the factor in global memory (row-major, stride w), each 32 x 32 diagonal block
// staged in T [32][33] before its triangular solve
struct FrontRowsGlobal {
  static constexpr bool kInPanel = false;
  const double* L;
  int w;
  double* T;
  __device__ __forceinline__ const double* row(int i) const { return L + (int64_t)i * w; }
  __device__ __forceinline__ const double* diag(int k0, int cw, int tid, int nthreads, int* ld) const {
    for (int e = tid; e < cw * cw; e += nthreads) {
      const int i = e / cw, j = e - i * cw;
      T[i * 33 + j] = L[(int64_t)(k0 + i) * w + k0 + j];
    }
    *ld = 33;
    return T;
  }
};
// ... and as the factor kernel reads them: in place in its shared-memory panel (row stride ldp, border rows shifted by w8 - w)
struct FrontRowsPanel {
  static constexpr bool kInPanel = true;
  const double* PN;
  int ldp, w, shift;
  __device__ __forceinline__ const double* row(int i) const { return PN + (i < w ? i : i + shift) * ldp; }
  __device__ __forceinline__ const double* diag(int k0, int, int, int, int* ld) const {
    *ld = ldp;
    return PN + k0 * ldp + k0;
  }
};

// Barrier over the GROUP threads that run front_forward_elim: the whole CTA, or -- a group of warps that works beside the rest of the
// CTA -- named barrier 1 (the host emulation has no named barriers and only runs the whole-CTA form)
template <int GROUP, bool WHOLE_CTA>
__device__ __forceinline__ void front_group_sync() {
#ifdef THB_SIMT_EMU
  static_assert(WHOLE_CTA, "the host emulation has no named barriers");
  __syncthreads();
#else
  if constexpr (WHOLE_CTA) __syncthreads();
  else asm volatile("bar.sync 1, %0;" ::"n"(GROUP) : "memory");
#endif
}

// GROUP threads (tid = 0 .. GROUP - 1: a whole CTA, or its first GROUP / 32 warps): u <- L^-1 u over the w pivot columns of a front of r
// rows, 32 columns at a time (u[i] at u[i * us]): a one-warp triangular solve on the chunk's diagonal block, then one row per thread for
// the rows below it.  The border part of u ends as u_b - P y.  Both the substitution kernel and the fused factor kernel run this same
// code (each row's sum in the same order, k ascending, whichever thread owns it), so their y and border vectors are bitwise equal.
template <int GROUP, bool WHOLE_CTA, typename Rows>
__device__ __forceinline__ void front_forward_elim(const Rows& R, double* u, int us, int w, int r, int tid, int lane) {
  for (int k0 = 0; k0 < w; k0 += 32) {
    const int cw = min(32, w - k0);
    int ld;
    const double* T = R.diag(k0, cw, tid, GROUP, &ld);
    front_group_sync<GROUP, WHOLE_CTA>();
    if (tid < 32) {
      const double ui = front_warp_trsv_lower(T, ld, lane < cw ? u[(k0 + lane) * us] : 0.0, cw, lane);
      if (lane < cw) u[(k0 + lane) * us] = ui;
    }
    front_group_sync<GROUP, WHOLE_CTA>();
    // rows below the chunk, one row per thread (from global memory: its 32 consecutive doubles are two cache lines, read once from DRAM)
    for (int i = k0 + cw + tid; i < r; i += GROUP) {
      const double* row = R.row(i) + k0;
      double s = 0.0;
      if constexpr (Rows::kInPanel) {
        // consecutive lanes own consecutive panel rows, whose stride is 4 mod 16 doubles: at equal k, lanes l, l + 4, l + 8, l + 12 of a
        // half-warp would hit the same banks.  Each of them runs its (unchanged, k ascending) sum one step later than the previous one.
        const int skew = (lane >> 2) & 3;
#pragma unroll 2   // the factor kernel's 64 registers: a deeper unroll spills
        for (int kk = 0; kk < cw + 3; kk++) {
          const int k = kk - skew;
          if ((unsigned)k < (unsigned)cw) s += row[k] * u[(k0 + k) * us];
        }
      } else {
        for (int k = 0; k < cw; k++) s += row[k] * u[(k0 + k) * us];
      }
      u[i * us] -= s;
    }
    front_group_sync<GROUP, WHOLE_CTA>();
  }
}

// Threads tid = 0 .. nthreads - 1: the factored panel (zeros above the diagonal of the pivot block) goes to the factor storage
__device__ __forceinline__ void front_store_panel(double* __restrict__ Lg, const double* __restrict__ PN, int ldp, int w, int w8, int r, int tid,
                                                  int nthreads) {
  int i = tid / w, j = tid - i * w;
  const int di = nthreads / w, dj = nthreads - di * w;
  for (int e = tid; e < r * w; e += nthreads) {
    Lg[e] = (j > i) ? 0.0 : PN[(i < w ? i : i + (w8 - w)) * ldp + j];
    i += di; j += dj;
    if (j >= w) { j -= w; i++; }
  }
}

// Threads tid = 0 .. nthreads - 1, after front_forward_elim on u = U[i * ldp]: y of the pivots -> work, the border vector -> the parent
__device__ __forceinline__ void front_store_forward(const FrontArgs& a, const double* U, int ldp, int64_t item, int t, int f_first, int w, int b,
                                                    int tid, int nthreads) {
  for (int i = tid; i < w; i += nthreads) a.work[item * a.p.n + f_first + i] = U[i * ldp];
  double* ub = a.v_cur + item * a.p.varena_size + a.p.f_u_off[t];
  for (int i = tid; i < b; i += nthreads) ub[i] = U[(w + i) * ldp];
}

// Warps of a front_small_kernel CTA that run the forward substitution while the others write the panel and form update-matrix tiles:
// four, or half the CTA in the 64- and 128-thread instances
__host__ __device__ constexpr int front_elim_warps(int threads) { return threads >= 256 ? 4 : threads / 64; }

// Registers are capped at 64 per thread (1 024 threads per SM): the kernel is bound by the latency chain of a CTA, so resident warps count.
template <int THREADS>
__global__ void __launch_bounds__(THREADS, 1024 / THREADS) front_small_kernel(FrontArgs a) {
  extern __shared__ double sm[];
  const thb_front_plan& p = a.p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = THREADS / 32;
  const int lr = lane >> 2, lc = lane & 3;
  const int64_t item = blockIdx.x;
  // flat descriptors (frontal.py): one record per front in LAUNCH order, one per (parent, child) pair in the parent's child order --
  // two dependent loads from kernel start to the first data load instead of five through the per-field arrays
  THB_PDL_TRIGGER();
  const int64_t* FD = p.fd + (int64_t)(a.s0 + blockIdx.y) * 8;
  const int t = (int)FD[0];
  const int w = (int)FD[1], b = (int)FD[2], r = w + b;
  const int f_first = (int)FD[3];
  const int64_t f_panel_off = FD[4];
  const int c_begin = (int)(FD[7] & 0xffffffffLL);
  const int nch = min((int)(FD[7] >> 32), FRONT_MAX_CHILDREN);
  const int b16 = (b + 15) & ~15, w8 = (w + 7) & ~7;
  const int ldp = front_pad_ld(w8);
  const int prow = w8 + b16 + 8;
  double* PN = sm;                          // [prow][ldp]
  double* Wd = PN + prow * ldp;             // [8][FRONT_WD_LD]
  FrontChild* ch = reinterpret_cast<FrontChild*>(Wd + 8 * FRONT_WD_LD);               // [FRONT_MAX_CHILDREN] (24 bytes each)
  int32_t* INV = reinterpret_cast<int32_t*>(Wd + 8 * FRONT_WD_LD + 3 * FRONT_MAX_CHILDREN);   // [nch][r] front row -> child row / -1
  // ---- children descriptors and inverse maps go to shared memory (one round trip, then every lookup is on chip): thread q reads child
  // q's record, every thread the inverse-map offsets of all children, then its entries of all the maps -- no load waits for another
  // child's ----
  if (tid < nch) {
    const int64_t* PC = p.pc + (int64_t)(c_begin + tid) * 6;   // (cb_off, cb_ld, lo, hi, inv_off, u_off) of this child
    ch[tid].src = a.arena_child + item * p.arena_size + PC[0];
    ch[tid].ldg = (int)(PC[1] & 0xffffffffLL);
    ch[tid].lo = (int)PC[2];
    ch[tid].hi = (int)PC[3];
    ch[tid].uoff = (int)PC[5];
  }
  {
    int64_t ioff[FRONT_MAX_CHILDREN];
#pragma unroll
    for (int q = 0; q < FRONT_MAX_CHILDREN; q++) ioff[q] = q < nch ? p.pc[(int64_t)(c_begin + q) * 6 + 4] : 0;
    for (int l = tid; l < r; l += THREADS) {
      int32_t iv[FRONT_MAX_CHILDREN];
#pragma unroll
      for (int q = 0; q < FRONT_MAX_CHILDREN; q++) iv[q] = q < nch ? front_ldg(p.c_inv + ioff[q] + l) : 0;
#pragma unroll
      for (int q = 0; q < FRONT_MAX_CHILDREN; q++)
        if (q < nch) INV[q * r + l] = iv[q];
    }
  }
  for (int e = tid; e < prow * ldp; e += THREADS) sm[e] = 0.0;
  int* next_tile = reinterpret_cast<int*>(Wd + 8);   // update-matrix tile counter, in a column of Wd's row padding that nothing else uses
  if (tid == 0) *next_tile = 0;
  THB_PDL_WAIT();   // everything above reads the plan only; below: the children's update matrices, AtA, and every global write
#ifndef THB_SIMT_EMU
  // forward substitution: the right-hand side of the pivots (through the permutation) and the children's border vectors are read once
  // the panel is assembled; ask L2 for them now (measured on H100: the fused substitution costs ~2 ms less per solve of C5 at batch 2048)
  if (a.rhs != nullptr) {
    for (int i = tid; i < w; i += THREADS) asm volatile("prefetch.global.L2 [%0];\n" ::"l"(a.rhs + item * p.n + p.perm[f_first + i]));
    for (int q = 0; q < nch; q++) {
      const int64_t* PC = p.pc + (int64_t)(c_begin + q) * 6;
      const double* cu = a.v_child + item * p.varena_size + PC[5];
      for (int off = tid * 16; off < (int)(PC[1] >> 32); off += THREADS * 16) asm volatile("prefetch.global.L2 [%0];\n" ::"l"(cu + off));
    }
  }
  // the children's update matrices (lower triangles) are read element by element by the gathers below: ask L2 for their lines now, so that
  // the gathers find them on chip (fire and forget: no register, no stall; opt-in, THB_FRONT_PREFETCH=1)
  for (int q = 0; a.prefetch != 0 && q < nch; q++) {
    const int64_t* PC = p.pc + (int64_t)(c_begin + q) * 6;
    const double* csrc = a.arena_child + item * p.arena_size + PC[0];
    const int cld = (int)(PC[1] & 0xffffffffLL), cbc = (int)(PC[1] >> 32);
    for (int off = tid * 16; off < cbc * cld; off += THREADS * 16) {
      const int i = off / cld, j = off - i * cld;
      if (j <= i) asm volatile("prefetch.global.L2 [%0];\n" ::"l"(csrc + off));
    }
  }
#endif
  __syncthreads();
  if (tid < w8 - w) PN[(w + tid) * ldp + w + tid] = 1.0;   // identity on the padding of the pivot block
  double* Lg = a.factor + item * p.data_size + f_panel_off;
  {
    const double al = a.alpha != nullptr ? a.alpha[item] : 0.0;
    const double be = a.beta != nullptr ? a.beta[item] : 0.0;
    const int total = r * w;
    // FRONT_PL panel elements per thread and pass.  Loads are issued in groups and summed only after the whole group: the FRONT_PL
    // pmap entries; the first two children's entries (they do not depend on pmap); the AtA values; then the next two children's
    // entries, and so on.  The sums keep their order: AtA + damping, then the children in list order.
    for (int e0 = tid; e0 < total; e0 += FRONT_PL * THREADS) {
      int ii[FRONT_PL], jj[FRONT_PL];
      double v[FRONT_PL];
#pragma unroll
      for (int u = 0; u < FRONT_PL; u++) {
        const int e = e0 + u * THREADS;
        ii[u] = e / w;
        jj[u] = e - ii[u] * w;
        if (e >= total || jj[u] > ii[u]) ii[u] = -1;   // outside, or above the diagonal of the pivot block
      }
      int32_t m[FRONT_PL];
#pragma unroll
      for (int u = 0; u < FRONT_PL; u++) m[u] = (a.ata != nullptr && ii[u] >= 0) ? front_ldg(p.pmap + f_panel_off + e0 + u * THREADS) : -1;
      double x[2][FRONT_PL];
      front_panel_gather2(ch, INV, r, nch, 0, ii, jj, x);
#pragma unroll
      for (int u = 0; u < FRONT_PL; u++) {
        if (a.ata != nullptr) v[u] = m[u] >= 0 ? front_ldg(a.ata + item * a.ata_stride + m[u]) : 0.0;
        else v[u] = ii[u] >= 0 ? Lg[e0 + u * THREADS] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < FRONT_PL; u++)
        if (ii[u] >= 0 && ii[u] == jj[u]) v[u] = v[u] + (al * v[u] + be);   // linear/utils.py:14-33: diag <- diag (1 + alpha) + beta
      for (int q = 0;;) {
#pragma unroll
        for (int u = 0; u < FRONT_PL; u++) v[u] = (v[u] + x[0][u]) + x[1][u];
        q += 2;
        if (q >= nch) break;
        front_panel_gather2(ch, INV, r, nch, q, ii, jj, x);
      }
#pragma unroll
      for (int u = 0; u < FRONT_PL; u++)
        if (ii[u] >= 0) PN[(ii[u] < w ? ii[u] : ii[u] + (w8 - w)) * ldp + jj[u]] = v[u];
    }
  }
  // forward substitution (a.rhs != null): u lives in column w8 of the panel (u[i] at U[i * ldp]), which neither the factorisation nor the
  // update-matrix tiles read (their columns stop at w8; ldp >= w8 + 4): no shared memory beyond the panel's.  u = [rhs of the pivots; 0]
  // + the children's border vectors, gathered through the inverse maps in list order -- front_forward_kernel's order
  double* U = PN + w8;
  if (a.rhs != nullptr) {
    for (int i = tid; i < r; i += THREADS) {
      double v = i < w ? a.rhs[item * p.n + p.perm[f_first + i]] : 0.0;
      for (int q = 0; q < nch; q++) {
        if (i >= ch[q].lo && i <= ch[q].hi) {
          const int k = INV[q * r + i];
          if (k >= 0) v += a.v_child[item * p.varena_size + ch[q].uoff + k];
        }
      }
      U[i * ldp] = v;
    }
  }
  __syncthreads();
  // ---- blocked left-looking factorisation of the panel, 8 columns at a time ----
  const int nbk = w8 / 8, nrt = (w8 + b16) / 8;
  // (A LOOK-AHEAD form -- warp 0 finishes row tile jb + 1 alone and factors the NEXT diagonal block while the other warps work through
  // block column jb, one barrier per step -- was built and gave no gain: with
  // <= 1 tile pair per warp the step is bound by tile -> diagonal block -> tile, look-ahead or not.  Removed; git history has it.)
  for (int jb = 0; jb < nbk; jb++) {
    if (warp == 0) front_diag_block(PN, ldp, jb, Wd, lane, w, f_first, a.info + item);
    __syncthreads();
    const int npair = (nrt - jb) / 2;   // row tiles jb+1 .. nrt-1 in pairs (an odd last tile pairs with the zero tile after the end)
    for (int q = warp; q < npair; q += NW) front_tile_column<true>(PN, ldp, jb, jb + 1 + 2 * q, Wd, lane);
    __syncthreads();
  }
  // ---- three consumers of the factored panel that share no data: the panel's copy to the factor storage (reads columns < w), the
  // forward substitution (reads the panel, owns column w8) and the update-matrix tiles (read the border rows, columns < w8).  In a
  // solve the first NE warps run the substitution behind their own barrier while the others write the panel and start on the tiles;
  // they join the tile loop when they are done.  Every tile is computed the same way whichever warp takes it. ----
#ifdef THB_SIMT_EMU   // no named barriers on the host emulation: the same three phases, each by the whole CTA, one after the other
  front_store_panel(Lg, PN, ldp, w, w8, r, tid, THREADS);
  if (a.rhs != nullptr) {
    front_forward_elim<THREADS, true>(FrontRowsPanel{PN, ldp, w, w8 - w}, U, ldp, w, r, tid, lane);
    front_store_forward(a, U, ldp, item, t, f_first, w, b, tid, THREADS);
  }
#else
  constexpr int NE = front_elim_warps(THREADS);
  if (a.rhs != nullptr && warp < NE) {
    front_forward_elim<32 * NE, false>(FrontRowsPanel{PN, ldp, w, w8 - w}, U, ldp, w, r, tid, lane);
    front_store_forward(a, U, ldp, item, t, f_first, w, b, tid, 32 * NE);
  } else {
    const int t0 = a.rhs != nullptr ? 32 * NE : 0;
    front_store_panel(Lg, PN, ldp, w, w8, r, tid - t0, THREADS - t0);
  }
#endif
  if (b == 0) return;
  // ---- update matrix: per 16 x 16 tile of the lower triangle  C = gathered children - P_I P_J^T, written once from registers; a warp
  // takes its next tile from a counter in shared memory, so the warps that come late from the substitution take fewer ----
  double* dst = a.arena_cur + item * p.arena_size + FD[5];   // (cb_off, cb_ld) are read here, not with the rest of the record: held in
  const int ldg_out = (int)FD[6];                            // registers across the phases above they spill
  const double* P = PN + w8 * ldp;
  const int nmt = b16 / 16;
  for (;;) {
    int q = 0;
    if (lane == 0) q = atomicAdd(next_tile, 1);
    q = __shfl_sync(0xffffffffu, q, 0);
    int R = (int)((sqrtf(8.0f * (float)q + 1.0f) - 1.0f) * 0.5f);   // tile q = (row R, column ct) of the lower triangle, row by row
    while ((R + 1) * (R + 2) / 2 <= q) R++;
    while (R * (R + 1) / 2 > q) R--;
    if (R >= nmt) break;
    const int ct = q - R * (R + 1) / 2;
    // Per element: ((0 + first child) + next child ...) - P_I P_J^T, over the children that reach the tile, in list order.  With one
    // such child its loads are issued before the DMMA loop and summed after it, in flight while the tensor pipe works on -P_I P_J^T.
    // With more, they are summed before the loop (the first two children's loads issued together, then one child per round trip):
    // the accumulators of the loop are not live yet, and under the 64-register cap there is no room for both.
    unsigned reach = 0;   // warp-uniform: the children whose rows meet this tile
    for (int qc = 0; qc < nch; qc++)
      if (w + 16 * R + 15 >= ch[qc].lo && w + 16 * ct <= ch[qc].hi) reach |= 1u << qc;
    double gch[2][2][2] = {{{-0.0, -0.0}, {-0.0, -0.0}}, {{-0.0, -0.0}, {-0.0, -0.0}}};
    const int li0 = w + 16 * R + lr, lj0 = w + 16 * ct + 2 * lc;   // front-local indices of this lane's 2 rows and 4 columns
    if (reach != 0) {
      const int qc = front_next_child(reach);
      front_tile_gather(ch[qc], INV + qc * r, r, li0, lj0, gch);
    }
    const bool summed = reach != 0;   // more than one child: the sum is complete before the DMMA loop
    for (bool first = true; reach != 0; first = false) {
      const int qc = front_next_child(reach);
      double x[2][2][2];
      front_tile_gather(ch[qc], INV + qc * r, r, li0, lj0, x);
#pragma unroll
      for (int mi = 0; mi < 2; mi++)
#pragma unroll
        for (int ni = 0; ni < 2; ni++)
#pragma unroll
          for (int u = 0; u < 2; u++) gch[mi][ni][u] = (first ? 0.0 + gch[mi][ni][u] : gch[mi][ni][u]) + x[mi][ni][u];
    }
    double acc[2][2][2] = {{{0.0, 0.0}, {0.0, 0.0}}, {{0.0, 0.0}, {0.0, 0.0}}};
    const double* Pa = P + (16 * R + lr) * ldp + lc;
    const double* Pb = P + (16 * ct + lr) * ldp + lc;
#pragma unroll 1   // w8 is a multiple of 8: no remainder loop, whose trip count spills
    for (int k8 = 0; k8 < w8; k8 += 8) {
#pragma unroll
      for (int k4 = k8; k4 < k8 + 8; k4 += 4) {
        const double a0 = Pa[k4], a1 = Pa[8 * ldp + k4];
        const double b0 = Pb[k4], b1 = Pb[8 * ldp + k4];
        front_mma884(acc[0][0][0], acc[0][0][1], a0, b0);
        front_mma884(acc[0][1][0], acc[0][1][1], a0, b1);
        front_mma884(acc[1][0][0], acc[1][0][1], a1, b0);
        front_mma884(acc[1][1][0], acc[1][1][1], a1, b1);
      }
    }
    if (!summed) {
#pragma unroll
      for (int mi = 0; mi < 2; mi++)
#pragma unroll
        for (int ni = 0; ni < 2; ni++)
#pragma unroll
          for (int u = 0; u < 2; u++) gch[mi][ni][u] = 0.0 + gch[mi][ni][u];
    }
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
      for (int ni = 0; ni < 2; ni++)
#pragma unroll
        for (int u = 0; u < 2; u++) acc[mi][ni][u] = gch[mi][ni][u] - acc[mi][ni][u];
#pragma unroll
    for (int mi = 0; mi < 2; mi++) {
      const int i = 16 * R + 8 * mi + lr;
      if (i < b) {
        double* drow = dst + (int64_t)i * ldg_out;
#pragma unroll
        for (int ni = 0; ni < 2; ni++)
#pragma unroll
          for (int u = 0; u < 2; u++) {
            const int jj = 16 * ct + 8 * ni + 2 * lc + u;
            if (jj <= i) drow[jj] = acc[mi][ni][u];
          }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ big fronts: assemble / extract
constexpr int ASM_ROWS = 16, ASM_THREADS = 256;

__device__ __forceinline__ int front_map_big(int l, int w, int wpad) { return l < w ? l : wpad + (l - w); }

// grid: x = item, y = row tile (np / ASM_ROWS).  Builds rows [R0, R0 + ASM_ROWS) of the padded front matrix F (np x np, row-major):
// zeros, identity on the padding, the panel's AtA entries (+ damping), the children's update matrices; written once.  Four CTAs per SM
// (64 registers): the grouped loads of the gather form would take 72 and leave room for three.
__global__ void __launch_bounds__(ASM_THREADS, 4) front_assemble_kernel(FrontArgs a, int t) {
  extern __shared__ double sm[];
  const thb_front_plan& p = a.p;
  const int tid = threadIdx.x;
  const int64_t item = blockIdx.x;
  const int w = p.f_w[t], b = p.f_b[t], r = w + b, wpad = p.f_wpad[t], np = p.f_np[t];
  const int R0 = blockIdx.y * ASM_ROWS;
  // the dense kernel reads 128 x 64 tiles (i, j <= 2 i + 1): of row R only the columns below 128 (R / 128 + 1) are ever read
  const int nc = min(np, 128 * (R0 / 128 + 1));
  const int c_first = p.child_ptr[t], n_children = p.child_ptr[t + 1] - c_first;
  if (n_children <= FRONT_MAX_CHILDREN) {
    // GATHER form (few children): every entry of the row tile is computed by one thread from the panel and the children's update
    // matrices through the inverse maps; independent loads, no shared memory, no barriers; children added in list order
    const double* Lgg = a.factor + item * p.data_size + p.f_panel_off[t];
    const double alg = a.alpha != nullptr ? a.alpha[item] : 0.0;
    const double beg = a.beta != nullptr ? a.beta[item] : 0.0;
    double* Fg = a.arena_cur + item * p.arena_size + p.f_fr_off[t] + (int64_t)R0 * np;
    // children descriptors once per CTA (the per-element chain child_list -> c_inv_ptr -> inv -> update matrix was four dependent
    // global loads per child and element); then four entries per thread and pass
    __shared__ const double* s_src[FRONT_MAX_CHILDREN];
    __shared__ const int32_t* s_inv[FRONT_MAX_CHILDREN];
    __shared__ int s_ld[FRONT_MAX_CHILDREN];
    if (tid < n_children) {
      const int c = p.child_list[c_first + tid];
      s_src[tid] = a.arena_child + item * p.arena_size + p.f_cb_off[c];
      s_inv[tid] = p.c_inv + p.c_inv_ptr[c];
      s_ld[tid] = p.f_cb_ld[c];
    }
    __syncthreads();
    const int64_t poff = p.f_panel_off[t];
    const int total = ASM_ROWS * nc;
    // children two at a time: the inverse-map entries of both, then their update-matrix entries (-0.0 where a child does not reach the
    // element), each group issued before any of it is used
    auto gather2 = [&](int q, const int (&li)[4], const int (&lj)[4], double (&x)[2][4]) {
      int ci[2][4], cj[2][4];
#pragma unroll
      for (int c = 0; c < 2; c++) {
        const int32_t* inv = q + c < n_children ? s_inv[q + c] : nullptr;
#pragma unroll
        for (int u = 0; u < 4; u++) {
          ci[c][u] = (inv != nullptr && li[u] >= 0) ? front_ldg(inv + li[u]) : -1;
          cj[c][u] = (inv != nullptr && li[u] >= 0) ? front_ldg(inv + lj[u]) : -1;
        }
      }
#pragma unroll
      for (int c = 0; c < 2; c++) {
        const double* src = q + c < n_children ? s_src[q + c] : nullptr;
        const int ldg = q + c < n_children ? s_ld[q + c] : 0;
#pragma unroll
        for (int u = 0; u < 4; u++) x[c][u] = (ci[c][u] >= 0 && cj[c][u] >= 0) ? front_ldg(src + (int64_t)ci[c][u] * ldg + cj[c][u]) : -0.0;
      }
    };
    for (int e0 = tid; e0 < total; e0 += 4 * ASM_THREADS) {
      int li[4], lj[4];
      int pe[4];   // panel element of the entry (its AtA value), or -1
      double v[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int e = e0 + u * ASM_THREADS;
        const int rr = e / nc, fc = e - rr * nc;
        const int fr = R0 + rr;
        li[u] = fr < w ? fr : ((fr >= wpad && fr - wpad + w < r) ? fr - wpad + w : -1);
        lj[u] = fc < w ? fc : ((fc >= wpad && fc - wpad + w < r) ? fc - wpad + w : -1);
        v[u] = 0.0;
        pe[u] = -1;
        if (e >= total) {
          li[u] = lj[u] = -2;                         // past the end: nothing to store
        } else if (li[u] < 0 || lj[u] < 0) {
          v[u] = (fr == fc) ? 1.0 : 0.0;              // identity on the padding
          li[u] = -1;
        } else if (lj[u] > li[u]) {
          li[u] = -1;                                 // above the diagonal: zero
        } else if (lj[u] < w) {
          pe[u] = li[u] * w + lj[u];
        }
      }
      int32_t m[4];
#pragma unroll
      for (int u = 0; u < 4; u++) m[u] = (a.ata != nullptr && pe[u] >= 0) ? front_ldg(p.pmap + poff + pe[u]) : -1;
      double x[2][4];
      gather2(0, li, lj, x);
#pragma unroll
      for (int u = 0; u < 4; u++) {
        if (a.ata != nullptr) { if (m[u] >= 0) v[u] = front_ldg(a.ata + item * a.ata_stride + m[u]); }
        else if (pe[u] >= 0) v[u] = Lgg[pe[u]];
      }
#pragma unroll
      for (int u = 0; u < 4; u++)
        if (li[u] >= 0 && li[u] == lj[u] && lj[u] < w) v[u] = v[u] + (alg * v[u] + beg);
      for (int q = 0;;) {
#pragma unroll
        for (int u = 0; u < 4; u++) v[u] = (v[u] + x[0][u]) + x[1][u];
        q += 2;
        if (q >= n_children) break;
        gather2(q, li, lj, x);
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int e = e0 + u * ASM_THREADS;
        if (e < total) Fg[e + (int64_t)(e / nc) * (np - nc)] = v[u];
      }
    }
    return;
  }
  double* buf = sm;   // [ASM_ROWS][nc]
  for (int e = tid; e < ASM_ROWS * nc; e += ASM_THREADS) buf[e] = 0.0;
  __syncthreads();
  const double* Lg = a.factor + item * p.data_size + p.f_panel_off[t];
  const double al = a.alpha != nullptr ? a.alpha[item] : 0.0;
  const double be = a.beta != nullptr ? a.beta[item] : 0.0;
  const int wlim = min(wpad, nc);
  for (int e = tid; e < ASM_ROWS * wlim; e += ASM_THREADS) {
    const int rr = e / wlim, j = e - rr * wlim;
    const int fr = R0 + rr;
    int i = -1;   // local front row
    if (fr < w) i = fr;
    else if (fr >= wpad && fr - wpad + w < r) i = fr - wpad + w;
    if (i >= 0) {
      if (j < w && !(i < w && j > i)) {
        double v = front_panel_in(a, Lg, p.f_panel_off[t], item, (int64_t)i * w + j);
        if (i == j) v = v + (al * v + be);
        buf[rr * nc + j] = v;
      }
    } else if (j == fr) {
      buf[rr * nc + j] = 1.0;   // padding inside the pivot columns
    }
  }
  for (int rr = tid; rr < ASM_ROWS; rr += ASM_THREADS) {
    const int fr = R0 + rr;
    if (fr >= wpad + b) buf[rr * nc + fr] = 1.0;   // padding after the border rows (fr < nc: the diagonal is always inside)
  }
  __syncthreads();
  for (int ci = p.child_ptr[t]; ci < p.child_ptr[t + 1]; ci++) {
    const int c = p.child_list[ci];
    const int bc = p.f_b[c], ldg = p.f_cb_ld[c];
    const int32_t* rel = p.f_rel + p.rel_ptr[c];
    // child rows whose image lies in this row tile: [i0, i1)  (rel is increasing)
    int lo = 0, hi = bc;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (front_map_big(rel[mid], w, wpad) < R0) lo = mid + 1; else hi = mid; }
    const int i0 = lo;
    hi = bc;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (front_map_big(rel[mid], w, wpad) < R0 + ASM_ROWS) lo = mid + 1; else hi = mid; }
    const int i1 = lo;
    if (i1 > i0) {
      const double* src = a.arena_child + item * p.arena_size + p.f_cb_off[c];
      for (int i = i0 + (tid >> 5); i < i1; i += ASM_THREADS / 32) {
        const int fr = front_map_big(rel[i], w, wpad) - R0;
        const double* srow = src + (int64_t)i * ldg;
        for (int j = tid & 31; j <= i; j += 32) buf[fr * nc + front_map_big(rel[j], w, wpad)] += srow[j];
      }
      __syncthreads();
    }
  }
  double* F = a.arena_cur + item * p.arena_size + p.f_fr_off[t] + (int64_t)R0 * np;
  for (int e = tid; e < ASM_ROWS * nc; e += ASM_THREADS) {
    const int rr = e / nc, c = e - rr * nc;
    F[(int64_t)rr * np + c] = buf[e];
  }
}

// grid: x = item, y = chunk.  factor panel <- the pivot columns of the factored front matrix
__global__ void __launch_bounds__(256) front_extract_kernel(FrontArgs a, int t) {
  const thb_front_plan& p = a.p;
  const int64_t item = blockIdx.x;
  const int w = p.f_w[t], b = p.f_b[t], r = w + b, wpad = p.f_wpad[t], np = p.f_np[t];
  const double* F = a.arena_cur + item * p.arena_size + p.f_fr_off[t];
  double* Lg = a.factor + item * p.data_size + p.f_panel_off[t];
  for (int e = blockIdx.y * blockDim.x + threadIdx.x; e < r * w; e += gridDim.y * blockDim.x) {
    const int i = e / w, j = e - i * w;
    const int fr = i < w ? i : wpad + (i - w);
    Lg[e] = (i < w && j > i) ? 0.0 : F[(int64_t)fr * np + j];
  }
}

// ------------------------------------------------------------------------------------------------ substitutions
struct FrontSolveArgs {
  thb_front_plan p;
  int s0;
  int64_t B;
  const double* factor;
  const double* rhs;        // [B, n] original order (forward)
  double* x;                // [B, n] original order (backward)
  double* work;             // [B, n] permuted: y after the forward pass, x after the backward pass
  double* v_cur;            // border vectors of this depth's parity
  const double* v_child;
  int stage_doubles;        // panels of at most this many doubles are staged in shared memory at kernel start (one coalesced pass) and
                            // every later read is on chip; larger panels are streamed chunk by chunk from global memory
};

// One warp: solve T^T x = t (upper triangular cw x cw, row stride 33) -- the forward direction is front_warp_trsv_lower above
__device__ __forceinline__ double front_warp_trsv_upper(const double* T, double ti, int cw, int lane) {
  const double rd = lane < cw ? 1.0 / T[lane * 33 + lane] : 0.0;
  for (int k = cw - 1; k >= 0; k--) {
    const double xk = __shfl_sync(0xffffffffu, ti * rd, k);
    if (lane == k) ti = xk;
    else if (lane < k) ti -= T[k * 33 + lane] * xk;
  }
  return ti;
}

template <int THREADS>
__global__ void __launch_bounds__(THREADS) front_forward_kernel(FrontSolveArgs a) {
  extern __shared__ double sm[];
  const thb_front_plan& p = a.p;
  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t item = blockIdx.x;
  THB_PDL_TRIGGER();
  const int64_t* FD = p.fd + (int64_t)(a.s0 + blockIdx.y) * 8;   // flat descriptor of the front (frontal.py)
  const int t = (int)FD[0];
  const int w = (int)FD[1], b = (int)FD[2], r = w + b, first = (int)FD[3];
  THB_PDL_WAIT();
  double* u = sm;            // [r]
  double* T = sm + ((r + 1) & ~1);   // [32][33]
  const double* Lg = a.factor + item * p.data_size + FD[4];
  if (r * w <= a.stage_doubles) {
    double* Ls = T + 32 * 33 + 1 + (THREADS & ~1) + 2;
    for (int e = tid; e < r * w; e += THREADS) Ls[e] = Lg[e];
    Lg = Ls;
  }
  {
    // u = [rhs of the pivots; 0] + the children's border vectors, GATHERED through the inverse maps (fixed child order, no barriers)
    const int c0 = (int)(FD[7] & 0xffffffffLL), nchild = (int)(FD[7] >> 32);
    for (int i = tid; i < r; i += THREADS) {
      double v = i < w ? a.rhs[item * p.n + p.perm[first + i]] : 0.0;
      for (int q = 0; q < nchild; q++) {
        const int64_t* PC = p.pc + (int64_t)(c0 + q) * 6;
        if (i >= (int)PC[2] && i <= (int)PC[3]) {
          const int k = p.c_inv[PC[4] + i];
          if (k >= 0) v += a.v_child[item * p.varena_size + PC[5] + k];
        }
      }
      u[i] = v;
    }
  }
  __syncthreads();
  front_forward_elim<THREADS, true>(FrontRowsGlobal{Lg, w, T}, u, 1, w, r, tid, lane);
  for (int i = tid; i < w; i += THREADS) a.work[item * p.n + first + i] = u[i];
  if (b > 0) {
    double* ub = a.v_cur + item * p.varena_size + p.f_u_off[t];
    for (int i = tid; i < b; i += THREADS) ub[i] = u[w + i];
  }
}

template <int THREADS>
__global__ void __launch_bounds__(THREADS) front_backward_kernel(FrontSolveArgs a) {
  extern __shared__ double sm[];
  const thb_front_plan& p = a.p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t item = blockIdx.x;
  THB_PDL_TRIGGER();
  const int64_t* FD = p.fd + (int64_t)(a.s0 + blockIdx.y) * 8;
  const int t = (int)FD[0];
  const int w = (int)FD[1], b = (int)FD[2], r = w + b, first = (int)FD[3];
  THB_PDL_WAIT();
  double* xf = sm;                       // [r] pivots (y, then x) followed by the border rows' x
  double* T = sm + ((r + 1) & ~1);       // [32][33]
  double* part = T + 32 * 33 + 1;        // [THREADS]
  const double* Lg = a.factor + item * p.data_size + FD[4];
  if (r * w <= a.stage_doubles) {
    double* Ls = T + 32 * 33 + 1 + (THREADS & ~1) + 2;
    for (int e = tid; e < r * w; e += THREADS) Ls[e] = Lg[e];
    Lg = Ls;
  }
  double* wk = a.work + item * p.n;
  const int32_t* rows = p.f_rows + p.rows_ptr[t];
  for (int i = tid; i < r; i += THREADS) xf[i] = i < w ? wk[first + i] : wk[rows[i - w]];
  __syncthreads();
  const int nchunk = (w + 31) / 32;
  for (int ch = nchunk - 1; ch >= 0; ch--) {
    const int k0 = ch * 32, cw = min(32, w - k0);
    // t_k = y_k - sum_{i >= k0 + cw} L[i][k0 + k] x_i : cw consecutive threads per row, THREADS / cw rows per pass
    const int RG = THREADS / cw;
    const int kk = tid % cw, rg = tid / cw;
    for (int e = tid; e < cw * cw; e += THREADS) {
      const int i = e / cw, j = e - i * cw;
      T[i * 33 + j] = Lg[(int64_t)(k0 + i) * w + k0 + j];
    }
    double acc = 0.0;
    if (rg < RG) {
      // four loads in flight per thread, summed in row order
      const double* col = Lg + k0 + kk;
      int i = k0 + cw + rg;
      for (; i + 3 * RG < r; i += 4 * RG) {
        const double l0 = col[(int64_t)i * w], l1 = col[(int64_t)(i + RG) * w], l2 = col[(int64_t)(i + 2 * RG) * w],
                     l3 = col[(int64_t)(i + 3 * RG) * w];
        acc += l0 * xf[i];
        acc += l1 * xf[i + RG];
        acc += l2 * xf[i + 2 * RG];
        acc += l3 * xf[i + 3 * RG];
      }
      for (; i < r; i += RG) acc += col[(int64_t)i * w] * xf[i];
    }
    part[tid] = acc;
    __syncthreads();
    if (warp == 0) {
      double tk = 0.0;
      if (lane < cw) {
        tk = xf[k0 + lane];
        for (int g = 0; g < RG; g++) tk -= part[g * cw + lane];
      }
      tk = front_warp_trsv_upper(T, tk, cw, lane);
      if (lane < cw) xf[k0 + lane] = tk;
    }
    __syncthreads();
  }
  for (int i = tid; i < w; i += THREADS) {
    const double v = xf[i];
    wk[first + i] = v;
    a.x[item * p.n + p.perm[first + i]] = v;
  }
}

// Big fronts: factored by the dense kernel straight into their panel (default), or -- THB_FRONT_BIG_DIRECT=0, read at every call: the
// reference the tests compare the direct form against -- assembled into the padded front matrix (front_assemble_kernel), factored in
// place and copied out (front_extract_kernel)
static inline bool front_big_direct() {
  const char* e = getenv("THB_FRONT_BIG_DIRECT");
  return !(e != nullptr && e[0] == '0');
}

static inline int front_threads_of_class(int cls) { return cls == 0 ? 64 : (cls == 1 ? 128 : 256); }

// Opt in to the launch's dynamic shared memory whenever it grows, not only above 48 KB: the 48 KB default limit also counts the kernel's
// static shared memory (front_assemble_kernel's children descriptors), so a launch of exactly 48 KB -- a big front with np = 384 -- failed.
template <typename K>
static inline int front_set_smem(K kernel, size_t bytes, size_t* cache) {
  if (bytes > *cache) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return (int)e;
    *cache = bytes;
  }
  return 0;
}

// One launch entry of the substitutions: pass 0 = forward (front_forward_kernel: y -> work, border vectors through varena), pass 1 =
// backward (front_backward_kernel: work -> x).  Forward launches go deepest first, backward ones roots first.
static int front_solve_launch(const thb_front_plan* p, const int64_t* L, int pass, const double* factor, const double* rhs, double* x,
                              double* work, double* varena, int64_t B, cudaStream_t cs) {
  static size_t fw_set[3] = {0, 0, 0}, bw_set[3] = {0, 0, 0};
  // tuning knob: largest panel (doubles) the substitution kernels stage in shared memory
  static const int64_t stage_cap = [] { const char* e = getenv("THB_SOLVE_STAGE"); return e != nullptr ? (int64_t)atoll(e) : (int64_t)0; }();
  const int depth = (int)L[0], cls = (int)L[1], begin = (int)L[2], count = (int)L[3];
  FrontSolveArgs a;
  a.p = *p; a.s0 = begin; a.B = B; a.factor = factor; a.rhs = rhs; a.x = x; a.work = work;
  a.v_cur = varena != nullptr ? varena + (int64_t)(depth & 1) * B * p->varena_size : nullptr;
  a.v_child = varena != nullptr ? varena + (int64_t)((depth + 1) & 1) * B * p->varena_size : nullptr;
  // (merging the launches of a depth into one was measured: slower -- small fronts on 256-thread CTAs)
  const int kc = cls > 2 ? 2 : cls;
  const int threads = front_threads_of_class(kc);
  const int64_t r_max = L[5];   // largest front of the launch (class-3 launches carry np >= r)
  // panels up to 40 KB are staged on chip (L[6] = largest r * w of a shared-memory launch; class-3 launches stream)
  const int64_t stage = (cls < 3 && L[6] > 0) ? (L[6] < stage_cap ? L[6] : stage_cap) : 0;
  a.stage_doubles = (int)stage;
  const size_t smem = (size_t)(((r_max + 1) & ~1LL) + 32 * 33 + 1 + threads + 2 + stage + 2) * 8;
  const dim3 grid((unsigned)B, (unsigned)count);
  if (pass == 0) {
    if (kc == 0) { int rc = front_set_smem(front_forward_kernel<64>, smem, &fw_set[0]); if (rc) return rc;
                   FRONT_LAUNCH(front_forward_kernel<64>, grid, 64, smem, cs, a); }
    else if (kc == 1) { int rc = front_set_smem(front_forward_kernel<128>, smem, &fw_set[1]); if (rc) return rc;
                        FRONT_LAUNCH(front_forward_kernel<128>, grid, 128, smem, cs, a); }
    else { int rc = front_set_smem(front_forward_kernel<256>, smem, &fw_set[2]); if (rc) return rc;
           FRONT_LAUNCH(front_forward_kernel<256>, grid, 256, smem, cs, a); }
  } else {
    if (kc == 0) { int rc = front_set_smem(front_backward_kernel<64>, smem, &bw_set[0]); if (rc) return rc;
                   FRONT_LAUNCH(front_backward_kernel<64>, grid, 64, smem, cs, a); }
    else if (kc == 1) { int rc = front_set_smem(front_backward_kernel<128>, smem, &bw_set[1]); if (rc) return rc;
                        FRONT_LAUNCH(front_backward_kernel<128>, grid, 128, smem, cs, a); }
    else { int rc = front_set_smem(front_backward_kernel<256>, smem, &bw_set[2]); if (rc) return rc;
           FRONT_LAUNCH(front_backward_kernel<256>, grid, 256, smem, cs, a); }
  }
  THB_CHECK_LAUNCH();
  return THB_OK;
}

// The numeric factorisation; with rhs != null also the forward substitution: fused into front_small_kernel for the shared-memory
// fronts, front_forward_kernel right after the dense kernel has written a big front's panel.
static int front_factor(const thb_front_plan* p, const int64_t* launches, int64_t num_launches, double* factor, const double* ata,
                        int64_t ata_stride, const double* alpha, const double* beta, double* arena, void* dense_ws, int64_t dense_ws_bytes,
                        int32_t* info, const double* rhs, double* work, double* varena, int64_t B, thb_stream_t stream) {
  if (p == nullptr || launches == nullptr || factor == nullptr || arena == nullptr || info == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || p->S == 0) return THB_OK;
  if (B > 65535LL * 32768LL) return THB_ERR_UNSUPPORTED;
  cudaStream_t cs = thb_cs(stream);
  THB_CUDA(cudaMemsetAsync(info, 0, (size_t)B * 4, cs));
  static size_t smem_set[5] = {0, 0, 0, 0, 0}, asm_set = 0;
  // tuning knobs: threads per CTA of the two smallest classes (THB_FRONT_T0: 64 | 128 | 256, THB_FRONT_T1: 128 | 256)
  static const int thr_cls[2] = {[] { const char* e = getenv("THB_FRONT_T0"); const int v = e ? atoi(e) : 64; return (v == 128 || v == 256) ? v : 64; }(),
                                 [] { const char* e = getenv("THB_FRONT_T1"); const int v = e ? atoi(e) : 128; return v == 256 ? 256 : 128; }()};
  static int front_prefetch_flag = -1;
  if (front_prefetch_flag < 0) {
    const char* e = getenv("THB_FRONT_PREFETCH");
    // opt-in: on H100 (C5, batch 2048) the prefetch made the factorisation slower, 175 -> 166 ms without it
    front_prefetch_flag = (e != nullptr && e[0] == '1') ? 1 : 0;
  }
  // largest CTA of front_small_kernel that runs the forward substitution itself (THB_FRONT_FUSE_MAX: 0 | 64 | ... | 1024); launches of
  // larger CTAs are followed by front_forward_kernel instead
  static const int fuse_max = [] { const char* e = getenv("THB_FRONT_FUSE_MAX"); return e != nullptr ? atoi(e) : 1024; }();
  for (int64_t l = 0; l < num_launches; l++) {
    const int64_t* L = launches + l * THB_FRONT_LAUNCH_COLS;
    const int depth = (int)L[0], cls = (int)L[1], begin = (int)L[2], count = (int)L[3];
    FrontArgs a;
    a.p = *p; a.s0 = begin; a.B = B; a.factor = factor; a.alpha = alpha; a.beta = beta; a.info = info;
    a.ata = (ata != nullptr && p->pmap != nullptr) ? ata : nullptr; a.ata_stride = ata_stride;
    a.prefetch = front_prefetch_flag;
    a.arena_cur = arena + (int64_t)(depth & 1) * B * p->arena_size;
    a.arena_child = arena + (int64_t)((depth + 1) & 1) * B * p->arena_size;
    a.rhs = rhs; a.work = work;
    a.v_cur = rhs != nullptr ? varena + (int64_t)(depth & 1) * B * p->varena_size : nullptr;
    a.v_child = rhs != nullptr ? varena + (int64_t)((depth + 1) & 1) * B * p->varena_size : nullptr;
    if (cls < 3) {
      const size_t smem = (size_t)L[4];
#ifndef THB_SIMT_EMU
      if (smem > 227 * 1024) return THB_ERR_UNSUPPORTED;
#endif
      const dim3 grid((unsigned)B, (unsigned)count);
      if (count > 65535) return THB_ERR_UNSUPPORTED;
      const int threads = (cls == 0 && thr_cls[0] == 64) ? 64
                          : ((cls == 0 && thr_cls[0] == 128) || (cls == 1 && thr_cls[1] == 128)) ? 128
                          : (cls <= 1 || smem <= 56 * 1024) ? 256 : (smem <= 113 * 1024 ? 512 : 1024);
      const bool fused = rhs != nullptr && threads <= fuse_max;
      if (!fused) a.rhs = nullptr;
      if (threads == 64) {
        int rc = front_set_smem(front_small_kernel<64>, smem, &smem_set[0]); if (rc) return rc;
        FRONT_LAUNCH(front_small_kernel<64>, grid, 64, smem, cs, a);
      } else if (threads == 128) {
        int rc = front_set_smem(front_small_kernel<128>, smem, &smem_set[1]); if (rc) return rc;
        FRONT_LAUNCH(front_small_kernel<128>, grid, 128, smem, cs, a);
      } else if (threads == 256) {   // class 2 (> 96 rows): threads so that ~32 warps are resident whatever the panel size
        int rc = front_set_smem(front_small_kernel<256>, smem, &smem_set[2]); if (rc) return rc;
        FRONT_LAUNCH(front_small_kernel<256>, grid, 256, smem, cs, a);
      } else if (threads == 512) {
        int rc = front_set_smem(front_small_kernel<512>, smem, &smem_set[3]); if (rc) return rc;
        FRONT_LAUNCH(front_small_kernel<512>, grid, 512, smem, cs, a);
      } else {                          // one CTA per SM: all 1 024 threads
        int rc = front_set_smem(front_small_kernel<1024>, smem, &smem_set[4]); if (rc) return rc;
        FRONT_LAUNCH(front_small_kernel<1024>, grid, 1024, smem, cs, a);
      }
      THB_CHECK_LAUNCH();
      if (rhs != nullptr && !fused) {
        const int rc = front_solve_launch(p, L, 0, factor, rhs, nullptr, work, varena, B, cs);
        if (rc != THB_OK) return rc;
      }
    } else {
      const int64_t np = L[5], nb_piv = L[6], fr_off = L[7], first = L[8];
      const int t = (int)L[9];
#ifdef THB_SIMT_EMU
      (void)np; (void)nb_piv; (void)fr_off; (void)first; (void)t; (void)dense_ws; (void)dense_ws_bytes; (void)asm_set;
      return THB_ERR_UNSUPPORTED;   // the DMMA dense kernel is not part of the host emulation
#else
      if (dense_ws == nullptr || np % 128 != 0 || np > 8192) return THB_ERR_BAD_ARG;
      const int32_t n_real = (int32_t)(nb_piv * 64 + L[11]);
      if (front_big_direct()) {
        // the dense kernel gathers the front's tiles from AtA and the children, and factors straight into the front's panel
        ThbCholDirect d;
        d.fd = p->fd + (int64_t)begin * 8; d.pc = p->pc; d.c_inv = p->c_inv; d.pmap = p->pmap;
        d.factor = factor; d.data_size = p->data_size;
        d.arena_child = a.arena_child; d.arena_size = p->arena_size;
        d.ata = a.ata; d.ata_stride = ata_stride; d.alpha = alpha; d.beta = beta;
        d.w = (int)L[10]; d.b = (int)L[11]; d.wpad = (int)(nb_piv * 64);
        int rc = thb_potrf_partial_direct_f64(a.arena_cur + fr_off, p->arena_size, np, (int32_t)nb_piv, n_real, (int32_t)first, info, B,
                                              dense_ws, dense_ws_bytes, &d, stream);
        if (rc != THB_OK) return rc;
        if (rhs != nullptr) {
          rc = front_solve_launch(p, L, 0, factor, rhs, nullptr, work, varena, B, cs);
          if (rc != THB_OK) return rc;
        }
        continue;
      }
      const size_t smem = (size_t)ASM_ROWS * np * 8;
      int rc = front_set_smem(front_assemble_kernel, smem, &asm_set); if (rc) return rc;
      front_assemble_kernel<<<dim3((unsigned)B, (unsigned)(np / ASM_ROWS)), ASM_THREADS, smem, cs>>>(a, t);
      THB_CHECK_LAUNCH();
      // w_real / n_real: the k loops stop at the real pivot columns, trailing tiles that lie in the padding are skipped
      rc = thb_potrf_partial_inplace_f64(a.arena_cur + fr_off, p->arena_size, np, (int32_t)nb_piv, (int32_t)L[10], n_real,
                                         (int32_t)first, info, B, dense_ws, dense_ws_bytes, stream);
      if (rc != THB_OK) return rc;
      front_extract_kernel<<<dim3((unsigned)B, 8), 256, 0, cs>>>(a, t);
      THB_CHECK_LAUNCH();
      if (rhs != nullptr) {   // the panel is in global memory now: the substitution kernel's forward launch for this front
        rc = front_solve_launch(p, L, 0, factor, rhs, nullptr, work, varena, B, cs);
        if (rc != THB_OK) return rc;
      }
#endif
    }
  }
  return THB_OK;
}

}  // namespace thb

extern "C" {

int64_t thb_front_small_smem_bytes(int32_t w, int32_t b, int32_t nchildren) { return thb::front_smem_doubles(w, b, nchildren) * 8; }

int thb_front_factor_f64(const thb_front_plan* p, const int64_t* launches, int64_t num_launches, double* factor, const double* ata,
                         int64_t ata_stride, const double* alpha, const double* beta, double* arena, void* dense_ws, int64_t dense_ws_bytes,
                         int32_t* info, int64_t B, thb_stream_t stream) {
  return thb::front_factor(p, launches, num_launches, factor, ata, ata_stride, alpha, beta, arena, dense_ws, dense_ws_bytes, info, nullptr,
                           nullptr, nullptr, B, stream);
}

int thb_front_factor_forward_f64(const thb_front_plan* p, const int64_t* launches, int64_t num_launches, double* factor, const double* ata,
                                 int64_t ata_stride, const double* alpha, const double* beta, double* arena, void* dense_ws,
                                 int64_t dense_ws_bytes, int32_t* info, const double* rhs, double* work, double* varena, int64_t B,
                                 thb_stream_t stream) {
  if (rhs == nullptr || work == nullptr || varena == nullptr) return THB_ERR_BAD_ARG;
  return thb::front_factor(p, launches, num_launches, factor, ata, ata_stride, alpha, beta, arena, dense_ws, dense_ws_bytes, info, rhs, work,
                           varena, B, stream);
}

int thb_front_solve_f64(const thb_front_plan* p, const int64_t* launches, int64_t num_launches, const double* factor, const double* rhs,
                        double* x, double* work, double* varena, int64_t B, thb_stream_t stream) {
  if (p == nullptr || launches == nullptr || factor == nullptr || rhs == nullptr || x == nullptr || work == nullptr || varena == nullptr ||
      B < 0)
    return THB_ERR_BAD_ARG;
  if (B == 0 || p->S == 0) return THB_OK;
  const int rc = thb_front_forward_f64(p, launches, num_launches, factor, rhs, work, varena, B, stream);
  if (rc != THB_OK) return rc;
  return thb_front_backward_f64(p, launches, num_launches, factor, x, work, B, stream);
}

int thb_front_forward_f64(const thb_front_plan* p, const int64_t* launches, int64_t num_launches, const double* factor, const double* rhs,
                          double* work, double* varena, int64_t B, thb_stream_t stream) {
  if (p == nullptr || launches == nullptr || factor == nullptr || rhs == nullptr || work == nullptr || varena == nullptr || B < 0)
    return THB_ERR_BAD_ARG;
  if (B == 0 || p->S == 0) return THB_OK;
  cudaStream_t cs = thb_cs(stream);
  for (int64_t q = 0; q < num_launches; q++) {   // deepest first
    const int rc = thb::front_solve_launch(p, launches + q * THB_FRONT_LAUNCH_COLS, 0, factor, rhs, nullptr, work, varena, B, cs);
    if (rc != THB_OK) return rc;
  }
  return THB_OK;
}

int thb_front_backward_f64(const thb_front_plan* p, const int64_t* launches, int64_t num_launches, const double* factor, double* x,
                           double* work, int64_t B, thb_stream_t stream) {
  if (p == nullptr || launches == nullptr || factor == nullptr || x == nullptr || work == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || p->S == 0) return THB_OK;
  cudaStream_t cs = thb_cs(stream);
  for (int64_t q = num_launches - 1; q >= 0; q--) {   // roots first
    const int rc = thb::front_solve_launch(p, launches + q * THB_FRONT_LAUNCH_COLS, 1, factor, nullptr, x, work, nullptr, B, cs);
    if (rc != THB_OK) return rc;
  }
  return THB_OK;
}

}  // extern "C"
