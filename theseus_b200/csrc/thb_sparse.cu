// Batched block-sparse Cholesky (factor + solve) over a batch-shared symbolic plan, fp64.
//
// Replaces the numeric half of the reference's sparse solvers: BaSpaCho `NumericDecomposition::{damp,factor,solve}`
// (theseus/extlib/baspacho_solver.cpp:93-257, baspacho_solver_cuda.cu:171-293), cusolverRf batched refactor/solve
// (extlib/cusolver_lu_solver.cpp:252-310) and the per-batch-item CHOLMOD loop (optimizer/autograd/cholmod_sparse_autograd.py:25-61).
// The symbolic plan (ordering, fill, elimination-tree levels, update lists, work items) is built on the host once per
// structure (theseus_b200/sparse.py); the factor storage [B, data_size] is filled by thb_gram (AtA blocks, no atomics).
//
// Execution model (round 1): one CTA per batch item walks the elimination-tree levels; inside a level every scalar of every
// block of the level's columns is an independent work item:
//   U: target(r,c) -= sum over update pairs (L_ik, L_jk) of <L_ik[r,:], L_jk[c,:]>   (left-looking, lists precomputed)
//   F: per column: Cholesky of the d x d diagonal block + its inverse W_j (d <= 16, registers/local memory)
//   T: per block row: L_ij[r,:] = U_ij[r,:] W_j^T
// Items of one level touch disjoint outputs and only read finished columns, so there are no atomics and the result is
// deterministic.  HBM/latency bound by construction (6x6 / 3x3 blocks, AI ~ 10 flop/B, SURVEY.md 8d): no tensor cores.
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

constexpr int SP_MAXD = 16;
constexpr int SP_THREADS = 512;

__global__ void __launch_bounds__(SP_THREADS) sparse_damp_kernel(thb_sparse_plan p, double* __restrict__ factor,
                                                                 const double* __restrict__ alpha, const double* __restrict__ beta, int64_t B) {
  // diag <- diag * (1 + alpha_b) + beta_b   (extlib/baspacho_solver.cpp:181-183, baspacho_solver_cuda.cu:171-185)
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * p.n) return;
  const int64_t b = t / p.n;
  const int64_t e = t - b * p.n;  // scalar index in the permuted vector
  // find column j with pstart[j] <= e < pstart[j]+dims[j] by bisection
  int lo = 0, hi = p.N;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (p.pstart[mid] <= e) lo = mid; else hi = mid;
  }
  const int d = p.dims[lo];
  const int r = (int)(e - p.pstart[lo]);
  double* D = factor + b * p.data_size + p.diag_off[lo] + (int64_t)r * d + r;
  const double a = alpha != nullptr ? alpha[b] : 0.0, be = beta != nullptr ? beta[b] : 0.0;
  *D = *D * (1.0 + a) + be;
}

// d x d Cholesky + inverse of one diagonal block held in registers (D known at compile time) or local memory (generic).
template <int D>
__device__ __noinline__ int potrf_inv_small(double* __restrict__ Dg, double* __restrict__ Wj, int d) {
  constexpr int LD = (D > 0) ? D : SP_MAXD;
  if (D > 0) d = D;
  double a[LD * LD];
#pragma unroll
  for (int r = 0; r < LD; r++)
#pragma unroll
    for (int c = 0; c < LD; c++)
      if (r < d && c <= r) a[r * LD + c] = Dg[r * d + c];
  int fail = 0;
#pragma unroll
  for (int c = 0; c < LD; c++) {
    if (c < d) {
      double dd = a[c * LD + c];
#pragma unroll
      for (int k = 0; k < LD; k++)
        if (k < c) dd -= a[c * LD + k] * a[c * LD + k];
      if (!(dd > 0.0) && fail == 0) fail = c + 1;
      const double inv = rsqrt(dd);
      a[c * LD + c] = dd * inv;
#pragma unroll
      for (int r = 0; r < LD; r++) {
        if (r > c && r < d) {
          double sacc = a[r * LD + c];
#pragma unroll
          for (int k = 0; k < LD; k++)
            if (k < c) sacc -= a[r * LD + k] * a[c * LD + k];
          a[r * LD + c] = sacc * inv;
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < LD; r++)
#pragma unroll
    for (int c = 0; c < LD; c++)
      if (r < d && c < d) Dg[r * d + c] = (c <= r) ? a[r * LD + c] : 0.0;
  // inverse of the lower-triangular block, column by column
#pragma unroll
  for (int c = 0; c < LD; c++) {
    if (c < d) {
      double x[LD];
#pragma unroll
      for (int r = 0; r < LD; r++) {
        if (r < d) {
          if (r < c) { x[r] = 0.0; }
          else {
            double sacc = (r == c) ? 1.0 : 0.0;
#pragma unroll
            for (int k = 0; k < LD; k++)
              if (k >= c && k < r) sacc -= a[r * LD + k] * x[k];
            x[r] = sacc / a[r * LD + r];
          }
          Wj[r * d + c] = x[r];
        }
      }
    }
  }
  return fail;
}

__global__ void __launch_bounds__(SP_THREADS) sparse_factor_kernel(thb_sparse_plan p, double* __restrict__ factor, double* __restrict__ winv,
                                                                   int32_t* __restrict__ info) {
  const int64_t b = blockIdx.x;
  double* F = factor + b * p.data_size;
  double* W = winv + b * p.winv_size;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = SP_THREADS / 32;
  __shared__ int s_fail;
  if (tid == 0) s_fail = 0;
  __syncthreads();
  for (int lv = 0; lv < p.num_levels; lv++) {
    // ---- U: updates.  One warp per block; lane l owns scalars l, l+32, ... of the block (u_r/u_c = rows/cols, u_ld = is-diagonal) ----
    {
      const int64_t e1 = p.u_ptr[lv + 1];
      for (int64_t e = p.u_ptr[lv] + warp; e < e1; e += NW) {
        const int di = p.u_r[e], dj = p.u_c[e];
        const bool diag = p.u_ld[e] != 0;
        const int64_t tgt = p.u_tgt[e];
        const int64_t q0 = p.u_p0[e], q1 = p.u_p1[e];
        for (int t = lane; t < di * dj; t += 32) {
          const int r = t / dj, c = t - r * dj;
          if (diag && c > r) continue;
          double acc0 = 0.0, acc1 = 0.0;
          int64_t q = q0;
          for (; q + 1 < q1; q += 2) {  // two independent update pairs in flight
            const int dk0 = p.up_k[q], dk1 = p.up_k[q + 1];
            const double* a0 = F + p.up_a[q] + r * dk0;
            const double* b0 = F + p.up_b[q] + c * dk0;
            const double* a1 = F + p.up_a[q + 1] + r * dk1;
            const double* b1 = F + p.up_b[q + 1] + c * dk1;
            for (int k = 0; k < dk0; k++) acc0 += a0[k] * b0[k];
            for (int k = 0; k < dk1; k++) acc1 += a1[k] * b1[k];
          }
          if (q < q1) {
            const int dk0 = p.up_k[q];
            const double* a0 = F + p.up_a[q] + r * dk0;
            const double* b0 = F + p.up_b[q] + c * dk0;
            for (int k = 0; k < dk0; k++) acc0 += a0[k] * b0[k];
          }
          F[tgt + t] -= (acc0 + acc1);
        }
      }
    }
    __syncthreads();
    // ---- F: diagonal blocks (one thread per column; 6x6 and 3x3 fully in registers) ----
    for (int64_t e = p.f_ptr[lv] + tid; e < p.f_ptr[lv + 1]; e += SP_THREADS) {
      const int d = p.f_dim[e];
      double* D = F + p.f_off[e];
      double* Wj = W + p.f_w[e];
      int fail;
      if (d == 6) fail = potrf_inv_small<6>(D, Wj, 6);
      else if (d == 3) fail = potrf_inv_small<3>(D, Wj, 3);
      else fail = potrf_inv_small<0>(D, Wj, d);
      if (fail != 0) record_first_failure(&s_fail, (int)(p.pstart[p.f_col[e]] + fail));
    }
    __syncthreads();
    // ---- T: L_ij[r,:] = U_ij[r,:] W_j^T ----
    for (int64_t e = p.t_ptr[lv] + tid; e < p.t_ptr[lv + 1]; e += SP_THREADS) {
      const int d = p.t_dim[e];
      double* row = F + p.t_off[e] + (int64_t)p.t_r[e] * d;
      const double* Wj = W + p.t_w[e];
      double u[SP_MAXD];
      for (int q = 0; q < d; q++) u[q] = row[q];
      for (int c = 0; c < d; c++) {
        double sacc = 0.0;
        for (int q = 0; q <= c; q++) sacc += u[q] * Wj[c * d + q];
        row[c] = sacc;
      }
    }
    __syncthreads();
  }
  if (tid == 0) info[b] = s_fail;
}

// x = (L L^T)^-1 rhs in the original variable order.  work [B,n] holds the permuted vector.
// One warp per column: the lanes split the column's block list, partial sums are combined with shuffles.
__global__ void __launch_bounds__(SP_THREADS) sparse_solve_kernel(thb_sparse_plan p, const double* __restrict__ factor,
                                                                  const double* __restrict__ winv, const double* __restrict__ rhs,
                                                                  double* __restrict__ x, double* __restrict__ work) {
  const int64_t b = blockIdx.x;
  const double* F = factor + b * p.data_size;
  const double* W = winv + b * p.winv_size;
  const double* rb = rhs + b * p.n;
  double* y = work + b * p.n;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = SP_THREADS / 32;
  // forward: y_j = W_j (rhs_j - sum_k L_jk y_k); the permutation is folded into the load (K8 scramble, baspacho_solver_cuda.cu:216-232)
  for (int lv = 0; lv < p.num_levels; lv++) {
    for (int64_t e = p.s_ptr[lv] + warp; e < p.s_ptr[lv + 1]; e += NW) {
      const int j = p.s_col[e];
      const int d = p.dims[j];
      double s[SP_MAXD];
#pragma unroll
      for (int r = 0; r < SP_MAXD; r++) s[r] = 0.0;
      for (int64_t q = p.fr_ptr[j] + lane; q < p.fr_ptr[j + 1]; q += 32) {
        const int k = p.fr_k[q];
        const int dk = p.dims[k];
        const double* L = F + p.fr_off[q];
        const double* yk = y + p.pstart[k];
#pragma unroll
        for (int r = 0; r < SP_MAXD; r++) {
          if (r < d) {
            double a = 0.0;
            for (int c = 0; c < dk; c++) a += L[r * dk + c] * yk[c];
            s[r] += a;
          }
        }
      }
#pragma unroll
      for (int r = 0; r < SP_MAXD; r++) {
        if (r < d) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) s[r] += __shfl_xor_sync(0xffffffffu, s[r], o);
          s[r] = rb[p.col_start[j] + r] - s[r];
        }
      }
      if (lane < d) {
        const double* Wj = W + p.winv_off[j];
        double a = 0.0;
#pragma unroll
        for (int c = 0; c < SP_MAXD; c++)
          if (c <= lane && c < d) a += Wj[lane * d + c] * s[c];
        y[p.pstart[j] + lane] = a;
      }
    }
    __syncthreads();
  }
  // backward: x_j = W_j^T (y_j - sum_i L_ij^T x_i)
  for (int lv = p.num_levels - 1; lv >= 0; lv--) {
    for (int64_t e = p.s_ptr[lv] + warp; e < p.s_ptr[lv + 1]; e += NW) {
      const int j = p.s_col[e];
      const int d = p.dims[j];
      double s[SP_MAXD];
#pragma unroll
      for (int r = 0; r < SP_MAXD; r++) s[r] = 0.0;
      for (int64_t q = p.bc_ptr[j] + lane; q < p.bc_ptr[j + 1]; q += 32) {
        const int i = p.bc_i[q];
        const int di = p.dims[i];
        const double* L = F + p.bc_off[q];
        const double* xi = y + p.pstart[i];
        for (int r = 0; r < di; r++) {
          const double xr = xi[r];
#pragma unroll
          for (int c = 0; c < SP_MAXD; c++)
            if (c < d) s[c] += L[r * d + c] * xr;
        }
      }
      double* yj = y + p.pstart[j];
#pragma unroll
      for (int c = 0; c < SP_MAXD; c++) {
        if (c < d) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) s[c] += __shfl_xor_sync(0xffffffffu, s[c], o);
          s[c] = yj[c] - s[c];
        }
      }
      __syncwarp();
      if (lane < d) {
        const double* Wj = W + p.winv_off[j];
        double a = 0.0;
#pragma unroll
        for (int r = 0; r < SP_MAXD; r++)
          if (r >= lane && r < d) a += Wj[r * d + lane] * s[r];
        yj[lane] = a;
        x[b * p.n + p.col_start[j] + lane] = a;  // un-permute on store (K8 unscramble, baspacho_solver_cuda.cu:234-250)
      }
    }
    __syncthreads();
  }
}

}  // namespace thb

extern "C" {

int thb_sparse_damp_f64(const thb_sparse_plan* p, double* factor, const double* alpha, const double* beta, int64_t B, thb_stream_t s) {
  if (p == nullptr || factor == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || p->n == 0) return THB_OK;
  const int64_t total = B * p->n;
  thb::sparse_damp_kernel<<<(unsigned)((total + 255) / 256), 256, 0, thb_cs(s)>>>(*p, factor, alpha, beta, B);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

int thb_sparse_factor_f64(const thb_sparse_plan* p, double* factor, double* winv, int32_t* info, int64_t B, thb_stream_t s) {
  if (p == nullptr || factor == nullptr || winv == nullptr || info == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (p->max_dim > thb::SP_MAXD) return THB_ERR_UNSUPPORTED;
  if (B == 0 || p->N == 0) return THB_OK;
  thb::sparse_factor_kernel<<<(unsigned)B, thb::SP_THREADS, 0, thb_cs(s)>>>(*p, factor, winv, info);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

int thb_sparse_solve_f64(const thb_sparse_plan* p, const double* factor, const double* winv, const double* rhs, double* x, double* work,
                         int64_t B, thb_stream_t s) {
  if (p == nullptr || factor == nullptr || winv == nullptr || rhs == nullptr || x == nullptr || work == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (p->max_dim > thb::SP_MAXD) return THB_ERR_UNSUPPORTED;
  if (B == 0 || p->N == 0) return THB_OK;
  thb::sparse_solve_kernel<<<(unsigned)B, thb::SP_THREADS, 0, thb_cs(s)>>>(*p, factor, winv, rhs, x, work);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

}  // extern "C"
