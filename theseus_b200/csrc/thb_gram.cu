// Gram assembly (AtA blocks, Atb, diag) from the batched-CSR Jacobian, and batched CSR mat-vec helpers.
//
// The Jacobian of these problems is block-sparse with 6x6 / 3x3 / 2xk blocks (SURVEY.md 8d): the
// Gram product is ~0.2 GFLOP of block products, not the 3.8 TFLOP dense bmm the reference runs
// (optimizer/dense_linearization.py:58-62).  It is an HBM-bound gather: every output scalar is the
// sum, over the cost functions touching that variable pair, of a short column-column dot product.
// Every output scalar is accumulated by one thread; contributions are visited in a fixed order, so the
// result is deterministic -- no fp64 atomics as in extlib/mat_mult.cu:36-79 /
// extlib/baspacho_solver_cuda.cu:96-134.  gram_staged_kernel (below) is the hot path.  Plans whose groups
// do not fit its shared-memory budget (a variable with many cost functions, e.g. the hub of a star) take
// gram_block_kernel when every block shape is one it is built for, else gram_kernel (one thread per output
// scalar and batch item), and atb_kernel; all give bitwise the same results.
#include "thb_common.cuh"

namespace thb {

template <typename T>
__global__ void __launch_bounds__(256) gram_kernel(thb_gram_plan p, int64_t B, const T* __restrict__ A_val, int64_t nnz,
                                                   T* __restrict__ out, int64_t out_bstride, T* __restrict__ diag) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.num_entries * B) return;
  const int64_t b = t / p.num_entries;
  const int64_t e = t - b * p.num_entries;
  const int blk = p.ent_blk[e];
  const int pp = p.ent_p[e], qq = p.ent_q[e];
  const T* A = A_val + b * nnz;
  T acc = T(0);
  const int c1 = p.blk_cptr[blk + 1];
  for (int c = p.blk_cptr[blk]; c < c1; c++) {
    const T* base = A + p.c_off[c];
    const int stride = p.c_stride[c];
    const int rows = p.c_rows[c];
    const int oa = p.c_bpa[c] + pp, ob = p.c_bpb[c] + qq;
    for (int r = 0; r < rows; r++) acc += base[r * stride + oa] * base[r * stride + ob];
  }
  T* o = out + b * out_bstride;
  const int ld = p.blk_ld[blk];
  o[p.blk_out[blk] + (int64_t)pp * ld + qq] = acc;
  const int64_t mo = p.blk_mirror[blk];
  if (mo >= 0) o[mo + (int64_t)qq * ld + pp] = acc;
}

template <typename T>
__global__ void __launch_bounds__(256) atb_kernel(thb_gram_plan p, int64_t B, const T* __restrict__ A_val, int64_t nnz,
                                                  const T* __restrict__ bvec, int64_t m, T* __restrict__ Atb, T* __restrict__ diag) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.n * B) return;
  const int64_t b = t / p.n;
  const int64_t col = t - b * p.n;
  const T* A = A_val + b * nnz;
  const T* bb = bvec + b * m;
  T acc = T(0), dacc = T(0);
  const int c1 = p.col_cptr[col + 1];
  for (int c = p.col_cptr[col]; c < c1; c++) {
    const T* base = A + p.cc_off[c];
    const int stride = p.cc_stride[c];
    const int rows = p.cc_rows[c];
    const T* br = bb + p.cc_row0[c];
    for (int r = 0; r < rows; r++) {
      const T a = base[r * stride];
      acc += a * br[r];
      dacc += a * a;
    }
  }
  Atb[b * p.n + col] = acc;
  if (diag != nullptr) diag[b * p.n + col] = dacc;
}

// y[b,row] = sum_k A_val[b,k] v[b,col_k]     (extlib/mat_mult.cu:134-163 semantics)
template <typename T>
__global__ void mat_vec_kernel(int64_t B, int64_t num_rows, int64_t num_cols, const int64_t* __restrict__ row_ptr,
                               const int64_t* __restrict__ col_ind, const T* __restrict__ A_val, const T* __restrict__ v,
                               T* __restrict__ y) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * num_rows) return;
  const int64_t b = t / num_rows, row = t - b * num_rows;
  const int64_t nnz = row_ptr[num_rows];
  const T* A = A_val + b * nnz;
  const T* vb = v + b * num_cols;
  T acc = T(0);
  for (int64_t k = row_ptr[row]; k < row_ptr[row + 1]; k++) acc += A[k] * vb[col_ind[k]];
  y[t] = acc;
}

// y[b,col] = sum over entries k in column col of A_val[b,k] v[b,row_k]   (extlib/mat_mult.cu:216-243 semantics).
// Generic entry point for arbitrary CSR patterns (tests, backward): one thread per (b, col) visits the rows
// in order and binary-searches the column, so the sum is deterministic (the reference uses fp64 atomicAdd).
// The per-iteration hot path does not use this: Atb comes from the Gram plan's precomputed columns.
template <typename T>
__global__ void tmat_vec_kernel(int64_t B, int64_t num_rows, int64_t num_cols, const int64_t* __restrict__ row_ptr,
                                const int64_t* __restrict__ col_ind, const T* __restrict__ A_val, const T* __restrict__ v,
                                T* __restrict__ y) {
  // one thread per (b, col): scan all rows' entries for this column using binary search in each row
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * num_cols) return;
  const int64_t b = t / num_cols, col = t - b * num_cols;
  const int64_t nnz = row_ptr[num_rows];
  const T* A = A_val + b * nnz;
  const T* vb = v + b * num_rows;
  T acc = T(0);
  for (int64_t row = 0; row < num_rows; row++) {
    int64_t lo = row_ptr[row], hi = row_ptr[row + 1];
    // columns inside a row are sorted (sparse_linearization.py:62-63)
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      const int64_t c = col_ind[mid];
      if (c < col) lo = mid + 1; else hi = mid;
    }
    if (lo < row_ptr[row + 1] && col_ind[lo] == col) acc += A[lo] * vb[row];
  }
  y[t] = acc;
}

// Backward of x = (AtA + D)^-1 At b with respect to A_val and b, given H = (AtA + D)^-1 grad_x:
//   b_grad = A H,   A_grad[r,c] = (b - A x)[r] H[c] - (A H)[r] x[c]  - 2 alpha H[c] x[c] A[r,c]
// (optimizer/autograd/common.py:11-48: a Python loop over the m rows there; derivation in baspacho_sparse_autograd.py:68-115).
// One thread per (batch item, row): the two row dot products and the row's slice of A_grad in one pass.
__global__ void __launch_bounds__(256) solve_backward_kernel(int64_t B, int64_t num_rows, int64_t num_cols, const int64_t* __restrict__ row_ptr,
                                                             const int64_t* __restrict__ col_ind, const double* __restrict__ A_val,
                                                             const double* __restrict__ bvec, const double* __restrict__ x,
                                                             const double* __restrict__ H, const double* __restrict__ alpha, int detach,
                                                             double* __restrict__ A_grad, double* __restrict__ b_grad) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * num_rows) return;
  const int64_t bi = t / num_rows, row = t - bi * num_rows;
  const int64_t nnz = row_ptr[num_rows];
  const double* A = A_val + bi * nnz;
  const double* xb = x + bi * num_cols;
  const double* Hb = H + bi * num_cols;
  const int64_t k0 = row_ptr[row], k1 = row_ptr[row + 1];
  double ah = 0.0, ax = 0.0;
  for (int64_t k = k0; k < k1; k++) {
    const int64_t c = col_ind[k];
    const double a = A[k];
    ah += a * Hb[c];
    ax += a * xb[c];
  }
  if (b_grad != nullptr) b_grad[t] = ah;
  if (A_grad == nullptr) return;
  const double res = detach ? bvec[t] : bvec[t] - ax;
  const double al2 = (alpha != nullptr) ? 2.0 * alpha[bi] : 0.0;
  double* G = A_grad + bi * nnz;
  for (int64_t k = k0; k < k1; k++) {
    const int64_t c = col_ind[k];
    const double h = Hb[c], xv = xb[c];
    double g = detach ? res * h : res * h - ah * xv;
    if (al2 > 0.0) g -= A[k] * al2 * h * xv;
    G[k] = g;
  }
}

}  // namespace thb

namespace thb {

// Block-per-thread Gram: one thread forms a whole DI x DJ block of AtA for one batch item in registers -- every Jacobian entry of a
// contribution is loaded once per block (12 loads for 36 FMAs with 6 x 6 blocks; the entry-per-thread kernel above issues 2 per FMA
// and is bound by load instructions at 0.14 of HBM) and the block's rows are written as DJ consecutive values.  Blocks are grouped by
// shape on the host (thb_gram_plan.segments); threads of a warp = consecutive blocks of ONE item, i.e. neighbouring cost functions'
// row blocks of A_val.  Contributions are visited in the plan's fixed order: deterministic, no atomics.
template <typename T, int DI, int DJ>
__global__ void __launch_bounds__(128, (DI * DJ > 18 ? 8 : 4)) gram_block_kernel(thb_gram_plan p, int64_t B, const T* __restrict__ A_val, int64_t nnz,
                                                                                 T* __restrict__ out, int64_t out_bstride, int seg_begin, int count) {
  // blocks with more than 18 entries are shared by two threads (rows [0, DI/2) and [DI/2, DI)): 18 accumulators + 9 operands fit 64
  // registers, so eight CTAs of 128 threads are resident and twice as many loads are in flight (the kernel is bound by memory latency)
  constexpr int SPLIT = (DI * DJ > 18 && DI % 2 == 0) ? 2 : 1;
  constexpr int RI = DI / SPLIT;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)count * B * SPLIT) return;
  const int64_t b = t / ((int64_t)count * SPLIT);
  const int rem = (int)(t - b * (int64_t)count * SPLIT);
  const int blk = p.blk_order[seg_begin + rem / SPLIT];
  const int r0 = (rem % SPLIT) * RI;
  const T* A = A_val + b * nnz;
  T acc[RI][DJ];
#pragma unroll
  for (int i = 0; i < RI; i++)
#pragma unroll
    for (int j = 0; j < DJ; j++) acc[i][j] = T(0);
  const int c1 = p.blk_cptr[blk + 1];
  for (int c = p.blk_cptr[blk]; c < c1; c++) {
    const T* base = A + p.c_off[c];
    const int stride = p.c_stride[c], rows = p.c_rows[c];
    const T* pa = base + p.c_bpa[c] + r0;
    const T* pb = base + p.c_bpb[c];
    for (int r = 0; r < rows; r++) {
      T av[RI], bv[DJ];
#pragma unroll
      for (int i = 0; i < RI; i++) av[i] = pa[r * stride + i];
#pragma unroll
      for (int j = 0; j < DJ; j++) bv[j] = pb[r * stride + j];
#pragma unroll
      for (int i = 0; i < RI; i++)
#pragma unroll
        for (int j = 0; j < DJ; j++) acc[i][j] += av[i] * bv[j];
    }
  }
  T* o = out + b * out_bstride;
  const int ld = p.blk_ld[blk];
  T* o0 = o + p.blk_out[blk];
#pragma unroll
  for (int i = 0; i < RI; i++)
#pragma unroll
    for (int j = 0; j < DJ; j++) o0[(int64_t)(r0 + i) * ld + j] = acc[i][j];
  const int64_t mo = p.blk_mirror[blk];
  if (mo >= 0) {
    T* o1 = o + mo;
#pragma unroll
    for (int j = 0; j < DJ; j++)
#pragma unroll
      for (int i = 0; i < RI; i++) o1[(int64_t)j * ld + r0 + i] = acc[i][j];
  }
}

template <typename T, int DI>
static int gram_block_launch_dj(int dj, const thb_gram_plan& p, int64_t B, const T* A_val, int64_t nnz, T* out, int64_t bs, int begin, int count,
                                cudaStream_t cs) {
  const int64_t total = (int64_t)count * B * ((DI * dj > 18 && DI % 2 == 0) ? 2 : 1);
  const unsigned grid = (unsigned)((total + 127) / 128);
  switch (dj) {
    case 1: gram_block_kernel<T, DI, 1><<<grid, 128, 0, cs>>>(p, B, A_val, nnz, out, bs, begin, count); return 1;
    case 2: gram_block_kernel<T, DI, 2><<<grid, 128, 0, cs>>>(p, B, A_val, nnz, out, bs, begin, count); return 1;
    case 3: gram_block_kernel<T, DI, 3><<<grid, 128, 0, cs>>>(p, B, A_val, nnz, out, bs, begin, count); return 1;
    case 6: gram_block_kernel<T, DI, 6><<<grid, 128, 0, cs>>>(p, B, A_val, nnz, out, bs, begin, count); return 1;
    default: return 0;
  }
}

}  // namespace thb

namespace thb {

// Staged Gram: one CTA per (batch item, group of consecutive variables).  The CTA first copies the rows of A and b of every cost
// function its group touches into shared memory (one warp per cost function, consecutive lanes on consecutive doubles: every load
// instruction reads whole sectors, and each cost function's rows are read once per CTA), then forms from shared memory every block
// whose row variable is in the group, and Atb / diag of the group's columns.  Neighbouring groups of one item run in neighbouring
// CTAs, so a cost function staged by two groups is read from HBM about once.
//
// Every output scalar is accumulated by one thread, over the plan's contributions in order and rows ascending, with the same
// `acc += a * b` as gram_kernel / atb_kernel: the results are bitwise those of the entry-per-thread kernels (which also serve plans
// whose groups do not fit the shared-memory budget).  A block task is one row p of one block and up to STAGE_COLS of its columns,
// so the row's value of A is read once per STAGE_COLS products.
constexpr int STAGE_COLS = 6;       // structure.GRAM_STAGE_COLS
constexpr int STAGE_THREADS = 256;

template <typename T>
__global__ void __launch_bounds__(STAGE_THREADS) gram_staged_kernel(thb_gram_plan p, const T* __restrict__ A_val, int64_t nnz,
                                                                    const T* __restrict__ bvec, int64_t m, T* __restrict__ out,
                                                                    int64_t out_bstride, T* __restrict__ Atb, T* __restrict__ diag) {
  extern __shared__ double2 gram_stage_raw[];
  T* sh = reinterpret_cast<T*>(gram_stage_raw);
  const int64_t b = blockIdx.x / p.num_groups;
  const int g = (int)(blockIdx.x - b * p.num_groups);
  const T* A = A_val + b * nnz;
  const T* bb = bvec + b * m;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const bool with_b = Atb != nullptr;
  for (int s = p.stage_ptr[g] + warp; s < p.stage_ptr[g + 1]; s += nwarps) {
    const T* src = A + p.st_off[s];
    const T* srcb = bb + p.st_row0[s];
    const int len = p.st_len[s];
    const int tot = with_b ? len + p.st_dim[s] : len;
    T* dst = sh + p.st_soff[s];
    for (int k0 = lane; k0 < tot; k0 += 4 * 32) {
      T v[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {     // four loads in flight per lane before the stores
        const int k = k0 + 32 * u;
        v[u] = k < len ? src[k] : (k < tot ? srcb[k - len] : T(0));
      }
#pragma unroll
      for (int u = 0; u < 4; u++)
        if (k0 + 32 * u < tot) dst[k0 + 32 * u] = v[u];
    }
  }
  __syncthreads();
  const int t0 = p.task_ptr[g];
  const int nbt = out != nullptr ? p.task_ptr[g + 1] - t0 : 0;
  const int col0 = p.grp_col[g];
  const int ncol = with_b ? p.grp_col[g + 1] - col0 : 0;
  for (int t = threadIdx.x; t < nbt + ncol; t += blockDim.x) {
    if (t < nbt) {
      const int blk = p.task_blk[t0 + t];
      const int pq = p.task_pq[t0 + t];
      const int pp = pq >> 16, q0 = pq & 0xffff;
      const int nq = min(STAGE_COLS, p.blk_cols[blk] - q0);
      T acc[STAGE_COLS];
#pragma unroll
      for (int q = 0; q < STAGE_COLS; q++) acc[q] = T(0);
      const int c1 = p.blk_cptr[blk + 1];
      for (int c = p.blk_cptr[blk]; c < c1; c++) {
        const T* base = sh + p.c_soff[c];
        const int stride = p.c_stride[c], rows = p.c_rows[c];
        const T* pa = base + p.c_bpa[c] + pp;
        const T* pb = base + p.c_bpb[c] + q0;
        for (int r = 0; r < rows; r++) {
          const T a = pa[r * stride];
#pragma unroll
          for (int q = 0; q < STAGE_COLS; q++)
            if (q < nq) acc[q] += a * pb[r * stride + q];
        }
      }
      T* o = out + b * out_bstride;
      const int ld = p.blk_ld[blk];
      T* o0 = o + p.blk_out[blk] + (int64_t)pp * ld + q0;
#pragma unroll
      for (int q = 0; q < STAGE_COLS; q++)
        if (q < nq) o0[q] = acc[q];
      const int64_t mo = p.blk_mirror[blk];
      if (mo >= 0) {
        T* o1 = o + mo + (int64_t)q0 * ld + pp;
#pragma unroll
        for (int q = 0; q < STAGE_COLS; q++)
          if (q < nq) o1[(int64_t)q * ld] = acc[q];
      }
    } else {
      const int64_t col = col0 + (t - nbt);
      T acc = T(0), dacc = T(0);
      const int c1 = p.col_cptr[col + 1];
      for (int c = p.col_cptr[col]; c < c1; c++) {
        const T* base = sh + p.cc_soff[c];
        const T* br = sh + p.cc_sb[c];
        const int stride = p.cc_stride[c], rows = p.cc_rows[c];
        for (int r = 0; r < rows; r++) {
          const T a = base[r * stride];
          acc += a * br[r];
          dacc += a * a;
        }
      }
      Atb[b * p.n + col] = acc;
      if (diag != nullptr) diag[b * p.n + col] = dacc;
    }
  }
}

}  // namespace thb

template <typename T>
static int gram_impl(const thb_gram_plan* p, int64_t B, const T* A_val, int64_t nnz, const T* b, int64_t m, T* out, int64_t out_bstride,
                     T* Atb, T* diag, thb_stream_t s) {
  if (p == nullptr || B < 0) return THB_ERR_BAD_ARG;
  if (B == 0) return THB_OK;
  cudaStream_t cs = thb_cs(s);
  const bool blocks = out != nullptr && p->num_entries > 0, cols = Atb != nullptr && p->n > 0;
  if (!blocks && !cols) return THB_OK;
  const int64_t smem = p->stage_elems * (int64_t)sizeof(T);
  if (p->num_groups > 0 && smem <= 48 * 1024) {
    const int64_t grid = p->num_groups * B;
    if (grid > 0x7fffffff) return THB_ERR_BAD_ARG;
    thb::gram_staged_kernel<T><<<(unsigned)grid, thb::STAGE_THREADS, (size_t)smem, cs>>>(*p, A_val, nnz, b, m, blocks ? out : nullptr,
                                                                                          out_bstride, cols ? Atb : nullptr, diag);
    THB_CHECK_LAUNCH();
    return THB_OK;
  }
  if (blocks && p->num_segments > 0 && p->segments != nullptr && p->blk_order != nullptr) {
    // every block shape is one the block-per-thread kernels are built for (the host only fills `segments` then)
    for (int64_t sgi = 0; sgi < p->num_segments; sgi++) {
      const int32_t* sg = p->segments + 4 * sgi;   // (di, dj, begin, end) into blk_order
      const int count = sg[3] - sg[2];
      if (count <= 0) continue;
      int ok = 0;
      switch (sg[0]) {
        case 1: ok = thb::gram_block_launch_dj<T, 1>(sg[1], *p, B, A_val, nnz, out, out_bstride, sg[2], count, cs); break;
        case 2: ok = thb::gram_block_launch_dj<T, 2>(sg[1], *p, B, A_val, nnz, out, out_bstride, sg[2], count, cs); break;
        case 3: ok = thb::gram_block_launch_dj<T, 3>(sg[1], *p, B, A_val, nnz, out, out_bstride, sg[2], count, cs); break;
        case 6: ok = thb::gram_block_launch_dj<T, 6>(sg[1], *p, B, A_val, nnz, out, out_bstride, sg[2], count, cs); break;
        default: ok = 0;
      }
      if (!ok) return THB_ERR_BAD_ARG;
      THB_CHECK_LAUNCH();
    }
  } else if (blocks) {
    const int64_t total = p->num_entries * B;
    thb::gram_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, cs>>>(*p, B, A_val, nnz, out, out_bstride, nullptr);
    THB_CHECK_LAUNCH();
  }
  if (cols) {
    const int64_t total = p->n * B;
    thb::atb_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, cs>>>(*p, B, A_val, nnz, b, m, Atb, diag);
    THB_CHECK_LAUNCH();
  }
  return THB_OK;
}

extern "C" {

int thb_gram_f64(const thb_gram_plan* p, int64_t B, const double* A_val, int64_t nnz, const double* b, int64_t m, double* out,
                 int64_t out_bstride, double* Atb, double* diag, thb_stream_t s) {
  return gram_impl<double>(p, B, A_val, nnz, b, m, out, out_bstride, Atb, diag, s);
}
int thb_gram_f32(const thb_gram_plan* p, int64_t B, const float* A_val, int64_t nnz, const float* b, int64_t m, float* out,
                 int64_t out_bstride, float* Atb, float* diag, thb_stream_t s) {
  return gram_impl<float>(p, B, A_val, nnz, b, m, out, out_bstride, Atb, diag, s);
}

int thb_mat_vec_f64(int64_t B, int64_t num_rows, int64_t num_cols, const int64_t* row_ptr, const int64_t* col_ind,
                    const double* A_val, const double* v, double* y, thb_stream_t s) {
  if (B <= 0 || num_rows <= 0) return THB_OK;
  const int64_t total = B * num_rows;
  thb::mat_vec_kernel<double><<<(unsigned)((total + 255) / 256), 256, 0, thb_cs(s)>>>(B, num_rows, num_cols, row_ptr, col_ind, A_val, v, y);
  THB_CHECK_LAUNCH();
  return THB_OK;
}
int thb_solve_backward_f64(int64_t B, int64_t num_rows, int64_t num_cols, const int64_t* row_ptr, const int64_t* col_ind,
                           const double* A_val, const double* b, const double* x, const double* H, const double* alpha,
                           int32_t detach_hessian, double* A_grad, double* b_grad, thb_stream_t s) {
  if (row_ptr == nullptr || col_ind == nullptr || A_val == nullptr || b == nullptr || x == nullptr || H == nullptr) return THB_ERR_BAD_ARG;
  if (B <= 0 || num_rows <= 0) return THB_OK;
  const int64_t total = B * num_rows;
  thb::solve_backward_kernel<<<(unsigned)((total + 255) / 256), 256, 0, thb_cs(s)>>>(B, num_rows, num_cols, row_ptr, col_ind, A_val, b, x, H, alpha,
                                                                                     detach_hessian, A_grad, b_grad);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

int thb_tmat_vec_f64(int64_t B, int64_t num_rows, int64_t num_cols, const int64_t* row_ptr, const int64_t* col_ind,
                     const double* A_val, const double* v, double* y, thb_stream_t s) {
  if (B <= 0 || num_cols <= 0) return THB_OK;
  const int64_t total = B * num_cols;
  thb::tmat_vec_kernel<double><<<(unsigned)((total + 255) / 256), 256, 0, thb_cs(s)>>>(B, num_rows, num_cols, row_ptr, col_ind, A_val, v, y);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

}  // extern "C"
