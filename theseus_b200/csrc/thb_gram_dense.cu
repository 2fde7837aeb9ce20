// Dense batched Gram  AtA[b] = A[b]^T A[b]  (fp64) for GENUINELY dense Jacobians, sm_90a: TMA-staged tiles + the FP64 tensor pipe.
//
// Replaces `At.bmm(A)` of theseus/optimizer/dense_linearization.py:58-62 for cost functions whose Jacobian is dense (AutoDiffCostFunction
// with dim >> dof: the block-sparse Gram of thb_gram.cu covers pose graphs / bundle adjustment, where A is 99 % structural zeros).
//   * A is [B, m, n] row-major.  One 3-D TMA tensor map over (n, m, B); boxes of (68 columns x 32 rows x 1 item): the 4 extra columns
//     give the staged tile a row pitch of 68 doubles (= 4 mod 16), which makes the DMMA fragment loads below bank-conflict free without a
//     swizzle; rows / columns past the matrix are zero-filled by the TMA unit, so ragged m and n need no special case in the main loop.
//   * CTA = one 64 x 64 tile (i-block, j-block <= i-block) of one item's AtA; 4 warps x (32 x 32) warp tiles; k runs over the m rows in
//     steps of 32 through a 3-stage ring: thread 0 arms an mbarrier with the stage's byte count and issues cp.async.bulk.tensor for the
//     two column blocks, everybody waits on the barrier's phase, multiplies (mma.sync m8n8k4 f64: wgmma has no fp64 kind) and meets at
//     a __syncthreads() before the slot is refilled.
//   * both operands come from the same rows of A: A-operand  a[i][k] = A[k][i0 + i], B-operand  b[k][j] = A[k][j0 + j].
//   * the tile is written to (i, j) and mirrored to (j, i): AtA is the full symmetric matrix like the reference's.
#include <cuda.h>

#include "thb_common.cuh"

namespace thb {

constexpr int GD_T = 64;          // output tile
constexpr int GD_BOX = 68;        // staged columns per block (row pitch in shared memory, doubles)
constexpr int GD_K = 32;          // rows of A per stage
constexpr int GD_STAGES = 3;
constexpr int GD_THREADS = 128;
constexpr int GD_STAGE_DOUBLES = 2 * GD_K * GD_BOX;                       // i-block + j-block
constexpr size_t GD_SMEM = (size_t)GD_STAGES * GD_STAGE_DOUBLES * 8 + 128 + 64;   // + alignment slack + barriers

__device__ __forceinline__ void gd_mma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ uint32_t gd_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void gd_mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(gd_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void gd_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(gd_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool gd_mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
      : "=r"(ok)
      : "r"(gd_smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void gd_tma_load_3d(void* dst, const CUtensorMap* tm, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];\n" ::"r"(gd_smem_u32(dst)),
      "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(gd_smem_u32(bar))
      : "memory");
}

__global__ void __launch_bounds__(GD_THREADS) gram_dense_kernel(const __grid_constant__ CUtensorMap tmap, double* __restrict__ AtA, int64_t m,
                                                                int64_t n, int nt) {
  extern __shared__ uint8_t gd_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(gd_raw) + 127) & ~uintptr_t(127));   // TMA destinations: 128-byte aligned
  double* stages = reinterpret_cast<double*>(base);
  uint64_t* full = reinterpret_cast<uint64_t*>(base + (size_t)GD_STAGES * GD_STAGE_DOUBLES * 8);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int lr = lane >> 2, lc = lane & 3;
  const int64_t item = blockIdx.y;
  // tile pair (ti >= tj) from the linear index
  int ti = (int)((sqrtf(8.0f * (float)blockIdx.x + 1.0f) - 1.0f) * 0.5f);
  while ((ti + 1) * (ti + 2) / 2 <= (int)blockIdx.x) ti++;
  while (ti * (ti + 1) / 2 > (int)blockIdx.x) ti--;
  const int tj = (int)blockIdx.x - ti * (ti + 1) / 2;
  (void)nt;
  const bool diag = (ti == tj);
  const int nk = (int)((m + GD_K - 1) / GD_K);
  const uint32_t stage_bytes = (uint32_t)((diag ? 1 : 2) * GD_K * GD_BOX * 8);
  if (tid == 0) {
    for (int s = 0; s < GD_STAGES; s++) gd_mbar_init(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int kt) {
    const int s = kt % GD_STAGES;
    double* dst = stages + (size_t)s * GD_STAGE_DOUBLES;
    gd_mbar_expect_tx(&full[s], stage_bytes);
    gd_tma_load_3d(dst, &tmap, ti * GD_T, kt * GD_K, (int)item, &full[s]);
    if (!diag) gd_tma_load_3d(dst + GD_K * GD_BOX, &tmap, tj * GD_T, kt * GD_K, (int)item, &full[s]);
  };
  if (tid == 0)
    for (int kt = 0; kt < GD_STAGES - 1 && kt < nk; kt++) issue(kt);
  const int wi = warp >> 1, wj = warp & 1;   // 2 x 2 warps, 32 x 32 each
  double acc[4][4][2];
#pragma unroll
  for (int mi = 0; mi < 4; mi++)
#pragma unroll
    for (int ni = 0; ni < 4; ni++) acc[mi][ni][0] = acc[mi][ni][1] = 0.0;
  for (int kt = 0; kt < nk; kt++) {
    if (tid == 0 && kt + GD_STAGES - 1 < nk) issue(kt + GD_STAGES - 1);   // refills the slot everybody left at the previous __syncthreads
    const int s = kt % GD_STAGES;
    const uint32_t parity = (uint32_t)((kt / GD_STAGES) & 1);
    while (!gd_mbar_try_wait(&full[s], parity)) {
    }
    const double* As = stages + (size_t)s * GD_STAGE_DOUBLES;
    const double* Bs = diag ? As : As + GD_K * GD_BOX;
#pragma unroll
    for (int k4 = 0; k4 < GD_K; k4 += 4) {
      double a[4], b[4];
#pragma unroll
      for (int mi = 0; mi < 4; mi++) a[mi] = As[(k4 + lc) * GD_BOX + wi * 32 + mi * 8 + lr];
#pragma unroll
      for (int ni = 0; ni < 4; ni++) b[ni] = Bs[(k4 + lc) * GD_BOX + wj * 32 + ni * 8 + lr];
#pragma unroll
      for (int mi = 0; mi < 4; mi++)
#pragma unroll
        for (int ni = 0; ni < 4; ni++) gd_mma884(acc[mi][ni][0], acc[mi][ni][1], a[mi], b[ni]);
    }
    __syncthreads();
  }
  double* C = AtA + item * n * n;
#pragma unroll
  for (int mi = 0; mi < 4; mi++) {
    const int64_t gi = (int64_t)ti * GD_T + wi * 32 + mi * 8 + lr;
#pragma unroll
    for (int ni = 0; ni < 4; ni++) {
#pragma unroll
      for (int u = 0; u < 2; u++) {
        const int64_t gj = (int64_t)tj * GD_T + wj * 32 + ni * 8 + lc * 2 + u;
        if (gi < n && gj < n) {
          const double v = acc[mi][ni][u];
          C[gi * n + gj] = v;
          if (!diag) C[gj * n + gi] = v;
        }
      }
    }
  }
}

typedef CUresult (*gd_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                 const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static gd_encode_fn gd_get_encode() {
  static gd_encode_fn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<gd_encode_fn>(p);
  }
  return fn;
}

}  // namespace thb

extern "C" {

/* AtA [B,n,n] = A^T A for A [B,m,n] row-major fp64 (dense_linearization.py:58-62).  n must be even (TMA: global strides are multiples of
 * 16 bytes) and A 16-byte aligned; the Python host pads an odd n with a zero column. */
int thb_gram_dense_f64(const double* A, double* AtA, int64_t B, int64_t m, int64_t n, thb_stream_t stream) {
  if (A == nullptr || AtA == nullptr || B < 0 || m < 0 || n < 0) return THB_ERR_BAD_ARG;
  if (B == 0 || n == 0) return THB_OK;
  if (m == 0) {
    THB_CUDA(cudaMemsetAsync(AtA, 0, (size_t)(B * n * n) * 8, thb_cs(stream)));
    return THB_OK;
  }
  if ((n & 1) != 0 || (reinterpret_cast<uintptr_t>(A) & 15) != 0 || B > 65535 || m >= (1LL << 31) || n >= (1LL << 31)) return THB_ERR_UNSUPPORTED;
  thb::gd_encode_fn encode = thb::gd_get_encode();
  if (encode == nullptr) return THB_ERR_UNSUPPORTED;
  CUtensorMap tm;
  const cuuint64_t gdim[3] = {(cuuint64_t)n, (cuuint64_t)m, (cuuint64_t)B};
  const cuuint64_t gstride[2] = {(cuuint64_t)n * 8, (cuuint64_t)m * (cuuint64_t)n * 8};
  const cuuint32_t box[3] = {(cuuint32_t)thb::GD_BOX, (cuuint32_t)thb::GD_K, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = encode(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, const_cast<double*>(A), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return THB_ERR_UNSUPPORTED;
  static bool attr_set = false;
  if (!attr_set) {
    THB_CUDA(cudaFuncSetAttribute(thb::gram_dense_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)thb::GD_SMEM));
    attr_set = true;
  }
  const int nt = (int)((n + thb::GD_T - 1) / thb::GD_T);
  const dim3 grid((unsigned)(nt * (nt + 1) / 2), (unsigned)B);
  thb::gram_dense_kernel<<<grid, thb::GD_THREADS, thb::GD_SMEM, thb_cs(stream)>>>(tm, AtA, m, n, nt);
  THB_CHECK_LAUNCH();
  return THB_OK;
}

}  // extern "C"
