// Shared helpers for libthb200 translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/thb200.h"

// every kernel launch of the library goes through this macro: it also counts launches (thb_launch_count)
extern "C" int64_t thb_launch_counter_;
#define THB_CHECK_LAUNCH()                               \
  do {                                                   \
    ++thb_launch_counter_;                               \
    cudaError_t _e = cudaGetLastError();                 \
    if (_e != cudaSuccess) return static_cast<int>(_e);  \
  } while (0)

#define THB_CUDA(x)                                      \
  do {                                                   \
    cudaError_t _e = (x);                                \
    if (_e != cudaSuccess) return static_cast<int>(_e);  \
  } while (0)

static inline cudaStream_t thb_cs(thb_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// Number of CTAs resident per SM is decided per kernel; grids are sized in multiples of the SM count
// where a grid-stride loop is used.
static inline int thb_sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Big fronts of the multifrontal factor (thb_front.cu) factored by the dense kernel of thb_chol_dense.cu straight into their panel in
// the factor storage: where that kernel gathers the front's initial tiles from and where the L of its pivot columns goes.
struct ThbCholDirect {
  const int64_t* fd;           // the front's flat descriptor (frontal.py): panel offset, children
  const int64_t* pc;           // per (parent, child) records: update-matrix offset and leading dimension, rows reached, inverse-map offset
  const int32_t* c_inv;        // inverse maps: front row -> child border row, or -1
  const int32_t* pmap;         // panel element -> compact AtA offset, or -1 (with ata)
  double* factor;              // [B, data_size]
  int64_t data_size;
  const double* arena_child;   // [B, arena_size] the children's update matrices
  int64_t arena_size;
  const double* ata;           // [B, ata_stride] compact AtA, or null: the panel holds AtA
  int64_t ata_stride;
  const double* alpha;         // [B] or null
  const double* beta;          // [B] or null
  int w, b, wpad;              // pivots, border rows, pivots padded to the 64-column block
};
extern "C" int thb_potrf_partial_direct_f64(double* F, int64_t bstride, int64_t np, int32_t nb_piv, int32_t n_real, int32_t info_base,
                                            int32_t* info, int64_t B, void* workspace, int64_t workspace_bytes, const ThbCholDirect* direct,
                                            thb_stream_t stream);
