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
