// Host emulation of the CUDA execution model for tests (NOT part of the product): the batch-lane kernels of
// theseus_b200/csrc/thb_sparse_lane.cu are compiled unchanged (tests/simt/build_emu.py rewrites only the <<<...>>> launches and the
// dynamic shared-memory declaration) and every CUDA thread of a block runs as an OS thread; __syncthreads() is a std::barrier from which
// exited threads drop out, like on the device.  Blocks run one after another.  This checks index arithmetic, work partitioning across
// warps, shared-memory layouts and barrier placement without a GPU; it says nothing about performance or about memory-model subtleties.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <barrier>
#include <memory>
#include <thread>
#include <vector>

#include "../../include/thb200.h"

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct double2 { double x, y; };
struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
inline thread_local dim3 threadIdx, blockIdx, blockDim, gridDim;
inline std::barrier<>* simt_block_barrier = nullptr;
// warp-level exchange for __shfl_*_sync: the 32 threads of a warp meet at their own barrier around a 32-slot buffer
struct SimtWarp {
  std::barrier<> bar;
  unsigned long long slot[32];
  explicit SimtWarp(int n) : bar(n) {}
};
inline thread_local SimtWarp* simt_warp = nullptr;
inline thread_local int simt_lane = 0;
template <typename T>
inline T __shfl_xor_sync(unsigned, T v, int lane_mask) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  memcpy(&simt_warp->slot[simt_lane], &v, sizeof(T));
  simt_warp->bar.arrive_and_wait();
  T r;
  memcpy(&r, &simt_warp->slot[(simt_lane ^ lane_mask) & 31], sizeof(T));
  simt_warp->bar.arrive_and_wait();
  return r;
}
template <typename T>
inline T __shfl_sync(unsigned, T v, int src_lane) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  memcpy(&simt_warp->slot[simt_lane], &v, sizeof(T));
  simt_warp->bar.arrive_and_wait();
  T r;
  memcpy(&r, &simt_warp->slot[src_lane & 31], sizeof(T));
  simt_warp->bar.arrive_and_wait();
  return r;
}
inline void __syncwarp(unsigned = 0xffffffffu) { simt_warp->bar.arrive_and_wait(); }
inline int atomicAdd(int* addr, int val) { return __sync_fetch_and_add(addr, val); }
inline char* simt_dyn_smem_ptr = nullptr;
inline void __syncthreads() { simt_block_barrier->arrive_and_wait(); }
template <typename T> inline T* simt_dyn_smem() { return reinterpret_cast<T*>(simt_dyn_smem_ptr); }

inline double rsqrt(double x) { return 1.0 / sqrt(x); }
inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
using std::max;
using std::min;
inline int atomicCAS(int* addr, int compare, int val) { return __sync_val_compare_and_swap(addr, compare, val); }

typedef void* cudaStream_t;
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaDevAttrMultiProcessorCount = 16 };
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, int, int) { *v = 132; return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
template <typename K> inline cudaError_t cudaFuncSetAttribute(K, int, int) { return cudaSuccess; }
extern "C" int64_t thb_launch_counter_;   // defined by thb_costs.cu, like in the product
#define THB_CHECK_LAUNCH() do { ++thb_launch_counter_; } while (0)
#define THB_CUDA(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return static_cast<int>(_e); } while (0)
static inline cudaStream_t thb_cs(thb_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

template <typename K, typename... A>
void simt_launch(K kernel, dim3 grid, dim3 block, size_t smem_bytes, A... args) {
  const unsigned nthreads = block.x * block.y * block.z;
  std::vector<char> smem(smem_bytes + 16);
  for (unsigned bz = 0; bz < grid.z; bz++)
    for (unsigned by = 0; by < grid.y; by++)
      for (unsigned bx = 0; bx < grid.x; bx++) {
        std::barrier<> bar(nthreads);
        simt_block_barrier = &bar;
        simt_dyn_smem_ptr = smem.data();
        std::vector<std::unique_ptr<SimtWarp>> warps;
        for (unsigned w = 0; w * 32 < nthreads; w++) warps.emplace_back(new SimtWarp((int)std::min(32u, nthreads - 32 * w)));
        std::vector<std::thread> ts;
        ts.reserve(nthreads);
        for (unsigned t = 0; t < nthreads; t++)
          ts.emplace_back([&, t]() {
            threadIdx = dim3(t % block.x, (t / block.x) % block.y, t / (block.x * block.y));
            blockIdx = dim3(bx, by, bz);
            blockDim = block;
            gridDim = grid;
            simt_warp = warps[t / 32].get();
            simt_lane = (int)(t % 32);
            kernel(args...);
            simt_warp->bar.arrive_and_drop();
            bar.arrive_and_drop();  // an exited thread no longer takes part in the block's barriers
          });
        for (auto& th : ts) th.join();
      }
}
#define SIMT_LAUNCH(kernel, grid, block, smem, ...) simt_launch(kernel, dim3(grid), dim3(block), (size_t)(smem), __VA_ARGS__)
