// Shared helpers for the vxm_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/vxm_b200.h"

namespace vxm {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
int check_launch(const char* what);  // cudaGetLastError -> VXM_OK / VXM_ERR_CUDA (+ counts one launch)
int sm_count();
int conv_ctas();                     // sm_count(), capped by VXM_B200_CONV_CTAS (tensor-core convolution grids)

#define VXM_REQUIRE(cond, ...)          \
  do {                                  \
    if (!(cond)) {                      \
      vxm::set_error(__VA_ARGS__);      \
      return VXM_ERR_ARG;               \
    }                                   \
  } while (0)

#define VXM_CUDA(call)                                                          \
  do {                                                                          \
    cudaError_t e_ = (call);                                                    \
    if (e_ != cudaSuccess) {                                                    \
      vxm::set_error("%s failed: %s", #call, cudaGetErrorString(e_));           \
      return VXM_ERR_CUDA;                                                      \
    }                                                                           \
  } while (0)

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// ------------------------------------------------------------------------------------
// Sampling-coordinate arithmetic of the reference resampler, replayed op for op in fp32
// with explicit round-to-nearest intrinsics (no FMA contraction):
//   layers.py:32   loc = grid + flow
//   layers.py:37   n   = 2 * (loc / (S-1) - 0.5)
//   ATen GridSampler.h:27-31 (align_corners)   coord = ((n + 1) / 2) * (Ssrc - 1)
// ------------------------------------------------------------------------------------
struct AxisNorm {
  float sm1;      // float(S_flow - 1)
  float inv_sm1;  // fl(1 / (S_flow - 1))
  float src_sm1;  // float(S_src - 1)
};

__host__ inline AxisNorm make_axis(int s_flow, int s_src) {
  AxisNorm a;
  a.sm1 = (float)(s_flow - 1);
  a.inv_sm1 = 1.0f / a.sm1;
  a.src_sm1 = (float)(s_src - 1);
  return a;
}

template <int ARITH>
__device__ __forceinline__ float sample_coord(float idx, float f, const AxisNorm& a) {
  float loc = __fadd_rn(idx, f);
  float t = (ARITH == VXM_ARITH_TRUE_DIV) ? __fdiv_rn(loc, a.sm1) : __fmul_rn(loc, a.inv_sm1);
  float u = __fsub_rn(t, 0.5f);
  float n = __fmul_rn(2.0f, u);
  float v = __fadd_rn(n, 1.0f);
  return __fmul_rn(__fmul_rn(v, 0.5f), a.src_sm1);
}

// float -> int with saturation (cvt.rzi saturates; NaN -> 0), safe for wild coordinates
__device__ __forceinline__ int f2i(float x) { return __float2int_rz(x); }

// ------------------------------------------------------------------------------------
// Block reduction (sum) in double; result valid in thread 0.
// ------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* smem /* >= 32 entries */) {
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
  lane = tid & 31;
  wid = tid >> 5;
  int nw = (blockDim.x * blockDim.y * blockDim.z + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  if (wid == 0) {
    v = (lane < nw) ? smem[lane] : T(0);
    v = warp_sum(v);
  }
  return v;
}

// Deterministic two-stage scalar reduction: every block writes its partial (double) to
// partials[blockIdx], the last block to finish (ticket counter) sums them in index order and
// writes  out[0] = float(scale * total).  `counter` must be zero on entry and is reset on exit.
struct ReduceWork {
  double* partials;       // >= grid size entries
  unsigned int* counter;  // 1 entry, zero-initialised once at allocation
};
constexpr int kMaxReduceBlocks = 4096;

__device__ __forceinline__ void finish_reduce(double block_total, const ReduceWork& rw, int nblocks,
                                              int bid, double scale, float* out, double* smem) {
  __shared__ bool is_last;
  int tid = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
  int nthreads = blockDim.x * blockDim.y * blockDim.z;
  if (tid == 0) {
    rw.partials[bid] = block_total;
    __threadfence();
    unsigned int t = atomicAdd(rw.counter, 1u);
    is_last = (t == (unsigned int)(nblocks - 1));
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    double acc = 0.0;
    for (int i = tid; i < nblocks; i += nthreads) acc += __ldcg(&rw.partials[i]);
    acc = block_sum<double>(acc, smem);
    if (tid == 0) {
      out[0] = (float)(acc * scale);
      *rw.counter = 0u;
    }
  }
}

}  // namespace vxm
