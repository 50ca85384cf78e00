// MeanStream (neurite's MeanStream(cap), the layer TemplateCreation wraps around the inverse flow): a capped running
// mean over every batch seen in training, carried as device state so that a step stays graph-capturable.
//
// For x (B, n) (n = nd * voxels, any dimensionality), state mean (n) and count (1):
//   S = sum_b x_b,  n' = count + B,  alpha = B / min(n', cap),  m' = mean (1 - alpha) + (S / B) alpha,
//   out = min(1, n' / cap) m'   (one copy; the caller broadcasts it over the batch),
//   training: mean <- m', count <- n'.   d out / d x_b = min(1, n' / cap) alpha / B  (nothing flows into the state).
//
// Both passes are memory bound: the forward moves 4 (B + 3) bytes per element with the commit (x, mean in, mean out,
// out), 4 (B + 2) without; the backward 8 B.  Sums over b run in a fixed order in fp32 (no data atomics): results are
// bit-reproducible.  count, alpha and the output scale never leave the device: every block reads the pre-step count
// from memory before it takes its ticket, and the block that takes the last ticket commits n', so no block can see the
// new count (the ticket counter is the reduce workspace's, zero on entry and reset on exit).
#include "common.cuh"

namespace vxm {

ReduceWork as_reduce_work(void* work);  // ncc.cu

struct MsScalars {
  float n1, alpha, scale;
};

__device__ __forceinline__ MsScalars ms_scalars(float count, int B, float cap) {
  MsScalars s;
  s.n1 = count + (float)B;
  s.alpha = (float)B / fminf(s.n1, cap);
  s.scale = fminf(1.f, s.n1 / cap);
  return s;
}

template <int V>
struct Vec;
template <>
struct Vec<1> {
  using T = float;
};
template <>
struct Vec<4> {
  using T = float4;
};

__device__ __forceinline__ float4 operator+(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 operator*(float a, float4 b) { return make_float4(a * b.x, a * b.y, a * b.z, a * b.w); }

// V floats per access (4 when n % 4 == 0: every x_b then starts 16-byte aligned); n is counted in V-wide elements
template <int V>
__global__ void __launch_bounds__(256) mean_stream_fwd_kernel(const typename Vec<V>::T* __restrict__ x,
                                                              typename Vec<V>::T* __restrict__ mean,
                                                              float* __restrict__ count, typename Vec<V>::T* __restrict__ out,
                                                              float* __restrict__ saved, unsigned int* __restrict__ ticket,
                                                              int B, size_t n, float cap, int commit) {
  using T = typename Vec<V>::T;
  __shared__ float s_count;
  if (threadIdx.x == 0) s_count = __ldcg(count);
  __syncthreads();
  const MsScalars s = ms_scalars(s_count, B, cap);
  const float invB = 1.f / (float)B, keep = 1.f - s.alpha;
  if (blockIdx.x == 0 && threadIdx.x == 0) saved[0] = s.scale * s.alpha * invB;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    T acc = __ldcs(x + i);
    for (int b = 1; b < B; ++b) acc = acc + __ldcs(x + (size_t)b * n + i);
    T m = keep * __ldcs(mean + i) + s.alpha * (invB * acc);
    if (commit) __stcs(mean + i, m);
    __stcs(out + i, s.scale * m);
  }
  if (!commit) return;
  // last-block commit: the ticket is taken after this block's read of count (thread 0, above), so the block that takes
  // the last one writes n' once every block has read the pre-step value
  if (threadIdx.x == 0) {
    __threadfence();
    unsigned int t = atomicAdd(ticket, 1u);
    if (t == gridDim.x - 1) {
      *count = s.n1;
      *ticket = 0u;
    }
  }
}

template <int V>
__global__ void __launch_bounds__(256) mean_stream_bwd_kernel(const typename Vec<V>::T* __restrict__ gout,
                                                              const float* __restrict__ saved,
                                                              typename Vec<V>::T* __restrict__ gx, int B, size_t n,
                                                              size_t gstride) {
  using T = typename Vec<V>::T;
  const float g = __ldg(saved);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    T acc = __ldcs(gout + i);
    for (int b = 1; b < B; ++b) acc = acc + __ldcs(gout + (size_t)b * gstride + i);
    T v = g * acc;
    for (int b = 0; b < B; ++b) __stcs(gx + (size_t)b * n + i, v);
  }
}

static int ms_grid(size_t n) {
  size_t b = (n + 255) / 256;
  size_t cap = (size_t)sm_count() * 8;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace vxm

using namespace vxm;

extern "C" int vxm_mean_stream_fwd(const float* x, float* mean, float* count, float* out, float* saved, void* work,
                                   int B, size_t n, float cap, int commit, void* stream) {
  VXM_REQUIRE(x && mean && count && out && saved && work, "mean_stream_fwd: null pointer");
  VXM_REQUIRE(B > 0 && n > 0, "mean_stream_fwd: non-positive size (B %d, n %zu)", B, n);
  VXM_REQUIRE(cap > 0.f, "mean_stream_fwd: cap must be positive, got %g", (double)cap);
  VXM_REQUIRE(commit == 0 || commit == 1, "mean_stream_fwd: commit must be 0 or 1, got %d", commit);
  unsigned int* ticket = as_reduce_work(work).counter;
  if (n % 4 == 0 && aligned16(x) && aligned16(mean) && aligned16(out)) {
    size_t n4 = n / 4;
    mean_stream_fwd_kernel<4><<<ms_grid(n4), 256, 0, as_stream(stream)>>>(
        (const float4*)x, (float4*)mean, count, (float4*)out, saved, ticket, B, n4, cap, commit);
  } else {
    mean_stream_fwd_kernel<1><<<ms_grid(n), 256, 0, as_stream(stream)>>>(x, mean, count, out, saved, ticket, B, n, cap,
                                                                         commit);
  }
  return check_launch("mean_stream_fwd");
}

extern "C" int vxm_mean_stream_bwd(const float* grad_out, const float* saved, float* grad_x, int B, size_t n,
                                   size_t gout_bstride, void* stream) {
  VXM_REQUIRE(grad_out && saved && grad_x, "mean_stream_bwd: null pointer");
  VXM_REQUIRE(B > 0 && n > 0, "mean_stream_bwd: non-positive size (B %d, n %zu)", B, n);
  VXM_REQUIRE(gout_bstride == 0 || gout_bstride == n, "mean_stream_bwd: grad_out batch stride must be 0 or n, got %zu",
              gout_bstride);
  if (n % 4 == 0 && aligned16(grad_out) && aligned16(grad_x)) {
    mean_stream_bwd_kernel<4><<<ms_grid(n / 4), 256, 0, as_stream(stream)>>>((const float4*)grad_out, saved,
                                                                             (float4*)grad_x, B, n / 4, gout_bstride / 4);
  } else {
    mean_stream_bwd_kernel<1><<<ms_grid(n), 256, 0, as_stream(stream)>>>(grad_out, saved, grad_x, B, n, gout_bstride);
  }
  return check_launch("mean_stream_bwd");
}
