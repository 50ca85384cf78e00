// HyperMorph (Hoopes et al., IPMI 2021; reference voxelmorph/tf/networks.py:1192-1231): a hypernetwork maps the
// regularisation weight(s) hyp (1, P) to every U-Net convolution weight and bias.
//
// The hypernetwork (one CTA each way): nb_layers Dense layers of U units, each followed by ReLU.  Weights are stored as
// torch.nn.Linear's (out, in): layer 0 is (U, P), the others (U, U).
//   pre_0[u] = b_0[u] + sum_p W_0[u,p] hyp[p],  pre_l[u] = b_l[u] + sum_k W_l[u,k] relu(pre_{l-1})[k]   (fma chains in
//   index order, starting from the bias),  h = relu(pre_{L-1})
// The backward takes dh and walks the layers down: g_pre = g (pre > 0), grad_b = g_pre, grad_W[u,k] = g_pre[u] x[k],
// g_x[k] = sum_u W[u,k] g_pre[u] (u order); no gradient is formed for hyp.
//
// The generated weights, for A = hyper_kernel (U, N) row-major and a = hyper_bias (N):
//   Wflat[j] = a[j] + sum_k h[k] A[k,j]                 (fma chain in k order, starting from a[j])
// and their backward, given the flat gradient dW (N):
//   grad_A[k,j] = h[k] dW[j],  grad_a[j] = dW[j],  dh[k] = sum_j A[k,j] dW[j]
// Both passes stream A once; threads run along j, so every row of A is read coalesced, with 16-, 8- or 4-byte loads
// (the widest that N and the pointers' alignment allow).  dh is summed per lane over a 1024-column tile, across the warp
// by a fixed shuffle tree, then over tiles in tile order in fp64 by a second one-CTA launch: bit-deterministic, and
// independent of the device's SM count.
#include "common.cuh"

namespace vxm {

constexpr int kHypMaxP = 16, kHypMaxU = 256, kHypMaxLayers = 8;
constexpr int kHypTile = 1024;     // columns per CTA of the weight backward: one dh partial per (tile, k)
constexpr int kHypThreads = 256;

struct HypMlp {
  const float* w[kHypMaxLayers];
  const float* b[kHypMaxLayers];
  float* gw[kHypMaxLayers];
  float* gb[kHypMaxLayers];
};

__global__ void __launch_bounds__(kHypThreads) hyper_mlp_fwd_kernel(HypMlp m, const float* __restrict__ hyp,
                                                                  float* __restrict__ pre, float* __restrict__ h,
                                                                  int P, int U, int L) {
  __shared__ float x[kHypMaxU];
  for (int l = 0; l < L; ++l) {
    const int in = l == 0 ? P : U;
    const float* src = l == 0 ? hyp : x;
    float acc = 0.f;
    const int u = threadIdx.x;
    if (u < U) {
      acc = m.b[l][u];
      for (int k = 0; k < in; ++k) acc = fmaf(m.w[l][(size_t)u * in + k], src[k], acc);
      pre[(size_t)l * U + u] = acc;
    }
    __syncthreads();                       // every thread has read x
    if (u < U) x[u] = fmaxf(acc, 0.f);
    __syncthreads();
  }
  if (threadIdx.x < U) h[threadIdx.x] = x[threadIdx.x];
}

__global__ void __launch_bounds__(kHypThreads) hyper_mlp_bwd_kernel(HypMlp m, const float* __restrict__ dh,
                                                                  const float* __restrict__ hyp,
                                                                  const float* __restrict__ pre, int P, int U, int L,
                                                                  int accumulate) {
  __shared__ float g[kHypMaxU], x[kHypMaxU];
  const int T = blockDim.x;
  for (int u = threadIdx.x; u < U; u += T) g[u] = dh[u];
  for (int l = L - 1; l >= 0; --l) {
    const int in = l == 0 ? P : U;
    __syncthreads();
    for (int u = threadIdx.x; u < U; u += T) {
      g[u] = pre[(size_t)l * U + u] > 0.f ? g[u] : 0.f;                      // TF's ReluGrad
      float* pb = m.gb[l] + u;
      *pb = accumulate ? __fadd_rn(*pb, g[u]) : g[u];
    }
    for (int k = threadIdx.x; k < in; k += T) x[k] = l == 0 ? hyp[k] : fmaxf(pre[(size_t)(l - 1) * U + k], 0.f);
    __syncthreads();
    for (int i = threadIdx.x; i < U * in; i += T) {
      const float v = __fmul_rn(g[i / in], x[i % in]);
      float* pw = m.gw[l] + i;
      *pw = accumulate ? __fadd_rn(*pw, v) : v;
    }
    if (l == 0) break;
    float s = 0.f;
    if (threadIdx.x < U)
      for (int u = 0; u < U; ++u) s = fmaf(m.w[l][(size_t)u * U + threadIdx.x], g[u], s);
    __syncthreads();                       // every thread has read g
    if (threadIdx.x < U) g[threadIdx.x] = s;
  }
}

template <int VEC>
struct VecT;
template <>
struct VecT<4> {
  using T = float4;
};
template <>
struct VecT<2> {
  using T = float2;
};
template <>
struct VecT<1> {
  using T = float;
};

template <int VEC>
__device__ __forceinline__ void vload(const float* p, float (&v)[VEC], bool stream) {
  using T = typename VecT<VEC>::T;
  const T t = stream ? __ldcs(reinterpret_cast<const T*>(p)) : *reinterpret_cast<const T*>(p);
  const float* f = reinterpret_cast<const float*>(&t);
#pragma unroll
  for (int i = 0; i < VEC; ++i) v[i] = f[i];
}

template <int VEC>
__device__ __forceinline__ void vstore(float* p, const float (&v)[VEC]) {
  using T = typename VecT<VEC>::T;
  T t;
  float* f = reinterpret_cast<float*>(&t);
#pragma unroll
  for (int i = 0; i < VEC; ++i) f[i] = v[i];
  *reinterpret_cast<T*>(p) = t;
}

template <int VEC>
__global__ void __launch_bounds__(kHypThreads) hyper_weights_fwd_kernel(const float* __restrict__ h,
                                                                      const float* __restrict__ A,
                                                                      const float* __restrict__ a,
                                                                      float* __restrict__ W, int U, size_t N) {
  __shared__ float sh[kHypMaxU];
  for (int k = threadIdx.x; k < U; k += blockDim.x) sh[k] = h[k];
  __syncthreads();
  const size_t j = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * VEC;
  if (j >= N) return;
  float acc[VEC];
  vload<VEC>(a + j, acc, false);
  const float* col = A + j;
  int k = 0;
  for (; k + 8 <= U; k += 8) {
    float v[8][VEC];
#pragma unroll
    for (int r = 0; r < 8; ++r) vload<VEC>(col + (size_t)(k + r) * N, v[r], true);
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] = fmaf(sh[k + r], v[r][i], acc[i]);
  }
  for (; k < U; ++k) {
    float v[VEC];
    vload<VEC>(col + (size_t)k * N, v, true);
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = fmaf(sh[k], v[i], acc[i]);
  }
  vstore<VEC>(W + j, acc);
}

// One CTA per kHypTile columns: the CTA stages dW of its tile in shared memory (and writes grad_a), then warp w takes rows
// k = w, w + 8, ...: its lanes stream A[k, tile] and write grad_A[k, tile], and the warp's dot product of the row with
// dW becomes partial[tile][k].
template <int VEC>
__global__ void __launch_bounds__(kHypThreads) hyper_weights_bwd_kernel(const float* __restrict__ h,
                                                                      const float* __restrict__ A,
                                                                      const float* __restrict__ dW,
                                                                      float* __restrict__ gA, float* __restrict__ ga,
                                                                      float* __restrict__ partial, int U, size_t N,
                                                                      int accumulate) {
  __shared__ __align__(16) float sdw[kHypTile];
  __shared__ float sh[kHypMaxU];
  const size_t c0 = (size_t)blockIdx.x * kHypTile;
  const int ncol = (int)(N - c0 < (size_t)kHypTile ? N - c0 : (size_t)kHypTile);
  for (int i = threadIdx.x; i < kHypTile; i += blockDim.x) {
    float d = 0.f;
    if (i < ncol) {
      d = dW[c0 + i];
      ga[c0 + i] = accumulate ? __fadd_rn(ga[c0 + i], d) : d;
    }
    sdw[i] = d;
  }
  for (int k = threadIdx.x; k < U; k += blockDim.x) sh[k] = h[k];
  __syncthreads();
  const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  constexpr int kIters = kHypTile / (32 * VEC);
  for (int k = threadIdx.x >> 5; k < U; k += nw) {
    const float hk = sh[k];
    const float* row = A + (size_t)k * N + c0;
    float* grow = gA + (size_t)k * N + c0;
    float s = 0.f;
#pragma unroll 4
    for (int it = 0; it < kIters; ++it) {
      const int c = (it * 32 + lane) * VEC;
      if (c >= ncol) break;
      float v[VEC], d[VEC], g[VEC];
      vload<VEC>(row + c, v, true);
#pragma unroll
      for (int i = 0; i < VEC; ++i) d[i] = sdw[c + i];
      if (accumulate) vload<VEC>(grow + c, g, false);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        s = fmaf(v[i], d[i], s);
        const float p = __fmul_rn(hk, d[i]);
        g[i] = accumulate ? __fadd_rn(g[i], p) : p;
      }
      vstore<VEC>(grow + c, g);
    }
    s = warp_sum(s);
    if (lane == 0) partial[(size_t)blockIdx.x * U + k] = s;
  }
}

__global__ void __launch_bounds__(kHypThreads) hyper_dh_reduce_kernel(const float* __restrict__ partial,
                                                                    float* __restrict__ dh, int U, int tiles) {
  for (int k = threadIdx.x; k < U; k += blockDim.x) {
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s += (double)partial[(size_t)t * U + k];
    dh[k] = (float)s;
  }
}

static int hyp_tiles(size_t N) { return (int)((N + kHypTile - 1) / kHypTile); }

static bool aligned(const void* p, size_t bytes) { return (reinterpret_cast<uintptr_t>(p) % bytes) == 0; }

// widest vector width that N and every row-streamed pointer allow
static int hyp_vec(size_t N, std::initializer_list<const void*> ptrs) {
  for (int vec : {4, 2}) {
    bool ok = N % vec == 0;
    for (const void* p : ptrs) ok = ok && aligned(p, sizeof(float) * vec);
    if (ok) return vec;
  }
  return 1;
}

static int hyp_check_mlp(int P, int U, int L, const char* what) {
  VXM_REQUIRE(P >= 1 && P <= kHypMaxP, "%s: P = %d hyperparameters, the kernel takes 1 to %d", what, P, kHypMaxP);
  VXM_REQUIRE(U >= 1 && U <= kHypMaxU, "%s: U = %d units, the kernel takes 1 to %d", what, U, kHypMaxU);
  VXM_REQUIRE(L >= 1 && L <= kHypMaxLayers, "%s: %d layers, the kernel takes 1 to %d", what, L, kHypMaxLayers);
  return VXM_OK;
}

static int hyp_check_weights(int U, size_t N, const char* what) {
  VXM_REQUIRE(U >= 1 && U <= kHypMaxU, "%s: U = %d units, the kernel takes 1 to %d", what, U, kHypMaxU);
  VXM_REQUIRE(N >= 1, "%s: N = 0 generated values", what);
  return VXM_OK;
}

}  // namespace vxm

using namespace vxm;

extern "C" size_t vxm_hyper_workspace_bytes(int U, size_t N) {
  if (U < 1 || U > kHypMaxU || N < 1) return 0;
  return sizeof(float) * (size_t)U * hyp_tiles(N);
}

extern "C" int vxm_hyper_mlp_fwd(const float* hyp, const float* const* weights, const float* const* biases, float* pre,
                                 float* h, int P, int U, int nb_layers, void* stream) {
  VXM_REQUIRE(hyp && weights && biases && pre && h, "hyper_mlp_fwd: null pointer");
  if (int rc = hyp_check_mlp(P, U, nb_layers, "hyper_mlp_fwd")) return rc;
  HypMlp m{};
  for (int l = 0; l < nb_layers; ++l) {
    VXM_REQUIRE(weights[l] && biases[l], "hyper_mlp_fwd: null pointer (layer %d)", l);
    m.w[l] = weights[l];
    m.b[l] = biases[l];
  }
  hyper_mlp_fwd_kernel<<<1, kHypThreads, 0, as_stream(stream)>>>(m, hyp, pre, h, P, U, nb_layers);
  return check_launch("hyper_mlp_fwd");
}

extern "C" int vxm_hyper_mlp_bwd(const float* grad_h, const float* hyp, const float* const* weights, const float* pre,
                                 float* const* grad_weights, float* const* grad_biases, int P, int U, int nb_layers,
                                 int accumulate, void* stream) {
  VXM_REQUIRE(grad_h && hyp && weights && pre && grad_weights && grad_biases, "hyper_mlp_bwd: null pointer");
  if (int rc = hyp_check_mlp(P, U, nb_layers, "hyper_mlp_bwd")) return rc;
  VXM_REQUIRE(accumulate == 0 || accumulate == 1, "hyper_mlp_bwd: accumulate must be 0 or 1, got %d", accumulate);
  HypMlp m{};
  for (int l = 0; l < nb_layers; ++l) {
    VXM_REQUIRE(weights[l] && grad_weights[l] && grad_biases[l], "hyper_mlp_bwd: null pointer (layer %d)", l);
    m.w[l] = weights[l];
    m.gw[l] = grad_weights[l];
    m.gb[l] = grad_biases[l];
  }
  hyper_mlp_bwd_kernel<<<1, kHypThreads, 0, as_stream(stream)>>>(m, grad_h, hyp, pre, P, U, nb_layers, accumulate);
  return check_launch("hyper_mlp_bwd");
}

extern "C" int vxm_hyper_weights_fwd(const float* h, const float* A, const float* a, float* W, int U, size_t N,
                                     void* stream) {
  VXM_REQUIRE(h && A && a && W, "hyper_weights_fwd: null pointer");
  if (int rc = hyp_check_weights(U, N, "hyper_weights_fwd")) return rc;
  const int vec = hyp_vec(N, {A, a, W});
  const size_t groups = N / vec;
  const unsigned grid = (unsigned)((groups + kHypThreads - 1) / kHypThreads);
  cudaStream_t s = as_stream(stream);
  if (vec == 4) hyper_weights_fwd_kernel<4><<<grid, kHypThreads, 0, s>>>(h, A, a, W, U, N);
  else if (vec == 2) hyper_weights_fwd_kernel<2><<<grid, kHypThreads, 0, s>>>(h, A, a, W, U, N);
  else hyper_weights_fwd_kernel<1><<<grid, kHypThreads, 0, s>>>(h, A, a, W, U, N);
  return check_launch("hyper_weights_fwd");
}

extern "C" int vxm_hyper_weights_bwd(const float* h, const float* A, const float* grad_W, float* grad_A, float* grad_a,
                                     float* grad_h, void* work, int U, size_t N, int accumulate, void* stream) {
  VXM_REQUIRE(h && A && grad_W && grad_A && grad_a && grad_h && work, "hyper_weights_bwd: null pointer");
  if (int rc = hyp_check_weights(U, N, "hyper_weights_bwd")) return rc;
  VXM_REQUIRE(accumulate == 0 || accumulate == 1, "hyper_weights_bwd: accumulate must be 0 or 1, got %d", accumulate);
  const int vec = hyp_vec(N, {A, grad_A});
  const int tiles = hyp_tiles(N);
  float* partial = static_cast<float*>(work);
  cudaStream_t s = as_stream(stream);
  if (vec == 4) hyper_weights_bwd_kernel<4><<<tiles, kHypThreads, 0, s>>>(h, A, grad_W, grad_A, grad_a, partial, U, N, accumulate);
  else if (vec == 2) hyper_weights_bwd_kernel<2><<<tiles, kHypThreads, 0, s>>>(h, A, grad_W, grad_A, grad_a, partial, U, N, accumulate);
  else hyper_weights_bwd_kernel<1><<<tiles, kHypThreads, 0, s>>>(h, A, grad_W, grad_A, grad_a, partial, U, N, accumulate);
  if (int rc = check_launch("hyper_weights_bwd")) return rc;
  hyper_dh_reduce_kernel<<<1, kHypThreads, 0, s>>>(partial, grad_h, U, tiles);
  return check_launch("hyper_dh_reduce");
}
