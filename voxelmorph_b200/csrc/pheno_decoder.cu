// The phenotype decoder of ConditionalTemplateCreation (reference voxelmorph/tf/networks.py:856-983): a rank-P Dense
// layer that expands the subject attributes into a full-resolution F-channel image, ELU, and neurite's conv_dec with no
// levels, i.e. one 1x1 convolution F -> F with bias and a linear activation.
//
// For pheno (B, P), W (P, F, V), bias (F, V), like_w (F, F) (output channel g, input channel f), like_b (F):
//   pre[b,f,v] = bias[f,v] + sum_p pheno[b,p] W[p,f,v]      (fma chain in p order, starting from bias)
//   h          = pre > 0 ? pre : expm1f(pre)                 (ELU, alpha 1)
//   out[b,g,v] = like_b[g] + sum_f like_w[g,f] h[b,f,v]      (fma chain in f order, starting from like_b)
// Backward (nothing is stored: pre and h are recomputed from W, bias and pheno in the forward's order, bit for bit):
//   g_h[b,f]  = sum_g like_w[g,f] g_out[b,g]                 (g order),  g_pre = g_h (h < 0 ? h + 1 : 1)   (TF EluGrad)
//   gW[p,f,v] = sum_b pheno[b,p] g_pre[b,f,v],  gbias[f,v] = sum_b g_pre[b,f,v]                        (b order)
//   g_like_w[g,f] = sum_{b,v} g_out[b,g,v] h[b,f,v],  g_like_b[g] = sum_{b,v} g_out[b,g,v]
// The two voxel sums run per thread in fp32, across a warp by a fixed shuffle tree, across warps and CTAs in fp64 in
// index order (one partial per CTA, summed by the CTA that takes the last ticket): the result is bit-deterministic.
//
// Both passes stream the per-voxel weights once: a thread owns voxels and loops over the batch inside, in chunks of BC
// entries whose accumulators stay in registers (BC F <= 64, so W is read once for B <= 64 / F, rounded down to 1, 2 or
// 4; a larger batch re-reads W once per chunk, and gW / gbias are then added to chunk by chunk).  Traffic per voxel, fp32: forward P F + F + B F words; backward
// P F + F + B F words read and P F + F written, twice P F + F more when it accumulates into existing gradients.
#include "common.cuh"

namespace vxm {

constexpr int kPdMaxP = 16, kPdMaxF = 32;
constexpr int kPdHeader = 256;  // workspace: ticket counter, then fp64 partials [grid][F F + F]
constexpr int kPdMaxCtas = 1024;  // backward grid cap: the workspace size is host arithmetic

__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : expm1f(x); }

struct PdArgs {
  const float *pheno, *W, *bias, *like_w, *like_b;
  int B, P, F;
  size_t V;
};

// FM >= F: the channel loops are unrolled over FM and guarded by F, so the per-thread arrays stay in registers
template <int FM, int BC>
__global__ void __launch_bounds__(256) pd_fwd_kernel(PdArgs a, float* __restrict__ out) {
  __shared__ float s_lw[FM * FM], s_lb[FM];
  const int F = a.F, P = a.P;
  for (int i = threadIdx.x; i < F * F; i += blockDim.x) s_lw[(i / F) * FM + i % F] = a.like_w[i];
  for (int i = threadIdx.x; i < F; i += blockDim.x) s_lb[i] = a.like_b[i];
  __syncthreads();
  const size_t V = a.V;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < V; v += (size_t)gridDim.x * blockDim.x) {
    for (int b0 = 0; b0 < a.B; b0 += BC) {
      const int nb = min(BC, a.B - b0);
      float acc[BC][FM];
#pragma unroll
      for (int j = 0; j < BC; ++j)
#pragma unroll
        for (int g = 0; g < FM; ++g) acc[j][g] = s_lb[g < F ? g : 0];
#pragma unroll
      for (int f = 0; f < FM; ++f) {
        if (f >= F) break;
        const float bf = __ldcs(a.bias + (size_t)f * V + v);
        float pre[BC];
#pragma unroll
        for (int j = 0; j < BC; ++j) pre[j] = bf;
        for (int p = 0; p < P; ++p) {
          const float w = __ldcs(a.W + ((size_t)p * F + f) * V + v);
#pragma unroll
          for (int j = 0; j < BC; ++j)
            if (j < nb) pre[j] = fmaf(__ldg(a.pheno + (size_t)(b0 + j) * P + p), w, pre[j]);
        }
#pragma unroll
        for (int j = 0; j < BC; ++j) {
          const float h = elu1(pre[j]);
#pragma unroll
          for (int g = 0; g < FM; ++g) acc[j][g] = fmaf(s_lw[g * FM + f], h, acc[j][g]);
        }
      }
#pragma unroll
      for (int j = 0; j < BC; ++j) {
        if (j >= nb) break;
#pragma unroll
        for (int g = 0; g < FM; ++g)
          if (g < F) __stcs(out + ((size_t)(b0 + j) * F + g) * V + v, acc[j][g]);
      }
    }
  }
}

// Per-thread accumulators of the 1x1 convolution's gradients: registers for FM <= 4, otherwise one shared-memory slot
// per (entry, thread), entry k = g F + f for like_w and F F + g for like_b
template <int FM, bool REG>
struct LikeAcc;
template <int FM>
struct LikeAcc<FM, true> {
  float w[FM][FM], b[FM];
  __device__ __forceinline__ void init(float*, int) {
#pragma unroll
    for (int g = 0; g < FM; ++g) {
      b[g] = 0.f;
#pragma unroll
      for (int f = 0; f < FM; ++f) w[g][f] = 0.f;
    }
  }
  __device__ __forceinline__ void add_w(int g, int f, float x) { w[g][f] += x; }
  __device__ __forceinline__ void add_b(int g, float x) { b[g] += x; }
  __device__ __forceinline__ float get(int k, int F) const {
    float r = 0.f;
#pragma unroll
    for (int g = 0; g < FM; ++g) {
      if (g >= F) break;
      if (k == F * F + g) r = b[g];
#pragma unroll
      for (int f = 0; f < FM; ++f)
        if (f < F && k == g * F + f) r = w[g][f];
    }
    return r;
  }
};
template <int FM>
struct LikeAcc<FM, false> {
  float* slot;  // [K][blockDim.x]
  int F, T;
  __device__ __forceinline__ void init(float* smem, int F_) {
    slot = smem + threadIdx.x;
    F = F_;
    T = blockDim.x;
    for (int k = 0; k < F * F + F; ++k) slot[(size_t)k * T] = 0.f;
  }
  __device__ __forceinline__ void add_w(int g, int f, float x) { slot[(size_t)(g * F + f) * T] += x; }
  __device__ __forceinline__ void add_b(int g, float x) { slot[(size_t)(F * F + g) * T] += x; }
  __device__ __forceinline__ float get(int k, int) const { return slot[(size_t)k * T]; }
};

template <int FM, int BC>
__global__ void __launch_bounds__(256) pd_bwd_kernel(PdArgs a, const float* __restrict__ gout, float* __restrict__ gW,
                                                     float* __restrict__ gbias, float* __restrict__ g_like_w,
                                                     float* __restrict__ g_like_b, unsigned char* __restrict__ work,
                                                     int accumulate) {
  constexpr bool REG = FM <= 4;
  extern __shared__ float dyn[];  // REG: [nwarps][K] warp sums; else [K][T] slots, then [nwarps][K]
  __shared__ float s_lw[FM * FM];
  __shared__ bool s_last;
  const int F = a.F, P = a.P, K = F * F + F, T = blockDim.x, nw = (T + 31) / 32;
  float* wsum = REG ? dyn : dyn + (size_t)K * T;
  for (int i = threadIdx.x; i < F * F; i += T) s_lw[(i / F) * FM + i % F] = a.like_w[i];
  LikeAcc<FM, REG> la;
  la.init(dyn, F);
  __syncthreads();
  const size_t V = a.V;
  for (size_t v = (size_t)blockIdx.x * T + threadIdx.x; v < V; v += (size_t)gridDim.x * T) {
    for (int b0 = 0; b0 < a.B; b0 += BC) {
      const int nb = min(BC, a.B - b0);
      const bool acc_old = accumulate || b0 > 0;
      float go[BC][FM];
#pragma unroll
      for (int j = 0; j < BC; ++j)
#pragma unroll
        for (int g = 0; g < FM; ++g) {
          go[j][g] = (j < nb && g < F) ? __ldcs(gout + ((size_t)(b0 + j) * F + g) * V + v) : 0.f;
          if (j < nb && g < F) la.add_b(g, go[j][g]);
        }
#pragma unroll
      for (int f = 0; f < FM; ++f) {
        if (f >= F) break;
        float pre[BC], gp[BC];
        const float bf = __ldcs(a.bias + (size_t)f * V + v);
#pragma unroll
        for (int j = 0; j < BC; ++j) pre[j] = bf;
        for (int p = 0; p < P; ++p) {
          const float w = __ldcs(a.W + ((size_t)p * F + f) * V + v);
#pragma unroll
          for (int j = 0; j < BC; ++j)
            if (j < nb) pre[j] = fmaf(__ldg(a.pheno + (size_t)(b0 + j) * P + p), w, pre[j]);
        }
#pragma unroll
        for (int j = 0; j < BC; ++j) {
          const float h = elu1(pre[j]);
          float gh = 0.f;
#pragma unroll
          for (int g = 0; g < FM; ++g)
            if (g < F) {
              gh = fmaf(s_lw[g * FM + f], go[j][g], gh);
              if (j < nb) la.add_w(g, f, go[j][g] * h);
            }
          gp[j] = j < nb ? gh * (h < 0.f ? h + 1.f : 1.f) : 0.f;
        }
        float sb = gp[0];
#pragma unroll
        for (int j = 1; j < BC; ++j)
          if (j < nb) sb += gp[j];
        float* pb = gbias + (size_t)f * V + v;
        *pb = acc_old ? *pb + sb : sb;
        for (int p = 0; p < P; ++p) {
          float s = __ldg(a.pheno + (size_t)b0 * P + p) * gp[0];
#pragma unroll
          for (int j = 1; j < BC; ++j)
            if (j < nb) s = fmaf(__ldg(a.pheno + (size_t)(b0 + j) * P + p), gp[j], s);
          float* pw = gW + ((size_t)p * F + f) * V + v;
          *pw = acc_old ? *pw + s : s;
        }
      }
    }
  }
  // CTA partials of the 1x1 convolution's gradients: warp shuffle tree, then warps in order, in fp64
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int k = 0; k < K; ++k) {
    float x = warp_sum(la.get(k, F));
    if (lane == 0) wsum[wid * K + k] = x;
  }
  __syncthreads();
  double* partials = reinterpret_cast<double*>(work + kPdHeader);
  for (int k = threadIdx.x; k < K; k += T) {
    double s = 0.0;
    for (int w = 0; w < nw; ++w) s += (double)wsum[w * K + k];
    partials[(size_t)blockIdx.x * K + k] = s;
  }
  __threadfence();
  __syncthreads();
  unsigned int* counter = reinterpret_cast<unsigned int*>(work);
  if (threadIdx.x == 0) {
    s_last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int k = threadIdx.x; k < K; k += T) {
    double s = 0.0;
    for (unsigned int c = 0; c < gridDim.x; ++c) s += __ldcg(partials + (size_t)c * K + k);
    float* dst = k < F * F ? g_like_w + k : g_like_b + (k - F * F);
    *dst = accumulate ? *dst + (float)s : (float)s;
  }
  if (threadIdx.x == 0) *counter = 0u;
}

static int pd_fm(int F) { return F <= 4 ? 4 : F <= 8 ? 8 : F <= 16 ? 16 : 32; }
static int pd_bc(int B, int FM) {
  int cap = 64 / FM < 4 ? 64 / FM : 4;
  int bc = B <= 1 ? 1 : B <= 2 ? 2 : 4;
  return bc < cap ? bc : cap;
}
static int pd_fwd_grid(size_t V) {
  size_t b = (V + 255) / 256, cap = (size_t)sm_count() * 8;
  return (int)(b > cap ? cap : b);
}
// backward CTA size: 256 threads, fewer when the shared-memory slots of F > 4 would exceed 100 KB
static int pd_bwd_threads(int F) {
  if (pd_fm(F) <= 4) return 256;
  int T = 256;
  const size_t K = (size_t)F * F + F;
  while (T > 32 && (size_t)T * K * 4 > 100 * 1024) T /= 2;
  return T;
}
static size_t pd_bwd_smem(int F, int T) {
  const size_t K = (size_t)F * F + F;
  return (pd_fm(F) <= 4 ? 0 : (size_t)T * K * 4) + (size_t)((T + 31) / 32) * K * 4;
}
static int pd_bwd_grid(size_t V, int T) {
  size_t b = (V + T - 1) / T, cap = (size_t)sm_count() * 4;
  cap = cap < (size_t)kPdMaxCtas ? cap : (size_t)kPdMaxCtas;
  return (int)(b > cap ? cap : b);
}

template <int FM, int BC>
static void pd_fwd_launch(const PdArgs& a, float* out, cudaStream_t s) {
  pd_fwd_kernel<FM, BC><<<pd_fwd_grid(a.V), 256, 0, s>>>(a, out);
}

template <int FM, int BC>
static int pd_bwd_launch(const PdArgs& a, const float* gout, float* gW, float* gbias, float* glw, float* glb, void* work,
                         int accumulate, cudaStream_t s) {
  const int T = pd_bwd_threads(a.F);
  const size_t smem = pd_bwd_smem(a.F, T);
  if (smem > 48 * 1024) VXM_CUDA(cudaFuncSetAttribute(pd_bwd_kernel<FM, BC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                      (int)smem));
  pd_bwd_kernel<FM, BC><<<pd_bwd_grid(a.V, T), T, smem, s>>>(a, gout, gW, gbias, glw, glb, (unsigned char*)work,
                                                             accumulate);
  return VXM_OK;
}

#define PD_DISPATCH(FN, ...)                                               \
  switch (pd_fm(a.F) * 8 + pd_bc(a.B, pd_fm(a.F))) {                        \
    case 4 * 8 + 1: FN<4, 1>(__VA_ARGS__); break;                           \
    case 4 * 8 + 2: FN<4, 2>(__VA_ARGS__); break;                           \
    case 4 * 8 + 4: FN<4, 4>(__VA_ARGS__); break;                           \
    case 8 * 8 + 1: FN<8, 1>(__VA_ARGS__); break;                           \
    case 8 * 8 + 2: FN<8, 2>(__VA_ARGS__); break;                           \
    case 8 * 8 + 4: FN<8, 4>(__VA_ARGS__); break;                           \
    case 16 * 8 + 1: FN<16, 1>(__VA_ARGS__); break;                         \
    case 16 * 8 + 2: FN<16, 2>(__VA_ARGS__); break;                         \
    case 16 * 8 + 4: FN<16, 4>(__VA_ARGS__); break;                         \
    case 32 * 8 + 1: FN<32, 1>(__VA_ARGS__); break;                         \
    default: FN<32, 2>(__VA_ARGS__); break;                                 \
  }

static int pd_check(int B, int P, int F, size_t V, const char* what) {
  VXM_REQUIRE(B > 0 && V > 0, "%s: non-positive size (B %d, V %zu)", what, B, V);
  VXM_REQUIRE(P >= 1 && P <= kPdMaxP, "%s: P = %d phenotype attributes, the kernel takes 1 to %d", what, P, kPdMaxP);
  VXM_REQUIRE(F >= 1 && F <= kPdMaxF, "%s: F = %d channels, the kernel takes 1 to %d", what, F, kPdMaxF);
  return VXM_OK;
}

}  // namespace vxm

using namespace vxm;

extern "C" size_t vxm_pheno_decoder_workspace_bytes(int F) {
  if (F < 1 || F > kPdMaxF) return 0;
  return kPdHeader + sizeof(double) * ((size_t)F * F + F) * kPdMaxCtas;
}

extern "C" int vxm_pheno_decoder_fwd(const float* pheno, const float* W, const float* bias, const float* like_w,
                                     const float* like_b, float* out, int B, int P, int F, size_t V, void* stream) {
  VXM_REQUIRE(pheno && W && bias && like_w && like_b && out, "pheno_decoder_fwd: null pointer");
  if (int rc = pd_check(B, P, F, V, "pheno_decoder_fwd")) return rc;
  PdArgs a{pheno, W, bias, like_w, like_b, B, P, F, V};
  PD_DISPATCH(pd_fwd_launch, a, out, as_stream(stream));
  return check_launch("pheno_decoder_fwd");
}

extern "C" int vxm_pheno_decoder_bwd(const float* grad_out, const float* pheno, const float* W, const float* bias,
                                     const float* like_w, float* grad_W, float* grad_bias, float* grad_like_w,
                                     float* grad_like_b, void* work, int B, int P, int F, size_t V, int accumulate,
                                     void* stream) {
  VXM_REQUIRE(grad_out && pheno && W && bias && like_w && grad_W && grad_bias && grad_like_w && grad_like_b && work,
              "pheno_decoder_bwd: null pointer");
  if (int rc = pd_check(B, P, F, V, "pheno_decoder_bwd")) return rc;
  VXM_REQUIRE(accumulate == 0 || accumulate == 1, "pheno_decoder_bwd: accumulate must be 0 or 1, got %d", accumulate);
  PdArgs a{pheno, W, bias, like_w, nullptr, B, P, F, V};
  int rc = VXM_OK;
  PD_DISPATCH(rc = pd_bwd_launch, a, grad_out, grad_W, grad_bias, grad_like_w, grad_like_b, work, accumulate,
              as_stream(stream));
  if (rc) return rc;
  return check_launch("pheno_decoder_bwd");
}
