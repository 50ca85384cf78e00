// The reparameterised sampler of probabilistic diffeomorphic VoxelMorph (reference voxelmorph/tf/networks.py:155-165,
// neurite's SampleNormalLogVar): z = mu + exp(logvar / 2) * eps, eps ~ N(0, 1), with eps drawn in the kernel from a
// counter-based generator, so that no noise tensor is stored and the backward regenerates it.
//
// Stream (restated in numpy by tests/probs_ref.py): Philox4x32-10 keyed by the 64-bit seed; element
// i = (b * nd + c) * V + v of z takes word i mod 4 of the block with counter (lo32(i / 4), hi32(i / 4), lo32(call),
// hi32(call)).  Box-Muller on the word pairs (0, 1) and (2, 3):
//   u1 = ((w_even >> 8) + 1) 2^-24 in (0, 1],  u2 = (w_odd >> 8) 2^-24 in [0, 1)   (both exact in fp32),
//   r = sqrt(-2 log u1),  eps_even = r cos(2 pi u2),  eps_odd = r sin(2 pi u2).
// eps depends on (seed, call, i) only: not on the launch geometry.
//
// State: noise_state = (seed, call) int64 on the device.  The forward reads call, writes it to an 8-byte ticket for its
// backward, and advances it by one; the block that takes the last ticket of the launch commits call + 1 once every block
// has read the old value (the counter is the reduce workspace's, zero on entry and reset on exit), so no host read is
// needed and a captured step draws fresh noise on every replay.
//
// Bytes per element of z: forward 12 (mu, logvar in; z out), backward 16 (dz, logvar in; dmu, dlogvar out).
#include "common.cuh"

namespace vxm {

ReduceWork as_reduce_work(void* work);  // ncc.cu

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, unsigned int k0, unsigned int k1) {
  const unsigned int M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += W0; k1 += W1; }
    unsigned int hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
    unsigned int hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

__device__ __forceinline__ float2 box_muller(unsigned int a, unsigned int b) {
  float u1 = (float)((a >> 8) + 1u) * 0x1p-24f;
  float u2 = (float)(b >> 8) * 0x1p-24f;
  float r = sqrtf(-2.f * logf(u1));
  float s, c;
  sincospif(2.f * u2, &s, &c);
  return make_float2(r * c, r * s);
}

// the four normals of counter block q
__device__ __forceinline__ float4 normals4(unsigned long long q, unsigned long long seed, unsigned long long call) {
  uint4 w = philox4x32_10(make_uint4((unsigned int)q, (unsigned int)(q >> 32), (unsigned int)call, (unsigned int)(call >> 32)),
                          (unsigned int)seed, (unsigned int)(seed >> 32));
  float2 e01 = box_muller(w.x, w.y), e23 = box_muller(w.z, w.w);
  return make_float4(e01.x, e01.y, e23.x, e23.y);
}

__device__ __forceinline__ float f4_get(const float4& v, int j) { return j == 0 ? v.x : (j == 1 ? v.y : (j == 2 ? v.z : v.w)); }

struct SampleGeom {
  size_t V, n;  // voxels per plane, elements of z (B * nd * V)
  int nd;
};

// offsets of mu and logvar of z element i in the (B, 2 nd, V) parameters
__device__ __forceinline__ size_t mu_off(size_t i, const SampleGeom& g) {
  size_t bc = i / g.V, v = i - bc * g.V, b = bc / g.nd;
  return (bc + b * g.nd) * g.V + v;
}

// VEC: V % 4 == 0, so the four elements of a counter block share one plane (float4 accesses)
template <bool VEC>
__global__ void __launch_bounds__(256) sample_fwd_kernel(const float* __restrict__ params, float* __restrict__ z,
                                                         long long* state, long long* __restrict__ ticket,
                                                         unsigned int* __restrict__ counter, SampleGeom g) {
  __shared__ unsigned long long s_seed, s_call;
  if (threadIdx.x == 0) {
    s_seed = (unsigned long long)__ldcg(state);
    s_call = (unsigned long long)__ldcg(state + 1);
  }
  __syncthreads();
  const unsigned long long seed = s_seed, call = s_call;
  const size_t nq = (g.n + 3) / 4, lv = (size_t)g.nd * g.V;
  for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += (size_t)gridDim.x * blockDim.x) {
    float4 e = normals4(q, seed, call);
    if (VEC) {
      size_t m = mu_off(4 * q, g);
      float4 mu = __ldcs(reinterpret_cast<const float4*>(params + m));
      float4 lv4 = __ldcs(reinterpret_cast<const float4*>(params + m + lv));
      float4 o = make_float4(fmaf(expf(0.5f * lv4.x), e.x, mu.x), fmaf(expf(0.5f * lv4.y), e.y, mu.y),
                             fmaf(expf(0.5f * lv4.z), e.z, mu.z), fmaf(expf(0.5f * lv4.w), e.w, mu.w));
      __stcs(reinterpret_cast<float4*>(z + 4 * q), o);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        size_t i = 4 * q + j;
        if (i < g.n) {
          size_t m = mu_off(i, g);
          z[i] = fmaf(expf(0.5f * __ldcs(params + m + lv)), f4_get(e, j), __ldcs(params + m));
        }
      }
    }
  }
  // last-block commit (see the header): every block has read call before it takes its ticket
  if (threadIdx.x == 0) {
    __threadfence();
    unsigned int t = atomicAdd(counter, 1u);
    if (t == gridDim.x - 1) {
      *ticket = (long long)call;
      state[1] = (long long)(call + 1);
      *counter = 0u;
    }
  }
}

template <bool VEC>
__global__ void __launch_bounds__(256) sample_bwd_kernel(const float* __restrict__ gz, const float* __restrict__ params,
                                                         const long long* __restrict__ state,
                                                         const long long* __restrict__ ticket,
                                                         float* __restrict__ gparams, SampleGeom g) {
  const unsigned long long seed = (unsigned long long)__ldg(state), call = (unsigned long long)__ldg(ticket);
  const size_t nq = (g.n + 3) / 4, lv = (size_t)g.nd * g.V;
  for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += (size_t)gridDim.x * blockDim.x) {
    float4 e = normals4(q, seed, call);
    if (VEC) {
      size_t m = mu_off(4 * q, g);
      float4 d = __ldcs(reinterpret_cast<const float4*>(gz + 4 * q));
      float4 l = __ldcs(reinterpret_cast<const float4*>(params + m + lv));
      __stcs(reinterpret_cast<float4*>(gparams + m), d);
      float4 o = make_float4(d.x * e.x * (0.5f * expf(0.5f * l.x)), d.y * e.y * (0.5f * expf(0.5f * l.y)),
                             d.z * e.z * (0.5f * expf(0.5f * l.z)), d.w * e.w * (0.5f * expf(0.5f * l.w)));
      __stcs(reinterpret_cast<float4*>(gparams + m + lv), o);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        size_t i = 4 * q + j;
        if (i < g.n) {
          size_t m = mu_off(i, g);
          float d = __ldcs(gz + i);
          gparams[m] = d;
          gparams[m + lv] = d * f4_get(e, j) * (0.5f * expf(0.5f * __ldcs(params + m + lv)));
        }
      }
    }
  }
}

static int sample_grid(size_t n) {
  size_t b = ((n + 3) / 4 + 255) / 256;
  size_t cap = (size_t)sm_count() * 8;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

static bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace vxm

using namespace vxm;

extern "C" int vxm_sample_normal_logvar_fwd(const float* params, float* z, long long* state, long long* ticket, void* work,
                                            int B, int nd, size_t V, void* stream) {
  VXM_REQUIRE(params && z && state && ticket && work, "sample_normal_logvar_fwd: null pointer");
  VXM_REQUIRE(B > 0 && nd > 0 && V > 0, "sample_normal_logvar_fwd: non-positive size (B %d, nd %d, V %zu)", B, nd, V);
  SampleGeom g{V, (size_t)B * nd * V, nd};
  unsigned int* counter = as_reduce_work(work).counter;
  if (V % 4 == 0 && aligned16(params) && aligned16(z))
    sample_fwd_kernel<true><<<sample_grid(g.n), 256, 0, as_stream(stream)>>>(params, z, state, ticket, counter, g);
  else
    sample_fwd_kernel<false><<<sample_grid(g.n), 256, 0, as_stream(stream)>>>(params, z, state, ticket, counter, g);
  return check_launch("sample_normal_logvar_fwd");
}

extern "C" int vxm_sample_normal_logvar_bwd(const float* grad_z, const float* params, const long long* state,
                                            const long long* ticket, float* grad_params, int B, int nd, size_t V,
                                            void* stream) {
  VXM_REQUIRE(grad_z && params && state && ticket && grad_params, "sample_normal_logvar_bwd: null pointer");
  VXM_REQUIRE(B > 0 && nd > 0 && V > 0, "sample_normal_logvar_bwd: non-positive size (B %d, nd %d, V %zu)", B, nd, V);
  SampleGeom g{V, (size_t)B * nd * V, nd};
  if (V % 4 == 0 && aligned16(grad_z) && aligned16(params) && aligned16(grad_params))
    sample_bwd_kernel<true><<<sample_grid(g.n), 256, 0, as_stream(stream)>>>(grad_z, params, state, ticket, grad_params, g);
  else
    sample_bwd_kernel<false><<<sample_grid(g.n), 256, 0, as_stream(stream)>>>(grad_z, params, state, ticket, grad_params, g);
  return check_launch("sample_normal_logvar_bwd");
}
