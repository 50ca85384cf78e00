// Channels-last bf16 glue kernels of the tensor-core U-Net engine: MaxPool(2) forward, and the two fused
// gradient-routing kernels of the backward pass (reference voxelmorph/torch/networks.py:126-138 under autograd):
//   sumpool_mask   : gradient through nearest-x2 upsampling (sum over the 2^nd children) times the LeakyReLU
//                    derivative of the (coarse) decoder activation it belongs to;
//   unpool_combine : gradient through MaxPool(2) (routed to the first maximal child, ATen's tie rule) plus the
//                    skip-connection gradient, times the LeakyReLU derivative of the encoder activation (a split
//                    variant routes to the child the split-precision pool chose on hi + lo).
// All tensors are bf16 (B, D, H, W, C) with C % 8 == 0; one thread moves 8 channels (16 bytes) per voxel.
// These are HBM-bound: algorithmic bytes = every operand once.
#include <cuda_bf16.h>

#include "common.cuh"

namespace vxm {

struct V8 {
  float v[8];
};
__device__ __forceinline__ V8 ld8(const __nv_bfloat16* p) {
  uint4 q = __ldg(reinterpret_cast<const uint4*>(p));
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
  V8 r;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __bfloat1622float2(h[i]);
    r.v[2 * i] = f.x;
    r.v[2 * i + 1] = f.y;
  }
  return r;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const V8& r) {
  uint4 q;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&q);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(r.v[2 * i], r.v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = q;
}

struct PoolGeom {
  int B, Dc, Hc, Wc, C8, fd;  // coarse dims, channel chunks, depth factor (2 or 1)
};

__device__ __forceinline__ bool decode(const PoolGeom& g, size_t i, int& b, int& d, int& h, int& w, int& c8) {
  size_t n = (size_t)g.B * g.Dc * g.Hc * g.Wc * g.C8;
  if (i >= n) return false;
  c8 = (int)(i % g.C8);
  size_t v = i / g.C8;
  w = (int)(v % g.Wc); v /= g.Wc;
  h = (int)(v % g.Hc); v /= g.Hc;
  d = (int)(v % g.Dc);
  b = (int)(v / g.Dc);
  return true;
}
__device__ __forceinline__ size_t fine_index(const PoolGeom& g, int b, int d, int h, int w, int kd, int kh, int kw) {
  return ((((size_t)b * (g.Dc * g.fd) + (d * g.fd + kd)) * (g.Hc * 2) + (h * 2 + kh)) * (size_t)(g.Wc * 2) + (w * 2 + kw));
}

__global__ void __launch_bounds__(256) pool_ndhwc_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, PoolGeom g) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int b, d, h, w, c8;
  if (!decode(g, i, b, d, h, w, c8)) return;
  const int C = g.C8 * 8;
  V8 m;
#pragma unroll
  for (int e = 0; e < 8; ++e) m.v[e] = -INFINITY;
  for (int kd = 0; kd < g.fd; ++kd)
    for (int kh = 0; kh < 2; ++kh)
      for (int kw = 0; kw < 2; ++kw) {
        V8 t = ld8(x + fine_index(g, b, d, h, w, kd, kh, kw) * C + c8 * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e) m.v[e] = (t.v[e] > m.v[e] || t.v[e] != t.v[e]) ? t.v[e] : m.v[e];
      }
  st8(y + ((((size_t)b * g.Dc + d) * g.Hc + h) * g.Wc + w) * C + c8 * 8, m);
}

__global__ void __launch_bounds__(256) sumpool_mask_kernel(const __nv_bfloat16* __restrict__ gf, const __nv_bfloat16* __restrict__ act,
                                                           __nv_bfloat16* __restrict__ out, PoolGeom g, float slope) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int b, d, h, w, c8;
  if (!decode(g, i, b, d, h, w, c8)) return;
  const int C = g.C8 * 8;
  V8 s;
#pragma unroll
  for (int e = 0; e < 8; ++e) s.v[e] = 0.f;
  for (int kd = 0; kd < g.fd; ++kd)
    for (int kh = 0; kh < 2; ++kh)
      for (int kw = 0; kw < 2; ++kw) {
        V8 t = ld8(gf + fine_index(g, b, d, h, w, kd, kh, kw) * C + c8 * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e) s.v[e] += t.v[e];
      }
  const size_t co = ((((size_t)b * g.Dc + d) * g.Hc + h) * g.Wc + w) * C + c8 * 8;
  if (act) {
    V8 a = ld8(act + co);
#pragma unroll
    for (int e = 0; e < 8; ++e) if (a.v[e] < 0.f) s.v[e] *= slope;
  }
  st8(out + co, s);
}

// The split-precision MaxPool's choice, shared by its forward (pool_split_ndhwc_kernel) and its backward
// (unpool_combine_kernel<true>): child (h, l) replaces the best so far when h + l is larger or NaN, so the first child with
// the largest h + l wins ties (ATen's rule on the value the pair carries).
__device__ __forceinline__ bool split_pool_takes(float h, float l, float& best) {
  const float t = h + l;
  if (t > best || t != t) {
    best = t;
    return true;
  }
  return false;
}

// SPLIT: the forward was the split-precision one, whose pool chose on hi + lo; e_fine holds hi and e_lo the lo parts.
// The LeakyReLU derivative reads the sign of hi, as every other mask of the (bf16-operand) backward does.
template <bool SPLIT>
__global__ void __launch_bounds__(256) unpool_combine_kernel(const __nv_bfloat16* __restrict__ e_fine, const __nv_bfloat16* __restrict__ g_skip,
                                                             const __nv_bfloat16* __restrict__ g_pool, __nv_bfloat16* __restrict__ out,
                                                             PoolGeom g, float slope, const __nv_bfloat16* __restrict__ e_lo) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int b, d, h, w, c8;
  if (!decode(g, i, b, d, h, w, c8)) return;
  const int C = g.C8 * 8;
  V8 ev[8];
  int arg[8];
  float best[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; arg[e] = 0; }
  const int nchild = g.fd * 4;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k < nchild) {
      const int kd = g.fd == 2 ? (k >> 2) : 0, kh = (k >> 1) & 1, kw = k & 1;
      ev[k] = ld8(e_fine + fine_index(g, b, d, h, w, kd, kh, kw) * C + c8 * 8);
      if constexpr (SPLIT) {
        const V8 el = ld8(e_lo + fine_index(g, b, d, h, w, kd, kh, kw) * C + c8 * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (split_pool_takes(ev[k].v[e], el.v[e], best[e])) arg[e] = k;
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (ev[k].v[e] > best[e] || ev[k].v[e] != ev[k].v[e]) { best[e] = ev[k].v[e]; arg[e] = k; }
      }
    }
  }
  V8 gp;
#pragma unroll
  for (int e = 0; e < 8; ++e) gp.v[e] = 0.f;
  if (g_pool) gp = ld8(g_pool + ((((size_t)b * g.Dc + d) * g.Hc + h) * g.Wc + w) * C + c8 * 8);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k < nchild) {
      const int kd = g.fd == 2 ? (k >> 2) : 0, kh = (k >> 1) & 1, kw = k & 1;
      const size_t fo = fine_index(g, b, d, h, w, kd, kh, kw) * C + c8 * 8;
      V8 r;
      if (g_skip) r = ld8(g_skip + fo);
      else {
#pragma unroll
        for (int e = 0; e < 8; ++e) r.v[e] = 0.f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (arg[e] == k) r.v[e] += gp.v[e];
        if (slope >= 0.f && ev[k].v[e] < 0.f) r.v[e] *= slope;
      }
      st8(out + fo, r);
    }
  }
}

struct PlanarSrc {
  const float* p[8];
  long long bstride[8];
  int n;
};
// out[(b*V + v)*8 + c] = bf16(plane_c[b][v]) for c < n, 0 otherwise
__global__ void __launch_bounds__(256) planar_to_ndhwc8_kernel(PlanarSrc src, __nv_bfloat16* __restrict__ out, int B, size_t V) {
  size_t n = (size_t)B * V;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    size_t b = i / V, v = i - b * V;
    V8 r;
#pragma unroll
    for (int c = 0; c < 8; ++c) r.v[c] = c < src.n ? __ldg(src.p[c] + b * src.bstride[c] + v) : 0.f;
    st8(out + i * 8, r);
  }
}

// "kd folded into the channels": out[b][d][hw][kd * n + p] = plane_p[b][d + kd - 1][hw] (0 outside the volume), kd = 0..2,
// channels >= 3n zero; COUT = 8 or 16.  A 3-D convolution with n <= COUT / 3 real input channels becomes a 2-D one over the
// folded tensor (3 instead of 9 MMA steps per tile), see engine_bf16.py.
// NP = number of planes (compile time: the channel index kd * NP + p must be a constant, a run-time index sends the
// register array to local memory — the first version of this kernel ran at a third of the HBM rate for that reason)
template <int COUT, int NP>
__global__ void __launch_bounds__(256) planar_fold_kd_kernel(PlanarSrc src, __nv_bfloat16* __restrict__ out, int D, int HW) {
  // grid = (HW / 256, D, B): no index divisions, 32-bit offsets inside one (batch item, slice)
  const int hw = blockIdx.x * 256 + threadIdx.x;
  if (hw >= HW) return;
  const int d = blockIdx.y, b = blockIdx.z;
  float r[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) r[c] = 0.f;
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    const float* q = src.p[p] + (size_t)b * src.bstride[p] + (size_t)d * HW + hw;
    if (d > 0) r[p] = __ldg(q - HW);
    r[NP + p] = __ldg(q);
    if (d + 1 < D) r[2 * NP + p] = __ldg(q + HW);
  }
  __nv_bfloat16* o = out + (((size_t)b * D + d) * HW + hw) * COUT;
  if constexpr (COUT == 16) {     // two adjacent 128-bit stores per voxel: one whole 32-byte sector
    uint32_t w[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      __nv_bfloat162 h = __floats2bfloat162_rn(r[2 * e], r[2 * e + 1]);
      w[e] = *reinterpret_cast<uint32_t*>(&h);
    }
    uint4* o4 = reinterpret_cast<uint4*>(o);
    o4[0] = make_uint4(w[0], w[1], w[2], w[3]);
    o4[1] = make_uint4(w[4], w[5], w[6], w[7]);
  } else {
    V8 t;
#pragma unroll
    for (int e = 0; e < 8; ++e) t.v[e] = r[e];
    st8(o, t);
  }
}

// split-precision (bf16x3) variants: a value is carried as a bf16 pair hi = bf16(x), lo = bf16(x - hi)  (16 mantissa bits)
__global__ void __launch_bounds__(256) planar_to_ndhwc8_split_kernel(PlanarSrc src, __nv_bfloat16* __restrict__ out_hi,
                                                                     __nv_bfloat16* __restrict__ out_lo, int B, size_t V) {
  size_t n = (size_t)B * V;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    size_t b = i / V, v = i - b * V;
    V8 h, l;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float x = c < src.n ? __ldg(src.p[c] + b * src.bstride[c] + v) : 0.f;
      h.v[c] = __bfloat162float(__float2bfloat16_rn(x));
      l.v[c] = x - h.v[c];
    }
    st8(out_hi + i * 8, h);
    st8(out_lo + i * 8, l);
  }
}

// MaxPool(2) of a (hi, lo) pair tensor: the maximum is taken on hi + lo, the winning child's pair is copied (first
// maximal child wins ties, like ATen; split_pool_takes)
__global__ void __launch_bounds__(256) pool_split_ndhwc_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl,
                                                               __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl, PoolGeom g) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  int b, d, h, w, c8;
  if (!decode(g, i, b, d, h, w, c8)) return;
  const int C = g.C8 * 8;
  V8 m, mh, ml;
#pragma unroll
  for (int e = 0; e < 8; ++e) { m.v[e] = -INFINITY; mh.v[e] = -INFINITY; ml.v[e] = 0.f; }
  for (int kd = 0; kd < g.fd; ++kd)
    for (int kh = 0; kh < 2; ++kh)
      for (int kw = 0; kw < 2; ++kw) {
        const size_t o = fine_index(g, b, d, h, w, kd, kh, kw) * C + c8 * 8;
        V8 th = ld8(xh + o), tl = ld8(xl + o);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (split_pool_takes(th.v[e], tl.v[e], m.v[e])) { mh.v[e] = th.v[e]; ml.v[e] = tl.v[e]; }
      }
  const size_t o = ((((size_t)b * g.Dc + d) * g.Hc + h) * g.Wc + w) * C + c8 * 8;
  st8(yh + o, mh);
  st8(yl + o, ml);
}

static int make_pool_geom(int B, int Dc, int Hc, int Wc, int C, int nd, PoolGeom* g) {
  VXM_REQUIRE(B > 0 && Dc > 0 && Hc > 0 && Wc > 0 && C > 0 && C % 8 == 0, "ndhwc op: bad dimensions (C must be a multiple of 8)");
  VXM_REQUIRE(nd == 2 || nd == 3, "ndhwc op: nd must be 2 or 3");
  VXM_REQUIRE(nd == 3 || Dc == 1, "ndhwc op: a 2-D problem must be passed with D == 1");
  g->B = B; g->Dc = Dc; g->Hc = Hc; g->Wc = Wc; g->C8 = C / 8; g->fd = nd == 3 ? 2 : 1;
  return VXM_OK;
}
static unsigned pool_grid(const PoolGeom& g) {
  size_t n = (size_t)g.B * g.Dc * g.Hc * g.Wc * g.C8;
  return (unsigned)((n + 255) / 256);
}

}  // namespace vxm

using namespace vxm;

extern "C" int vxm_pool2_ndhwc_bf16(const void* x, void* y, int B, int Dc, int Hc, int Wc, int C, int nd, void* stream) {
  PoolGeom g;
  int rc = make_pool_geom(B, Dc, Hc, Wc, C, nd, &g);
  if (rc) return rc;
  VXM_REQUIRE(x && y, "pool2_ndhwc: null pointer");
  pool_ndhwc_kernel<<<pool_grid(g), 256, 0, as_stream(stream)>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, g);
  return check_launch("pool2_ndhwc");
}

extern "C" int vxm_sumpool_mask_ndhwc_bf16(const void* g_fine, const void* act_coarse, void* out, int B, int Dc, int Hc, int Wc, int C,
                                           int nd, float slope, void* stream) {
  PoolGeom g;
  int rc = make_pool_geom(B, Dc, Hc, Wc, C, nd, &g);
  if (rc) return rc;
  VXM_REQUIRE(g_fine && out, "sumpool_mask: null pointer");
  sumpool_mask_kernel<<<pool_grid(g), 256, 0, as_stream(stream)>>>((const __nv_bfloat16*)g_fine, (const __nv_bfloat16*)act_coarse,
                                                                   (__nv_bfloat16*)out, g, slope);
  return check_launch("sumpool_mask");
}

extern "C" int vxm_unpool_combine_ndhwc_bf16(const void* e_fine, const void* g_skip, const void* g_pool, void* out, int B, int Dc, int Hc,
                                             int Wc, int C, int nd, float slope, void* stream) {
  PoolGeom g;
  int rc = make_pool_geom(B, Dc, Hc, Wc, C, nd, &g);
  if (rc) return rc;
  VXM_REQUIRE(e_fine && out && (g_skip || g_pool), "unpool_combine: null pointer");
  unpool_combine_kernel<false><<<pool_grid(g), 256, 0, as_stream(stream)>>>((const __nv_bfloat16*)e_fine, (const __nv_bfloat16*)g_skip,
                                                                            (const __nv_bfloat16*)g_pool, (__nv_bfloat16*)out, g, slope, nullptr);
  return check_launch("unpool_combine");
}

extern "C" int vxm_unpool_combine_split_ndhwc_bf16(const void* e_hi, const void* e_lo, const void* g_skip, const void* g_pool, void* out,
                                                   int B, int Dc, int Hc, int Wc, int C, int nd, float slope, void* stream) {
  PoolGeom g;
  int rc = make_pool_geom(B, Dc, Hc, Wc, C, nd, &g);
  if (rc) return rc;
  VXM_REQUIRE(e_hi && e_lo && out && (g_skip || g_pool), "unpool_combine_split: null pointer");
  unpool_combine_kernel<true><<<pool_grid(g), 256, 0, as_stream(stream)>>>((const __nv_bfloat16*)e_hi, (const __nv_bfloat16*)g_skip,
                                                                           (const __nv_bfloat16*)g_pool, (__nv_bfloat16*)out, g, slope,
                                                                           (const __nv_bfloat16*)e_lo);
  return check_launch("unpool_combine_split");
}

extern "C" int vxm_planar_to_ndhwc8_bf16(const float* const* planes, const long long* bstrides, int nplanes, void* out, int B, size_t V,
                                         void* stream) {
  VXM_REQUIRE(planes && bstrides && out && nplanes > 0 && nplanes <= 8 && B > 0 && V > 0, "planar_to_ndhwc8: bad argument");
  PlanarSrc src{};
  src.n = nplanes;
  for (int i = 0; i < nplanes; ++i) { src.p[i] = planes[i]; src.bstride[i] = bstrides[i]; }
  size_t n = (size_t)B * V;
  size_t blocks = (n + 255) / 256;
  size_t cap = (size_t)sm_count() * 16;
  planar_to_ndhwc8_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, as_stream(stream)>>>(src, (__nv_bfloat16*)out, B, V);
  return check_launch("planar_to_ndhwc8");
}

extern "C" int vxm_planar_fold_kd_bf16(const float* const* planes, const long long* bstrides, int nplanes, void* out, int B, int D,
                                       size_t HW, int cout, void* stream) {
  VXM_REQUIRE(planes && bstrides && out && nplanes > 0 && B > 0 && D > 0 && HW > 0, "planar_fold_kd: bad argument");
  VXM_REQUIRE((cout == 8 || cout == 16) && 3 * nplanes <= cout, "planar_fold_kd: %d planes x 3 do not fit %d channels", nplanes, cout);
  PlanarSrc src{};
  src.n = nplanes;
  for (int i = 0; i < nplanes; ++i) { src.p[i] = planes[i]; src.bstride[i] = bstrides[i]; }
  VXM_REQUIRE(D <= 65535 && B <= 65535 && HW < (1u << 30), "planar_fold_kd: volume exceeds the launch grid limits");
  const dim3 grid((unsigned)((HW + 255) / 256), (unsigned)D, (unsigned)B);
  cudaStream_t st = as_stream(stream);
  __nv_bfloat16* o = (__nv_bfloat16*)out;
  const int hw = (int)HW;
  switch (cout * 8 + nplanes) {
    case 8 * 8 + 1: planar_fold_kd_kernel<8, 1><<<grid, 256, 0, st>>>(src, o, D, hw); break;
    case 8 * 8 + 2: planar_fold_kd_kernel<8, 2><<<grid, 256, 0, st>>>(src, o, D, hw); break;
    case 16 * 8 + 1: planar_fold_kd_kernel<16, 1><<<grid, 256, 0, st>>>(src, o, D, hw); break;
    case 16 * 8 + 2: planar_fold_kd_kernel<16, 2><<<grid, 256, 0, st>>>(src, o, D, hw); break;
    case 16 * 8 + 3: planar_fold_kd_kernel<16, 3><<<grid, 256, 0, st>>>(src, o, D, hw); break;
    case 16 * 8 + 4: planar_fold_kd_kernel<16, 4><<<grid, 256, 0, st>>>(src, o, D, hw); break;
    default: planar_fold_kd_kernel<16, 5><<<grid, 256, 0, st>>>(src, o, D, hw); break;
  }
  return check_launch("planar_fold_kd");
}

extern "C" int vxm_planar_to_ndhwc8_split_bf16(const float* const* planes, const long long* bstrides, int nplanes, void* out_hi,
                                               void* out_lo, int B, size_t V, void* stream) {
  VXM_REQUIRE(planes && bstrides && out_hi && out_lo && nplanes > 0 && nplanes <= 8 && B > 0 && V > 0, "planar_to_ndhwc8_split: bad argument");
  PlanarSrc src{};
  src.n = nplanes;
  for (int i = 0; i < nplanes; ++i) { src.p[i] = planes[i]; src.bstride[i] = bstrides[i]; }
  size_t n = (size_t)B * V;
  size_t blocks = (n + 255) / 256;
  size_t cap = (size_t)sm_count() * 16;
  planar_to_ndhwc8_split_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, as_stream(stream)>>>(
      src, (__nv_bfloat16*)out_hi, (__nv_bfloat16*)out_lo, B, V);
  return check_launch("planar_to_ndhwc8_split");
}

extern "C" int vxm_pool2_split_ndhwc_bf16(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int B, int Dc, int Hc, int Wc,
                                          int C, int nd, void* stream) {
  PoolGeom g;
  int rc = make_pool_geom(B, Dc, Hc, Wc, C, nd, &g);
  if (rc) return rc;
  VXM_REQUIRE(x_hi && x_lo && y_hi && y_lo, "pool2_split_ndhwc: null pointer");
  pool_split_ndhwc_kernel<<<pool_grid(g), 256, 0, as_stream(stream)>>>((const __nv_bfloat16*)x_hi, (const __nv_bfloat16*)x_lo,
                                                                       (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo, g);
  return check_launch("pool2_split_ndhwc");
}
