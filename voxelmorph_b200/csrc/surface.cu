// Surface-point registration (reference voxelmorph/tf/networks.py:391-486): the point warp
// (point_spatial_transformer, voxelmorph/tf/utils/utils.py:465-499) and the distance lookup (value_at_location,
// utils.py:71-88), both sampling with neurite's clamped interpn (ClampCell, sampler.cuh).
//
// Point warp.  q = p + r * interp(flow, p) per point, one thread per point; the label column passes through.  Its
// flow gradient scatters N points into a dense field without float atomics: every (point, corner) pair writes its
// voxel key and its index, a stable radix sort (CUB) groups the pairs by voxel with the indices in order, and one
// thread per run sums that voxel's contributions in point order (fp64) and adds the sum to the caller's buffer.  No
// host synchronisation: the result is bit-reproducible and the calls can be captured in a CUDA graph.
//
// Distance lookup.  |interp(sdt, q)| in nd + 1 dimensions, the label index the last coordinate; a label tap of
// weight 0 is not read, so an integral label reads one channel.  Its gradient is sign(v) * d interp / d q over the nd
// spatial coordinates (the label column gets 0); one thread per point.
#include <climits>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "sampler.cuh"

namespace vxm {
namespace surf {

constexpr int NT = 256;

struct Geo {
  int B, N, D, H, W, nd;
  size_t V;  // D * H * W
};

// the cell of a point whose spatial coordinates start at p (3-D: z, y, x; 2-D: y, x)
template <bool IS3D>
__device__ __forceinline__ ClampCell<IS3D> point_cell(const float* p, const Geo& g) {
  return IS3D ? clamp_cell<IS3D>(p[0], p[1], p[2], g.D, g.H, g.W) : clamp_cell<IS3D>(0.f, p[0], p[1], g.D, g.H, g.W);
}

template <bool IS3D>
__global__ void __launch_bounds__(NT) warp_fwd_kernel(const float* __restrict__ pts, const float* __restrict__ flow,
                                                      float* __restrict__ out, Geo g, float r) {
  constexpr int ND = IS3D ? 3 : 2;
  const size_t i = (size_t)blockIdx.x * NT + threadIdx.x;
  if (i >= (size_t)g.B * g.N) return;
  const size_t b = i / g.N;
  const float* p = pts + i * (ND + 1);
  const ClampCell<IS3D> c = point_cell<IS3D>(p, g);
  float* q = out + i * (ND + 1);
#pragma unroll
  for (int d = 0; d < ND; ++d) q[d] = p[d] + r * c.value(flow + (b * ND + d) * g.V);
  q[ND] = p[ND];
}

// one (key, index, weight) triple per (point, corner); key = b * V + voxel
template <bool IS3D>
__global__ void __launch_bounds__(NT) warp_pairs_kernel(const float* __restrict__ pts, Geo g, float r,
                                                        uint32_t* __restrict__ keys, uint32_t* __restrict__ idx,
                                                        float* __restrict__ w) {
  constexpr int ND = IS3D ? 3 : 2, K = IS3D ? 8 : 4;
  const size_t i = (size_t)blockIdx.x * NT + threadIdx.x;
  if (i >= (size_t)g.B * g.N) return;
  const size_t b = i / g.N;
  const ClampCell<IS3D> c = point_cell<IS3D>(pts + i * (ND + 1), g);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const size_t j = i * K + k;
    keys[j] = (uint32_t)(b * g.V + (size_t)c.off(k));
    idx[j] = (uint32_t)j;
    w[j] = r * c.weight(k);
  }
}

// one thread per run of equal keys in the sorted pairs: grad_flow[b, :, voxel] += sum of w * grad_out in pair order
template <int ND>
__global__ void __launch_bounds__(NT) warp_runsum_kernel(const uint32_t* __restrict__ keys,
                                                         const uint32_t* __restrict__ idx, const float* __restrict__ w,
                                                         const float* __restrict__ gout, float* __restrict__ gflow,
                                                         size_t M, size_t V) {
  constexpr int K = ND == 3 ? 8 : 4;
  const size_t i = (size_t)blockIdx.x * NT + threadIdx.x;
  if (i >= M) return;
  const uint32_t key = keys[i];
  if (i > 0 && keys[i - 1] == key) return;
  double acc[ND] = {};
  for (size_t j = i; j < M && keys[j] == key; ++j) {
    const uint32_t e = idx[j];
    const double we = (double)w[e];
    const float* go = gout + (size_t)(e / K) * (ND + 1);
#pragma unroll
    for (int d = 0; d < ND; ++d) acc[d] += we * (double)go[d];
  }
  const size_t b = key / V, v = key % V;
#pragma unroll
  for (int d = 0; d < ND; ++d) {
    float* dst = gflow + (b * ND + d) * V + v;
    *dst += (float)acc[d];
  }
}

// value of the SDT at one point (signed); fills the label taps and the spatial cell for the backward
template <bool IS3D>
__device__ __forceinline__ float sdt_value(const float* sdt, const float* q, const Geo& g, int L, ClampTap& tl,
                                           ClampCell<IS3D>& c, const float*& p0, const float*& p1) {
  constexpr int ND = IS3D ? 3 : 2;
  c = point_cell<IS3D>(q, g);
  tl = clamp_tap(q[ND], L);
  p0 = sdt + tl.i0 * g.V;
  p1 = sdt + tl.i1 * g.V;
  float v = 0.f;
  if (tl.w0 != 0.f) v = tl.w0 * c.value(p0);
  if (tl.w1 != 0.f) v = fmaf(tl.w1, c.value(p1), v);
  return v;
}

template <bool IS3D>
__global__ void __launch_bounds__(NT) value_fwd_kernel(const float* __restrict__ sdt, const float* __restrict__ pts,
                                                       float* __restrict__ out, Geo g, int L) {
  constexpr int ND = IS3D ? 3 : 2;
  const size_t i = (size_t)blockIdx.x * NT + threadIdx.x;
  if (i >= (size_t)g.B * g.N) return;
  const size_t b = i / g.N;
  ClampTap tl;
  ClampCell<IS3D> c;
  const float *p0, *p1;
  out[i] = fabsf(sdt_value<IS3D>(sdt + b * L * g.V, pts + i * (ND + 1), g, L, tl, c, p0, p1));
}

template <bool IS3D>
__global__ void __launch_bounds__(NT) value_bwd_kernel(const float* __restrict__ sdt, const float* __restrict__ pts,
                                                       const float* __restrict__ gout, float* __restrict__ gpts, Geo g,
                                                       int L) {
  constexpr int ND = IS3D ? 3 : 2;
  const size_t i = (size_t)blockIdx.x * NT + threadIdx.x;
  if (i >= (size_t)g.B * g.N) return;
  const size_t b = i / g.N;
  ClampTap tl;
  ClampCell<IS3D> c;
  const float *p0, *p1;
  const float v = sdt_value<IS3D>(sdt + b * L * g.V, pts + i * (ND + 1), g, L, tl, c, p0, p1);
  const float s = (v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f)) * gout[i];
  float gz = 0.f, gy = 0.f, gx = 0.f;
  if (tl.w0 != 0.f) c.grad(p0, s * tl.w0, gz, gy, gx);
  if (tl.w1 != 0.f) c.grad(p1, s * tl.w1, gz, gy, gx);
  float* dst = gpts + i * (ND + 1);
  if (IS3D) {
    dst[0] = gz; dst[1] = gy; dst[2] = gx;
  } else {
    dst[0] = gy; dst[1] = gx;
  }
  dst[ND] = 0.f;
}

int check_geo(const Geo& g, const char* what) {
  VXM_REQUIRE(g.nd == 2 || g.nd == 3, "%s: nd must be 2 or 3 (got %d)", what, g.nd);
  VXM_REQUIRE(g.B > 0 && g.N > 0 && g.D > 0 && g.H > 0 && g.W > 0, "%s: sizes must be positive", what);
  VXM_REQUIRE(g.nd == 3 || g.D == 1, "%s: a 2-D problem is passed with D == 1", what);
  VXM_REQUIRE((size_t)g.H * g.W * g.D <= (size_t)INT_MAX, "%s: volume too large", what);
  return VXM_OK;
}

unsigned grid_of(size_t n) { return (unsigned)((n + NT - 1) / NT); }

// sort sizing: M pairs, keys below B * V
struct SortPlan {
  size_t M;
  int end_bit;
};

int sort_plan(const Geo& g, SortPlan& s) {
  const size_t keys = (size_t)g.B * g.V;
  s.M = (size_t)g.B * g.N * (g.nd == 3 ? 8 : 4);
  VXM_REQUIRE(keys <= (size_t)UINT32_MAX && s.M <= (size_t)INT_MAX,
              "point_warp_bwd: B * volume (%zu) must stay below 2^32 and B * N * 2^nd (%zu) below 2^31", keys, s.M);
  s.end_bit = 1;
  while (s.end_bit < 32 && ((size_t)1 << s.end_bit) < keys) ++s.end_bit;
  return VXM_OK;
}

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

// workspace: keys, keys', indices, indices', weights (M each), then CUB's scratch
size_t sort_temp_bytes(const SortPlan& s) {
  size_t bytes = 0;
  if (cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                      (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)s.M, 0, s.end_bit) !=
      cudaSuccess)
    return 0;
  return bytes;
}

size_t workspace_bytes(const SortPlan& s, size_t& temp) {
  temp = sort_temp_bytes(s);
  return temp ? 5 * align256(s.M * 4) + align256(temp) : 0;
}

}  // namespace surf
}  // namespace vxm

using namespace vxm;
using namespace vxm::surf;

extern "C" size_t vxm_point_warp_workspace_bytes(int B, int N, int D, int H, int W, int nd) {
  Geo g{B, N, D, H, W, nd, (size_t)D * H * W};
  SortPlan s;
  if (check_geo(g, "point_warp_workspace") || sort_plan(g, s)) return 0;
  size_t temp;
  return workspace_bytes(s, temp);
}

extern "C" int vxm_point_warp_fwd(const float* points, const float* flow, float* out, int B, int N, int D, int H,
                                  int W, int nd, float r, void* stream) {
  Geo g{B, N, D, H, W, nd, (size_t)D * H * W};
  int rc = check_geo(g, "point_warp_fwd");
  if (rc) return rc;
  VXM_REQUIRE(points && flow && out, "point_warp_fwd: null pointer");
  const size_t n = (size_t)B * N;
  if (nd == 3)
    warp_fwd_kernel<true><<<grid_of(n), NT, 0, as_stream(stream)>>>(points, flow, out, g, r);
  else
    warp_fwd_kernel<false><<<grid_of(n), NT, 0, as_stream(stream)>>>(points, flow, out, g, r);
  return check_launch("point_warp_fwd");
}

extern "C" int vxm_point_warp_bwd(const float* points, const float* grad_out, float* grad_flow, void* work,
                                  size_t work_bytes, int B, int N, int D, int H, int W, int nd, float r, void* stream) {
  Geo g{B, N, D, H, W, nd, (size_t)D * H * W};
  int rc = check_geo(g, "point_warp_bwd");
  if (rc) return rc;
  SortPlan s;
  rc = sort_plan(g, s);
  if (rc) return rc;
  VXM_REQUIRE(points && grad_out && grad_flow && work, "point_warp_bwd: null pointer");
  size_t temp;
  const size_t need = workspace_bytes(s, temp);
  VXM_REQUIRE(need && work_bytes >= need, "point_warp_bwd: workspace of %zu bytes, %zu needed", work_bytes, need);
  cudaStream_t st = as_stream(stream);
  char* ws = (char*)work;
  const size_t a = align256(s.M * 4);
  uint32_t *k0 = (uint32_t*)ws, *k1 = (uint32_t*)(ws + a), *i0 = (uint32_t*)(ws + 2 * a), *i1 = (uint32_t*)(ws + 3 * a);
  float* w = (float*)(ws + 4 * a);
  const size_t n = (size_t)B * N;
  if (nd == 3)
    warp_pairs_kernel<true><<<grid_of(n), NT, 0, st>>>(points, g, r, k0, i0, w);
  else
    warp_pairs_kernel<false><<<grid_of(n), NT, 0, st>>>(points, g, r, k0, i0, w);
  rc = check_launch("point_warp_pairs");
  if (rc) return rc;
  VXM_CUDA(cub::DeviceRadixSort::SortPairs(ws + 5 * a, temp, k0, k1, i0, i1, (int)s.M, 0, s.end_bit, st));
  rc = check_launch("point_warp_sort");
  if (rc) return rc;
  if (nd == 3)
    warp_runsum_kernel<3><<<grid_of(s.M), NT, 0, st>>>(k1, i1, w, grad_out, grad_flow, s.M, g.V);
  else
    warp_runsum_kernel<2><<<grid_of(s.M), NT, 0, st>>>(k1, i1, w, grad_out, grad_flow, s.M, g.V);
  return check_launch("point_warp_runsum");
}

extern "C" int vxm_value_at_fwd(const float* sdt, const float* points, float* out, int B, int N, int L, int D, int H,
                                int W, int nd, void* stream) {
  Geo g{B, N, D, H, W, nd, (size_t)D * H * W};
  int rc = check_geo(g, "value_at_fwd");
  if (rc) return rc;
  VXM_REQUIRE(L > 0, "value_at_fwd: L must be positive");
  VXM_REQUIRE(sdt && points && out, "value_at_fwd: null pointer");
  const size_t n = (size_t)B * N;
  if (nd == 3)
    value_fwd_kernel<true><<<grid_of(n), NT, 0, as_stream(stream)>>>(sdt, points, out, g, L);
  else
    value_fwd_kernel<false><<<grid_of(n), NT, 0, as_stream(stream)>>>(sdt, points, out, g, L);
  return check_launch("value_at_fwd");
}

extern "C" int vxm_value_at_bwd(const float* sdt, const float* points, const float* grad_out, float* grad_points, int B,
                                int N, int L, int D, int H, int W, int nd, void* stream) {
  Geo g{B, N, D, H, W, nd, (size_t)D * H * W};
  int rc = check_geo(g, "value_at_bwd");
  if (rc) return rc;
  VXM_REQUIRE(L > 0, "value_at_bwd: L must be positive");
  VXM_REQUIRE(sdt && points && grad_out && grad_points, "value_at_bwd: null pointer");
  const size_t n = (size_t)B * N;
  if (nd == 3)
    value_bwd_kernel<true><<<grid_of(n), NT, 0, as_stream(stream)>>>(sdt, points, grad_out, grad_points, g, L);
  else
    value_bwd_kernel<false><<<grid_of(n), NT, 0, as_stream(stream)>>>(sdt, points, grad_out, grad_points, g, L);
  return check_launch("value_at_bwd");
}
