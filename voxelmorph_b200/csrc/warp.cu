// SpatialTransformer forward / backward (reference voxelmorph/torch/layers.py:30-48).
//
// One thread per output voxel, x fastest (coalesced flow reads / output writes); the 8-corner
// gather goes through the read-only path and is served by L1/L2 (neighbouring threads touch
// neighbouring source lines because registration flows are smooth).  The identity grid the
// reference materialises as a buffer (layers.py:17-28, 82.6 MB at 160x192x224) is never built:
// p is the thread's own index.  The trilinear arithmetic of both paths lives in sampler.cuh.
//
// Algorithmic HBM bytes per output voxel (fp32): 4*C (src) + 4*nd (flow) + 4*C (out).
#include "sampler.cuh"

namespace vxm {

constexpr int TX = 32, TY = 8;

struct WarpGeom {
  Vol src, dst;
  AxisNorm ax, ay, az;
  int B, C, nd;
};

// exact (and nearest) path: the reference's coordinate replay and ATen's corner arithmetic
template <bool IS3D, int MODE, int ARITH>
__global__ void __launch_bounds__(TX* TY) warp_fwd_kernel(const float* __restrict__ src,
                                                          const float* __restrict__ flow,
                                                          float* __restrict__ out, WarpGeom g) {
  int x = blockIdx.x * TX + threadIdx.x;
  int y = blockIdx.y * TY + threadIdx.y;
  int zb = blockIdx.z;
  int z = zb % g.dst.D, b = zb / g.dst.D;
  if (x >= g.dst.W || y >= g.dst.H) return;
  size_t p = ((size_t)z * g.dst.H + y) * g.dst.W + x;
  float fv[3], cz, cy, cx;
  exact_coords<IS3D, ARITH>(flow + (size_t)b * g.nd * g.dst.DHW + p, g.dst.DHW, z, y, x, g, fv, cz, cy, cx);
  const float* sb = src + (size_t)b * g.C * g.src.DHW;
  float* ob = out + (size_t)b * g.C * g.dst.DHW + p;
  if (MODE == VXM_MODE_NEAREST) {
    ptrdiff_t idx = nearest_index<IS3D>(cx, cy, cz, g.src);
    for (int c = 0; c < g.C; ++c) ob[(size_t)c * g.dst.DHW] = idx >= 0 ? __ldg(sb + (size_t)c * g.src.DHW + idx) : 0.0f;
  } else {
    const ExactCell<IS3D> cell = exact_cell<IS3D>(cz, cy, cx, g.src.D, g.src.H, g.src.W);
    for (int c = 0; c < g.C; ++c)
      ob[(size_t)c * g.dst.DHW] = exact_sample<IS3D, true>(sb + (size_t)c * g.src.DHW, cell);
  }
}

template <bool IS3D, int MODE, int ARITH>
__global__ void __launch_bounds__(TX* TY) warp_bwd_kernel(const float* __restrict__ gout,
                                                          const float* __restrict__ src,
                                                          const float* __restrict__ flow,
                                                          float* __restrict__ gsrc,
                                                          float* __restrict__ gflow, WarpGeom g,
                                                          float mz, float my, float mx) {
  int x = blockIdx.x * TX + threadIdx.x;
  int y = blockIdx.y * TY + threadIdx.y;
  int zb = blockIdx.z;
  int z = zb % g.dst.D, b = zb / g.dst.D;
  if (x >= g.dst.W || y >= g.dst.H) return;
  size_t p = ((size_t)z * g.dst.H + y) * g.dst.W + x;
  float fv[3], cz, cy, cx;
  exact_coords<IS3D, ARITH>(flow + (size_t)b * g.nd * g.dst.DHW + p, g.dst.DHW, z, y, x, g, fv, cz, cy, cx);
  const float* sb = src + (size_t)b * g.C * g.src.DHW;
  float* gsb = gsrc ? gsrc + (size_t)b * g.C * g.src.DHW : nullptr;
  const float* gob = gout + (size_t)b * g.C * g.dst.DHW + p;
  float gx = 0.f, gy = 0.f, gz = 0.f;
  if (MODE == VXM_MODE_NEAREST) {
    ptrdiff_t idx = nearest_index<IS3D>(cx, cy, cz, g.src);
    if (gsb && idx >= 0)
      for (int c = 0; c < g.C; ++c) atomicAdd(gsb + (size_t)c * g.src.DHW + idx, __ldg(gob + (size_t)c * g.dst.DHW));
  } else {
    const ExactCell<IS3D> cell = exact_cell<IS3D>(cz, cy, cx, g.src.D, g.src.H, g.src.W);
    for (int c = 0; c < g.C; ++c) {
      const float go = __ldg(gob + (size_t)c * g.dst.DHW);
      const float* plane = sb + (size_t)c * g.src.DHW;
      if (gflow) exact_grad(cell, [&](int off) { return __ldg(plane + off) * go; }, gz, gy, gx);
      if (gsb) exact_scatter(cell, gsb + (size_t)c * g.src.DHW, go);
    }
  }
  if (gflow) {
    float* gf = gflow + (size_t)b * g.nd * g.dst.DHW + p;
    if (IS3D) {
      gf[0] = gz * mz;
      gf[g.dst.DHW] = gy * my;
      gf[2 * g.dst.DHW] = gx * mx;
    } else {
      gf[0] = gy * my;
      gf[g.dst.DHW] = gx * mx;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// FAST linear path (arith == VXM_ARITH_FAST).  north_star asks the linear resampler for 1e-4 relative accuracy,
// not for a replay of torch's coordinate round trip (layers.py:37 + GridSampler.h:27-31), which costs a true
// fp32 division and ~10 dependent roundings per axis and made the exact kernel instruction bound (336 executed
// instructions per voxel, 15 % of HBM peak).  Here  coord = (p + flow) * (Ssrc-1)/(S-1)  (the same map in exact
// arithmetic; identity scale when src and flow grids agree, which is the only case the reference uses), and the
// cell is sampler.cuh's FastCell: a lerp-tree blend of zero-padded corners, read without per-corner predicates
// when the cell lies inside the volume.  Each thread walks ZU consecutive slices and issues all of their flow
// loads before the first gather so that enough bytes are in flight.
// Deviation from the exact path: <= a few 1e-6 of the value range (tests/test_gpu_ops.py).
// ------------------------------------------------------------------------------------------------------------
constexpr int ZU = 4;

struct FastGeom {
  int D, H, W, Ds, Hs, Ws, B, C, nd, nzc;
  float rz, ry, rx;
};

template <bool IS3D, bool C1>
__global__ void __launch_bounds__(TX* TY) warp_fwd_fast_kernel(const float* __restrict__ src, const float* __restrict__ flow,
                                                               float* __restrict__ out, FastGeom g) {
  const int x = blockIdx.x * TX + threadIdx.x;
  const int y = blockIdx.y * TY + threadIdx.y;
  const int zc = blockIdx.z % g.nzc, b = blockIdx.z / g.nzc;
  if (x >= g.W || y >= g.H) return;
  const int HW = g.H * g.W, DHW = g.D * HW;
  const int sDHW = g.Ds * g.Hs * g.Ws;
  const int C = C1 ? 1 : g.C;
  const float* fb = flow + (size_t)b * g.nd * DHW + y * g.W + x;
  const float* sb = src + (size_t)b * C * sDHW;
  float* ob = out + (size_t)b * C * DHW + y * g.W + x;
  const int z0c = zc * ZU;
  float f[ZU][3];
#pragma unroll
  for (int u = 0; u < ZU; ++u) {
    const int z = z0c + u;
    if (z < g.D) {
      const float* q = fb + z * HW;
      if (IS3D) { f[u][0] = __ldg(q); f[u][1] = __ldg(q + DHW); f[u][2] = __ldg(q + 2 * DHW); }
      else { f[u][0] = 0.f; f[u][1] = __ldg(q); f[u][2] = __ldg(q + DHW); }
    }
  }
#pragma unroll
  for (int u = 0; u < ZU; ++u) {
    const int z = z0c + u;
    if (z >= g.D) break;
    const float cz = IS3D ? ((float)z + f[u][0]) * g.rz : 0.f;
    const float cy = ((float)y + f[u][1]) * g.ry;
    const float cx = ((float)x + f[u][2]) * g.rx;
    const FastCell<IS3D> cell = fast_cell<IS3D>(cz, cy, cx, g.Ds, g.Hs, g.Ws);
    for (int c = 0; c < C; ++c) {
      float v[8];
      cell.fetch(sb + (size_t)c * sDHW, v);
      ob[(size_t)c * DHW + z * HW] = cell.blend(v);
    }
  }
}

// backward of the fast path: d out / d flow from the lerp tree of the same corners, d out / d src as a scatter
// (red.global.add) only when the caller asks for it.  NOSRC: no gradient w.r.t. the source (the moving image of the
// training step), the variant the step runs.
template <bool IS3D, bool NOSRC>
__global__ void __launch_bounds__(TX* TY, NOSRC ? 3 : 2) warp_bwd_fast_kernel(const float* __restrict__ gout, const float* __restrict__ src,
                                                               const float* __restrict__ flow, float* __restrict__ gsrc,
                                                               float* __restrict__ gflow, FastGeom g) {
  const int x = blockIdx.x * TX + threadIdx.x;
  const int y = blockIdx.y * TY + threadIdx.y;
  const int zc = blockIdx.z % g.nzc, b = blockIdx.z / g.nzc;
  if (x >= g.W || y >= g.H) return;
  const int HW = g.H * g.W, DHW = g.D * HW;
  const int sDHW = g.Ds * g.Hs * g.Ws;
  const float* fb = flow + (size_t)b * g.nd * DHW + y * g.W + x;
  const float* sb = src + (size_t)b * g.C * sDHW;
  float* gsb = (!NOSRC && gsrc) ? gsrc + (size_t)b * g.C * sDHW : nullptr;
  const float* gob = gout + (size_t)b * g.C * DHW + y * g.W + x;
  const int z0c = zc * ZU;
  float f[ZU][3];
#pragma unroll
  for (int u = 0; u < ZU; ++u) {
    const int z = z0c + u;
    if (z < g.D) {
      const float* q = fb + z * HW;
      if (IS3D) { f[u][0] = __ldg(q); f[u][1] = __ldg(q + DHW); f[u][2] = __ldg(q + 2 * DHW); }
      else { f[u][0] = 0.f; f[u][1] = __ldg(q); f[u][2] = __ldg(q + DHW); }
    }
  }
#pragma unroll
  for (int u = 0; u < ZU; ++u) {
    const int z = z0c + u;
    if (z >= g.D) break;
    const float cz = IS3D ? ((float)z + f[u][0]) * g.rz : 0.f;
    const float cy = ((float)y + f[u][1]) * g.ry;
    const float cx = ((float)x + f[u][2]) * g.rx;
    const FastCell<IS3D> cell = fast_cell<IS3D>(cz, cy, cx, g.Ds, g.Hs, g.Ws);
    float gx = 0.f, gy = 0.f, gz = 0.f;
    for (int c = 0; c < g.C; ++c) {
      const float go = __ldg(gob + (size_t)c * DHW + z * HW);
      if (NOSRC || gflow) {
        float v[8], dz, dy, dx;
        cell.fetch(sb + (size_t)c * sDHW, v);
        cell.grad(v, dz, dy, dx);
        gx = fmaf(go, dx, gx);
        gy = fmaf(go, dy, gy);
        if (IS3D) gz = fmaf(go, dz, gz);
      }
      if (gsb) cell.scatter(gsb + (size_t)c * sDHW, go);
    }
    if (gflow) {
      float* gf = gflow + (size_t)b * g.nd * DHW + z * HW + y * g.W + x;
      if (IS3D) { gf[0] = gz * g.rz; gf[DHW] = gy * g.ry; gf[2 * DHW] = gx * g.rx; }
      else { gf[0] = gy * g.ry; gf[DHW] = gx * g.rx; }
    }
  }
}

static FastGeom make_fast_geom(int B, int C, int Ds, int Hs, int Ws, int D, int H, int W, int nd) {
  FastGeom g;
  g.D = D; g.H = H; g.W = W; g.Ds = Ds; g.Hs = Hs; g.Ws = Ws; g.B = B; g.C = C; g.nd = nd;
  g.nzc = (D + ZU - 1) / ZU;
  auto ratio = [](int s_src, int s) { return s > 1 ? (float)(s_src - 1) / (float)(s - 1) : 0.f; };
  g.rz = nd == 3 ? ratio(Ds, D) : 0.f; g.ry = ratio(Hs, H); g.rx = ratio(Ws, W);
  return g;
}

static int check_geom(int B, int C, int Ds, int Hs, int Ws, int D, int H, int W, int nd) {
  VXM_REQUIRE(nd == 2 || nd == 3, "warp: nd must be 2 or 3 (reference layers.py:41-46), got %d", nd);
  VXM_REQUIRE(B > 0 && C > 0 && Ds > 0 && Hs > 0 && Ws > 0 && D > 0 && H > 0 && W > 0, "warp: non-positive dimension");
  VXM_REQUIRE(nd == 3 || (D == 1 && Ds == 1), "warp: a 2-D problem must be passed with D == 1");
  VXM_REQUIRE((size_t)D * B <= 65535u, "warp: D*B exceeds the launch grid limit (65535)");
  VXM_REQUIRE((size_t)Ds * Hs * Ws < (1u << 31) && (size_t)D * H * W < (1u << 31), "warp: volume exceeds 2^31 voxels");
  return VXM_OK;
}

static WarpGeom make_geom(int B, int C, int Ds, int Hs, int Ws, int D, int H, int W, int nd) {
  WarpGeom g;
  g.src = make_vol(Ds, Hs, Ws);
  g.dst = make_vol(D, H, W);
  g.ax = make_axis(W, Ws);
  g.ay = make_axis(H, Hs);
  g.az = make_axis(D, Ds);
  g.B = B; g.C = C; g.nd = nd;
  return g;
}

#define WARP_DISPATCH(KERNEL, ...)                                                                  \
  do {                                                                                              \
    bool is3d = (nd == 3);                                                                          \
    bool near = (mode == VXM_MODE_NEAREST);                                                         \
    bool rec = (arith == VXM_ARITH_RECIPROCAL);                                                     \
    if (is3d && !near && !rec) KERNEL<true, 0, 0><<<grid, block, 0, st>>>(__VA_ARGS__);             \
    else if (is3d && !near && rec) KERNEL<true, 0, 1><<<grid, block, 0, st>>>(__VA_ARGS__);         \
    else if (is3d && near && !rec) KERNEL<true, 1, 0><<<grid, block, 0, st>>>(__VA_ARGS__);         \
    else if (is3d && near && rec) KERNEL<true, 1, 1><<<grid, block, 0, st>>>(__VA_ARGS__);          \
    else if (!is3d && !near && !rec) KERNEL<false, 0, 0><<<grid, block, 0, st>>>(__VA_ARGS__);      \
    else if (!is3d && !near && rec) KERNEL<false, 0, 1><<<grid, block, 0, st>>>(__VA_ARGS__);       \
    else if (!is3d && near && !rec) KERNEL<false, 1, 0><<<grid, block, 0, st>>>(__VA_ARGS__);       \
    else KERNEL<false, 1, 1><<<grid, block, 0, st>>>(__VA_ARGS__);                                  \
  } while (0)

}  // namespace vxm

using namespace vxm;

extern "C" int vxm_warp_fwd(const float* src, const float* flow, float* out, int B, int C, int Ds,
                            int Hs, int Ws, int D, int H, int W, int nd, int mode, int arith,
                            void* stream) {
  int rc = check_geom(B, C, Ds, Hs, Ws, D, H, W, nd);
  if (rc) return rc;
  VXM_REQUIRE(src && flow && out, "warp_fwd: null pointer");
  VXM_REQUIRE(mode == VXM_MODE_LINEAR || mode == VXM_MODE_NEAREST, "warp_fwd: bad mode %d", mode);
  VXM_REQUIRE(arith == VXM_ARITH_TRUE_DIV || arith == VXM_ARITH_RECIPROCAL || (arith == VXM_ARITH_FAST && mode == VXM_MODE_LINEAR),
              "warp_fwd: bad arith %d (VXM_ARITH_FAST is for the linear mode only)", arith);
  cudaStream_t st = as_stream(stream);
  if (arith == VXM_ARITH_FAST) {
    FastGeom fg = make_fast_geom(B, C, Ds, Hs, Ws, D, H, W, nd);
    VXM_REQUIRE((size_t)fg.nzc * B <= 65535u, "warp: D*B exceeds the launch grid limit");
    dim3 block(TX, TY, 1), grid((W + TX - 1) / TX, (H + TY - 1) / TY, fg.nzc * B);
    if (nd == 3 && C == 1) warp_fwd_fast_kernel<true, true><<<grid, block, 0, st>>>(src, flow, out, fg);
    else if (nd == 3) warp_fwd_fast_kernel<true, false><<<grid, block, 0, st>>>(src, flow, out, fg);
    else warp_fwd_fast_kernel<false, false><<<grid, block, 0, st>>>(src, flow, out, fg);
    return check_launch("warp_fwd");
  }
  WarpGeom g = make_geom(B, C, Ds, Hs, Ws, D, H, W, nd);
  dim3 block(TX, TY, 1), grid((W + TX - 1) / TX, (H + TY - 1) / TY, D * B);
  WARP_DISPATCH(warp_fwd_kernel, src, flow, out, g);
  return check_launch("warp_fwd");
}

extern "C" int vxm_warp_bwd(const float* grad_out, const float* src, const float* flow,
                            float* grad_src, float* grad_flow, int B, int C, int Ds, int Hs, int Ws,
                            int D, int H, int W, int nd, int mode, int arith, void* stream) {
  int rc = check_geom(B, C, Ds, Hs, Ws, D, H, W, nd);
  if (rc) return rc;
  VXM_REQUIRE(grad_out && src && flow, "warp_bwd: null pointer");
  VXM_REQUIRE(arith == VXM_ARITH_TRUE_DIV || arith == VXM_ARITH_RECIPROCAL || (arith == VXM_ARITH_FAST && mode == VXM_MODE_LINEAR),
              "warp_bwd: bad arith %d (VXM_ARITH_FAST is for the linear mode only)", arith);
  if (arith == VXM_ARITH_FAST) {
    FastGeom fg = make_fast_geom(B, C, Ds, Hs, Ws, D, H, W, nd);
    dim3 block(TX, TY, 1), grid((W + TX - 1) / TX, (H + TY - 1) / TY, fg.nzc * B);
    cudaStream_t st = as_stream(stream);
    const bool nosrc = grad_src == nullptr && grad_flow != nullptr;
    if (nd == 3 && nosrc) warp_bwd_fast_kernel<true, true><<<grid, block, 0, st>>>(grad_out, src, flow, grad_src, grad_flow, fg);
    else if (nd == 3) warp_bwd_fast_kernel<true, false><<<grid, block, 0, st>>>(grad_out, src, flow, grad_src, grad_flow, fg);
    else if (nosrc) warp_bwd_fast_kernel<false, true><<<grid, block, 0, st>>>(grad_out, src, flow, grad_src, grad_flow, fg);
    else warp_bwd_fast_kernel<false, false><<<grid, block, 0, st>>>(grad_out, src, flow, grad_src, grad_flow, fg);
    return check_launch("warp_bwd");
  }
  WarpGeom g = make_geom(B, C, Ds, Hs, Ws, D, H, W, nd);
  // d coord / d flow = ((Ssrc-1)/2) * 2 / (Sflow-1)   (GridSampler.h:45-47 and layers.py:37)
  float mx = (g.ax.src_sm1 * 0.5f) * 2.0f / g.ax.sm1;
  float my = (g.ay.src_sm1 * 0.5f) * 2.0f / g.ay.sm1;
  float mz = nd == 3 ? (g.az.src_sm1 * 0.5f) * 2.0f / g.az.sm1 : 0.f;
  dim3 block(TX, TY, 1), grid((W + TX - 1) / TX, (H + TY - 1) / TY, D * B);
  cudaStream_t st = as_stream(stream);
  WARP_DISPATCH(warp_bwd_kernel, grad_out, src, flow, grad_src, grad_flow, g, mz, my, mx);
  return check_launch("warp_bwd");
}
