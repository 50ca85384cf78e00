// VecInt — scaling and squaring (reference voxelmorph/torch/layers.py:51-68).
//
// The reference issues ~7 launches per squaring step (add grid, normalise x3, permute, index,
// grid_sample, add).  Here ALL nsteps squarings run in ONE cooperative launch: a persistent grid
// walks the field, `grid.sync()` separates the steps, and the (B,nd,D,H,W) field (10.3 MB at
// 80x96x112) stays L2-resident between steps.  The backward runs the reversed chain in one
// cooperative launch as well.  The trilinear arithmetic of both paths lives in sampler.cuh.
//
// Algorithmic bytes (fp32) per voxel per step: forward 4*nd read + 4*nd write;
// backward 4*nd (v_k) + 4*nd (g_{k+1}) read + 4*nd (g_k) write.
#include <cooperative_groups.h>

#include "sampler.cuh"

namespace cg = cooperative_groups;

namespace vxm {

struct VecGeom {
  Vol vol;
  AxisNorm ax, ay, az;
  int B, nd;
  size_t N;  // B * nd * DHW
};

// step == -1: scaling pass; 0 <= step < nsteps: one squaring
template <bool IS3D, int ARITH>
__global__ void __launch_bounds__(256) vecint_fwd_kernel(const float* __restrict__ vel, float* out,
                                                         float* states, float* work, VecGeom g,
                                                         int nsteps, float scale) {
  cg::grid_group grid = cg::this_grid();
  const size_t tid0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t nvox = (size_t)g.B * g.vol.DHW;
  auto buf = [&](int k) -> float* {
    if (k == nsteps) return out;
    if (states) return states + (size_t)k * g.N;
    return ((nsteps - k) & 1) ? work : out;
  };
  for (int s = -1; s < nsteps; ++s) {
    if (s < 0) {
      float* dst = buf(0);
      for (size_t i = tid0; i < g.N; i += stride) dst[i] = __fmul_rn(vel[i], scale);
    } else {
      const float* cur = buf(s);
      float* nxt = buf(s + 1);
      for (size_t q = tid0; q < nvox; q += stride) {
        int b = (int)(q / g.vol.DHW);
        size_t p = q - (size_t)b * g.vol.DHW;
        int z = (int)(p / g.vol.HW);
        int r = (int)(p - (size_t)z * g.vol.HW);
        int y = r / g.vol.W, x = r - y * g.vol.W;
        const float* fb = cur + (size_t)b * g.nd * g.vol.DHW;
        float fv[3], cz, cy, cx;
        exact_coords<IS3D, ARITH>(fb + p, g.vol.DHW, z, y, x, g, fv, cz, cy, cx);
        const ExactCell<IS3D> cell = exact_cell<IS3D>(cz, cy, cx, g.vol.D, g.vol.H, g.vol.W);
        float* ob = nxt + (size_t)b * g.nd * g.vol.DHW + p;
#pragma unroll
        for (int c = 0; c < (IS3D ? 3 : 2); ++c) {
          // plain (coherent) loads: `cur` was written earlier in this same launch
          ob[(size_t)c * g.vol.DHW] = __fadd_rn(fv[c], exact_sample<IS3D, false>(fb + (size_t)c * g.vol.DHW, cell));
        }
      }
    }
    if (s + 1 < nsteps) grid.sync();
  }
}

// phase 0: G_cur = g_next + (d warp / d flow)^T g_next     (gather, plain stores)
// phase 1: G_cur += (d warp / d src)^T g_next               (scatter, fp32 atomics)
// phase 2 (after step 0): grad_vel = G_0 * scale
template <bool IS3D, int ARITH>
__global__ void __launch_bounds__(256) vecint_bwd_kernel(const float* __restrict__ gout,
                                                         const float* __restrict__ states,
                                                         float* grad_vel, float* work, VecGeom g,
                                                         int nsteps, float scale, float mz, float my, float mx) {
  cg::grid_group grid = cg::this_grid();
  const size_t tid0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t nvox = (size_t)g.B * g.vol.DHW;
  constexpr int NCH = IS3D ? 3 : 2;
  // work items: for k = nsteps-1 .. 0: (phase 0, phase 1); then the final scaling pass
  // item index it = 2*(nsteps-1-k) + phase, final = 2*nsteps
  for (int it = 0; it <= 2 * nsteps; ++it) {
    if (it == 2 * nsteps) {
      const float* G0 = nsteps == 0 ? gout : (((nsteps - 1) & 1) ? work + g.N : work);
      for (size_t i = tid0; i < g.N; i += stride) grad_vel[i] = G0[i] * scale;
    } else {
      int j = it >> 1, phase = it & 1;     // j-th processed step, k = nsteps-1-j
      int k = nsteps - 1 - j;
      const float* gn = (j == 0) ? gout : (((j - 1) & 1) ? work + g.N : work);
      float* gc = (j & 1) ? work + g.N : work;
      const float* v = states + (size_t)k * g.N;
      for (size_t q = tid0; q < nvox; q += stride) {
        int b = (int)(q / g.vol.DHW);
        size_t p = q - (size_t)b * g.vol.DHW;
        int z = (int)(p / g.vol.HW);
        int r = (int)(p - (size_t)z * g.vol.HW);
        int y = r / g.vol.W, x = r - y * g.vol.W;
        const float* fb = v + (size_t)b * g.nd * g.vol.DHW;
        float fv[3], cz, cy, cx;
        exact_coords<IS3D, ARITH>(fb + p, g.vol.DHW, z, y, x, g, fv, cz, cy, cx);
        const ExactCell<IS3D> cell = exact_cell<IS3D>(cz, cy, cx, g.vol.D, g.vol.H, g.vol.W);
        const float* gnb = gn + (size_t)b * g.nd * g.vol.DHW + p;
        float go[NCH];
#pragma unroll
        for (int c = 0; c < NCH; ++c) go[c] = gnb[(size_t)c * g.vol.DHW];
        if (phase == 0) {
          float gx = 0.f, gy = 0.f, gz = 0.f;
          exact_grad(cell, [&](int off) {
            float vg = 0.f;
#pragma unroll
            for (int c = 0; c < NCH; ++c) vg += __ldg(fb + (size_t)c * g.vol.DHW + off) * go[c];
            return vg;
          }, gz, gy, gx);
          float* gcb = gc + (size_t)b * g.nd * g.vol.DHW + p;
          if (IS3D) {
            gcb[0] = go[0] + gz * mz;
            gcb[g.vol.DHW] = go[1] + gy * my;
            gcb[2 * g.vol.DHW] = go[2] + gx * mx;
          } else {
            gcb[0] = go[0] + gy * my;
            gcb[g.vol.DHW] = go[1] + gx * mx;
          }
        } else {
          float* gcb = gc + (size_t)b * g.nd * g.vol.DHW;
#pragma unroll
          for (int c = 0; c < NCH; ++c) exact_scatter(cell, gcb + (size_t)c * g.vol.DHW, go[c]);
        }
      }
    }
    if (it < 2 * nsteps) grid.sync();
  }
}

// ------------------------------------------------------------------------------------------------------------
// FAST path (arith == VXM_ARITH_FAST, 3-D): same algorithm, but
//  * the field lives in an INTERLEAVED float4 (z, y, x, 0) layout inside the launch: a squaring step is one
//    16-byte own load, eight 16-byte gathers and one 16-byte store per voxel instead of 3 + 24 + 3 four-byte
//    accesses (the planar layout is only read in the scaling pass and written by the last step);
//  * coordinates are p + v directly (no replay of the reference's normalise / un-normalise round trip), and the cell
//    is sampler.cuh's FastCell, as in the fast warp;
//  * the backward scatters d/d(src) with ONE red.global.add.v4.f32 per corner (8 + 1 vector reductions per voxel
//    and step instead of 24 scalar atomics), rotating three float4 gradient buffers so that every step is one
//    phase (one grid.sync) instead of two.
// Agreement with the exact path: ~1e-6 of the field's range per step (tests/test_gpu_ops.py).
// ------------------------------------------------------------------------------------------------------------
struct FastDiv {
  unsigned mul, shr;
  int d;
};
static FastDiv make_fastdiv(int d) {
  FastDiv f;
  f.d = d;
  if (d == 1) { f.mul = 0; f.shr = 0; return f; }
  unsigned lg = 0;
  while ((1u << lg) < (unsigned)d) ++lg;
  const unsigned p = 31 + lg;
  f.mul = (unsigned)(((1ull << p) + (unsigned)d - 1) / (unsigned)d);
  f.shr = p - 32;
  return f;
}
__device__ __forceinline__ int fdiv(int n, const FastDiv& f) { return f.d == 1 ? n : (int)(__umulhi((unsigned)n, f.mul) >> f.shr); }

struct VecFast {
  int B, D, H, W, HW, DHW, nvox;
  FastDiv dW, dH, dD;
};

// Work decomposition of the forward: the field is cut into 512-voxel blocks; CTA c owns the contiguous run of blocks
// [c * nblk / grid, (c + 1) * nblk / grid) (so consecutive iterations of a CTA touch neighbouring rows: L1 reuse), and a thread
// carries TWO voxels (blocks blk, blk + 1) per iteration with all 16 gathers in flight — at 16 warps per SM the kernel is bound by
// the L2 round trip of its gathers otherwise.  The gathers read the clamped corners of FastCell and blend them with its
// branch-free weighted_blend, so interior and border voxels issue the same loads.
// SAVE: every intermediate field v_0 .. v_{n-1} is kept (states, for the backward); otherwise two buffers ping-pong
template <bool SAVE>
__global__ void __launch_bounds__(512) vecint_fwd_fast_kernel(const float* __restrict__ vel, float* __restrict__ out, float4* buf,
                                                              VecFast g, int nsteps, float scale) {
  cg::grid_group grid = cg::this_grid();
  const int nblk = (g.nvox + 511) >> 9;
  const int blk0 = (int)((long long)blockIdx.x * nblk / gridDim.x), blk1 = (int)((long long)(blockIdx.x + 1) * nblk / gridDim.x);
  auto field = [&](int k) -> float4* { return buf + (size_t)(SAVE ? k : (k & 1)) * g.nvox; };
  {
    float4* f0 = field(0);
    for (int blk = blk0; blk < blk1; ++blk) {
      const int q = (blk << 9) + threadIdx.x;
      if (q < g.nvox) {
        const int b = q / g.DHW;
        const int p = q - b * g.DHW;
        const float* vb = vel + (size_t)b * 3 * g.DHW + p;
        f0[q] = make_float4(__ldg(vb) * scale, __ldg(vb + g.DHW) * scale, __ldg(vb + 2 * g.DHW) * scale, 0.f);
      }
    }
  }
  grid.sync();
  for (int s = 0; s < nsteps; ++s) {
    const float4* __restrict__ cur = field(s);
    float4* __restrict__ nxt = field(s + 1);
    const bool last = s + 1 == nsteps;
    for (int blk = blk0; blk < blk1; blk += 2) {
      int q[2];
      bool has[2];
      float4 v[2];
      FastCell<true> f[2];
      float4 u[2][8];
      int bb[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        q[e] = ((blk + e) << 9) + threadIdx.x;
        has[e] = blk + e < blk1 && q[e] < g.nvox;
        if (!has[e]) q[e] = 0;
        v[e] = cur[q[e]];
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int t1 = fdiv(q[e], g.dW), x = q[e] - t1 * g.W;
        const int t2 = fdiv(t1, g.dH), y = t1 - t2 * g.H;
        const int b = fdiv(t2, g.dD), z = t2 - b * g.D;
        bb[e] = b;
        const float4* cb = cur + (size_t)b * g.DHW;
        f[e] = fast_cell<true>((float)z + v[e].x, (float)y + v[e].y, (float)x + v[e].z, g.D, g.H, g.W);
#pragma unroll
        for (int k = 0; k < 8; ++k) u[e][k] = cb[f[e].off(k)];
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float4 r = f[e].weighted_blend(u[e]);
        const float4 o = make_float4(v[e].x + r.x, v[e].y + r.y, v[e].z + r.z, 0.f);
        if (has[e]) {
          if (last) {
            const int p = q[e] - bb[e] * g.DHW;
            float* ob = out + (size_t)bb[e] * 3 * g.DHW + p;
            ob[0] = o.x; ob[g.DHW] = o.y; ob[2 * g.DHW] = o.z;
          } else {
            nxt[q[e]] = o;
          }
        }
      }
    }
    if (!last) grid.sync();
  }
}

// The backward walks the field grid-stride, loading the next voxel's own data ahead of this one's gathers.  Three rotating
// float4 gradient buffers G[0..2] (work): step j reads G[j%3], reduces into G[(j+1)%3] (zero on entry) and zeroes G[(j+2)%3]
// for the step after.
__global__ void __launch_bounds__(512) vecint_bwd_fast_kernel(const float* __restrict__ gout, const float4* __restrict__ states,
                                                              float* __restrict__ grad_vel, float4* G, VecFast g, int nsteps, float scale) {
  cg::grid_group grid = cg::this_grid();
  const int tid0 = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  const int stride = (int)(gridDim.x * blockDim.x);
  float4* G0 = G;
  float4* G1 = G + (size_t)g.nvox;
  float4* G2 = G + 2 * (size_t)g.nvox;
  for (int q = tid0; q < g.nvox; q += stride) {
    const int b = q / g.DHW, p = q - b * g.DHW;
    const float* gb = gout + (size_t)b * 3 * g.DHW + p;
    G0[q] = make_float4(__ldg(gb), __ldg(gb + g.DHW), __ldg(gb + 2 * g.DHW), 0.f);
    G1[q] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  grid.sync();
  for (int j = 0; j < nsteps; ++j) {
    const int k = nsteps - 1 - j;
    const float4* __restrict__ v = states + (size_t)k * g.nvox;
    const float4* __restrict__ gn = j % 3 == 0 ? G0 : (j % 3 == 1 ? G1 : G2);
    float4* gc = j % 3 == 0 ? G1 : (j % 3 == 1 ? G2 : G0);
    float4* __restrict__ gz = j % 3 == 0 ? G2 : (j % 3 == 1 ? G0 : G1);
    float4 own_next = make_float4(0.f, 0.f, 0.f, 0.f), go_next = own_next;
    if (tid0 < g.nvox) { own_next = v[tid0]; go_next = gn[tid0]; }
    for (int q = tid0; q < g.nvox; q += stride) {
      const int t1 = fdiv(q, g.dW), x = q - t1 * g.W;
      const int t2 = fdiv(t1, g.dH), y = t1 - t2 * g.H;
      const int b = fdiv(t2, g.dD), z = t2 - b * g.D;
      const float4 own = own_next;
      const float4 go = go_next;
      if (q + stride < g.nvox) { own_next = v[q + stride]; go_next = gn[q + stride]; }   // next iteration's own data, ahead of this one's gathers
      gz[q] = make_float4(0.f, 0.f, 0.f, 0.f);
      const FastCell<true> cell = fast_cell<true>((float)z + own.x, (float)y + own.y, (float)x + own.z, g.D, g.H, g.W);
      float4 u[8];
      cell.fetch(v + (size_t)b * g.DHW, u);
      // <corner, go>: the scalar field whose position-gradient is the flow gradient of this voxel
      float s[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) s[c] = fmaf(u[c].x, go.x, fmaf(u[c].y, go.y, u[c].z * go.z));
      float dz, dy, dx;
      cell.grad(s, dz, dy, dx);
      cell.scatter(gc + (size_t)b * g.DHW, go);
      atomicAdd(gc + q, make_float4(go.x + dz, go.y + dy, go.z + dx, 0.f));
    }
    grid.sync();
  }
  const float4* Gf = nsteps % 3 == 0 ? G0 : (nsteps % 3 == 1 ? G1 : G2);
  for (int q = tid0; q < g.nvox; q += stride) {
    const int b = q / g.DHW, p = q - b * g.DHW;
    const float4 r = Gf[q];
    float* o = grad_vel + (size_t)b * 3 * g.DHW + p;
    o[0] = r.x * scale; o[g.DHW] = r.y * scale; o[2 * g.DHW] = r.z * scale;
  }
}

// measurement aid (tools/r2_memprof.py): a cooperative launch of the same shape that only synchronises
__global__ void __launch_bounds__(512) gridsync_probe_kernel(int nsync, unsigned* sink) {
  cg::grid_group grid = cg::this_grid();
  for (int i = 0; i < nsync; ++i) grid.sync();
  if (sink && blockIdx.x == 0 && threadIdx.x == 0) *sink = (unsigned)nsync;
}

static VecFast make_vfast(int B, int D, int H, int W) {
  VecFast g;
  g.B = B; g.D = D; g.H = H; g.W = W; g.HW = H * W; g.DHW = D * H * W; g.nvox = B * D * H * W;
  g.dW = make_fastdiv(W); g.dH = make_fastdiv(H); g.dD = make_fastdiv(D);
  return g;
}

static VecGeom make_vgeom(int B, int D, int H, int W, int nd) {
  VecGeom g;
  g.vol = make_vol(D, H, W);
  g.ax = make_axis(W, W);
  g.ay = make_axis(H, H);
  g.az = make_axis(D, D);
  g.B = B; g.nd = nd;
  g.N = (size_t)B * nd * g.vol.DHW;
  return g;
}

// grid of a cooperative launch: as many CTAs as fit on the device at once, but no more than max_ctas
template <typename K>
static int coop_grid(K kernel, int threads, size_t max_ctas, int* grid_out) {
  int dev = 0, nsm = 0, coop = 0, per_sm = 0;
  VXM_CUDA(cudaGetDevice(&dev));
  VXM_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  VXM_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  VXM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0));
  if (!coop || per_sm < 1) {
    set_error("vecint: cooperative launch unavailable on this device");
    return VXM_ERR_UNSUPPORTED;
  }
  const size_t cap = (size_t)nsm * per_sm;
  *grid_out = (int)(max_ctas < cap ? max_ctas : cap);
  return VXM_OK;
}

}  // namespace vxm

using namespace vxm;

extern "C" size_t vxm_vecint_workspace_bytes(int B, int D, int H, int W, int nd, int nsteps) {
  (void)nsteps;
  return (size_t)B * nd * D * H * W * sizeof(float);
}

extern "C" size_t vxm_vecint_fast_states_bytes(int B, int D, int H, int W, int nsteps) {
  return (size_t)(nsteps > 0 ? nsteps : 0) * B * D * H * W * sizeof(float4);
}
extern "C" size_t vxm_vecint_fast_work_bytes(int B, int D, int H, int W, int backward) {
  return (size_t)(backward ? 3 : 2) * B * D * H * W * sizeof(float4);
}

extern "C" int vxm_debug_gridsync(int nsync, int ctas_per_sm, void* stream) {
  int grid = 0;
  int rc = coop_grid(gridsync_probe_kernel, 512, SIZE_MAX, &grid);
  if (rc) return rc;
  if (ctas_per_sm > 0 && ctas_per_sm * sm_count() < grid) grid = ctas_per_sm * sm_count();
  unsigned* sink = nullptr;
  void* args[] = {(void*)&nsync, (void*)&sink};
  VXM_CUDA(cudaLaunchCooperativeKernel((void*)gridsync_probe_kernel, dim3(grid), dim3(512), args, 0, as_stream(stream)));
  return check_launch("debug_gridsync");
}

static int vecint_fast_check(int B, int D, int H, int W, int nd, int nsteps) {
  VXM_REQUIRE(nd == 3, "vecint (fast): 3-D fields only");
  VXM_REQUIRE(nsteps >= 1 && nsteps < 31, "vecint (fast): nsteps must be in 1..30, found: %d", nsteps);
  VXM_REQUIRE(B > 0 && D > 1 && H > 1 && W > 1, "vecint (fast): every spatial size must be > 1");
  VXM_REQUIRE((size_t)B * D * H * W < (1u << 30), "vecint (fast): field exceeds 2^30 voxels");
  return VXM_OK;
}

static int vecint_fwd_fast(const float* vel, float* out, void* states, void* work, int B, int D, int H, int W, int nd, int nsteps, cudaStream_t st) {
  int rc = vecint_fast_check(B, D, H, W, nd, nsteps);
  if (rc) return rc;
  VXM_REQUIRE(states || work, "vecint_fwd (fast): need `states` or `work`");
  VecFast g = make_vfast(B, D, H, W);
  float scale = 1.0f / (float)(1u << nsteps);
  float4* buf = (float4*)(states ? states : work);
  auto kern = states ? vecint_fwd_fast_kernel<true> : vecint_fwd_fast_kernel<false>;
  int grid = 0;
  rc = coop_grid(kern, 512, SIZE_MAX, &grid);
  if (rc) return rc;
  void* args[] = {(void*)&vel, (void*)&out, (void*)&buf, (void*)&g, (void*)&nsteps, (void*)&scale};
  VXM_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(grid), dim3(512), args, 0, st));
  return check_launch("vecint_fwd");
}

static int vecint_bwd_fast(const float* gout, const void* states, float* grad_vel, void* work, int B, int D, int H, int W, int nd, int nsteps, cudaStream_t st) {
  int rc = vecint_fast_check(B, D, H, W, nd, nsteps);
  if (rc) return rc;
  VXM_REQUIRE(states && work, "vecint_bwd (fast): need `states` and `work`");
  VecFast g = make_vfast(B, D, H, W);
  float scale = 1.0f / (float)(1u << nsteps);
  const float4* sp = (const float4*)states;
  float4* G = (float4*)work;
  int grid = 0;
  rc = coop_grid(vecint_bwd_fast_kernel, 512, SIZE_MAX, &grid);
  if (rc) return rc;
  void* args[] = {(void*)&gout, (void*)&sp, (void*)&grad_vel, (void*)&G, (void*)&g, (void*)&nsteps, (void*)&scale};
  VXM_CUDA(cudaLaunchCooperativeKernel((void*)vecint_bwd_fast_kernel, dim3(grid), dim3(512), args, 0, st));
  return check_launch("vecint_bwd");
}

template <bool IS3D, int ARITH>
static int vecint_fwd_launch(const float* vel, float* out, float* states, float* work, VecGeom g,
                             int nsteps, float scale, cudaStream_t st) {
  auto kern = vecint_fwd_kernel<IS3D, ARITH>;
  int grid = 0;
  int rc = coop_grid(kern, 256, ((size_t)g.B * g.vol.DHW + 255) / 256, &grid);
  if (rc) return rc;
  void* args[] = {(void*)&vel, (void*)&out, (void*)&states, (void*)&work, (void*)&g, (void*)&nsteps, (void*)&scale};
  VXM_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(grid), dim3(256), args, 0, st));
  return check_launch("vecint_fwd");
}

extern "C" int vxm_vecint_fwd(const float* vel, float* out, float* states, void* work, int B, int D,
                              int H, int W, int nd, int nsteps, int arith, void* stream) {
  VXM_REQUIRE(nd == 2 || nd == 3, "vecint: nd must be 2 or 3");
  VXM_REQUIRE(nsteps >= 0 && nsteps < 31, "vecint: nsteps should be >= 0, found: %d", nsteps);  // layers.py:59
  VXM_REQUIRE(vel && out, "vecint_fwd: null pointer");
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "vecint: non-positive dimension");
  VXM_REQUIRE(nd == 3 || D == 1, "vecint: a 2-D problem must be passed with D == 1");
  VXM_REQUIRE(states || work || nsteps == 0, "vecint_fwd: need `states` or `work`");
  if (arith == VXM_ARITH_FAST) return vecint_fwd_fast(vel, out, states, work, B, D, H, W, nd, nsteps, as_stream(stream));
  VecGeom g = make_vgeom(B, D, H, W, nd);
  float scale = 1.0f / (float)(1u << nsteps);
  cudaStream_t st = as_stream(stream);
  bool rec = arith == VXM_ARITH_RECIPROCAL;
  if (nd == 3) return rec ? vecint_fwd_launch<true, 1>(vel, out, states, (float*)work, g, nsteps, scale, st)
                          : vecint_fwd_launch<true, 0>(vel, out, states, (float*)work, g, nsteps, scale, st);
  return rec ? vecint_fwd_launch<false, 1>(vel, out, states, (float*)work, g, nsteps, scale, st)
             : vecint_fwd_launch<false, 0>(vel, out, states, (float*)work, g, nsteps, scale, st);
}

template <bool IS3D, int ARITH>
static int vecint_bwd_launch(const float* gout, const float* states, float* grad_vel, float* work,
                             VecGeom g, int nsteps, float scale, cudaStream_t st) {
  auto kern = vecint_bwd_kernel<IS3D, ARITH>;
  int grid = 0;
  int rc = coop_grid(kern, 256, ((size_t)g.B * g.vol.DHW + 255) / 256, &grid);
  if (rc) return rc;
  float mx = (g.ax.src_sm1 * 0.5f) * 2.0f / g.ax.sm1;
  float my = (g.ay.src_sm1 * 0.5f) * 2.0f / g.ay.sm1;
  float mz = IS3D ? (g.az.src_sm1 * 0.5f) * 2.0f / g.az.sm1 : 0.f;
  void* args[] = {(void*)&gout, (void*)&states, (void*)&grad_vel, (void*)&work, (void*)&g, (void*)&nsteps,
                  (void*)&scale, (void*)&mz, (void*)&my, (void*)&mx};
  VXM_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(grid), dim3(256), args, 0, st));
  return check_launch("vecint_bwd");
}

extern "C" int vxm_vecint_bwd(const float* grad_out, const float* states, float* grad_vel, void* work,
                              int B, int D, int H, int W, int nd, int nsteps, int arith, void* stream) {
  VXM_REQUIRE(nd == 2 || nd == 3, "vecint: nd must be 2 or 3");
  VXM_REQUIRE(nsteps >= 0 && nsteps < 31, "vecint: nsteps should be >= 0, found: %d", nsteps);
  VXM_REQUIRE(grad_out && grad_vel, "vecint_bwd: null pointer");
  VXM_REQUIRE(nsteps == 0 || (states && work), "vecint_bwd: need `states` and `work`");
  VXM_REQUIRE(nd == 3 || D == 1, "vecint: a 2-D problem must be passed with D == 1");
  if (arith == VXM_ARITH_FAST) return vecint_bwd_fast(grad_out, states, grad_vel, work, B, D, H, W, nd, nsteps, as_stream(stream));
  VecGeom g = make_vgeom(B, D, H, W, nd);
  float scale = 1.0f / (float)(1u << nsteps);
  cudaStream_t st = as_stream(stream);
  bool rec = arith == VXM_ARITH_RECIPROCAL;
  if (nd == 3) return rec ? vecint_bwd_launch<true, 1>(grad_out, states, grad_vel, (float*)work, g, nsteps, scale, st)
                          : vecint_bwd_launch<true, 0>(grad_out, states, grad_vel, (float*)work, g, nsteps, scale, st);
  return rec ? vecint_bwd_launch<false, 1>(grad_out, states, grad_vel, (float*)work, g, nsteps, scale, st)
             : vecint_bwd_launch<false, 0>(grad_out, states, grad_vel, (float*)work, g, nsteps, scale, st);
}
