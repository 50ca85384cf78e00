// Trilinear / nearest sampling shared by the warp and VecInt kernels, written once per arithmetic mode.
//
// Reference semantics: voxelmorph/torch/layers.py:30-48 -> F.grid_sample(align_corners=True, padding_mode='zeros').
// Corners are numbered in ATen's order: bit0 = x+1, bit1 = y+1, bit2 = z+1; a corner outside the volume reads as 0
// and receives no gradient.
//
// * Exact mode (VXM_ARITH_TRUE_DIV / VXM_ARITH_RECIPROCAL): the reference's coordinate replay (`exact_coords`),
//   ATen grid_sampler_3d's corner weights (products (x1-x)(y1-y)(z1-z) ...) and accumulation order, every product
//   and sum an explicit _rn intrinsic so that the result does not depend on FMA contraction.  The linear path
//   reproduces the torch CPU reference to the bit on every input we have tried; the nearest path is bit-exact by
//   construction.  This is the reference mode the bit-exact tests compare against.
// * Fast mode (VXM_ARITH_FAST): coordinates (p + v)·r computed by the caller, the blend and its gradient as lerp
//   trees, and cells that lie inside the volume (all but a one-voxel shell for registration flows) read their
//   corners without per-corner predicates.
#pragma once
#include "common.cuh"

namespace vxm {

struct Vol {
  int D, H, W;
  size_t HW, DHW;
};
__host__ __device__ inline Vol make_vol(int D, int H, int W) {
  Vol v;
  v.D = D; v.H = H; v.W = W;
  v.HW = (size_t)H * W;
  v.DHW = (size_t)D * H * W;
  return v;
}

// ------------------------------------------------------------------------------------------------------------
// Exact mode
// ------------------------------------------------------------------------------------------------------------

// Replays the reference's sampling coordinates of voxel (z, y, x).  f points at the voxel's first field channel,
// cs is the channel stride (channel order D, H, W for 3-D; H, W for 2-D); fv receives the field's own values.
// G is any geometry with the AxisNorms ax, ay, az.  Plain loads: VecInt reads fields written earlier in its launch.
template <bool IS3D, int ARITH, class G>
__device__ __forceinline__ void exact_coords(const float* f, size_t cs, int z, int y, int x, const G& g, float fv[3],
                                             float& cz, float& cy, float& cx) {
  if (IS3D) {
    fv[0] = f[0]; fv[1] = f[cs]; fv[2] = f[2 * cs];
    cz = sample_coord<ARITH>((float)z, fv[0], g.az);
    cy = sample_coord<ARITH>((float)y, fv[1], g.ay);
    cx = sample_coord<ARITH>((float)x, fv[2], g.ax);
  } else {
    fv[0] = f[0]; fv[1] = f[cs]; fv[2] = 0.f;
    cz = 0.f;
    cy = sample_coord<ARITH>((float)y, fv[0], g.ay);
    cx = sample_coord<ARITH>((float)x, fv[1], g.ax);
  }
}

// The trilinear cell of one exact-mode sample point: per corner a clamped offset (always loadable) and a weight, per
// axis the two tap weights, and the mask of the corners inside the volume.  A tap outside the volume has weight 0.
template <bool IS3D>
struct ExactCell {
  int off[8];
  float w[8];      // (x-weight * y-weight) * z-weight, each product rounded (ATen order)
  float wx[2], wy[2], wz[2];
  unsigned mask;   // bit k set <=> corner k inside the volume
};

template <bool IS3D>
__device__ __forceinline__ ExactCell<IS3D> exact_cell(float cz, float cy, float cx, int D, int H, int W) {
  ExactCell<IS3D> c;
  const float fx = floorf(cx), fy = floorf(cy);
  const int x0 = f2i(fx), y0 = f2i(fy);
  const bool xok[2] = {(unsigned)x0 < (unsigned)W, (unsigned)(x0 + 1) < (unsigned)W};
  const bool yok[2] = {(unsigned)y0 < (unsigned)H, (unsigned)(y0 + 1) < (unsigned)H};
  bool zok[2] = {true, false};
  c.wx[0] = xok[0] ? __fsub_rn(__fadd_rn(fx, 1.0f), cx) : 0.f;
  c.wx[1] = xok[1] ? __fsub_rn(cx, fx) : 0.f;
  c.wy[0] = yok[0] ? __fsub_rn(__fadd_rn(fy, 1.0f), cy) : 0.f;
  c.wy[1] = yok[1] ? __fsub_rn(cy, fy) : 0.f;
  const int ox[2] = {min(max(x0, 0), W - 1), min(max(x0, -1) + 1, W - 1)};
  const int oy[2] = {min(max(y0, 0), H - 1) * W, min(max(y0, -1) + 1, H - 1) * W};
  int oz[2] = {0, 0};
  c.wz[0] = 1.0f; c.wz[1] = 0.0f;
  if (IS3D) {
    const float fz = floorf(cz);
    const int z0 = f2i(fz);
    zok[0] = (unsigned)z0 < (unsigned)D;
    zok[1] = (unsigned)(z0 + 1) < (unsigned)D;
    c.wz[0] = zok[0] ? __fsub_rn(__fadd_rn(fz, 1.0f), cz) : 0.f;
    c.wz[1] = zok[1] ? __fsub_rn(cz, fz) : 0.f;
    oz[0] = min(max(z0, 0), D - 1) * (H * W); oz[1] = min(max(z0, -1) + 1, D - 1) * (H * W);
  }
  c.mask = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    c.off[k] = oz[k >> 2] + oy[(k >> 1) & 1] + ox[k & 1];
    const float w = __fmul_rn(c.wx[k & 1], c.wy[(k >> 1) & 1]);
    c.w[k] = IS3D ? __fmul_rn(w, c.wz[k >> 2]) : w;
    c.mask |= (zok[k >> 2] && yok[(k >> 1) & 1] && xok[k & 1]) ? (1u << k) : 0u;
  }
  return c;
}

// Value of one channel plane at the cell, branch free: a corner outside the volume has weight 0 and acc + v*0 leaves
// acc unchanged, so this equals the masked sum bit for bit (for finite inputs).  READONLY: the plane is not written
// during the launch, so it may go through the read-only path.
template <bool IS3D, bool READONLY>
__device__ __forceinline__ float exact_sample(const float* __restrict__ plane, const ExactCell<IS3D>& c) {
  float acc = 0.0f;
#pragma unroll
  for (int k = 0; k < (IS3D ? 8 : 4); ++k) {
    const float v = READONLY ? __ldg(plane + c.off[k]) : plane[c.off[k]];
    acc = __fadd_rn(acc, __fmul_rn(v, c.w[k]));
  }
  return acc;
}

// d(value)/d(coordinate) in signed-sum form, added to (gz, gy, gx).  s(off) is the scalar corner k carries: its value
// times an adjoint, or its channels dotted with one.
template <bool IS3D, class S>
__device__ __forceinline__ void exact_grad(const ExactCell<IS3D>& c, S s, float& gz, float& gy, float& gx) {
#pragma unroll
  for (int k = 0; k < (IS3D ? 8 : 4); ++k) {
    if (c.mask & (1u << k)) {
      const float v = s(c.off[k]);
      const float wx = c.wx[k & 1], wy = c.wy[(k >> 1) & 1], wz = IS3D ? c.wz[k >> 2] : 1.0f;
      gx += ((k & 1) ? v : -v) * wy * wz;
      gy += ((k & 2) ? v : -v) * wx * wz;
      if (IS3D) gz += ((k & 4) ? v : -v) * wx * wy;
    }
  }
}

// d(value)/d(plane): adds weight(k) * go to every corner inside the volume (fp32 atomics)
template <bool IS3D>
__device__ __forceinline__ void exact_scatter(const ExactCell<IS3D>& c, float* plane, float go) {
#pragma unroll
  for (int k = 0; k < (IS3D ? 8 : 4); ++k)
    if (c.mask & (1u << k)) atomicAdd(plane + c.off[k], c.w[k] * go);
}

// nearest index (round half to even) or -1 when outside the volume
template <bool IS3D>
__device__ __forceinline__ ptrdiff_t nearest_index(float cx, float cy, float cz, const Vol& s) {
  int x = f2i(rintf(cx)), y = f2i(rintf(cy));
  int z = IS3D ? f2i(rintf(cz)) : 0;
  bool ok = (unsigned)x < (unsigned)s.W && (unsigned)y < (unsigned)s.H && (unsigned)z < (unsigned)s.D;
  return ok ? ((ptrdiff_t)z * s.H + y) * (ptrdiff_t)s.W + x : (ptrdiff_t)-1;
}

// ------------------------------------------------------------------------------------------------------------
// Fast mode
// ------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ float scaled(float g, float w) { return w * g; }
__device__ __forceinline__ float4 scaled(const float4& g, float w) { return make_float4(w * g.x, w * g.y, w * g.z, 0.f); }

// The trilinear cell of one fast-mode sample point.  Corner values are per channel plane (float) or per voxel of an
// interleaved field (float4); the blend and gradient take scalars.
template <bool IS3D>
struct FastCell {
  int x0, y0, z0;                // integer corner
  float tx, ty, tz;              // fractions
  bool inx[2], iny[2], inz[2];   // is the lower / upper tap of each axis inside the volume
  int ox[2], oy[2], oz[2];       // clamped per-axis offsets (always loadable; rows and planes pre-multiplied)
  bool interior;                 // all 8 corners inside: they lie at base + step(k)
  int base, W, HW;

  __device__ __forceinline__ int off(int k) const { return oz[k >> 2] + oy[(k >> 1) & 1] + ox[k & 1]; }
  __device__ __forceinline__ int step(int k) const { return (k & 1) + ((k >> 1) & 1) * W + (k >> 2) * HW; }
  __device__ __forceinline__ bool inside(int k) const { return inz[k >> 2] && iny[(k >> 1) & 1] && inx[k & 1]; }
  __device__ __forceinline__ float weight(int k) const {
    const float wx = (k & 1) ? tx : 1.f - tx, wy = (k & 2) ? ty : 1.f - ty;
    return IS3D ? ((k & 4) ? tz : 1.f - tz) * wy * wx : wy * wx;
  }

  // the corner values of a plane that is not written during the launch, 0 outside the volume
  template <class T>
  __device__ __forceinline__ void fetch(const T* __restrict__ plane, T (&u)[8]) const {
    if (interior) {
      const T* s = plane + base;
#pragma unroll
      for (int k = 0; k < (IS3D ? 8 : 4); ++k) u[k] = __ldg(s + step(k));
    } else {
#pragma unroll
      for (int k = 0; k < (IS3D ? 8 : 4); ++k) u[k] = inside(k) ? __ldg(plane + off(k)) : T();
    }
  }

  // three nested lerps: along x, then y, then z
  __device__ __forceinline__ float blend(const float (&u)[8]) const {
    const float r0 = fmaf(tx, u[1] - u[0], u[0]), r1 = fmaf(tx, u[3] - u[2], u[2]);
    float v = fmaf(ty, r1 - r0, r0);
    if (IS3D) {
      const float q0 = fmaf(tx, u[5] - u[4], u[4]), q1 = fmaf(tx, u[7] - u[6], u[6]);
      const float v1 = fmaf(ty, q1 - q0, q0);
      v = fmaf(tz, v1 - v, v);
    }
    return v;
  }

  // d(blend)/d(coordinate) from the same lerp tree; d/dx is lerp_z(lerp_y(upper - lower along x)), d/dy and d/dz alike
  __device__ __forceinline__ void grad(const float (&u)[8], float& dz, float& dy, float& dx) const {
    const float ex0 = u[1] - u[0], ex1 = u[3] - u[2];
    const float dxa = fmaf(ty, ex1 - ex0, ex0);
    const float ra0 = fmaf(tx, ex0, u[0]), ra1 = fmaf(tx, ex1, u[2]);
    const float dya = ra1 - ra0;
    if (IS3D) {
      const float fx0 = u[5] - u[4], fx1 = u[7] - u[6];
      const float dxb = fmaf(ty, fx1 - fx0, fx0);
      const float rb0 = fmaf(tx, fx0, u[4]), rb1 = fmaf(tx, fx1, u[6]);
      const float dyb = rb1 - rb0;
      dx = fmaf(tz, dxb - dxa, dxa);
      dy = fmaf(tz, dyb - dya, dya);
      dz = fmaf(ty, rb1 - rb0, rb0) - fmaf(ty, ra1 - ra0, ra0);
    } else {
      dx = dxa;
      dy = dya;
      dz = 0.f;
    }
  }

  // d(blend)/d(plane): adds weight(k) * go to every corner inside the volume (fp32 atomics; a float4 adjoint is one
  // red.global.add.v4.f32 per corner)
  template <class T>
  __device__ __forceinline__ void scatter(T* plane, const T& go) const {
    if (interior) {
      T* s = plane + base;
#pragma unroll
      for (int k = 0; k < (IS3D ? 8 : 4); ++k) atomicAdd(s + step(k), scaled(go, weight(k)));
    } else {
#pragma unroll
      for (int k = 0; k < (IS3D ? 8 : 4); ++k)
        if (inside(k)) atomicAdd(plane + off(k), scaled(go, weight(k)));
    }
  }

  // VecInt's branch-free blend of the float4 values at the clamped offsets off(k): every tap is weighted by (1 - t, t),
  // or 0 outside the volume, so interior and border voxels run the same code and the gathers of several voxels can be
  // in flight together
  __device__ __forceinline__ float4 weighted_blend(const float4 (&u)[8]) const {
    const float wx[2] = {inx[0] ? 1.f - tx : 0.f, inx[1] ? tx : 0.f};
    const float wy[2] = {iny[0] ? 1.f - ty : 0.f, iny[1] ? ty : 0.f};
    const float wz[2] = {inz[0] ? 1.f - tz : 0.f, inz[1] ? tz : 0.f};
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int zz = 0; zz < 2; ++zz) {
      float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int yy = 0; yy < 2; ++yy) {
        const float4& a = u[zz * 4 + yy * 2], & b = u[zz * 4 + yy * 2 + 1];
        const float qx = fmaf(wx[1], b.x, wx[0] * a.x), qy = fmaf(wx[1], b.y, wx[0] * a.y), qz = fmaf(wx[1], b.z, wx[0] * a.z);
        p.x = fmaf(wy[yy], qx, p.x); p.y = fmaf(wy[yy], qy, p.y); p.z = fmaf(wy[yy], qz, p.z);
      }
      r.x = fmaf(wz[zz], p.x, r.x); r.y = fmaf(wz[zz], p.y, r.y); r.z = fmaf(wz[zz], p.z, r.z);
    }
    return r;
  }
};

template <bool IS3D>
__device__ __forceinline__ FastCell<IS3D> fast_cell(float cz, float cy, float cx, int D, int H, int W) {
  FastCell<IS3D> c;
  const float fx = floorf(cx), fy = floorf(cy), fz = IS3D ? floorf(cz) : 0.f;
  c.x0 = f2i(fx); c.y0 = f2i(fy); c.z0 = IS3D ? f2i(fz) : 0;
  c.tx = cx - fx; c.ty = cy - fy; c.tz = IS3D ? cz - fz : 0.f;
  c.inx[0] = (unsigned)c.x0 < (unsigned)W; c.inx[1] = (unsigned)(c.x0 + 1) < (unsigned)W;
  c.iny[0] = (unsigned)c.y0 < (unsigned)H; c.iny[1] = (unsigned)(c.y0 + 1) < (unsigned)H;
  c.inz[0] = !IS3D || (unsigned)c.z0 < (unsigned)D; c.inz[1] = IS3D && (unsigned)(c.z0 + 1) < (unsigned)D;
  c.W = W; c.HW = H * W;
  c.ox[0] = min(max(c.x0, 0), W - 1); c.ox[1] = min(max(c.x0, -1) + 1, W - 1);
  c.oy[0] = min(max(c.y0, 0), H - 1) * W; c.oy[1] = min(max(c.y0, -1) + 1, H - 1) * W;
  c.oz[0] = IS3D ? min(max(c.z0, 0), D - 1) * c.HW : 0; c.oz[1] = IS3D ? min(max(c.z0, -1) + 1, D - 1) * c.HW : 0;
  c.interior = (unsigned)c.x0 < (unsigned)(W - 1) && (unsigned)c.y0 < (unsigned)(H - 1) &&
               (!IS3D || (unsigned)c.z0 < (unsigned)(D - 1));
  c.base = (c.z0 * H + c.y0) * W + c.x0;
  return c;
}

// ------------------------------------------------------------------------------------------------------------
// Clamped mode: neurite's ne.utils.interpn(vol, loc, 'linear', fill_value=None), which the reference's surface
// utilities sample with (voxelmorph/tf/utils/utils.py:71-88, 465-499).  Per axis of size n at coordinate x:
//   c = clip(x, 0, n-1),  i0 = clip(floor(x), 0, n-1),  i1 = clip(i0 + 1, 0, n-1),
//   weight (i1 - c) on i0 and 1 - (i1 - c) on i1; the axis weights multiply.
// Outside the volume the value is the border value.  d/dx is the cell's difference along the axis where
// 0 <= x <= n-1 (both ends included: the clip passes its gradient there) and 0 elsewhere; at an integer k < n-1 that
// is the forward difference v[k+1] - v[k], at n-1 it is 0 (i0 == i1).
// ------------------------------------------------------------------------------------------------------------

struct ClampTap {
  int i0, i1;      // the two taps (equal on the last voxel)
  float w0, w1;    // their weights
  float pass;      // 1 where the clip passes the gradient, else 0
};

__device__ __forceinline__ ClampTap clamp_tap(float x, int n) {
  ClampTap t;
  const float hi = (float)(n - 1);
  const float c = fminf(fmaxf(x, 0.f), hi);
  t.i0 = (int)fminf(fmaxf(floorf(x), 0.f), hi);   // clip before the cast: wild coordinates stay in range
  t.i1 = min(t.i0 + 1, n - 1);
  t.w0 = (float)t.i1 - c;
  t.w1 = 1.f - t.w0;
  t.pass = (x >= 0.f && x <= hi) ? 1.f : 0.f;
  return t;
}

// The clamped cell of one point over an (D, H, W) plane (2-D: D == 1, only the y and x taps are read).  Corners are
// numbered as in the other cells: bit0 = x+1, bit1 = y+1, bit2 = z+1; every corner is inside the volume.
template <bool IS3D>
struct ClampCell {
  ClampTap tz, ty, tx;
  int W, HW;

  __device__ __forceinline__ int off(int k) const {
    const int z = IS3D ? ((k & 4) ? tz.i1 : tz.i0) : 0, y = (k & 2) ? ty.i1 : ty.i0, x = (k & 1) ? tx.i1 : tx.i0;
    return z * HW + y * W + x;
  }
  // (z-weight * y-weight) * x-weight: interpn's product in axis order
  __device__ __forceinline__ float weight(int k) const {
    const float wy = (k & 2) ? ty.w1 : ty.w0, wx = (k & 1) ? tx.w1 : tx.w0;
    return IS3D ? (((k & 4) ? tz.w1 : tz.w0) * wy) * wx : wy * wx;
  }
  __device__ __forceinline__ float value(const float* __restrict__ plane) const {
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < (IS3D ? 8 : 4); ++k) v = fmaf(weight(k), __ldg(plane + off(k)), v);
    return v;
  }
  // d(value)/d(coordinate), scaled by s, added to (gz, gy, gx)
  __device__ __forceinline__ void grad(const float* __restrict__ plane, float s, float& gz, float& gy, float& gx) const {
    float dz = 0.f, dy = 0.f, dx = 0.f;
#pragma unroll
    for (int k = 0; k < (IS3D ? 8 : 4); ++k) {
      const float v = __ldg(plane + off(k));
      const float wz = IS3D ? ((k & 4) ? tz.w1 : tz.w0) : 1.f, wy = (k & 2) ? ty.w1 : ty.w0, wx = (k & 1) ? tx.w1 : tx.w0;
      dx = fmaf((k & 1) ? v : -v, wz * wy, dx);
      dy = fmaf((k & 2) ? v : -v, wz * wx, dy);
      if (IS3D) dz = fmaf((k & 4) ? v : -v, wy * wx, dz);
    }
    gx = fmaf(s * tx.pass, dx, gx);
    gy = fmaf(s * ty.pass, dy, gy);
    if (IS3D) gz = fmaf(s * tz.pass, dz, gz);
  }
};

template <bool IS3D>
__device__ __forceinline__ ClampCell<IS3D> clamp_cell(float cz, float cy, float cx, int D, int H, int W) {
  ClampCell<IS3D> c;
  c.tz = IS3D ? clamp_tap(cz, D) : ClampTap{0, 0, 1.f, 0.f, 0.f};
  c.ty = clamp_tap(cy, H);
  c.tx = clamp_tap(cx, W);
  c.W = W;
  c.HW = H * W;
  return c;
}

}  // namespace vxm
