// 3x3x3 (or 1x3x3 for 2-D) convolution, stride 1, zero pad 1, + bias + LeakyReLU(0.2):
// reference voxelmorph/torch/networks.py:290-305 (ConvBlock) and :210-215,257 (flow head).
//
// This is the fp32 "parity" engine (CUDA-core FFMA, NCDHW planar): it reproduces the reference's
// fp32 convolution to ~1e-6 relative so that the 1e-4 flow / moved-image tolerance holds through
// the 12-layer U-Net.  The bf16 wgmma implicit-GEMM engine (conv3d_tc.cu) is the
// throughput path.
//
// forward / dgrad share one kernel: dgrad is the same convolution with the roles of Cin / Cout
// swapped and the taps flipped, its input (grad_y) masked on load by the LeakyReLU derivative
// taken from the saved activation y.  wgrad is a split-K reduction over voxels with a
// deterministic second-stage sum.
#include "common.cuh"

namespace vxm {

constexpr int CTW = 32, CTH = 16, CCK = 4;   // output tile 32 x 16 (x 1 slice), 4 input channels per stage
constexpr int CSW = CTW + 2 + 1;             // padded smem row

struct ConvArgs {
  const float* x;       // input  (B, Cin, D, H, W)
  const float* mask;    // optional: same shape as x; x is scaled by (mask < 0 ? slope : 1) on load
  const float* w;       // weights, original layout (Co_orig, Ci_orig, KD, 3, 3)
  const float* bias;    // optional (Cout)
  float* y;             // output (B, Cout, D, H, W)
  int B, Cin, Cout, D, H, W;
  int transposed;       // 1: dgrad addressing  w'[in][tap][out] = w[(in*Cout + out)*T + (T-1-tap)]
  float slope;          // epilogue LeakyReLU slope (<0: none); also the mask slope
  int tiles_w;
};

template <int KD, int COB>
__global__ void __launch_bounds__(256) conv_fwd_kernel(ConvArgs a) {
  constexpr int T = KD * 9;
  __shared__ float s_x[CCK][KD][CTH + 2][CSW];
  __shared__ __align__(16) float s_w[CCK][T][COB];

  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;  // ty 0..7 -> rows ty, ty+8
  const int tile = blockIdx.x, tw = tile % a.tiles_w, th = tile / a.tiles_w;
  const int w0 = tw * CTW, h0 = th * CTH, z = blockIdx.y;
  const int ncob = (a.Cout + COB - 1) / COB;
  const int cob = blockIdx.z % ncob, b = blockIdx.z / ncob;
  const int co0 = cob * COB;
  const size_t HW = (size_t)a.H * a.W, DHW = HW * a.D;
  const float* xb = a.x + (size_t)b * a.Cin * DHW;
  const float* mb = a.mask ? a.mask + (size_t)b * a.Cin * DHW : nullptr;

  float acc0[COB], acc1[COB];
#pragma unroll
  for (int i = 0; i < COB; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }

  for (int c0 = 0; c0 < a.Cin; c0 += CCK) {
    // ---- stage input chunk (zero padded, optional LeakyReLU-derivative mask) ----
    constexpr int NX = CCK * KD * (CTH + 2) * (CTW + 2);
    for (int idx = tid; idx < NX; idx += 256) {
      int c = idx % (CTW + 2);
      int r = (idx / (CTW + 2)) % (CTH + 2);
      int k = (idx / ((CTW + 2) * (CTH + 2))) % KD;
      int ci = idx / ((CTW + 2) * (CTH + 2) * KD);
      int zz = z + k - (KD / 2), hh = h0 + r - 1, ww = w0 + c - 1;
      float v = 0.f;
      if (c0 + ci < a.Cin && zz >= 0 && zz < a.D && hh >= 0 && hh < a.H && ww >= 0 && ww < a.W) {
        size_t off = (size_t)(c0 + ci) * DHW + (size_t)zz * HW + (size_t)hh * a.W + ww;
        v = __ldg(xb + off);
        if (mb && __ldg(mb + off) < 0.f) v *= a.slope;
      }
      s_x[ci][k][r][c] = v;
    }
    // ---- stage weights chunk ----
    for (int idx = tid; idx < CCK * T * COB; idx += 256) {
      int co = idx % COB, t = (idx / COB) % T, ci = idx / (COB * T);
      float v = 0.f;
      if (c0 + ci < a.Cin && co0 + co < a.Cout) {
        if (!a.transposed) v = __ldg(a.w + ((size_t)(co0 + co) * a.Cin + (c0 + ci)) * T + t);
        else v = __ldg(a.w + ((size_t)(c0 + ci) * a.Cout + (co0 + co)) * T + (T - 1 - t));
      }
      s_w[ci][t][co] = v;
    }
    __syncthreads();
#pragma unroll
    for (int ci = 0; ci < CCK; ++ci) {
#pragma unroll
      for (int k = 0; k < KD; ++k) {
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            float x0 = s_x[ci][k][ty + kh][tx + kw];
            float x1 = s_x[ci][k][ty + 8 + kh][tx + kw];
            const float4* wp = reinterpret_cast<const float4*>(&s_w[ci][k * 9 + kh * 3 + kw][0]);
#pragma unroll
            for (int q = 0; q < COB / 4; ++q) {
              float4 wv = wp[q];
              acc0[4 * q + 0] = fmaf(x0, wv.x, acc0[4 * q + 0]);
              acc0[4 * q + 1] = fmaf(x0, wv.y, acc0[4 * q + 1]);
              acc0[4 * q + 2] = fmaf(x0, wv.z, acc0[4 * q + 2]);
              acc0[4 * q + 3] = fmaf(x0, wv.w, acc0[4 * q + 3]);
              acc1[4 * q + 0] = fmaf(x1, wv.x, acc1[4 * q + 0]);
              acc1[4 * q + 1] = fmaf(x1, wv.y, acc1[4 * q + 1]);
              acc1[4 * q + 2] = fmaf(x1, wv.z, acc1[4 * q + 2]);
              acc1[4 * q + 3] = fmaf(x1, wv.w, acc1[4 * q + 3]);
            }
          }
        }
      }
    }
    __syncthreads();
  }
  // ---- epilogue: bias + LeakyReLU ----
  const int w = w0 + tx;
  if (w < a.W) {
    float* yb = a.y + (size_t)b * a.Cout * DHW + (size_t)z * HW + w;
#pragma unroll
    for (int co = 0; co < COB; ++co) {
      if (co0 + co < a.Cout) {
        float bv = a.bias ? __ldg(a.bias + co0 + co) : 0.f;
        float v0 = acc0[co] + bv, v1 = acc1[co] + bv;
        if (a.slope >= 0.f && !a.transposed) {
          v0 = v0 >= 0.f ? v0 : v0 * a.slope;
          v1 = v1 >= 0.f ? v1 : v1 * a.slope;
        }
        int h = h0 + ty;
        if (h < a.H) yb[(size_t)(co0 + co) * DHW + (size_t)h * a.W] = v0;
        if (h + 8 < a.H) yb[(size_t)(co0 + co) * DHW + (size_t)(h + 8) * a.W] = v1;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// wgrad:  gw[co][ci][tap] = sum_{b,v} gz[b,co,v] * x[b,ci,v + tap - 1],  gz = gy * lrelu'(y)
// Block = 288 threads = 4 co-groups(4 co) x 8 ci x 9 (kd,kh) ; each thread owns 4 co x 3 kw.
// grid.x = spatial splits (persistent over tiles), grid.y = (Cout/16) * (Cin/8) channel blocks.
// Partials go to work[split][Cout*Cin*T]; a second kernel sums splits in order (deterministic).
// ---------------------------------------------------------------------------------------------
constexpr int WTW = 32, WTH = 8, WCO = 16, WCI = 8;

struct WgradArgs {
  const float* gy; const float* y; const float* x;
  float* partial;     // [nsplit][Cout][Cin][T]
  float* gbias_part;  // [nsplit][Cout] (written by channel block ci==0) or null
  int B, Cin, Cout, D, H, W;
  float slope;
  int tiles_w, tiles_h, ntiles;  // tiles over (b, z, th, tw)
};

template <int KD>
__global__ void __launch_bounds__(288) conv_wgrad_kernel(WgradArgs a) {
  constexpr int T = KD * 9;
  __shared__ float s_g[WCO][WTH][WTW];
  __shared__ float s_x[WCI][KD][WTH + 2][WTW + 2];
  const int tid = threadIdx.x;
  const int kk = tid % 9;            // kd*3 + kh   (kd < KD)
  const int ci = (tid / 9) % WCI;
  const int cog = tid / (9 * WCI);   // 0..3
  const int kd = kk / 3, kh = kk % 3;
  const bool active = kd < KD;
  const int nci = (a.Cin + WCI - 1) / WCI;
  const int cib = blockIdx.y % nci, cob = blockIdx.y / nci;
  const int ci0 = cib * WCI, co0 = cob * WCO;
  const size_t HW = (size_t)a.H * a.W, DHW = HW * a.D;

  float acc[4][3];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) acc[i][j] = 0.f;
  float bacc = 0.f;  // bias gradient: thread (co = tid < 16) sums gz over its tiles

  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    int tw = tile % a.tiles_w;
    int th = (tile / a.tiles_w) % a.tiles_h;
    int z = (tile / (a.tiles_w * a.tiles_h)) % a.D;
    int b = tile / (a.tiles_w * a.tiles_h * a.D);
    int w0 = tw * WTW, h0 = th * WTH;
    const float* gb = a.gy + (size_t)b * a.Cout * DHW;
    const float* yb = a.y ? a.y + (size_t)b * a.Cout * DHW : nullptr;
    const float* xb = a.x + (size_t)b * a.Cin * DHW;
    for (int idx = tid; idx < WCO * WTH * WTW; idx += 288) {
      int c = idx % WTW, r = (idx / WTW) % WTH, co = idx / (WTW * WTH);
      int hh = h0 + r, ww = w0 + c;
      float v = 0.f;
      if (co0 + co < a.Cout && hh < a.H && ww < a.W) {
        size_t off = (size_t)(co0 + co) * DHW + (size_t)z * HW + (size_t)hh * a.W + ww;
        v = __ldg(gb + off);
        if (yb && a.slope >= 0.f && __ldg(yb + off) < 0.f) v *= a.slope;
      }
      s_g[co][r][c] = v;
    }
    constexpr int NX = WCI * KD * (WTH + 2) * (WTW + 2);
    for (int idx = tid; idx < NX; idx += 288) {
      int c = idx % (WTW + 2);
      int r = (idx / (WTW + 2)) % (WTH + 2);
      int k = (idx / ((WTW + 2) * (WTH + 2))) % KD;
      int cc = idx / ((WTW + 2) * (WTH + 2) * KD);
      int zz = z + k - (KD / 2), hh = h0 + r - 1, ww = w0 + c - 1;
      float v = 0.f;
      if (ci0 + cc < a.Cin && zz >= 0 && zz < a.D && hh >= 0 && hh < a.H && ww >= 0 && ww < a.W)
        v = __ldg(xb + (size_t)(ci0 + cc) * DHW + (size_t)zz * HW + (size_t)hh * a.W + ww);
      s_x[cc][k][r][c] = v;
    }
    __syncthreads();
    if (active) {
      for (int r = 0; r < WTH; ++r) {
        const float* xr = &s_x[ci][kd][r + kh][0];
        float xa = xr[0], xb2 = xr[1];
#pragma unroll 8
        for (int c = 0; c < WTW; ++c) {
          float xc = xr[c + 2];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float g = s_g[cog * 4 + i][r][c];
            acc[i][0] = fmaf(g, xa, acc[i][0]);
            acc[i][1] = fmaf(g, xb2, acc[i][1]);
            acc[i][2] = fmaf(g, xc, acc[i][2]);
          }
          xa = xb2; xb2 = xc;
        }
      }
    }
    if (a.gbias_part && cib == 0 && tid < WCO) {
      for (int r = 0; r < WTH; ++r)
        for (int c = 0; c < WTW; ++c) bacc += s_g[tid][r][(c + tid) & (WTW - 1)];
    }
    __syncthreads();
  }
  float* part = a.partial + (size_t)blockIdx.x * a.Cout * a.Cin * T;
  if (active && ci0 + ci < a.Cin) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int co = co0 + cog * 4 + i;
      if (co < a.Cout) {
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) part[((size_t)co * a.Cin + ci0 + ci) * T + kd * 9 + kh * 3 + kw] = acc[i][kw];
      }
    }
  }
  if (a.gbias_part && cib == 0 && tid < WCO && co0 + tid < a.Cout) a.gbias_part[(size_t)blockIdx.x * a.Cout + co0 + tid] = bacc;
}

__global__ void __launch_bounds__(256) split_reduce_kernel(const float* __restrict__ partial, float* __restrict__ out,
                                                           int n, int nsplit) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = 0.f;
  for (int s = 0; s < nsplit; ++s) acc += partial[(size_t)s * n + i];
  out[i] += acc;  // accumulate into the (zero-filled once per step) gradient buffer
}

static int wgrad_splits() { return 2 * sm_count(); }

template <int KD>
static void launch_fwd(const ConvArgs& a, dim3 grid, cudaStream_t st) {
  if (a.Cout <= 8) conv_fwd_kernel<KD, 8><<<dim3(grid.x, grid.y, a.B * ((a.Cout + 7) / 8)), 256, 0, st>>>(a);
  else if (a.Cout <= 16) conv_fwd_kernel<KD, 16><<<dim3(grid.x, grid.y, a.B), 256, 0, st>>>(a);
  else conv_fwd_kernel<KD, 32><<<dim3(grid.x, grid.y, a.B * ((a.Cout + 31) / 32)), 256, 0, st>>>(a);
}

static int conv_check(int B, int Cin, int Cout, int D, int H, int W, int kd) {
  VXM_REQUIRE(B > 0 && Cin > 0 && Cout > 0 && D > 0 && H > 0 && W > 0, "conv3d: non-positive dimension");
  VXM_REQUIRE(kd == 1 || kd == 3, "conv3d: kd must be 1 or 3");
  VXM_REQUIRE(D <= 65535 && (size_t)B * ((Cout + 7) / 8) <= 65535u, "conv3d: dimension exceeds launch grid limits");
  return VXM_OK;
}

}  // namespace vxm

using namespace vxm;

extern "C" int vxm_conv3d_fwd_f32(const float* x, const float* w, const float* bias, float* y, int B, int Cin,
                                  int Cout, int D, int H, int W, int kd, float leaky_slope, void* stream) {
  int rc = conv_check(B, Cin, Cout, D, H, W, kd);
  if (rc) return rc;
  VXM_REQUIRE(x && w && y, "conv3d_fwd: null pointer");
  ConvArgs a{};
  a.x = x; a.w = w; a.bias = bias; a.y = y; a.mask = nullptr;
  a.B = B; a.Cin = Cin; a.Cout = Cout; a.D = D; a.H = H; a.W = W;
  a.transposed = 0; a.slope = leaky_slope;
  a.tiles_w = (W + CTW - 1) / CTW;
  dim3 grid(a.tiles_w * ((H + CTH - 1) / CTH), D, 1);
  if (kd == 3) launch_fwd<3>(a, grid, as_stream(stream)); else launch_fwd<1>(a, grid, as_stream(stream));
  return check_launch("conv3d_fwd_f32");
}

extern "C" size_t vxm_conv3d_bwd_workspace_bytes(int B, int Cin, int Cout, int D, int H, int W, int kd) {
  (void)B; (void)D; (void)H; (void)W;
  // worst-case split count (device independent upper bound: 2 * 256 SMs)
  return (size_t)512 * ((size_t)Cout * Cin * kd * 9 + Cout) * sizeof(float);
}

extern "C" int vxm_conv3d_bwd_f32(const float* grad_y, const float* y, const float* x, const float* w, float* grad_x,
                                  float* grad_w, float* grad_b, void* work, int B, int Cin, int Cout, int D, int H,
                                  int W, int kd, float leaky_slope, void* stream) {
  int rc = conv_check(B, Cin, Cout, D, H, W, kd);
  if (rc) return rc;
  VXM_REQUIRE(grad_y && w, "conv3d_bwd: null pointer");
  VXM_REQUIRE(leaky_slope < 0.f || y, "conv3d_bwd: the saved activation is required for the LeakyReLU mask");
  cudaStream_t st = as_stream(stream);
  if (grad_x) {  // dgrad: roles swapped, taps flipped, mask applied on load
    ConvArgs a{};
    a.x = grad_y; a.mask = leaky_slope >= 0.f ? y : nullptr; a.w = w; a.bias = nullptr; a.y = grad_x;
    a.B = B; a.Cin = Cout; a.Cout = Cin; a.D = D; a.H = H; a.W = W;
    a.transposed = 1; a.slope = leaky_slope;
    a.tiles_w = (W + CTW - 1) / CTW;
    dim3 grid(a.tiles_w * ((H + CTH - 1) / CTH), D, 1);
    if (kd == 3) launch_fwd<3>(a, grid, st); else launch_fwd<1>(a, grid, st);
    rc = check_launch("conv3d_dgrad_f32");
    if (rc) return rc;
  }
  if (grad_w) {
    VXM_REQUIRE(x && work, "conv3d_bwd: wgrad needs x and work");
    WgradArgs a{};
    a.gy = grad_y; a.y = leaky_slope >= 0.f ? y : nullptr; a.x = x;
    a.B = B; a.Cin = Cin; a.Cout = Cout; a.D = D; a.H = H; a.W = W; a.slope = leaky_slope;
    a.tiles_w = (W + WTW - 1) / WTW; a.tiles_h = (H + WTH - 1) / WTH;
    a.ntiles = a.tiles_w * a.tiles_h * D * B;
    int T = kd * 9;
    int nsplit = wgrad_splits();
    if (nsplit > a.ntiles) nsplit = a.ntiles;
    if (nsplit > 512) nsplit = 512;
    size_t nW = (size_t)Cout * Cin * T;
    a.partial = (float*)work;
    a.gbias_part = grad_b ? (float*)work + (size_t)nsplit * nW : nullptr;
    dim3 grid(nsplit, ((Cout + WCO - 1) / WCO) * ((Cin + WCI - 1) / WCI));
    if (kd == 3) conv_wgrad_kernel<3><<<grid, 288, 0, st>>>(a); else conv_wgrad_kernel<1><<<grid, 288, 0, st>>>(a);
    rc = check_launch("conv3d_wgrad_f32");
    if (rc) return rc;
    split_reduce_kernel<<<(int)((nW + 255) / 256), 256, 0, st>>>(a.partial, grad_w, (int)nW, nsplit);
    rc = check_launch("conv3d_wgrad_reduce");
    if (rc) return rc;
    if (grad_b) {
      split_reduce_kernel<<<(Cout + 255) / 256, 256, 0, st>>>(a.gbias_part, grad_b, Cout, nsplit);
      rc = check_launch("conv3d_bgrad_reduce");
      if (rc) return rc;
    }
  }
  return VXM_OK;
}
