// Grad / MSE / Dice losses (reference voxelmorph/torch/losses.py:70-135): fused stencil+reduce
// kernels.  Reductions are deterministic (fixed block partial order, double accumulation).
//
// Algorithmic bytes (fp32): Grad 4*C B/voxel fwd (+ 8*C bwd); MSE 8 B/elem fwd (+ 12 bwd);
// Dice 8 B/elem fwd (+ 8 bwd); KL 4 B/elem of flow_params fwd (+ 8 bwd).
#include "common.cuh"

namespace vxm {

ReduceWork as_reduce_work(void* work);  // ncc.cu

struct GradGeom {
  int B, C, D, H, W;
  size_t HW, DHW;
  double cz, cy, cx;  // mult / (nd * B * count_axis); 0 for an unused axis
};

template <int P>
__device__ __forceinline__ float pen(float d) { return P == 1 ? fabsf(d) : d * d; }
template <int P>
__device__ __forceinline__ float dpen(float d) {
  return P == 1 ? (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) : 2.f * d;
}

template <int P>
__global__ void __launch_bounds__(256) gradloss_fwd_kernel(const float* __restrict__ y, float* __restrict__ loss,
                                                           GradGeom g, ReduceWork rw) {
  __shared__ double s_red[32];
  size_t n = (size_t)g.B * g.C * g.DHW;
  double accz = 0, accy = 0, accx = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    size_t p = i % g.DHW;
    int z = (int)(p / g.HW);
    int r = (int)(p - (size_t)z * g.HW);
    int yy = r / g.W, x = r - yy * g.W;
    float v = __ldg(y + i);
    if (x + 1 < g.W) accx += pen<P>(__ldg(y + i + 1) - v);
    if (yy + 1 < g.H) accy += pen<P>(__ldg(y + i + g.W) - v);
    if (z + 1 < g.D) accz += pen<P>(__ldg(y + i + g.HW) - v);
  }
  double tot = block_sum<double>(accz * g.cz + accy * g.cy + accx * g.cx, s_red);
  finish_reduce(tot, rw, gridDim.x, blockIdx.x, 1.0, loss, s_red);
}

template <int P>
__global__ void __launch_bounds__(256) gradloss_bwd_kernel(const float* __restrict__ y, const float* __restrict__ gl,
                                                           float* __restrict__ gy, GradGeom g) {
  size_t n = (size_t)g.B * g.C * g.DHW;
  float s = __ldg(gl);
  float cz = (float)g.cz, cy = (float)g.cy, cx = (float)g.cx;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    size_t p = i % g.DHW;
    int z = (int)(p / g.HW);
    int r = (int)(p - (size_t)z * g.HW);
    int yy = r / g.W, x = r - yy * g.W;
    float v = __ldg(y + i), acc = 0.f;
    if (x > 0) acc += cx * dpen<P>(v - __ldg(y + i - 1));
    if (x + 1 < g.W) acc -= cx * dpen<P>(__ldg(y + i + 1) - v);
    if (yy > 0) acc += cy * dpen<P>(v - __ldg(y + i - g.W));
    if (yy + 1 < g.H) acc -= cy * dpen<P>(__ldg(y + i + g.W) - v);
    if (z > 0) acc += cz * dpen<P>(v - __ldg(y + i - g.HW));
    if (z + 1 < g.D) acc -= cz * dpen<P>(__ldg(y + i + g.HW) - v);
    gy[i] = s * acc;
  }
}

// KL of probabilistic VoxelMorph (reference voxelmorph/tf/losses.py:247-349) on flow_params (B, 2 nd, D, H, W): channels
// [0, nd) the mean mu, [nd, 2 nd) l = log sigma^2.  With deg(v) the number of in-volume axial neighbours of v,
//   loss = 0.5 / (B V) sum (lambda deg e^l - l)  +  sum_axes c_axis sum (mu_{x + e_axis} - mu_x)^2,
// c_axis = lambda / (4 * count_axis), count_axis = B nd (n_axis - 1) V / n_axis (0 for an axis of size 1).
struct KlGeom {
  int B, nd, D, H, W;
  size_t HW, DHW;
  float lam;
  double cz, cy, cx, cs;
};

__device__ __forceinline__ int kl_degree(int z, int yy, int x, const KlGeom& g) {
  return (x > 0) + (x + 1 < g.W) + (yy > 0) + (yy + 1 < g.H) + (z > 0) + (z + 1 < g.D);
}

// one (b, channel) plane per blockIdx.y (mu or l: uniform per block), 32-bit voxel indices within it
__global__ void __launch_bounds__(256) kl_fwd_kernel(const float* __restrict__ y, float* __restrict__ loss, KlGeom g,
                                                     ReduceWork rw) {
  __shared__ double s_red[32];
  const int V = (int)g.DHW, HW = (int)g.HW;
  const float* yp = y + (size_t)blockIdx.y * g.DHW;
  const bool is_mu = (int)(blockIdx.y % (2 * g.nd)) < g.nd;
  double accz = 0, accy = 0, accx = 0, accs = 0;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < V; p += gridDim.x * blockDim.x) {
    int z = p / HW;
    int r = p - z * HW;
    int yy = r / g.W, x = r - yy * g.W;
    float v = __ldg(yp + p);
    if (is_mu) {
      if (x + 1 < g.W) accx += pen<2>(__ldg(yp + p + 1) - v);
      if (yy + 1 < g.H) accy += pen<2>(__ldg(yp + p + g.W) - v);
      if (z + 1 < g.D) accz += pen<2>(__ldg(yp + p + HW) - v);
    } else {
      accs += g.lam * (float)kl_degree(z, yy, x, g) * expf(v) - v;
    }
  }
  double tot = block_sum<double>(accz * g.cz + accy * g.cy + accx * g.cx + accs * g.cs, s_red);
  finish_reduce(tot, rw, gridDim.x * gridDim.y, blockIdx.y * gridDim.x + blockIdx.x, 1.0, loss, s_red);
}

__global__ void __launch_bounds__(256) kl_bwd_kernel(const float* __restrict__ y, const float* __restrict__ gl,
                                                     float* __restrict__ gy, KlGeom g) {
  const int V = (int)g.DHW, HW = (int)g.HW;
  const float* yp = y + (size_t)blockIdx.y * g.DHW;
  float* gp = gy + (size_t)blockIdx.y * g.DHW;
  const bool is_mu = (int)(blockIdx.y % (2 * g.nd)) < g.nd;
  const float s = __ldg(gl);
  const float cz = (float)g.cz, cy = (float)g.cy, cx = (float)g.cx, cs = (float)g.cs;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < V; p += gridDim.x * blockDim.x) {
    int z = p / HW;
    int r = p - z * HW;
    int yy = r / g.W, x = r - yy * g.W;
    float v = __ldg(yp + p), acc;
    if (is_mu) {   // the 2 nd-point Laplacian of mu, each axis scaled by its own count
      acc = 0.f;
      if (x > 0) acc += cx * dpen<2>(v - __ldg(yp + p - 1));
      if (x + 1 < g.W) acc -= cx * dpen<2>(__ldg(yp + p + 1) - v);
      if (yy > 0) acc += cy * dpen<2>(v - __ldg(yp + p - g.W));
      if (yy + 1 < g.H) acc -= cy * dpen<2>(__ldg(yp + p + g.W) - v);
      if (z > 0) acc += cz * dpen<2>(v - __ldg(yp + p - HW));
      if (z + 1 < g.D) acc -= cz * dpen<2>(__ldg(yp + p + HW) - v);
    } else {
      acc = cs * (g.lam * (float)kl_degree(z, yy, x, g) * expf(v) - 1.f);
    }
    gp[p] = s * acc;
  }
}

__global__ void __launch_bounds__(256) mse_fwd_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                      float* __restrict__ loss, size_t n, double scale, ReduceWork rw) {
  __shared__ double s_red[32];
  double acc = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float d = __ldg(a + i) - __ldg(b + i);
    acc += (double)(d * d);
  }
  double tot = block_sum<double>(acc, s_red);
  finish_reduce(tot, rw, gridDim.x, blockIdx.x, scale / (double)n, loss, s_red);
}

__global__ void __launch_bounds__(256) mse_bwd_kernel(const float* __restrict__ yt, const float* __restrict__ yp,
                                                      const float* __restrict__ gl, float* __restrict__ gp, size_t n,
                                                      double scale) {
  float s = __ldg(gl) * (float)(2.0 * scale / (double)n);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    gp[i] = s * (__ldg(yp + i) - __ldg(yt + i));
}

constexpr int DICE_CHUNKS = 64;

__global__ void __launch_bounds__(256) dice_partial_kernel(const float* __restrict__ yt, const float* __restrict__ yp,
                                                           double* __restrict__ partials, size_t V) {
  __shared__ double s_red[32];
  int bl = blockIdx.y, ch = blockIdx.x;
  size_t per = (V + DICE_CHUNKS - 1) / DICE_CHUNKS;
  size_t lo = (size_t)ch * per, hi = lo + per < V ? lo + per : V;
  const float* t = yt + (size_t)bl * V;
  const float* p = yp + (size_t)bl * V;
  double top = 0, bot = 0;
  for (size_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    float a = __ldg(t + i), b = __ldg(p + i);
    top += (double)(a * b);
    bot += (double)(a + b);
  }
  top = block_sum<double>(top, s_red);
  bot = block_sum<double>(bot, s_red);
  if (threadIdx.x == 0) {
    partials[((size_t)bl * DICE_CHUNKS + ch) * 2] = top;
    partials[((size_t)bl * DICE_CHUNKS + ch) * 2 + 1] = bot;
  }
}

__global__ void __launch_bounds__(256) dice_final_kernel(const double* __restrict__ partials, float* __restrict__ loss,
                                                         float* __restrict__ sums, int BL) {
  __shared__ double s_red[32];
  double acc = 0;
  for (int bl = threadIdx.x; bl < BL; bl += blockDim.x) {
    double top = 0, bot = 0;
    for (int c = 0; c < DICE_CHUNKS; ++c) {
      top += partials[((size_t)bl * DICE_CHUNKS + c) * 2];
      bot += partials[((size_t)bl * DICE_CHUNKS + c) * 2 + 1];
    }
    float ftop = 2.f * (float)top, fbot = (float)bot;
    if (sums) { sums[2 * bl] = ftop; sums[2 * bl + 1] = fbot; }
    acc += (double)(ftop / fmaxf(fbot, 1e-5f));
  }
  double tot = block_sum<double>(acc, s_red);
  if (threadIdx.x == 0) loss[0] = (float)(-tot / BL);
}

__global__ void __launch_bounds__(256) dice_bwd_kernel(const float* __restrict__ yt, const float* __restrict__ sums,
                                                       const float* __restrict__ gl, float* __restrict__ gp, size_t V, int BL) {
  int bl = blockIdx.y;
  float top = __ldg(sums + 2 * bl), bot = __ldg(sums + 2 * bl + 1);
  float bc = fmaxf(bot, 1e-5f);
  float s = -__ldg(gl) / (float)BL;
  float k1 = s * 2.f / bc;
  // torch.clamp(min=1e-5) passes the gradient where its input is >= the floor (ATen clamp_backward), the floor included
  float k2 = bot >= 1e-5f ? s * top / (bc * bc) : 0.f;
  const float* t = yt + (size_t)bl * V;
  float* o = gp + (size_t)bl * V;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (size_t)gridDim.x * blockDim.x)
    o[i] = k1 * __ldg(t + i) - k2;
}

static int reduce_grid(size_t n) {
  size_t b = (n + 256 * 8 - 1) / (256 * 8);
  int cap = sm_count() * 8;
  if (cap > kMaxReduceBlocks) cap = kMaxReduceBlocks;
  return (int)(b < 1 ? 1 : (b > (size_t)cap ? cap : b));
}

static int make_grad_geom(int B, int C, int D, int H, int W, int nd, float mult, GradGeom* g) {
  VXM_REQUIRE(B > 0 && C > 0 && D > 0 && H > 0 && W > 0, "gradloss: non-positive dimension");
  VXM_REQUIRE(nd == 2 || nd == 3, "gradloss: nd must be 2 or 3");
  VXM_REQUIRE(nd == 3 || D == 1, "gradloss: a 2-D problem must be passed with D == 1");
  g->B = B; g->C = C; g->D = D; g->H = H; g->W = W;
  g->HW = (size_t)H * W; g->DHW = g->HW * D;
  double base = (double)mult / ((double)nd * B);
  auto coef = [&](int s, double others) { return s > 1 ? base / ((double)C * (s - 1) * others) : 0.0; };
  g->cx = coef(W, (double)D * H);
  g->cy = coef(H, (double)D * W);
  g->cz = nd == 3 ? coef(D, (double)H * W) : 0.0;
  return VXM_OK;
}

static int make_kl_geom(int B, int D, int H, int W, int nd, float lam, KlGeom* g) {
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "kl: non-positive dimension");
  VXM_REQUIRE(nd == 2 || nd == 3, "kl: nd must be 2 or 3");
  VXM_REQUIRE(nd == 3 || D == 1, "kl: a 2-D problem must be passed with D == 1");
  VXM_REQUIRE((size_t)D * H * W < (1u << 31), "kl: at most 2^31 - 1 voxels per volume");
  VXM_REQUIRE(2 * nd * B <= kMaxReduceBlocks, "kl: at most %d (batch, channel) planes, got %d", kMaxReduceBlocks, 2 * nd * B);
  g->B = B; g->nd = nd; g->D = D; g->H = H; g->W = W; g->lam = lam;
  g->HW = (size_t)H * W; g->DHW = g->HW * D;
  double V = (double)g->DHW;
  auto coef = [&](int s) { return s > 1 ? (double)lam / (4.0 * B * nd * (s - 1) * (V / s)) : 0.0; };
  g->cx = coef(W);
  g->cy = coef(H);
  g->cz = nd == 3 ? coef(D) : 0.0;
  g->cs = 0.5 / ((double)B * V);
  return VXM_OK;
}

// blocks per plane: about 8 blocks per SM over all planes (fwd: at most kMaxReduceBlocks partials in all)
static dim3 kl_grid(const KlGeom& g) {
  int planes = 2 * g.nd * g.B;
  size_t want = (g.DHW + 256 * 8 - 1) / (256 * 8);
  int cap = sm_count() * 8 / planes;
  if (cap > kMaxReduceBlocks / planes) cap = kMaxReduceBlocks / planes;
  if (cap < 1) cap = 1;
  return dim3((unsigned)(want < 1 ? 1 : (want > (size_t)cap ? cap : want)), (unsigned)planes);
}

}  // namespace vxm

using namespace vxm;

extern "C" int vxm_gradloss_fwd(const float* y, float* loss, void* work, int B, int C, int D, int H, int W,
                                int nd, int penalty, float mult, void* stream) {
  GradGeom g;
  int rc = make_grad_geom(B, C, D, H, W, nd, mult, &g);
  if (rc) return rc;
  VXM_REQUIRE(y && loss && work, "gradloss_fwd: null pointer");
  VXM_REQUIRE(penalty == 1 || penalty == 2, "penalty can only be l1 or l2. Got: %d", penalty);  // losses.py:126
  int grid = reduce_grid((size_t)B * C * g.DHW);
  ReduceWork rw = as_reduce_work(work);
  if (penalty == 1) gradloss_fwd_kernel<1><<<grid, 256, 0, as_stream(stream)>>>(y, loss, g, rw);
  else gradloss_fwd_kernel<2><<<grid, 256, 0, as_stream(stream)>>>(y, loss, g, rw);
  return check_launch("gradloss_fwd");
}

extern "C" int vxm_gradloss_bwd(const float* y, const float* grad_loss, float* grad_y, int B, int C, int D,
                                int H, int W, int nd, int penalty, float mult, void* stream) {
  GradGeom g;
  int rc = make_grad_geom(B, C, D, H, W, nd, mult, &g);
  if (rc) return rc;
  VXM_REQUIRE(y && grad_loss && grad_y, "gradloss_bwd: null pointer");
  VXM_REQUIRE(penalty == 1 || penalty == 2, "penalty can only be l1 or l2. Got: %d", penalty);
  int grid = reduce_grid((size_t)B * C * g.DHW);
  if (penalty == 1) gradloss_bwd_kernel<1><<<grid, 256, 0, as_stream(stream)>>>(y, grad_loss, grad_y, g);
  else gradloss_bwd_kernel<2><<<grid, 256, 0, as_stream(stream)>>>(y, grad_loss, grad_y, g);
  return check_launch("gradloss_bwd");
}

extern "C" int vxm_mse_fwd(const float* y_true, const float* y_pred, float* loss, void* work, size_t n, void* stream) {
  VXM_REQUIRE(y_true && y_pred && loss && work && n > 0, "mse_fwd: bad argument");
  mse_fwd_kernel<<<reduce_grid(n), 256, 0, as_stream(stream)>>>(y_true, y_pred, loss, n, 1.0, as_reduce_work(work));
  return check_launch("mse_fwd");
}

extern "C" int vxm_mse_bwd(const float* y_true, const float* y_pred, const float* grad_loss, float* grad_pred,
                           size_t n, void* stream) {
  VXM_REQUIRE(y_true && y_pred && grad_loss && grad_pred && n > 0, "mse_bwd: bad argument");
  mse_bwd_kernel<<<reduce_grid(n), 256, 0, as_stream(stream)>>>(y_true, y_pred, grad_loss, grad_pred, n, 1.0);
  return check_launch("mse_bwd");
}

extern "C" int vxm_mse_scaled_fwd(const float* y_true, const float* y_pred, float* loss, void* work, size_t n, double scale,
                                  void* stream) {
  VXM_REQUIRE(y_true && y_pred && loss && work && n > 0, "mse_scaled_fwd: bad argument");
  mse_fwd_kernel<<<reduce_grid(n), 256, 0, as_stream(stream)>>>(y_true, y_pred, loss, n, scale, as_reduce_work(work));
  return check_launch("mse_scaled_fwd");
}

extern "C" int vxm_mse_scaled_bwd(const float* y_true, const float* y_pred, const float* grad_loss, float* grad_pred,
                                  size_t n, double scale, void* stream) {
  VXM_REQUIRE(y_true && y_pred && grad_loss && grad_pred && n > 0, "mse_scaled_bwd: bad argument");
  mse_bwd_kernel<<<reduce_grid(n), 256, 0, as_stream(stream)>>>(y_true, y_pred, grad_loss, grad_pred, n, scale);
  return check_launch("mse_scaled_bwd");
}

extern "C" int vxm_kl_fwd(const float* params, float* loss, void* work, int B, int D, int H, int W, int nd,
                          float prior_lambda, void* stream) {
  KlGeom g;
  int rc = make_kl_geom(B, D, H, W, nd, prior_lambda, &g);
  if (rc) return rc;
  VXM_REQUIRE(params && loss && work, "kl_fwd: null pointer");
  kl_fwd_kernel<<<kl_grid(g), 256, 0, as_stream(stream)>>>(params, loss, g, as_reduce_work(work));
  return check_launch("kl_fwd");
}

extern "C" int vxm_kl_bwd(const float* params, const float* grad_loss, float* grad_params, int B, int D, int H, int W,
                          int nd, float prior_lambda, void* stream) {
  KlGeom g;
  int rc = make_kl_geom(B, D, H, W, nd, prior_lambda, &g);
  if (rc) return rc;
  VXM_REQUIRE(params && grad_loss && grad_params, "kl_bwd: null pointer");
  kl_bwd_kernel<<<kl_grid(g), 256, 0, as_stream(stream)>>>(params, grad_loss, grad_params, g);
  return check_launch("kl_bwd");
}

extern "C" size_t vxm_dice_workspace_bytes(int BL) { return (size_t)BL * DICE_CHUNKS * 2 * sizeof(double); }

extern "C" int vxm_dice_fwd(const float* y_true, const float* y_pred, float* loss, float* sums, void* work, int BL,
                            size_t V, void* stream) {
  VXM_REQUIRE(y_true && y_pred && loss && work && BL > 0 && V > 0 && BL <= 65535, "dice_fwd: bad argument");
  dice_partial_kernel<<<dim3(DICE_CHUNKS, BL), 256, 0, as_stream(stream)>>>(y_true, y_pred, (double*)work, V);
  int rc = check_launch("dice_partial");
  if (rc) return rc;
  dice_final_kernel<<<1, 256, 0, as_stream(stream)>>>((const double*)work, loss, sums, BL);
  return check_launch("dice_final");
}

extern "C" int vxm_dice_bwd(const float* y_true, const float* sums, const float* grad_loss, float* grad_pred, int BL,
                            size_t V, void* stream) {
  VXM_REQUIRE(y_true && sums && grad_loss && grad_pred && BL > 0 && V > 0 && BL <= 65535, "dice_bwd: bad argument");
  int gx = (int)((V + 2047) / 2048);
  if (gx > 1024) gx = 1024;
  dice_bwd_kernel<<<dim3(gx, BL), 256, 0, as_stream(stream)>>>(y_true, sums, grad_loss, grad_pred, V, BL);
  return check_launch("dice_bwd");
}
