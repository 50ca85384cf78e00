// MutualInformation (reference voxelmorph/tf/losses.py:352-367, a subclass of neurite's soft-binned MI): the loss
// and its exact gradient, fused so that no per-voxel [V, B] bin array is ever stored.
//
// For t in {x = y_true, y = y_pred}: centres c (given, or linspace(min t, max t, B) over the whole batch),
// t~ = clip(t, min_clip, max_clip), w_vb = softmax_b(-alpha (t~_v - c_b)^2).  Per item n, with eps = 1e-7:
//   P = sum_v wx_v wy_v^T,  pxy = P / (sum P + eps),  px = sx / (sum sx + eps) with sx = sum_v wx_v (py likewise),
//   MI_n = sum_bc pxy log(pxy / (px py^T + eps) + eps),  loss = -mean_n MI_n.
//
// Launches.  Forward: [min/max, data-driven centres only] -> joint histogram (per-CTA partials of P, sx, sy and the
// tie counts at the min and max; fp32 products summed over one tile, then fp64) -> fixed-order fp64 reduction of
// the partials -> finalize (one CTA: loss and the B x B table dMI/dP plus dMI/dsx, dMI/dsy of every item).
// Backward: one per-voxel pass (recompute w, a = Gp wy + gsx, softmax backward, write gx and/or gy and per-CTA
// partials of dL/dc) -> [data-driven only] fixed-order reduction of dL/dc to dL/dlo, dL/dhi -> the tie share added to
// the voxels at the min and max (torch.amin/amax's equal split).  No host synchronisation; no float atomics.
//
// Bins are padded to BP = 16, 32, 48 or 64; padded bins carry weight 0 and stay out of every softmax sum.
#include <math.h>

#include "common.cuh"

namespace vxm {

ReduceWork as_reduce_work(void* work);  // ncc.cu

namespace mi {

constexpr int NT = 256;      // threads per CTA (every kernel)
constexpr int TF = 128;      // voxels per forward tile: one (tensor, voxel) softmax per thread
constexpr int TB = 64;       // voxels per backward tile
constexpr double EPS = 1e-7; // Keras' epsilon
constexpr int NSTAT = 16;    // doubles: lo/hi x,y | tie counts | dL/dlo, dL/dhi x,y

// stats[]: 0 xlo, 1 xhi, 2 ylo, 3 yhi, 4 x#lo, 5 x#hi, 6 y#lo, 7 y#hi, 8 dL/dxlo, 9 dL/dxhi, 10 dL/dylo, 11 dL/dyhi

struct Args {
  const float* x;
  const float* y;
  const float* centers;  // B given centres (both tensors), or null: data-driven
  int N, B;
  size_t V;
  float alpha, clip_lo, clip_hi;
};

__host__ __device__ constexpr int tpp(int bp) { return (bp / 4) * (bp / 4); }
__host__ __device__ constexpr int groups(int bp) { return tpp(bp) >= NT ? 1 : NT / tpp(bp); }
__host__ __device__ constexpr int rec_len(int bp) { return bp * bp + 2 * bp + 4; }   // P, sx, sy, ties
__host__ __device__ constexpr int tab_len(int bp) { return bp * bp + 2 * bp; }       // dMI/dP, dMI/dsx, dMI/dsy

template <int BP>
constexpr size_t fwd_smem() { return sizeof(float) * 2 * TF * (BP + 4); }
template <int BP>
constexpr size_t bwd_smem() { return sizeof(float) * (4 * BP * (TB + 4) + 2 * BP * BP); }

// centres of both tensors into sc[2][BP] (padded entries 0)
template <int BP>
__device__ __forceinline__ void load_centres(const Args& a, const double* stats, float* sc) {
  for (int i = threadIdx.x; i < 2 * BP; i += NT) {
    int side = i / BP, b = i % BP;
    float c = 0.f;
    if (b < a.B) {
      if (a.centers) {
        c = __ldg(a.centers + b);
      } else {
        double lo = stats[2 * side], hi = stats[2 * side + 1];
        c = (float)(lo + (hi - lo) * (double)b / (double)(a.B - 1));
      }
    }
    sc[i] = c;
  }
}

__device__ __forceinline__ float clip(float t, const Args& a) { return fminf(fmaxf(t, a.clip_lo), a.clip_hi); }

// ---- min / max of x and y over all N V elements (data-driven centres only) --------------------------------------
__device__ __forceinline__ void block_minmax4(float v[4], float (*s)[4]) {
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v[0] = fminf(v[0], __shfl_xor_sync(0xffffffffu, v[0], o));
    v[1] = fmaxf(v[1], __shfl_xor_sync(0xffffffffu, v[1], o));
    v[2] = fminf(v[2], __shfl_xor_sync(0xffffffffu, v[2], o));
    v[3] = fmaxf(v[3], __shfl_xor_sync(0xffffffffu, v[3], o));
  }
  __syncthreads();
  if (lane == 0)
    for (int j = 0; j < 4; ++j) s[wid][j] = v[j];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < NT / 32; ++w) {
      v[0] = fminf(v[0], s[w][0]); v[1] = fmaxf(v[1], s[w][1]);
      v[2] = fminf(v[2], s[w][2]); v[3] = fmaxf(v[3], s[w][3]);
    }
}

__global__ void __launch_bounds__(NT) minmax_kernel(const float* __restrict__ x, const float* __restrict__ y, size_t n,
                                                    ReduceWork rw, double* __restrict__ stats) {
  __shared__ float s[NT / 32][4];
  __shared__ bool is_last;
  float v[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
  for (size_t i = (size_t)blockIdx.x * NT + threadIdx.x; i < n; i += (size_t)gridDim.x * NT) {
    float a = __ldg(x + i), b = __ldg(y + i);
    v[0] = fminf(v[0], a); v[1] = fmaxf(v[1], a);
    v[2] = fminf(v[2], b); v[3] = fmaxf(v[3], b);
  }
  block_minmax4(v, s);
  if (threadIdx.x == 0) {
    for (int j = 0; j < 4; ++j) rw.partials[4 * blockIdx.x + j] = (double)v[j];
    __threadfence();
    is_last = atomicAdd(rw.counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  float u[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
  for (int i = threadIdx.x; i < (int)gridDim.x; i += NT) {
    u[0] = fminf(u[0], (float)__ldcg(&rw.partials[4 * i + 0]));
    u[1] = fmaxf(u[1], (float)__ldcg(&rw.partials[4 * i + 1]));
    u[2] = fminf(u[2], (float)__ldcg(&rw.partials[4 * i + 2]));
    u[3] = fmaxf(u[3], (float)__ldcg(&rw.partials[4 * i + 3]));
  }
  block_minmax4(u, s);
  if (threadIdx.x == 0) {
    for (int j = 0; j < 4; ++j) stats[j] = (double)u[j];
    *rw.counter = 0u;
  }
}

// ---- joint histogram: per-(item, CTA, voxel group) partials of P, sx, sy and the tie counts ------------------------
// Stage 1: thread (side, v) writes the softmax weights of one voxel, row v of sw[side] (BP + 4 floats: float4 stores
// land in distinct bank quads).  Stage 2: G groups of (BP/4)^2 threads, each thread a 4 x 4 block of P over the voxels
// v = g (mod G) of the tile, summed in fp32 over the tile and then into fp64 registers.
template <int BP>
__global__ void __launch_bounds__(NT) hist_kernel(Args a, const double* __restrict__ stats, double* __restrict__ part) {
  constexpr int LD = BP + 4, R4 = BP / 4, TPP = tpp(BP), G = groups(BP), R = rec_len(BP);
  extern __shared__ __align__(16) float sw[];   // [2][TF][LD]
  __shared__ float sc[2 * BP];
  __shared__ unsigned int s_ties[4];
  const int n = blockIdx.y, k = blockIdx.x, K = gridDim.x, tid = threadIdx.x;
  const bool data = a.centers == nullptr;
  load_centres<BP>(a, stats, sc);
  if (tid < 4) s_ties[tid] = 0u;
  // stage-1 role
  const int side = tid / TF, v1 = tid % TF;
  const float* src = (side ? a.y : a.x) + (size_t)n * a.V;
  const float lo = data ? (float)stats[2 * side] : 0.f, hi = data ? (float)stats[2 * side + 1] : 0.f;
  unsigned int tie_lo = 0, tie_hi = 0;
  // stage-2 role
  const int g = tid / TPP, p = tid % TPP, bi = p / R4, ci = p % R4;
  const bool acc_role = g < G;
  double dP[4][4] = {}, dsx[4] = {}, dsy[4] = {};
  __syncthreads();
  const float* cs = sc + side * BP;
  const size_t ntile = (a.V + TF - 1) / TF;
  for (size_t tile = k; tile < ntile; tile += K) {
    {
      const size_t idx = tile * TF + v1;
      float* row = sw + (size_t)(side * TF + v1) * LD;
      if (idx < a.V) {
        const float t = __ldg(src + idx);
        tie_lo += data && t == lo;
        tie_hi += data && t == hi;
        const float tc = clip(t, a);
        float m = -INFINITY;
        for (int b = 0; b < a.B; ++b) {
          float d = tc - cs[b];
          m = fmaxf(m, -a.alpha * d * d);
        }
        float sum = 0.f;
#pragma unroll 4
        for (int b = 0; b < BP; b += 4) {
          float e[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float d = tc - cs[b + j];
            e[j] = b + j < a.B ? __expf(-a.alpha * d * d - m) : 0.f;
            sum += e[j];
          }
          *reinterpret_cast<float4*>(row + b) = make_float4(e[0], e[1], e[2], e[3]);
        }
        const float inv = 1.f / sum;
#pragma unroll 4
        for (int b = 0; b < BP; b += 4) {
          float4 q = *reinterpret_cast<float4*>(row + b);
          q.x *= inv; q.y *= inv; q.z *= inv; q.w *= inv;
          *reinterpret_cast<float4*>(row + b) = q;
        }
      } else {
#pragma unroll 4
        for (int b = 0; b < BP; b += 4) *reinterpret_cast<float4*>(row + b) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    __syncthreads();
    if (acc_role) {
      float f[4][4] = {}, fx[4] = {}, fy[4] = {};
      for (int v = g; v < TF; v += G) {
        const float4 wx4 = *reinterpret_cast<const float4*>(sw + (size_t)v * LD + bi * 4);
        const float4 wy4 = *reinterpret_cast<const float4*>(sw + (size_t)(TF + v) * LD + ci * 4);
        const float wx[4] = {wx4.x, wx4.y, wx4.z, wx4.w}, wy[4] = {wy4.x, wy4.y, wy4.z, wy4.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) f[i][j] = fmaf(wx[i], wy[j], f[i][j]);
        if (ci == 0)
#pragma unroll
          for (int i = 0; i < 4; ++i) fx[i] += wx[i];
        if (bi == 0)
#pragma unroll
          for (int j = 0; j < 4; ++j) fy[j] += wy[j];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) dP[i][j] += (double)f[i][j];
        dsx[i] += (double)fx[i];
        dsy[i] += (double)fy[i];
      }
    }
    __syncthreads();
  }
  if (data) {   // integer shared atomics: order-free and exact
    if (tie_lo) atomicAdd(&s_ties[2 * side], tie_lo);
    if (tie_hi) atomicAdd(&s_ties[2 * side + 1], tie_hi);
  }
  __syncthreads();
  if (!acc_role) return;
  double* rec = part + ((size_t)(n * K + k) * G + g) * R;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) rec[(bi * 4 + i) * BP + ci * 4 + j] = dP[i][j];
  if (ci == 0)
    for (int i = 0; i < 4; ++i) rec[BP * BP + bi * 4 + i] = dsx[i];
  if (bi == 0)
    for (int j = 0; j < 4; ++j) rec[BP * BP + BP + ci * 4 + j] = dsy[j];
  if (p == 0)
    for (int j = 0; j < 4; ++j) rec[BP * BP + 2 * BP + j] = g == 0 ? (double)s_ties[j] : 0.0;
}

// red[n][e] = sum over the item's records in record order (fp64)
__global__ void __launch_bounds__(NT) reduce_kernel(const double* __restrict__ part, double* __restrict__ red, int nrec,
                                                    int R) {
  const int n = blockIdx.y, e = blockIdx.x * NT + threadIdx.x;
  if (e >= R) return;
  const double* p = part + (size_t)n * nrec * R + e;
  double s = 0.0;
  for (int r = 0; r < nrec; ++r) s += p[(size_t)r * R];
  red[(size_t)n * R + e] = s;
}

__device__ __forceinline__ double bcast_sum(double v, double* s_red, double* s_b) {
  v = block_sum<double>(v, s_red);
  if (threadIdx.x == 0) *s_b = v;
  __syncthreads();
  v = *s_b;
  __syncthreads();
  return v;
}

// One CTA: for every item, MI_n and the tables dMI/dP (B x B), dMI/dsx, dMI/dsy (fp64 math, fp32 tables; padded
// entries 0).  loss = -mean_n MI_n; the tie counts of the whole batch go to stats[4..7].
template <int BP>
__global__ void __launch_bounds__(NT) finalize_kernel(const double* __restrict__ red, float* __restrict__ tab,
                                                      double* __restrict__ stats, float* __restrict__ loss, int N, int B) {
  constexpr int R = rec_len(BP), TL = tab_len(BP);
  __shared__ double sP[BP * BP];
  __shared__ double ssx[BP], ssy[BP], spx[BP], spy[BP], sgx[BP], sgy[BP];
  __shared__ double s_red[32], s_b;
  const int tid = threadIdx.x;
  double mi_tot = 0.0, ties = 0.0;
  for (int n = 0; n < N; ++n) {
    const double* r = red + (size_t)n * R;
    for (int e = tid; e < BP * BP; e += NT) sP[e] = r[e];
    for (int b = tid; b < BP; b += NT) { ssx[b] = r[BP * BP + b]; ssy[b] = r[BP * BP + BP + b]; }
    if (tid < 4) ties += r[BP * BP + 2 * BP + tid];
    __syncthreads();
    double acc = 0.0;
    for (int e = tid; e < BP * BP; e += NT) acc += sP[e];
    const double S1 = bcast_sum(acc, s_red, &s_b) + EPS, iS = __drcp_rn(S1);
    const double SX1 = bcast_sum(tid < B ? ssx[tid] : 0.0, s_red, &s_b) + EPS, iX = __drcp_rn(SX1);
    const double SY1 = bcast_sum(tid < B ? ssy[tid] : 0.0, s_red, &s_b) + EPS, iY = __drcp_rn(SY1);
    if (tid < B) { spx[tid] = ssx[tid] * iX; spy[tid] = ssy[tid] * iY; }
    __syncthreads();
    // per entry: pxy, den = px py + eps, r = pxy / den, lg = log(r + eps);  MI term pxy lg,
    // dMI/dpxy = lg + pxy / ((r + eps) den) = A,  dMI/d(px py) = -pxy^2 / ((r + eps) den^2) = Q
    double mi = 0.0, ap = 0.0;
    for (int e = tid; e < BP * BP; e += NT) {
      const int b = e / BP, c = e % BP;
      if (b >= B || c >= B) continue;
      const double pxy = sP[e] * iS, den = spx[b] * spy[c] + EPS, rr = pxy * __drcp_rn(den), lg = log(rr + EPS);
      mi += pxy * lg;
      ap += (lg + pxy * __drcp_rn((rr + EPS) * den)) * sP[e];
    }
    mi = bcast_sum(mi, s_red, &s_b);
    const double AP = bcast_sum(ap, s_red, &s_b);
    // dMI/dpx_b = sum_c Q_bc py_c (threads [0, B)), dMI/dpy_c = sum_b Q_bc px_b (threads [BP, BP + B))
    if (tid < B || (tid >= BP && tid < BP + B)) {
      const bool row = tid < BP;
      const int i = row ? tid : tid - BP;
      double s = 0.0;
      for (int j = 0; j < B; ++j) {
        const int b = row ? i : j, c = row ? j : i;
        const double pxy = sP[b * BP + c] * iS, den = spx[b] * spy[c] + EPS, rr = pxy * __drcp_rn(den);
        s += -pxy * pxy * __drcp_rn((rr + EPS) * den * den) * (row ? spy[c] : spx[b]);
      }
      if (row) sgx[i] = s;
      else sgy[i] = s;
    }
    __syncthreads();
    const double GX = bcast_sum(tid < B ? sgx[tid] * ssx[tid] : 0.0, s_red, &s_b);
    const double GY = bcast_sum(tid < B ? sgy[tid] * ssy[tid] : 0.0, s_red, &s_b);
    float* t = tab + (size_t)n * TL;
    for (int e = tid; e < BP * BP; e += NT) {
      const int b = e / BP, c = e % BP;
      double gp = 0.0;
      if (b < B && c < B) {
        const double pxy = sP[e] * iS, den = spx[b] * spy[c] + EPS, rr = pxy * __drcp_rn(den), lg = log(rr + EPS);
        gp = (lg + pxy * __drcp_rn((rr + EPS) * den)) * iS - AP * iS * iS;
      }
      t[e] = (float)gp;
    }
    for (int b = tid; b < BP; b += NT) {
      t[BP * BP + b] = b < B ? (float)(sgx[b] * iX - GX * iX * iX) : 0.f;
      t[BP * BP + BP + b] = b < B ? (float)(sgy[b] * iY - GY * iY * iY) : 0.f;
    }
    mi_tot += mi;
    __syncthreads();
  }
  if (tid < 4) stats[4 + tid] = ties;
  if (tid == 0) loss[0] = (float)(-mi_tot / N);
}

// ---- backward: one pass over the voxels -------------------------------------------------------------------------
// Per tile: (1) thread (side, v) writes w of one voxel, column v of sw[side][BP][TB + 4]; (2) each thread a 4 bins x
// 4 voxels block of a_x = Gp wy + gsx and/or a_y = Gp^T wx + gsy into sa; (3) thread (side, v): d_b = w_b (a_b -
// sum_k w_k a_k), e_b = s d_b 2 alpha (t~ - c_b) back into sa, g_v = -mask sum_b e_b; (4) thread (side, b) adds row b
// of e (dL/dc_b of the tile, in voxel order) to its fp64 partial.
template <int BP>
__global__ void __launch_bounds__(NT) bwd_kernel(Args a, const double* __restrict__ stats, const float* __restrict__ tab,
                                                 const float* __restrict__ gl, float* __restrict__ gx,
                                                 float* __restrict__ gy, int which, double* __restrict__ dcpart) {
  constexpr int LD = TB + 4, TL = tab_len(BP), NQ = (TB / 4) * (BP / 4);
  extern __shared__ __align__(16) float sm[];
  float* sw = sm;                          // [2][BP][LD]
  float* sa = sw + 2 * BP * LD;            // [2][BP][LD]
  float* sG = sa + 2 * BP * LD;            // [BP][BP]: Gp[b][c]
  float* sGT = sG + BP * BP;               // [BP][BP]: Gp[c][b]
  __shared__ float sc[2 * BP], sgs[2 * BP], st[2][TB];
  __shared__ bool smk[2][TB];
  const int n = blockIdx.y, k = blockIdx.x, K = gridDim.x, tid = threadIdx.x;
  const bool data = a.centers == nullptr;
  load_centres<BP>(a, stats, sc);
  const float* tn = tab + (size_t)n * TL;
  for (int e = tid; e < BP * BP; e += NT) {
    const float v = __ldg(tn + e);
    sG[e] = v;
    sGT[(e % BP) * BP + e / BP] = v;
  }
  for (int i = tid; i < 2 * BP; i += NT) sgs[i] = __ldg(tn + BP * BP + i);
  const float s = __ldg(gl) * (float)(-1.0 / a.N);
  const float two_alpha = 2.f * a.alpha;
  double dacc = 0.0;
  // sides to run: 0 = x (bit 0), 1 = y (bit 1)
  const int nsides = (which & 1) + ((which >> 1) & 1), side0 = (which & 1) ? 0 : 1;
  __syncthreads();
  const size_t ntile = (a.V + TB - 1) / TB;
  for (size_t tile = k; tile < ntile; tile += K) {
    if (tid < 2 * TB) {   // (1)
      const int side = tid / TB, v = tid % TB;
      const size_t idx = tile * TB + v;
      const float* cs = sc + side * BP;
      float* col = sw + side * BP * LD + v;
      if (idx < a.V) {
        const float t = __ldg((side ? a.y : a.x) + (size_t)n * a.V + idx), tc = clip(t, a);
        st[side][v] = tc;
        smk[side][v] = t >= a.clip_lo && t <= a.clip_hi;
        float m = -INFINITY;
        for (int b = 0; b < a.B; ++b) {
          float d = tc - cs[b];
          m = fmaxf(m, -a.alpha * d * d);
        }
        float sum = 0.f;
        for (int b = 0; b < a.B; ++b) {
          float d = tc - cs[b];
          float e = __expf(-a.alpha * d * d - m);
          col[b * LD] = e;
          sum += e;
        }
        const float inv = 1.f / sum;
        for (int b = 0; b < a.B; ++b) col[b * LD] *= inv;
      } else {
        st[side][v] = 0.f;
        smk[side][v] = false;
        for (int b = 0; b < a.B; ++b) col[b * LD] = 0.f;
      }
      for (int b = a.B; b < BP; ++b) col[b * LD] = 0.f;
    }
    __syncthreads();
    for (int q = tid; q < nsides * NQ; q += NT) {   // (2)
      const int side = q < NQ ? side0 : 1, r = q % NQ, v0 = (r % (TB / 4)) * 4, b0 = (r / (TB / 4)) * 4;
      const float* gm = side ? sG : sGT;                    // row k: Gp[k][.] (y side) or Gp[.][k] (x side)
      const float* wo = sw + (1 - side) * BP * LD;          // the other tensor's weights
      float f[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float g0 = sgs[side * BP + b0 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) f[i][j] = g0;
      }
#pragma unroll 4
      for (int kk = 0; kk < BP; ++kk) {
        const float4 g4 = *reinterpret_cast<const float4*>(gm + kk * BP + b0);
        const float4 w4 = *reinterpret_cast<const float4*>(wo + kk * LD + v0);
        const float gg[4] = {g4.x, g4.y, g4.z, g4.w}, ww[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) f[i][j] = fmaf(gg[i], ww[j], f[i][j]);
      }
      float* dst = sa + side * BP * LD + b0 * LD + v0;
#pragma unroll
      for (int i = 0; i < 4; ++i) *reinterpret_cast<float4*>(dst + i * LD) = make_float4(f[i][0], f[i][1], f[i][2], f[i][3]);
    }
    __syncthreads();
    if (tid < 2 * TB && ((which >> (tid / TB)) & 1)) {   // (3)
      const int side = tid / TB, v = tid % TB;
      const size_t idx = tile * TB + v;
      const float* w = sw + side * BP * LD + v;
      float* ae = sa + side * BP * LD + v;
      const float* cs = sc + side * BP;
      const float tc = st[side][v];
      float dot = 0.f;
      for (int b = 0; b < a.B; ++b) dot = fmaf(w[b * LD], ae[b * LD], dot);
      float gsum = 0.f;
      for (int b = 0; b < a.B; ++b) {
        const float d = w[b * LD] * (ae[b * LD] - dot);
        const float e = s * d * two_alpha * (tc - cs[b]);
        ae[b * LD] = e;
        gsum -= e;
      }
      if (idx < a.V) (side ? gy : gx)[(size_t)n * a.V + idx] = smk[side][v] ? gsum : 0.f;
    }
    if (data) {
      __syncthreads();
      if (tid < 2 * BP) {   // (4)
        const int side = tid / BP, b = tid % BP;
        if (((which >> side) & 1) && b < a.B) {
          const float* row = sa + side * BP * LD + b * LD;
          float f = 0.f;
          for (int v = 0; v < TB; ++v) f += row[v];
          dacc += (double)f;
        }
      }
    }
    __syncthreads();
  }
  if (data && tid < 2 * BP) {
    const int side = tid / BP, b = tid % BP;
    if ((which >> side) & 1) dcpart[((size_t)(side * a.N + n) * K + k) * BP + b] = dacc;
  }
}

// dL/dc_b of each side summed over (item, CTA) in order, then dL/dlo = sum_b dL/dc_b (1 - b/(B-1)) and dL/dhi =
// sum_b dL/dc_b b/(B-1) into stats[8..11]
__global__ void __launch_bounds__(NT) dc_kernel(const double* __restrict__ dcpart, double* __restrict__ stats, int N,
                                                int K, int B, int BP, int which) {
  __shared__ double s_red[32], s_b;
  const int tid = threadIdx.x;
  for (int side = 0; side < 2; ++side) {
    if (!((which >> side) & 1)) continue;
    double lo = 0.0, hi = 0.0;
    if (tid < B) {
      double dc = 0.0;
      for (int r = 0; r < N * K; ++r) dc += dcpart[((size_t)side * N * K + r) * BP + tid];
      const double f = (double)tid / (double)(B - 1);
      lo = dc * (1.0 - f);
      hi = dc * f;
    }
    lo = bcast_sum(lo, s_red, &s_b);
    hi = bcast_sum(hi, s_red, &s_b);
    if (tid == 0) { stats[8 + 2 * side] = lo; stats[9 + 2 * side] = hi; }
  }
}

// the tie share: every voxel equal to the min gets dL/dlo / #min, every voxel equal to the max dL/dhi / #max
__global__ void __launch_bounds__(NT) ties_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                  float* __restrict__ gx, float* __restrict__ gy,
                                                  const double* __restrict__ stats, size_t n) {
  const int side = blockIdx.y;
  const float* t = side ? y : x;
  float* g = side ? gy : gx;
  if (g == nullptr) return;
  const float lo = (float)stats[2 * side], hi = (float)stats[2 * side + 1];
  const double slo = stats[8 + 2 * side] / stats[4 + 2 * side], shi = stats[9 + 2 * side] / stats[5 + 2 * side];
  for (size_t i = (size_t)blockIdx.x * NT + threadIdx.x; i < n; i += (size_t)gridDim.x * NT) {
    const float v = __ldg(t + i);
    if (v == lo || v == hi) g[i] += (float)((v == lo ? slo : 0.0) + (v == hi ? shi : 0.0));
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------
static int pad_bins(int B) { return (B + 15) / 16 * 16; }

struct Layout {
  int BP, G, R, Kf, Kb;
  size_t stats, tab, part, red, dc, total;   // byte offsets
};

static size_t align256(size_t b) { return (b + 255) / 256 * 256; }

static int ctas_per_item(int N, size_t V, int tile) {
  size_t want = ((size_t)2 * sm_count() + N - 1) / N, tiles = (V + tile - 1) / tile;
  if (want > tiles) want = tiles;
  return (int)(want < 1 ? 1 : want);
}

static Layout layout(int N, size_t V, int B) {
  Layout L;
  L.BP = pad_bins(B);
  L.G = groups(L.BP);
  L.R = rec_len(L.BP);
  L.Kf = ctas_per_item(N, V, TF);
  L.Kb = ctas_per_item(N, V, TB);
  size_t off = 0;
  L.stats = off; off += align256(sizeof(double) * NSTAT);
  L.tab = off;   off += align256(sizeof(float) * N * tab_len(L.BP));
  L.part = off;  off += align256(sizeof(double) * N * L.Kf * L.G * L.R);
  L.red = off;   off += align256(sizeof(double) * N * L.R);
  L.dc = off;    off += align256(sizeof(double) * 2 * N * L.Kb * L.BP);
  L.total = off;
  return L;
}

static int check_args(const Args& a, const char* what) {
  VXM_REQUIRE(a.x && a.y, "%s: null input", what);
  VXM_REQUIRE(a.N > 0 && a.N <= 65535 && a.V > 0, "%s: bad shape (N = %d, V = %zu)", what, a.N, a.V);
  VXM_REQUIRE(a.B >= 2 && a.B <= 64, "%s: nb_bins must be in [2, 64], got %d", what, a.B);
  VXM_REQUIRE(isfinite(a.alpha) && a.alpha > 0.f, "%s: soft_bin_alpha must be finite and positive", what);
  return VXM_OK;
}

template <int BP>
static int fwd_impl(const Args& a, const Layout& L, char* ws, float* loss, cudaStream_t st) {
  double* stats = (double*)(ws + L.stats);
  VXM_CUDA(cudaFuncSetAttribute(hist_kernel<BP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<BP>()));
  hist_kernel<BP><<<dim3(L.Kf, a.N), NT, fwd_smem<BP>(), st>>>(a, stats, (double*)(ws + L.part));
  int rc = check_launch("mi_hist");
  if (rc) return rc;
  reduce_kernel<<<dim3((L.R + NT - 1) / NT, a.N), NT, 0, st>>>((const double*)(ws + L.part), (double*)(ws + L.red),
                                                                L.Kf * L.G, L.R);
  rc = check_launch("mi_reduce");
  if (rc) return rc;
  finalize_kernel<BP><<<1, NT, 0, st>>>((const double*)(ws + L.red), (float*)(ws + L.tab), stats, loss, a.N, a.B);
  return check_launch("mi_finalize");
}

template <int BP>
static int bwd_impl(const Args& a, const Layout& L, char* ws, const float* gl, float* gx, float* gy, int which,
                    cudaStream_t st) {
  double* stats = (double*)(ws + L.stats);
  VXM_CUDA(cudaFuncSetAttribute(bwd_kernel<BP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<BP>()));
  bwd_kernel<BP><<<dim3(L.Kb, a.N), NT, bwd_smem<BP>(), st>>>(a, stats, (const float*)(ws + L.tab), gl, gx, gy, which,
                                                              (double*)(ws + L.dc));
  return check_launch("mi_bwd");
}

}  // namespace mi
}  // namespace vxm

using namespace vxm;
using namespace vxm::mi;

extern "C" size_t vxm_mi_workspace_bytes(int N, size_t V, int nbins) {
  if (N <= 0 || V == 0 || nbins < 2 || nbins > 64) return 0;
  return layout(N, V, nbins).total;
}

extern "C" int vxm_mi_fwd(const float* y_true, const float* y_pred, const float* centers, float* loss, void* work,
                          void* reduce_work, int N, size_t V, int nbins, float alpha, float min_clip, float max_clip,
                          void* stream) {
  Args a{y_true, y_pred, centers, N, nbins, V, alpha, min_clip, max_clip};
  int rc = check_args(a, "mi_fwd");
  if (rc) return rc;
  VXM_REQUIRE(loss && work, "mi_fwd: null pointer");
  VXM_REQUIRE(centers || reduce_work, "mi_fwd: data-driven centres need the reduce workspace");
  const Layout L = layout(N, V, nbins);
  cudaStream_t st = as_stream(stream);
  char* ws = (char*)work;
  if (!centers) {
    const size_t n = (size_t)N * V;
    size_t grid = (n + NT * 8 - 1) / (NT * 8);
    size_t cap = (size_t)sm_count() * 4;
    if (cap > (size_t)kMaxReduceBlocks / 4) cap = kMaxReduceBlocks / 4;
    if (grid > cap) grid = cap;
    minmax_kernel<<<(unsigned)(grid < 1 ? 1 : grid), NT, 0, st>>>(y_true, y_pred, n, as_reduce_work(reduce_work),
                                                                  (double*)(ws + L.stats));
    rc = check_launch("mi_minmax");
    if (rc) return rc;
  }
  switch (L.BP) {
    case 16: return fwd_impl<16>(a, L, ws, loss, st);
    case 32: return fwd_impl<32>(a, L, ws, loss, st);
    case 48: return fwd_impl<48>(a, L, ws, loss, st);
    default: return fwd_impl<64>(a, L, ws, loss, st);
  }
}

extern "C" int vxm_mi_bwd(const float* y_true, const float* y_pred, const float* centers, const float* grad_loss,
                          float* grad_true, float* grad_pred, void* work, int N, size_t V, int nbins, float alpha,
                          float min_clip, float max_clip, void* stream) {
  Args a{y_true, y_pred, centers, N, nbins, V, alpha, min_clip, max_clip};
  int rc = check_args(a, "mi_bwd");
  if (rc) return rc;
  VXM_REQUIRE(grad_loss && work, "mi_bwd: null pointer");
  const int which = (grad_true ? 1 : 0) | (grad_pred ? 2 : 0);
  if (!which) return VXM_OK;
  const Layout L = layout(N, V, nbins);
  cudaStream_t st = as_stream(stream);
  char* ws = (char*)work;
  switch (L.BP) {
    case 16: rc = bwd_impl<16>(a, L, ws, grad_loss, grad_true, grad_pred, which, st); break;
    case 32: rc = bwd_impl<32>(a, L, ws, grad_loss, grad_true, grad_pred, which, st); break;
    case 48: rc = bwd_impl<48>(a, L, ws, grad_loss, grad_true, grad_pred, which, st); break;
    default: rc = bwd_impl<64>(a, L, ws, grad_loss, grad_true, grad_pred, which, st); break;
  }
  if (rc || centers) return rc;
  double* stats = (double*)(ws + L.stats);
  dc_kernel<<<1, NT, 0, st>>>((const double*)(ws + L.dc), stats, N, L.Kb, nbins, L.BP, which);
  rc = check_launch("mi_dc");
  if (rc) return rc;
  const size_t n = (size_t)N * V;
  size_t grid = (n + NT * 8 - 1) / (NT * 8);
  if (grid > (size_t)sm_count() * 8) grid = (size_t)sm_count() * 8;
  ties_kernel<<<dim3((unsigned)(grid < 1 ? 1 : grid), 2), NT, 0, st>>>(y_true, y_pred, grad_true, grad_pred, stats, n);
  return check_launch("mi_ties");
}
