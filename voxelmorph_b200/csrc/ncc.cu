// Local normalised cross-correlation loss (reference voxelmorph/torch/losses.py:15-67).
//
// The reference forms five zero-padded box sums with five dense F.conv3d calls against a
// ones(1,1,9,9,9) filter (50 GFLOP of multiply-by-one at 160x192x224) plus ~15 elementwise
// kernels.  Here one kernel does everything: each CTA owns a (16 x 32) column of the volume and
// marches along D; per input slice it stages I and J (with halo) in shared memory, forms the
// products, runs the W pass and the H pass through shared memory, keeps the last `wd` slice sums
// in a register ring for the D pass, evaluates cc exactly as losses.py:57-65 does and reduces.
// Box sums are direct sums (no running prefix), zero padded, divisor prod(win) everywhere.
//
// Backward (closed form, see oracle/spec_np.ncc_grad_pred): with den = Ivar*Jvar + 1e-5,
//   A = 2 cross/den,  Bq = -cross^2 Ivar/den^2,  T = A u_I + 2 Bq u_J
//   dL/dJ = -(1/N) [ I S(A) + 2 J S(Bq) - S(T) ]
// The forward stores A, Bq, T (3 fields); the backward box-sums them with the same machinery.
//
// By the symmetry of cc in (I, J) the gradient w.r.t. I is the same expression with the roles swapped:
//   Bp = -cross^2 Jvar/den^2,  Tp = A u_J + 2 Bp u_I
//   dL/dI = -(1/N) [ J S(A) + 2 I S(Bp) - S(Tp) ]
// The two-sided entry points (vxm_ncc_fwd2 / vxm_ncc_bwd2) store A, Bq, T, Bp, Tp and box-sum the five fields in one
// launch (S(A) is shared); with y_true alone they store A, Bp, Tp and run the three-field backward with I and J swapped.
//
// Algorithmic bytes (fp32): forward 8 B/voxel (read I, J); backward 12 B/voxel (I, J, dJ)
// (+ 12 B/voxel written and read again for the three saved fields in training).  Two-sided: backward 16 B/voxel
// (I, J, dI, dJ) + 20 B/voxel of saved fields.
//
// Kernel MODE: 0 forward (saves A, Bq, T), 1 backward over three fields, 2 forward saving for y_true (`which`),
// 3 backward over five fields -> dJ and dI.
#include "common.cuh"

namespace vxm {

constexpr int NTH = 16, NTW = 32, NHALO = 4;        // tile and max halo (window <= 9)
constexpr int NIH = NTH + 2 * NHALO, NIW = NTW + 2 * NHALO;
// Depth chunk per CTA.  Every chunk re-reads wd - 1 halo slices, and the grid should fill the 2-CTA-per-SM slots in
// whole waves: pick the chunk count that minimises waves x (slices per chunk + halo).  VXM_B200_NCC_ZCHUNK overrides.
static int ncc_zchunk(int D, long long tiles, int wd) {
  const char* e = getenv("VXM_B200_NCC_ZCHUNK");
  if (e && atoi(e) >= 4) return atoi(e);
  const long long slots = 2LL * sm_count();
  int best = D;
  double best_cost = 1e300;
  for (int nch = 1; nch <= D; ++nch) {
    const int zc = (D + nch - 1) / nch;
    if (zc < 8 && nch > 1) break;
    const long long ctas = tiles * ((D + zc - 1) / zc);
    if (ctas > kMaxReduceBlocks) break;      // the deterministic reduction holds one partial per CTA
    const double cost = (double)((ctas + slots - 1) / slots) * (zc + wd - 1);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = zc; }
  }
  return best;
}

struct NccArgs {
  const float* I;
  const float* J;
  const float* saved_in;   // bwd: A, Bq, T
  float* saved_out;        // fwd: A, Bq, T (may be null)
  float* out;              // fwd: loss scalar ; bwd: grad_J
  const float* grad_loss;  // bwd
  ReduceWork rw;
  int B, D, H, W, wd, wh, ww, zchunk;
  float nwin;              // prod(win)
  double scale;            // -1 / (B*D*H*W)
  float* out2;             // bwd over five fields: grad_I (`out` is grad_J)
  int which;               // MODE 2: 1 = save A, Bp, Tp (y_true alone), 3 = save A, Bq, T, Bp, Tp
};

constexpr bool ncc_is_fwd(int mode) { return mode == 0 || mode == 2; }
constexpr int ncc_fields(int mode) { return mode == 1 ? 3 : 5; }     // box-summed fields of a kernel mode

// The saved fields of one voxel (MODE 2; MODE 0 stores A, Bq, T in place).
__device__ __forceinline__ void ncc_save2(float* so, size_t DHW, int which, float A, float Bq, float T, float Bp, float Tp) {
  so[0] = A;
  if (which == 3) { so[DHW] = Bq; so[2 * DHW] = T; so[3 * DHW] = Bp; so[4 * DHW] = Tp; }
  else { so[DHW] = Bp; so[2 * DHW] = Tp; }
}

template <int MODE, int WD>
__global__ void __launch_bounds__(256, 2) ncc_kernel(NccArgs a) {   // 2 CTAs per SM: the per-slice barriers of one overlap the loads of the other
  constexpr bool FWD = ncc_is_fwd(MODE);
  constexpr int NS = ncc_fields(MODE);
  constexpr int NF = FWD ? 2 : NS;
  __shared__ __align__(16) float s_in[NF][NIH][NIW];
  __shared__ __align__(16) float s_w[NS][NIH + 2][NTW];
  __shared__ double s_red[32];

  const int tid = threadIdx.x;
  const int tx = tid & 31, ty = tid >> 5;  // ty in 0..7 -> rows ty and ty+8
  const int w0 = blockIdx.x * NTW, h0 = blockIdx.y * NTH;
  const int nchunks = (a.D + a.zchunk - 1) / a.zchunk;
  const int chunk = blockIdx.z % nchunks, b = blockIdx.z / nchunks;
  const int z0 = chunk * a.zchunk, z1 = min(z0 + a.zchunk, a.D);
  const int pd = WD / 2, ph = a.wh / 2, pw = a.ww / 2;
  const size_t HW = (size_t)a.H * a.W, DHW = HW * a.D;
  const float* f0 = (FWD ? a.I : a.saved_in) + (size_t)b * (FWD ? 1 : NS) * DHW;
  const float* f1 = FWD ? a.J + (size_t)b * DHW : f0 + DHW;      // backward: field f at f0 + f * DHW

  float ring[2][WD][NS];
#pragma unroll
  for (int o = 0; o < 2; ++o)
#pragma unroll
    for (int j = 0; j < WD; ++j)
#pragma unroll
      for (int s = 0; s < NS; ++s) ring[o][j][s] = 0.f;

  double local = 0.0;
  const int rows_in = NTH + 2 * ph, cols_in = NTW + 2 * pw;

  for (int base = z0 - pd; base < z1 + pd; base += WD) {
#pragma unroll
    for (int j = 0; j < WD; ++j) {
      const int zi = base + j;
      if (zi < z1 + pd) {  // block-uniform
        const bool inside = zi >= 0 && zi < a.D;
        if (inside) {
          // ---- stage the slice (zero padded) ----
          for (int idx = tid; idx < rows_in * cols_in; idx += 256) {
            int r = idx / cols_in, c = idx - r * cols_in;
            int h = h0 - ph + r, w = w0 - pw + c;
            bool ok = h >= 0 && h < a.H && w >= 0 && w < a.W;
            size_t off = (size_t)zi * HW + (size_t)h * a.W + w;
            s_in[0][r][c] = ok ? __ldg(f0 + off) : 0.f;
            s_in[1][r][c] = ok ? __ldg(f1 + off) : 0.f;
#pragma unroll
            for (int f = 2; f < NF; ++f) s_in[f][r][c] = ok ? __ldg(f0 + f * DHW + off) : 0.f;
          }
          __syncthreads();
          // ---- W pass: each thread forms 4 adjacent window sums of one row from 12 staged values (register blocked) ----
          if (tid < rows_in * (NTW / 4)) {
            const int r = tid >> 3, c4 = (tid & 7) * 4;
            float x[NF][12];
#pragma unroll
            for (int f = 0; f < NF; ++f)
#pragma unroll
              for (int q = 0; q < 3; ++q) {
                const float4 a4 = *reinterpret_cast<const float4*>(&s_in[f][r][c4 + 4 * q]);
                x[f][4 * q] = a4.x; x[f][4 * q + 1] = a4.y; x[f][4 * q + 2] = a4.z; x[f][4 * q + 3] = a4.w;
              }
            float acc[NS][4];
#pragma unroll
            for (int s = 0; s < NS; ++s)
#pragma unroll
              for (int o = 0; o < 4; ++o) acc[s][o] = 0.f;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
              if (k < a.ww) {
#pragma unroll
                for (int o = 0; o < 4; ++o) {
                  if (FWD) {
                    const float u = x[0][o + k], v = x[1][o + k];
                    acc[0][o] += u; acc[1][o] += v; acc[2][o] += u * u; acc[3][o] += v * v; acc[4][o] += u * v;
                  } else {
#pragma unroll
                    for (int s = 0; s < NS; ++s) acc[s][o] += x[s][o + k];
                  }
                }
              }
            }
#pragma unroll
            for (int s = 0; s < NS; ++s)
              *reinterpret_cast<float4*>(&s_w[s][r][c4]) = make_float4(acc[s][0], acc[s][1], acc[s][2], acc[s][3]);
          }
          __syncthreads();
          // ---- H pass -> ring slot j: two ADJACENT rows per thread share their 10 loads ----
#pragma unroll
          for (int s = 0; s < NS; ++s) {
            float col[10];
#pragma unroll
            for (int k = 0; k < 10; ++k) col[k] = s_w[s][2 * ty + k][tx];
            float a0 = 0.f, a1 = 0.f;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
              if (k < a.wh) { a0 += col[k]; a1 += col[k + 1]; }
            }
            ring[0][j][s] = a0;
            ring[1][j][s] = a1;
          }
        } else {
#pragma unroll
          for (int o = 0; o < 2; ++o)
#pragma unroll
            for (int s = 0; s < NS; ++s) ring[o][j][s] = 0.f;
        }
        // ---- D pass + pointwise for output slice zo ----
        const int zo = zi - pd;
        if (zo >= z0) {
#pragma unroll
          for (int o = 0; o < 2; ++o) {
            int h = h0 + 2 * ty + o, w = w0 + tx;
            if (h < a.H && w < a.W) {
              float S[NS];
#pragma unroll
              for (int s = 0; s < NS; ++s) {
                float acc = 0.f;
#pragma unroll
                for (int q = 0; q < WD; ++q) acc += ring[o][q][s];
                S[s] = acc;
              }
              size_t off = (size_t)zo * HW + (size_t)h * a.W + w;
              if (FWD) {
                // losses.py:57-65, evaluated left to right with one rounding per op
                float Is = S[0], Js = S[1], I2s = S[2], J2s = S[3], IJs = S[4];
                float uI = __fdiv_rn(Is, a.nwin), uJ = __fdiv_rn(Js, a.nwin);
                float cross = __fadd_rn(__fsub_rn(__fsub_rn(IJs, __fmul_rn(uJ, Is)), __fmul_rn(uI, Js)),
                                        __fmul_rn(__fmul_rn(uI, uJ), a.nwin));
                float Ivar = __fadd_rn(__fsub_rn(I2s, __fmul_rn(__fmul_rn(2.f, uI), Is)),
                                       __fmul_rn(__fmul_rn(uI, uI), a.nwin));
                float Jvar = __fadd_rn(__fsub_rn(J2s, __fmul_rn(__fmul_rn(2.f, uJ), Js)),
                                       __fmul_rn(__fmul_rn(uJ, uJ), a.nwin));
                float den = __fadd_rn(__fmul_rn(Ivar, Jvar), 1e-5f);
                float cc = __fdiv_rn(__fmul_rn(cross, cross), den);
                local += (double)cc;
                if (a.saved_out) {
                  float A = 2.f * cross / den;
                  float Bq = -(cross * cross) * Ivar / (den * den);
                  float T = A * uI + 2.f * Bq * uJ;
                  if (MODE == 0) {
                    float* so = a.saved_out + (size_t)b * 3 * DHW + off;
                    so[0] = A; so[DHW] = Bq; so[2 * DHW] = T;
                  } else {
                    float Bp = -(cross * cross) * Jvar / (den * den);
                    float Tp = A * uJ + 2.f * Bp * uI;
                    ncc_save2(a.saved_out + (size_t)b * (a.which == 3 ? 5 : 3) * DHW + off, DHW, a.which, A, Bq, T, Bp, Tp);
                  }
                }
              } else {
                float Iv = __ldg(a.I + (size_t)b * DHW + off), Jv = __ldg(a.J + (size_t)b * DHW + off);
                float gl = __ldg(a.grad_loss) * (float)a.scale;
                a.out[(size_t)b * DHW + off] = gl * (Iv * S[0] + 2.f * Jv * S[1] - S[2]);
                if (MODE == 3) a.out2[(size_t)b * DHW + off] = gl * (Jv * S[0] + 2.f * Iv * S[3] - S[4]);
              }
            }
          }
        }
        __syncthreads();  // s_in / s_w reuse in the next slice
      }
    }
  }
  if (FWD) {
    double tot = block_sum<double>(local, s_red);
    int nblocks = gridDim.x * gridDim.y * gridDim.z;
    int bid = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
    finish_reduce(tot, a.rw, nblocks, bid, a.scale, a.out, s_red);
  }
}

// ------------------------------------------------------------------------------------------------------------
// 9x9(x9) window fast path (the reference default, losses.py:26) — `ncc9_kernel`.
//
// The generic kernel above spends ~290 instructions per voxel (direct 9-tap sums in all three passes, a 16x32 tile
// whose 24x40 halo'd slab is re-staged and re-filtered for every one of its zchunk + 8 slices) and two-plus
// barriers per slice on 252 CTAs: 0.04 of the HBM roofline.  This kernel
//   * runs the D pass FIRST, so the z halo slices cost loads, not a W and an H pass.  The forward sums every halo'd
//     column directly over the window's slices, re-read from L1 / L2: a running sum's rounding residue would be as
//     large as the true sums in background and rim windows, and the pointwise stage divides by den ~ 1e-5 there.
//     The backward's box sums of A, Bq, T feed no division; there the window slides, S += P(z+4) - P(z-5) in shared
//     memory, and the leading halo slices cost a load and 3 adds per column;
//   * runs the W and H passes on the D-summed slice in registers, 8 / 4 outputs per thread, each window the sum of
//     a suffix sum of the first half and a prefix sum of the second (22 / 14 adds instead of 72 / 36, no subtraction),
//     so every box sum is a sum of the window's own values and a window of zeros sums to exactly 0, as in the reference;
//   * uses a 32 x 56 tile (halo overhead 1.43x instead of 1.88x; 224 = 4 x 56), 512 threads, 2 CTAs per SM,
//     bank-conflict-free pitches (68 / 60 floats) for the 16-byte shared-memory accesses of the W pass;
//   * is persistent over (tile, depth-chunk) items, so any volume fits the reduction workspace.
// tests/test_gpu_fp32_step_kernels.py holds the loss and the gradient to twice the fp64 distance of the
// reference's own fp32 arithmetic (+1e-6), on smooth, skull-stripped and offset images.
// ------------------------------------------------------------------------------------------------------------
namespace ncc9 {
constexpr int TH = 32, TW = 56, HR = TH + 8, HC = TW + 8, PD = 68, PW = 60, NT = 512;
constexpr int KC = HR * HC / NT;   // halo'd columns per thread (5)
static_assert(HR * HC % NT == 0, "column ownership must be exact");

struct Args9 {
  NccArgs a;
  int tiles_w, tiles_h, nchunks, nitems;
};

template <int MODE>
constexpr size_t smem_bytes() { return (size_t)ncc_fields(MODE) * HR * (PD + PW) * sizeof(float); }

template <int MODE, int WD>
__global__ void __launch_bounds__(NT, 2) ncc9_kernel(const Args9 q) {
  constexpr bool FWD = ncc_is_fwd(MODE);
  constexpr int NS = ncc_fields(MODE);
  constexpr int PDZ = WD / 2;
  const NccArgs& a = q.a;
  extern __shared__ __align__(16) float sm9[];
  float* s_d = sm9;                   // [NS][HR][PD]  D-summed fields of the current window
  float* s_w = sm9 + NS * HR * PD;    // [NS][HR][PW]  ... after the W pass
  __shared__ double s_red[32];
  const int tid = threadIdx.x;
  const size_t HW = (size_t)a.H * a.W, DHW = HW * a.D;
  const float inv_n = 1.0f / a.nwin;
  double local = 0.0;

  for (int item = blockIdx.x; item < q.nitems; item += gridDim.x) {
    const int wt = item % q.tiles_w, ht = (item / q.tiles_w) % q.tiles_h;
    const int ch = (item / (q.tiles_w * q.tiles_h)) % q.nchunks, b = item / (q.tiles_w * q.tiles_h * q.nchunks);
    const int z0 = ch * a.zchunk, z1 = min(z0 + a.zchunk, a.D);
    const int h0 = ht * TH - 4, w0 = wt * TW - 4;
    const float* f0 = (FWD ? a.I : a.saved_in) + (size_t)b * (FWD ? 1 : NS) * DHW;
    const float* f1 = FWD ? a.J + (size_t)b * DHW : f0 + DHW;    // backward: field f at f0 + f * DHW
    const float* f2 = FWD ? nullptr : f0 + 2 * DHW;
    int goff[KC], soff[KC];
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      const int idx = tid + k * NT, r = idx >> 6, c = idx & 63;
      const int h = h0 + r, w = w0 + c;
      goff[k] = (h >= 0 && h < a.H && w >= 0 && w < a.W) ? h * a.W + w : -1;
      soff[k] = r * PD + c;
    }
    if (!FWD) {
      for (int i = tid; i < NS * HR * PD; i += NT) s_d[i] = 0.f;
      __syncthreads();
    }
    // forward: one iteration per output slice; backward: the window's leading halo slices first (running sum)
    for (int zi = FWD ? z0 + PDZ : z0 - PDZ; zi < z1 + PDZ; ++zi) {
      const int zo = zi - PDZ;
      if (FWD) {
        // ---------------- D pass (forward): every halo'd column summed directly over the WD slices of the window ----
        // (zero padded).  A running sum (S += new - old) keeps the rounding of the larger values it slid past: where a
        // window then holds only zeros or faint values (the background and rims of skull-stripped images) that residue
        // is as large as the true sums, and den = Ivar * Jvar + 1e-5 turns it into large errors in cc, A and Bq.
#pragma unroll
        for (int k = 0; k < KC; ++k) {
          float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
          if (goff[k] >= 0) {
            float u[WD], v[WD];
#pragma unroll
            for (int j = 0; j < WD; ++j) {
              const int zj = zo - PDZ + j;
              u[j] = v[j] = 0.f;
              if (zj >= 0 && zj < a.D) {
                const size_t o = (size_t)zj * HW + goff[k];
                u[j] = __ldg(f0 + o); v[j] = __ldg(f1 + o);
              }
            }
#pragma unroll
            for (int j = 0; j < WD; ++j) {
              acc[0] += u[j]; acc[1] += v[j]; acc[2] += u[j] * u[j]; acc[3] += v[j] * v[j]; acc[4] += u[j] * v[j];
            }
          }
          float* d = s_d + soff[k];
#pragma unroll
          for (int f = 0; f < 5; ++f) d[f * HR * PD] = acc[f];
        }
      } else {
        // ---------------- D pass (backward): slide the window of every halo'd column by one slice ----------------
        // S += P(zi) - P(zi - WD) over the saved fields.  No division follows, so the residue of this running sum stays
        // at the rounding level of the values it slid past (the test suite checks d/dJ on skull-stripped images).
        // The two-sided backward slides Bp, Tp in a second pass, so that no more than 30 values are in flight per thread.
        const int zold = zi - WD;
        const bool has_new = zi >= 0 && zi < a.D;
        const bool has_old = WD > 1 && zold >= z0 - PDZ && zold >= 0;   // it was added earlier in this chunk
        float un[KC], vn[KC], tn[KC], uo[KC], vo[KC], to[KC];
#pragma unroll
        for (int k = 0; k < KC; ++k) {
          un[k] = vn[k] = tn[k] = uo[k] = vo[k] = to[k] = 0.f;
          if (goff[k] >= 0) {
            if (has_new) {
              const size_t o = (size_t)zi * HW + goff[k];
              un[k] = __ldg(f0 + o); vn[k] = __ldg(f1 + o); tn[k] = __ldg(f2 + o);
            }
            if (has_old) {
              const size_t o = (size_t)zold * HW + goff[k];
              uo[k] = __ldg(f0 + o); vo[k] = __ldg(f1 + o); to[k] = __ldg(f2 + o);
            }
          }
        }
#pragma unroll
        for (int k = 0; k < KC; ++k) {
          if (goff[k] >= 0) {
            float* d = s_d + soff[k];
            const float dl[3] = {un[k] - uo[k], vn[k] - vo[k], tn[k] - to[k]};
#pragma unroll
            for (int f = 0; f < 3; ++f) {
              if (WD > 1) d[f * HR * PD] += dl[f]; else d[f * HR * PD] = dl[f];
            }
          }
        }
        if (MODE == 3) {
          const float* f3 = f0 + 3 * DHW;
          const float* f4 = f0 + 4 * DHW;
#pragma unroll
          for (int k = 0; k < KC; ++k) {
            un[k] = vn[k] = uo[k] = vo[k] = 0.f;
            if (goff[k] >= 0) {
              if (has_new) {
                const size_t o = (size_t)zi * HW + goff[k];
                un[k] = __ldg(f3 + o); vn[k] = __ldg(f4 + o);
              }
              if (has_old) {
                const size_t o = (size_t)zold * HW + goff[k];
                uo[k] = __ldg(f3 + o); vo[k] = __ldg(f4 + o);
              }
            }
          }
#pragma unroll
          for (int k = 0; k < KC; ++k) {
            if (goff[k] >= 0) {
              float* d = s_d + 3 * HR * PD + soff[k];
              const float dl[2] = {un[k] - uo[k], vn[k] - vo[k]};
#pragma unroll
              for (int f = 0; f < 2; ++f) {
                if (WD > 1) d[f * HR * PD] += dl[f]; else d[f * HR * PD] = dl[f];
              }
            }
          }
        }
      }
      __syncthreads();
      if (zo >= z0) {   // block-uniform
        // ---------------- W pass: 8 adjacent window sums per work item from 16 staged values ----------------
        for (int it = tid; it < NS * 7 * HR; it += NT) {
          const int r = it % HR, t = it / HR, seg = t % 7, f = t / 7;
          const float4* src = reinterpret_cast<const float4*>(s_d + (f * HR + r) * PD + seg * 8);
          const float4 x0 = src[0], x1 = src[1], x2 = src[2], x3 = src[3];
          const float x[16] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w, x2.x, x2.y, x2.z, x2.w, x3.x, x3.y, x3.z, x3.w};
          // o[j] = x[j..j+8] = (x[j] + .. + x[7]) + (x[8] + .. + x[8+j]): suffix sums of the first half plus prefix sums
          // of the second, no subtraction, so a window of zeros sums to exactly 0
          float sfx[8], pfx[8], o[8];
          sfx[7] = x[7];
          pfx[0] = x[8];
#pragma unroll
          for (int j = 6; j >= 0; --j) sfx[j] = x[j] + sfx[j + 1];
#pragma unroll
          for (int j = 1; j < 8; ++j) pfx[j] = pfx[j - 1] + x[j + 8];
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = sfx[j] + pfx[j];
          float4* dst = reinterpret_cast<float4*>(s_w + (f * HR + r) * PW + seg * 8);
          dst[0] = make_float4(o[0], o[1], o[2], o[3]);
          dst[1] = make_float4(o[4], o[5], o[6], o[7]);
        }
        __syncthreads();
        // ---------------- H pass (4 outputs of one column per thread) + pointwise ----------------
        if (tid < TW * (TH / 4)) {
          const int wl = tid % TW, hq = tid / TW;
          float S[NS][4];
#pragma unroll
          for (int f = 0; f < NS; ++f) {
            const float* colp = s_w + (f * HR + hq * 4) * PW + wl;
            float col[12];
#pragma unroll
            for (int j = 0; j < 12; ++j) col[j] = colp[j * PW];
            // S[j] = col[j..j+8] = (col[j] + .. + col[7]) + (col[8] + .. + col[8+j]), as in the W pass
            float sfx = col[3] + ((col[4] + col[5]) + (col[6] + col[7])), pfx = col[8];
            S[f][3] = sfx;
#pragma unroll
            for (int j = 2; j >= 0; --j) { sfx = col[j] + sfx; S[f][j] = sfx; }
            S[f][0] += pfx;
#pragma unroll
            for (int j = 1; j < 4; ++j) { pfx += col[j + 8]; S[f][j] += pfx; }
          }
          const int w = wt * TW + wl;
          if (w < a.W) {
            float gl = 0.f;
            if (!FWD) gl = __ldg(a.grad_loss) * (float)a.scale;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int h = ht * TH + hq * 4 + j;
              if (h < a.H) {
                const size_t off = (size_t)zo * HW + (size_t)h * a.W + w;
                if (FWD) {
                  // losses.py:57-65
                  const float Is = S[0][j], Js = S[1][j], I2s = S[2][j], J2s = S[3][j], IJs = S[4][j];
                  const float uI = Is * inv_n, uJ = Js * inv_n;
                  const float cross = IJs - uJ * Is - uI * Js + uI * uJ * a.nwin;
                  const float Ivar = I2s - 2.f * uI * Is + uI * uI * a.nwin;
                  const float Jvar = J2s - 2.f * uJ * Js + uJ * uJ * a.nwin;
                  const float den = Ivar * Jvar + 1e-5f;
                  const float rden = 1.0f / den;
                  const float cc = cross * cross * rden;
                  local += (double)cc;
                  if (a.saved_out) {
                    const float A = 2.f * cross * rden;
                    const float Bq = -cc * Ivar * rden;
                    const float T = A * uI + 2.f * Bq * uJ;
                    if (MODE == 0) {
                      float* so = a.saved_out + (size_t)b * 3 * DHW + off;
                      so[0] = A; so[DHW] = Bq; so[2 * DHW] = T;
                    } else {
                      const float Bp = -cc * Jvar * rden;
                      const float Tp = A * uJ + 2.f * Bp * uI;
                      ncc_save2(a.saved_out + (size_t)b * (a.which == 3 ? 5 : 3) * DHW + off, DHW, a.which, A, Bq, T, Bp, Tp);
                    }
                  }
                } else {
                  const float Iv = __ldg(a.I + (size_t)b * DHW + off), Jv = __ldg(a.J + (size_t)b * DHW + off);
                  a.out[(size_t)b * DHW + off] = gl * (Iv * S[0][j] + 2.f * Jv * S[1][j] - S[2][j]);
                  if (MODE == 3) a.out2[(size_t)b * DHW + off] = gl * (Jv * S[0][j] + 2.f * Iv * S[3][j] - S[4][j]);
                }
              }
            }
          }
        }
      }
    }
    __syncthreads();   // every thread is done with s_w / s_d before the next item writes them
  }
  if (FWD) {
    double tot = block_sum<double>(local, s_red);
    finish_reduce(tot, a.rw, gridDim.x, blockIdx.x, a.scale, a.out, s_red);
  }
}

// depth chunks: fill 2 CTAs per SM in whole waves, every chunk re-reads wd - 1 halo slices (D pass only)
static int pick_zchunk(int D, long long tiles, int wd) {
  const char* e = getenv("VXM_B200_NCC_ZCHUNK");
  if (e && atoi(e) >= 1) return atoi(e);
  if (wd == 1) return D;
  const long long slots = 2LL * sm_count();
  int best = D;
  double best_cost = 1e300;
  for (int nch = 1; nch <= D; ++nch) {
    const int zc = (D + nch - 1) / nch;
    if (zc < 4 && nch > 1) break;
    const long long ctas = tiles * ((D + zc - 1) / zc);
    // a slice of the chunk costs ~3 units (D + W + H passes), a halo slice ~1 (D pass only)
    const double cost = (double)((ctas + slots - 1) / slots) * (3.0 * zc + (wd - 1));
    if (cost < best_cost - 1e-9) { best_cost = cost; best = zc; }
  }
  return best;
}

template <int MODE>
static int launch(NccArgs a, cudaStream_t st) {
  Args9 q;
  q.tiles_w = (a.W + TW - 1) / TW; q.tiles_h = (a.H + TH - 1) / TH;
  a.zchunk = pick_zchunk(a.D, (long long)a.B * q.tiles_w * q.tiles_h, a.wd);
  q.nchunks = (a.D + a.zchunk - 1) / a.zchunk;
  const long long items = (long long)a.B * q.tiles_w * q.tiles_h * q.nchunks;
  VXM_REQUIRE(items < (1LL << 31) && (size_t)a.H * a.W < (1u << 31), "ncc: volume too large");
  q.nitems = (int)items;
  q.a = a;
  const int cap = 2 * sm_count() < kMaxReduceBlocks ? 2 * sm_count() : kMaxReduceBlocks;
  const int grid = q.nitems < cap ? q.nitems : cap;
  const size_t smem = smem_bytes<MODE>();
  if (a.wd == 9) {
    VXM_CUDA(cudaFuncSetAttribute(ncc9_kernel<MODE, 9>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ncc9_kernel<MODE, 9><<<grid, NT, smem, st>>>(q);
  } else {
    VXM_CUDA(cudaFuncSetAttribute(ncc9_kernel<MODE, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ncc9_kernel<MODE, 1><<<grid, NT, smem, st>>>(q);
  }
  return check_launch(ncc_is_fwd(MODE) ? "ncc_fwd" : "ncc_bwd");
}
static bool applies(int wd, int wh, int ww) {
  const char* e = getenv("VXM_B200_NCC_KERNEL");
  if (e && e[0] == 'g') return false;      // "generic": A/B switch
  return wh == 9 && ww == 9 && (wd == 9 || wd == 1);
}
}  // namespace ncc9

template <int MODE>
static int ncc_launch(const NccArgs& a, dim3 grid, cudaStream_t st) {
  switch (a.wd) {
    case 1: ncc_kernel<MODE, 1><<<grid, 256, 0, st>>>(a); break;
    case 3: ncc_kernel<MODE, 3><<<grid, 256, 0, st>>>(a); break;
    case 5: ncc_kernel<MODE, 5><<<grid, 256, 0, st>>>(a); break;
    case 7: ncc_kernel<MODE, 7><<<grid, 256, 0, st>>>(a); break;
    case 9: ncc_kernel<MODE, 9><<<grid, 256, 0, st>>>(a); break;
    default: set_error("ncc: unsupported window depth %d", a.wd); return VXM_ERR_UNSUPPORTED;
  }
  return check_launch(ncc_is_fwd(MODE) ? "ncc_fwd" : "ncc_bwd");
}

static int ncc_check(int B, int D, int H, int W, int wd, int wh, int ww, dim3* grid, int* zchunk) {
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "ncc: non-positive dimension");
  auto okw = [](int w) { return w >= 1 && w <= 9 && (w & 1); };
  if (!(okw(wd) && okw(wh) && okw(ww))) {
    set_error("ncc: window (%d,%d,%d) unsupported (odd sizes 1..9 only)", wd, wh, ww);
    return VXM_ERR_UNSUPPORTED;
  }
  const int zc = ncc_zchunk(D, (long long)B * ((W + NTW - 1) / NTW) * ((H + NTH - 1) / NTH), wd);
  *zchunk = zc;
  int nchunks = (D + zc - 1) / zc;
  *grid = dim3((W + NTW - 1) / NTW, (H + NTH - 1) / NTH, nchunks * B);
  VXM_REQUIRE((size_t)grid->x * grid->y * grid->z <= (size_t)kMaxReduceBlocks && grid->z <= 65535u,
              "ncc: volume too large for the reduction workspace");
  return VXM_OK;
}

}  // namespace vxm

using namespace vxm;

extern "C" size_t vxm_reduce_workspace_bytes(void) { return sizeof(double) * kMaxReduceBlocks + 256; }

namespace vxm {
ReduceWork as_reduce_work(void* work) {
  ReduceWork rw;
  rw.counter = reinterpret_cast<unsigned int*>(work);
  rw.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(work) + 256);
  return rw;
}
}  // namespace vxm

static int ncc_window_check(int wd, int wh, int ww) {
  auto okw = [](int w) { return w >= 1 && w <= 9 && (w & 1); };
  if (!(okw(wd) && okw(wh) && okw(ww))) {
    set_error("ncc: window (%d,%d,%d) unsupported (odd sizes 1..9 only)", wd, wh, ww);
    return VXM_ERR_UNSUPPORTED;
  }
  return VXM_OK;
}

extern "C" int vxm_ncc_fwd(const float* I, const float* J, float* loss, float* saved, void* work, int B,
                           int D, int H, int W, int wd, int wh, int ww, void* stream) {
  if (int rcw = ncc_window_check(wd, wh, ww)) return rcw;
  VXM_REQUIRE(I && J && loss && work, "ncc_fwd: null pointer");
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "ncc: non-positive dimension");
  NccArgs a{};
  a.I = I; a.J = J; a.saved_out = saved; a.out = loss; a.rw = as_reduce_work(work);
  a.B = B; a.D = D; a.H = H; a.W = W; a.wd = wd; a.wh = wh; a.ww = ww;
  a.nwin = (float)(wd * wh * ww);
  a.scale = -1.0 / ((double)B * D * H * W);
  if (ncc9::applies(wd, wh, ww)) return ncc9::launch<0>(a, as_stream(stream));
  dim3 grid;
  int zchunk = 0;
  int rc = ncc_check(B, D, H, W, wd, wh, ww, &grid, &zchunk);
  if (rc) return rc;
  a.zchunk = zchunk;
  return ncc_launch<0>(a, grid, as_stream(stream));
}

extern "C" int vxm_ncc_bwd(const float* I, const float* J, const float* saved, const float* grad_loss,
                           float* grad_J, int B, int D, int H, int W, int wd, int wh, int ww, void* stream) {
  if (int rcw = ncc_window_check(wd, wh, ww)) return rcw;
  VXM_REQUIRE(I && J && saved && grad_loss && grad_J, "ncc_bwd: null pointer");
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "ncc: non-positive dimension");
  NccArgs a{};
  a.I = I; a.J = J; a.saved_in = saved; a.out = grad_J; a.grad_loss = grad_loss;
  a.B = B; a.D = D; a.H = H; a.W = W; a.wd = wd; a.wh = wh; a.ww = ww;
  a.nwin = (float)(wd * wh * ww);
  a.scale = -1.0 / ((double)B * D * H * W);
  if (ncc9::applies(wd, wh, ww)) return ncc9::launch<1>(a, as_stream(stream));
  dim3 grid;
  int zchunk = 0;
  int rc = ncc_check(B, D, H, W, wd, wh, ww, &grid, &zchunk);
  if (rc) return rc;
  a.zchunk = zchunk;
  return ncc_launch<1>(a, grid, as_stream(stream));
}

// Two-sided NCC.  `which`: bit 0 = y_true (I) needs a gradient, bit 1 = y_pred (J).  The forward saves, per voxel,
// which == 2: A, Bq, T (exactly vxm_ncc_fwd); 1: A, Bp, Tp; 3: A, Bq, T, Bp, Tp — `saved` holds that many fields of B*D*H*W.
extern "C" int vxm_ncc_fwd2(const float* I, const float* J, float* loss, float* saved, void* work, int which, int B,
                            int D, int H, int W, int wd, int wh, int ww, void* stream) {
  VXM_REQUIRE(which >= 1 && which <= 3, "ncc_fwd2: which must be 1 (y_true), 2 (y_pred) or 3 (both), got %d", which);
  if (which == 2) return vxm_ncc_fwd(I, J, loss, saved, work, B, D, H, W, wd, wh, ww, stream);
  if (int rcw = ncc_window_check(wd, wh, ww)) return rcw;
  VXM_REQUIRE(I && J && loss && saved && work, "ncc_fwd2: null pointer");
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "ncc: non-positive dimension");
  NccArgs a{};
  a.I = I; a.J = J; a.saved_out = saved; a.out = loss; a.rw = as_reduce_work(work); a.which = which;
  a.B = B; a.D = D; a.H = H; a.W = W; a.wd = wd; a.wh = wh; a.ww = ww;
  a.nwin = (float)(wd * wh * ww);
  a.scale = -1.0 / ((double)B * D * H * W);
  if (ncc9::applies(wd, wh, ww)) return ncc9::launch<2>(a, as_stream(stream));
  dim3 grid;
  int zchunk = 0;
  int rc = ncc_check(B, D, H, W, wd, wh, ww, &grid, &zchunk);
  if (rc) return rc;
  a.zchunk = zchunk;
  return ncc_launch<2>(a, grid, as_stream(stream));
}

// grad_I / grad_J = grad_loss[0] * d(-mean cc)/d(I | J) from the fields vxm_ncc_fwd2 saved with the same `which`; the
// pointer of a gradient that is not asked for is ignored.  which == 3 is one launch over five box sums.
extern "C" int vxm_ncc_bwd2(const float* I, const float* J, const float* saved, const float* grad_loss, float* grad_I,
                            float* grad_J, int which, int B, int D, int H, int W, int wd, int wh, int ww, void* stream) {
  VXM_REQUIRE(which >= 1 && which <= 3, "ncc_bwd2: which must be 1 (y_true), 2 (y_pred) or 3 (both), got %d", which);
  if (which == 2) return vxm_ncc_bwd(I, J, saved, grad_loss, grad_J, B, D, H, W, wd, wh, ww, stream);
  // y_true alone: A, Bp, Tp are what the three-field backward expects once I and J trade places
  if (which == 1) return vxm_ncc_bwd(J, I, saved, grad_loss, grad_I, B, D, H, W, wd, wh, ww, stream);
  if (int rcw = ncc_window_check(wd, wh, ww)) return rcw;
  VXM_REQUIRE(I && J && saved && grad_loss && grad_I && grad_J, "ncc_bwd2: null pointer");
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "ncc: non-positive dimension");
  NccArgs a{};
  a.I = I; a.J = J; a.saved_in = saved; a.out = grad_J; a.out2 = grad_I; a.grad_loss = grad_loss; a.which = which;
  a.B = B; a.D = D; a.H = H; a.W = W; a.wd = wd; a.wh = wh; a.ww = ww;
  a.nwin = (float)(wd * wh * ww);
  a.scale = -1.0 / ((double)B * D * H * W);
  if (ncc9::applies(wd, wh, ww)) return ncc9::launch<3>(a, as_stream(stream));
  dim3 grid;
  int zchunk = 0;
  int rc = ncc_check(B, D, H, W, wd, wh, ww, &grid, &zchunk);
  if (rc) return rc;
  a.zchunk = zchunk;
  return ncc_launch<3>(a, grid, as_stream(stream));
}
