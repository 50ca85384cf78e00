// Weight gradient of the k=3 convolution on the Hopper tensor cores (wgmma):
//     gw[tap][ci][co] = sum_{b,v} x[b, v + tap - 1, ci] * gz[b, v, co]          (gz = grad wrt the conv output)
// (autograd of nn.Conv3d at reference voxelmorph/torch/networks.py:299,211).  The general path: planar fp32 sources and
// channel counts conv3d_tc_wgrad2.cu does not take.
//
// Per (tap, 16 voxels) one MMA  D[64 x N] += A^T[64 ch x 16 vox] * B[16 vox x N]  with both operands
// "MN-major" straight out of the channels-last slabs the forward kernel also uses:
//   A = x slab  [Cin/8][180 rows][8 ch]  (halo'd 18 x 10 voxels of one input slice; the tap is a start-address
//       offset; K = voxels: 8 consecutive w are 16 B apart = one core matrix, the next K group is the next h row)
//   B = gz tile [Cout/8][128 rows][8 ch] (16 x 8 voxels, no halo)
// The nine (kh, kw) tap accumulators of one kd (9 x 64 x N fp32) stay in the registers of two MMA warpgroups for the
// CTA's whole lifetime (grid.y = kd); each CTA streams its share of the volume, then writes its taps of ONE partial
// [27][64][N]; a second kernel reduces the partials over CTAs in fixed order (deterministic) into the fp32
// (Cout,Cin,kd,3,3) gradient.
#include <type_traits>

#include "tc_common.cuh"

namespace vxm {
namespace tc {

constexpr int WTH = 16, WTW = 8, WSW = WTW + 2, WSH = WTH + 2;
constexpr int WROWS = WSH * WSW, WPLANE = WROWS * 16;   // x slab plane: 180 rows
constexpr int GPLANE = 128 * 16;                        // gz tile plane: 128 rows
constexpr int WMAXSLOT = 8, WNG = 4, WKMAX = 12;
constexpr int WNLOADER = 128, WNTHREADS = 384;   // warps 0-3 / 4-7: MMA warpgroups (0-3 also sum the bias), 8-11: loader

struct WgradTcArgs {
  const __nv_bfloat16* xa; const __nv_bfloat16* xb;
  const float* xf[4]; long long xf_bs[4]; int nplanar_x;
  int Ca, Cb, up, upd;
  const __nv_bfloat16* gz; int Cg;
  const float* gf[4]; long long gf_bs[4]; int nplanar_g;
  float* partial;
  float* bias_partial;   // [grid][NP]
  int B, D, H, W, KD, NP;
  int tiles_h, tiles_w, dchunk, nchunks, nitems, nslot;
};

// Grid (gx, KD): CTA (x, kd) accumulates the nine (kh, kw) taps of input-slice offset kd over its share x of the volume
// (the x slabs of a share are staged once per kd), split over its two MMA warpgroups (taps 0-4 / 5-8): all nine
// M = 64 x N = NP accumulators stay in registers for the CTA's lifetime.
template <int KD, int NP>
__global__ void __launch_bounds__(WNTHREADS, 1) wgrad_tc_kernel(const WgradTcArgs a) {
  constexpr int NTAP = 5;                                  // accumulators per warpgroup (taps 5g .. 5g + 4, < 9)
  extern __shared__ __align__(128) uint8_t smem[];
  const bool px = a.nplanar_x > 0, pg = a.nplanar_g > 0;
  const int nc8 = px ? 1 : (a.Ca + a.Cb) / 8;
  const int ncg = pg ? 1 : a.Cg / 8;
  const uint32_t slab_bytes = (uint32_t)nc8 * WPLANE;
  const uint32_t gt_bytes = (uint32_t)ncg * GPLANE;
  uint8_t* s_slab = smem;
  const int WNSLOT = a.nslot;
  // tail padding so that the M=64 operand (8 channel planes) never reads past the allocation
  uint8_t* s_g = s_slab + WNSLOT * slab_bytes + 16 * WPLANE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_g + WNG * gt_bytes + 4 * GPLANE);
  uint64_t* xfull = bars;
  uint64_t* xempty = bars + WMAXSLOT;
  uint64_t* gfull = bars + 2 * WMAXSLOT;
  uint64_t* gempty = gfull + WNG;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = KD * 9;
  const int kdc = blockIdx.y;                              // this CTA's kd tap

  if (threadIdx.x == 0) {
    // one arrival per warp of both MMA warpgroups, after its last MMA reading the slab has completed
    for (int i = 0; i < WNSLOT; ++i) { mbar_init(&xfull[i], WNLOADER); mbar_init(&xempty[i], 8); }
    for (int i = 0; i < WNG; ++i) { mbar_init(&gfull[i], WNLOADER); mbar_init(&gempty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  const int HW_tiles = a.tiles_h * a.tiles_w;
  const bool has_work = blockIdx.x < a.nitems;

  if (warp >= 8) {
    // ================================ LOADER ================================
    const int lt = threadIdx.x - 8 * 32;
    uint32_t xcnt = 0, gcnt = 0;
    const int Da = a.upd ? a.D >> 1 : a.D, Ha = a.up ? a.H >> 1 : a.H, Wa = a.up ? a.W >> 1 : a.W;
    const int nca8 = a.Ca >> 3;
    const int nchunk = nc8 * WROWS, ngchunk = ncg * 128;
    for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
      const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
      const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
      const int h0 = ht * WTH, w0 = wt * WTW, d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, a.D);
      const int s_begin = KD == 3 ? d0 - 1 : d0, s_end = KD == 3 ? d1 + 1 : d1;
      int soff[WKMAX];
      uint32_t doff[WKMAX];
      if (!px) {
#pragma unroll
        for (int k = 0; k < WKMAX; ++k) {
          const int id = lt + k * WNLOADER;
          soff[k] = -1;
          doff[k] = 0;
          if (id < nchunk) {
            const int c8 = id % nc8, row = id / nc8;
            const int r = row / WSW, c = row - r * WSW;
            const int h = h0 - 1 + r, w = w0 - 1 + c;
            doff[k] = (uint32_t)c8 * WPLANE + (uint32_t)row * 16u;
            if (h >= 0 && h < a.H && w >= 0 && w < a.W) {
              if (c8 < nca8) soff[k] = (((a.up ? h >> 1 : h) * Wa + (a.up ? w >> 1 : w)) * a.Ca + c8 * 8) << 1;
              else soff[k] = (((h * a.W + w) * a.Cb + (c8 - nca8) * 8) << 1) | 1;
            }
          }
        }
      }
      int goff[4];
      uint32_t gdoff[4];
      if (!pg) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int id = lt + k * WNLOADER;
          goff[k] = -1;
          gdoff[k] = 0;
          if (id < ngchunk) {
            const int c8 = id % ncg, row = id / ncg;
            const int h = h0 + (row >> 3), w = w0 + (row & 7);
            gdoff[k] = (uint32_t)c8 * GPLANE + (uint32_t)row * 16u;
            if (h < a.H && w < a.W) goff[k] = (h * a.W + w) * a.Cg + c8 * 8;
          }
        }
      }
      for (int ds = s_begin; ds < s_end; ++ds) {
        // ---- x slab of input slice ds ----
        const int slot = xcnt % WNSLOT;
        mbar_wait(&xempty[slot], ((xcnt / WNSLOT) & 1) ^ 1);
        uint8_t* slab = s_slab + (size_t)slot * slab_bytes;
        const bool dok = ds >= 0 && ds < a.D;
        if (!px) {
          const __nv_bfloat16* baseA = a.xa ? a.xa + (((size_t)b * Da + (dok ? (a.upd ? ds >> 1 : ds) : 0)) * Ha * Wa) * a.Ca : nullptr;
          const __nv_bfloat16* baseB = a.xb ? a.xb + (((size_t)b * a.D + (dok ? ds : 0)) * a.H * a.W) * a.Cb : nullptr;
          const __nv_bfloat16* dummy = a.xa ? a.xa : a.xb;
#pragma unroll
          for (int k = 0; k < WKMAX; ++k) {
            if (lt + k * WNLOADER < nchunk) {
              const bool ok = dok && soff[k] >= 0;
              const __nv_bfloat16* src = ok ? ((soff[k] & 1) ? baseB : baseA) + (soff[k] >> 1) : dummy;
              cp_async16(slab + doff[k], src, ok ? 16u : 0u);
            }
          }
          cp_async_arrive_noinc(&xfull[slot]);
        } else {
          for (int row = lt; row < WROWS; row += WNLOADER) {
            const int r = row / WSW, c = row - r * WSW;
            const int h = h0 - 1 + r, w = w0 - 1 + c;
            const bool ok = dok && h >= 0 && h < a.H && w >= 0 && w < a.W;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            if (ok) {
              const size_t off = ((size_t)ds * a.H + h) * a.W + w;
              for (int p = 0; p < a.nplanar_x; ++p) v[p] = __ldg(a.xf[p] + (size_t)b * a.xf_bs[p] + off);
            }
            const uint4 q = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), 0u, 0u);
            *reinterpret_cast<uint4*>(slab + row * 16) = q;
          }
          fence_proxy_async();
          mbar_arrive(&xfull[slot]);
        }
        ++xcnt;
        // ---- gz tile of OUTPUT slice dg (the slice whose window this x slab completes) ----
        const int dg = KD == 3 ? ds - 1 : ds;
        if (dg >= d0 && dg < d1) {
          const int gslot = gcnt % WNG;
          mbar_wait(&gempty[gslot], ((gcnt / WNG) & 1) ^ 1);
          uint8_t* gt = s_g + (size_t)gslot * gt_bytes;
          if (!pg) {
            const __nv_bfloat16* baseG = a.gz + (((size_t)b * a.D + dg) * a.H * a.W) * a.Cg;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              if (lt + k * WNLOADER < ngchunk) {
                const bool ok = goff[k] >= 0;
                cp_async16(gt + gdoff[k], ok ? baseG + goff[k] : a.gz, ok ? 16u : 0u);
              }
            }
            cp_async_arrive_noinc(&gfull[gslot]);
          } else {
            for (int row = lt; row < 128; row += WNLOADER) {
              const int h = h0 + (row >> 3), w = w0 + (row & 7);
              float v[4] = {0.f, 0.f, 0.f, 0.f};
              if (h < a.H && w < a.W) {
                const size_t off = ((size_t)dg * a.H + h) * a.W + w;
                for (int p = 0; p < a.nplanar_g; ++p) v[p] = __ldg(a.gf[p] + (size_t)b * a.gf_bs[p] + off);
              }
              *reinterpret_cast<uint4*>(gt + row * 16) = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), 0u, 0u);
            }
            fence_proxy_async();
            mbar_arrive(&gfull[gslot]);
          }
          ++gcnt;
        }
      }
    }
  } else {
    // ================================ MMA WARPGROUPS ================================
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    const int tap0 = wg * NTAP, ntap = wg == 0 ? NTAP : 9 - NTAP;
    float acc[NTAP][NP / 2];
    // warpgroup 0 of the kd = 0 CTAs also folds the bias gradient out of the staged gz tiles: thread t owns tile row t
    float bsum[NP];
#pragma unroll
    for (int c = 0; c < NP; ++c) bsum[c] = 0.f;
    const bool do_bias = wg == 0 && kdc == 0;
    if (has_work) {
      const uint32_t slab_u32 = smem_u32(s_slab), g_u32 = smem_u32(s_g);
      uint32_t xbase = 0, gcnt = 0;
      uint32_t acc0 = 0;                // 0 only for the very first tile of this CTA
      for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
        const int ch = (item / HW_tiles) % a.nchunks;
        const int d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, a.D);
        const int nd = d1 - d0;
        for (int j = 0; j < nd; ++j) {
          if (KD == 3) {
            if (j == 0) for (int q = 0; q < 2; ++q) { uint32_t c = xbase + q; mbar_wait(&xfull[c % WNSLOT], (c / WNSLOT) & 1); }
            uint32_t c = xbase + j + 2;
            mbar_wait(&xfull[c % WNSLOT], (c / WNSLOT) & 1);
          } else {
            uint32_t c = xbase + j;
            mbar_wait(&xfull[c % WNSLOT], (c / WNSLOT) & 1);
          }
          const uint32_t gs = gcnt % WNG;
          mbar_wait(&gfull[gs], (gcnt / WNG) & 1);
          const uint64_t bdesc0 = make_desc_mnmajor_noswz(g_u32 + gs * gt_bytes, 128u, (uint32_t)GPLANE);
          const uint64_t adesc = make_desc_mnmajor_noswz(slab_u32 + ((xbase + j + kdc) % WNSLOT) * slab_bytes, (uint32_t)WSW * 16u, (uint32_t)WPLANE);
          // one straight-line wgmma chain per warpgroup (no warpgroup-divergent branch inside a chain): NT taps from tap0
          auto chain = [&](auto nt) {
            constexpr int NT = decltype(nt)::value;
            wg_fence();
#pragma unroll
            for (int s = 0; s < NT; ++s) {
              const int t9 = tap0 + s, kh = t9 / 3, kw = t9 % 3;
#pragma unroll
              for (int i = 0; i < 8; ++i) {   // 8 x 16 voxels = the 128-voxel tile; 16-byte address units
                const uint64_t ad = adesc + (uint64_t)((kh + 2 * i) * WSW + kw);
                const uint64_t bd = bdesc0 + (uint64_t)(2 * i * 128 / 16);
                Wgmma<NP, 1, 1>::mma(acc[s], ad, bd, i == 0 ? acc0 : 1u);
              }
            }
            wg_commit();
          };
          if (wg == 0) chain(std::integral_constant<int, NTAP>{});
          else chain(std::integral_constant<int, 9 - NTAP>{});
          if (do_bias) {
            const uint8_t* gt = s_g + (size_t)gs * gt_bytes + t * 16;
#pragma unroll
            for (int c8 = 0; c8 < NP / 8; ++c8) {
              const uint4 q = *reinterpret_cast<const uint4*>(gt + (size_t)c8 * GPLANE);
              const __nv_bfloat162* hq = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 f = __bfloat1622float2(hq[e]);
                bsum[c8 * 8 + 2 * e] += f.x;
                bsum[c8 * 8 + 2 * e + 1] += f.y;
              }
            }
          }
          wg_wait<0>();
          if (lane == 0) {
            mbar_arrive(&xempty[(xbase + j) % WNSLOT]);
            mbar_arrive(&gempty[gs]);
          }
          acc0 = 1u;
          ++gcnt;
        }
        if (KD == 3) {
          if (lane == 0) {
            mbar_arrive(&xempty[(xbase + nd) % WNSLOT]);
            mbar_arrive(&xempty[(xbase + nd + 1) % WNSLOT]);
          }
          xbase += nd + 2;
        } else {
          xbase += nd;
        }
      }
    }
    // partial[x][tap][ci][co]: fragment (row ci, column co) of the accumulator of tap kd * 9 + t9
    float* part = a.partial + (size_t)blockIdx.x * T * 64 * NP;
    const int w4 = t >> 5, qr = lane >> 2, pc = lane & 3;
#pragma unroll
    for (int s = 0; s < NTAP; ++s) {
      if (s >= ntap) break;
      const int tap = kdc * 9 + tap0 + s;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int ci = 16 * w4 + 8 * i + qr;
#pragma unroll
        for (int jn = 0; jn < NP / 8; ++jn) {
          const int co = 8 * jn + 2 * pc;
          *reinterpret_cast<float2*>(part + ((size_t)tap * 64 + ci) * NP + co) =
              has_work ? make_float2(acc[s][4 * jn + 2 * i], acc[s][4 * jn + 2 * i + 1]) : make_float2(0.f, 0.f);
        }
      }
    }
    // bias partial of this CTA: deterministic reduction over the 128 rows through shared memory (the slab ring is idle
    // once both warpgroups have passed their last wgmma wait)
    if (kdc == 0) {
      named_bar(1, 256);
      if (wg == 0) {
        float* s_b = reinterpret_cast<float*>(s_slab);
#pragma unroll
        for (int c = 0; c < NP; ++c) s_b[t * (NP + 1) + c] = bsum[c];
        named_bar(2, 128);
        if (t < NP) {
          float sum = 0.f;
          for (int r2 = 0; r2 < 128; ++r2) sum += s_b[r2 * (NP + 1) + t];
          a.bias_partial[(size_t)blockIdx.x * NP + t] = sum;
        }
      }
    }
  }
}

// gw[co][ci][tap] (+)= sum_cta partial[cta][tap][ci][co]   (fixed order -> deterministic).  Threads walk the partial
// layout (co fastest) so the ncta reads per element are coalesced; the small transposed write is scattered.
__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ gw, int ncta, int T, int NP, int Cout, int Cin,
                                    const float* __restrict__ bias_partial, float* __restrict__ gb, int accumulate) {
  if (gb && blockIdx.x == 0 && threadIdx.x < Cout) {
    float acc = accumulate ? gb[threadIdx.x] : 0.f;
    for (int c = 0; c < ncta; ++c) acc += bias_partial[(size_t)c * NP + threadIdx.x];
    gb[threadIdx.x] = acc;
  }
  const int per_cta = T * 64 * NP;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < per_cta; j += gridDim.x * blockDim.x) {
    const int co = j % NP, ci = (j / NP) % 64, tap = j / (NP * 64);
    if (co >= Cout || ci >= Cin) continue;
    float acc = 0.f;
    for (int c = 0; c < ncta; ++c) acc += partial[(size_t)c * per_cta + j];
    float* dst = gw + ((size_t)co * Cin + ci) * T + tap;
    *dst = (accumulate ? *dst : 0.f) + acc;
  }
}

// bias gradient from a bf16 NDHWC tensor: gb[c] = sum_v gz[v][c]; two-stage, deterministic
__global__ void __launch_bounds__(256) bias_grad_partial_kernel(const __nv_bfloat16* __restrict__ gz, float* __restrict__ part, size_t V, int C) {
  // thread t handles channel t % C of voxels t / C, t / C + stride...
  __shared__ float s[256];
  const int c = threadIdx.x % C, lane_v = threadIdx.x / C, vper = 256 / C;
  float acc = 0.f;
  if (lane_v < vper)
    for (size_t v = (size_t)blockIdx.x * vper + lane_v; v < V; v += (size_t)gridDim.x * vper) acc += __bfloat162float(gz[v * C + c]);
  s[threadIdx.x] = lane_v < vper ? acc : 0.f;
  __syncthreads();
  if (threadIdx.x < C) {
    float t = 0.f;
    for (int k = 0; k < vper; ++k) t += s[k * C + threadIdx.x];
    part[(size_t)blockIdx.x * C + threadIdx.x] = t;
  }
}
__global__ void bias_grad_final_kernel(const float* __restrict__ part, float* __restrict__ gb, int nblocks, int C, int Creal) {
  const int c = threadIdx.x;
  if (c >= Creal) return;
  float acc = 0.f;
  for (int b = 0; b < nblocks; ++b) acc += part[(size_t)b * C + c];
  gb[c] = acc;
}

}  // namespace tc
}  // namespace vxm

using namespace vxm;
using namespace vxm::tc;

namespace vxm {
namespace tcw {   // conv3d_tc_wgrad2.cu: the kw-stacked Toeplitz formulation (channels-last bf16 sources only)
bool wgrad2_supported(int Ca, int Cb, int Cg);
int wgrad2_launch(const void* x, int Cx, int up, const void* gz, int Cg, float* grad_w, float* grad_b, void* work, int B, int D, int H, int W,
                  int kd, int Cout_real, int Cin_total, int ci_off, int ci_cnt, int accumulate, cudaStream_t st, ReduceDesc* desc,
                  size_t* work_used, bool khm, int x_pitch, int g_pitch, int co_off);
int wgrad2_reduce(const ReduceDesc* d, int n, cudaStream_t st);
}
}

static int wgrad_np(int cg) { return cg <= 8 ? 8 : cg <= 16 ? 16 : 32; }

extern "C" size_t vxm_conv3d_tc_wgrad_workspace_bytes(int kd) {
  // worst case: 256 CTAs x 27 taps x 64 rows x 32 cols fp32, + bias partials
  return (size_t)256 * kd * 9 * 64 * 32 * sizeof(float) + 1024 * 32 * sizeof(float);
}

extern "C" int vxm_conv3d_tc_wgrad(const void* xa, const void* xb, const float* const* xf, const long long* xf_bs, int nplanar_x,
                                   const void* gz, const float* const* gf, const long long* gf_bs, int nplanar_g,
                                   float* grad_w, float* grad_b, void* work, int B, int D, int H, int W, int Ca, int Cb, int up,
                                   int Cin_real, int Cg, int Cout_real, int kd, int accumulate, void* stream) {
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0 && grad_w && work, "conv3d_tc_wgrad: bad argument");
  VXM_REQUIRE(kd == 1 || kd == 3, "conv3d_tc_wgrad: kd must be 1 or 3");
  WgradTcArgs a{};
  int Cin;
  if (nplanar_x > 0) {
    VXM_REQUIRE(nplanar_x <= 4 && xf && xf_bs, "conv3d_tc_wgrad: at most 4 planar x sources");
    for (int i = 0; i < nplanar_x; ++i) { a.xf[i] = xf[i]; a.xf_bs[i] = xf_bs[i]; }
    a.nplanar_x = nplanar_x;
    Cin = 8;
  } else {
    VXM_REQUIRE(Ca % 8 == 0 && Cb % 8 == 0 && Ca + Cb >= 8 && Ca + Cb <= 64, "conv3d_tc_wgrad: channel counts (%d,%d) unsupported", Ca, Cb);
    VXM_REQUIRE((Ca == 0 || xa) && (Cb == 0 || xb), "conv3d_tc_wgrad: missing source tensor");
    Cin = Ca + Cb;
  }
  VXM_REQUIRE(Cin_real <= Cin && Cin_real > 0, "conv3d_tc_wgrad: Cin_real out of range");
  if (nplanar_g > 0) {
    VXM_REQUIRE(nplanar_g <= 4 && gf && gf_bs, "conv3d_tc_wgrad: at most 4 planar gz sources");
    for (int i = 0; i < nplanar_g; ++i) { a.gf[i] = gf[i]; a.gf_bs[i] = gf_bs[i]; }
    a.nplanar_g = nplanar_g;
    Cg = 8;
  } else {
    VXM_REQUIRE(gz && Cg % 8 == 0 && Cg >= 8 && Cg <= 32, "conv3d_tc_wgrad: gz channels %d unsupported", Cg);
  }
  VXM_REQUIRE(Cout_real > 0 && Cout_real <= Cg, "conv3d_tc_wgrad: Cout_real out of range");
  if (nplanar_x == 0 && nplanar_g == 0 && tcw::wgrad2_supported(Ca, Cb, Cg)) {
    // one launch per source tensor of the (virtual) concatenation: xa -> weights [0, Ca), xb -> [Ca, Ca + Cb), then one
    // reduction of both.  Their partials, 2 x (256 x kd x 9 x 32 x 32 + 256 x 32) floats + 2 x 255 bytes of rounding at
    // most, fit the 256 x kd x 9 x 64 x 32 + 1024 x 32 floats of vxm_conv3d_tc_wgrad_workspace_bytes(kd).
    cudaStream_t st2 = as_stream(stream);
    tcw::ReduceDesc d[2];
    int n = 0;
    size_t used = 0, used_b = 0;
    if (Ca) {
      const int cnt = Cin_real < Ca ? Cin_real : Ca;
      int rc = tcw::wgrad2_launch(xa, Ca, up, gz, Cg, grad_w, grad_b, work, B, D, H, W, kd, Cout_real, Cin_real, 0, cnt, accumulate, st2,
                                  &d[n++], &used, false, 0, 0, 0);
      if (rc) return rc;
    }
    if (Cb && Cin_real > Ca) {
      const int cnt = Cin_real - Ca < Cb ? Cin_real - Ca : Cb;
      int rc = tcw::wgrad2_launch(xb, Cb, 0, gz, Cg, grad_w, Ca ? nullptr : grad_b, (char*)work + used, B, D, H, W, kd, Cout_real, Cin_real, Ca,
                                  cnt, accumulate, st2, &d[n++], &used_b, false, 0, 0, 0);
      if (rc) return rc;
    }
    return tcw::wgrad2_reduce(d, n, st2);
  }
  a.xa = (const __nv_bfloat16*)xa; a.xb = (const __nv_bfloat16*)xb; a.gz = (const __nv_bfloat16*)gz;
  a.Ca = Ca; a.Cb = Cb; a.up = up; a.upd = (up && kd == 3) ? 1 : 0; a.Cg = Cg;
  a.B = B; a.D = D; a.H = H; a.W = W; a.KD = kd; a.NP = wgrad_np(Cg);
  VXM_REQUIRE(a.NP == Cg, "conv3d_tc_wgrad: gz channels must be 8, 16 or 32");
  a.tiles_h = (H + WTH - 1) / WTH; a.tiles_w = (W + WTW - 1) / WTW;
  int nsm = sm_count();
  int dchunk = D;
  auto items = [&](int dc) { return (long long)B * a.tiles_h * a.tiles_w * ((D + dc - 1) / dc); };
  while (items(dchunk) < 4LL * nsm && dchunk > 8) dchunk = (dchunk + 1) / 2;
  a.dchunk = dchunk; a.nchunks = (D + dchunk - 1) / dchunk;
  a.nitems = (int)items(dchunk);
  int grid = a.nitems < nsm ? a.nitems : nsm;
  if (grid > 256) grid = 256;
  a.partial = (float*)work;
  a.bias_partial = (float*)work + (size_t)256 * kd * 9 * 64 * 32;
  int nc8 = nplanar_x > 0 ? 1 : Cin / 8, ncg = nplanar_g > 0 ? 1 : Cg / 8;
  VXM_REQUIRE(nc8 * WROWS <= WKMAX * WNLOADER && ncg * 128 <= 4 * WNLOADER, "conv3d_tc_wgrad: tile too large for the loader table");
  size_t fixed = 16 * WPLANE + (size_t)WNG * ncg * GPLANE + 4 * GPLANE + 512;
  int nslot = (int)((200 * 1024 - fixed) / ((size_t)nc8 * WPLANE));
  if (nslot > WMAXSLOT) nslot = WMAXSLOT;
  VXM_REQUIRE(nslot >= 4, "conv3d_tc_wgrad: not enough shared memory for the slab ring");
  a.nslot = nslot;
  size_t smem = fixed + (size_t)nslot * nc8 * WPLANE;
  cudaStream_t st = as_stream(stream);
  const dim3 grid2(grid, kd);
#define VXM_WG_LAUNCH(KD_, NP_)                                                                                        \
  do {                                                                                                                 \
    VXM_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<KD_, NP_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    wgrad_tc_kernel<KD_, NP_><<<grid2, WNTHREADS, smem, st>>>(a);                                                       \
  } while (0)
#define VXM_WG_NP(KD_)                                                                                            \
  do { if (a.NP == 8) VXM_WG_LAUNCH(KD_, 8); else if (a.NP == 16) VXM_WG_LAUNCH(KD_, 16); else VXM_WG_LAUNCH(KD_, 32); } while (0)
  if (kd == 3) VXM_WG_NP(3);
  else VXM_WG_NP(1);
  int rc = check_launch("conv3d_tc_wgrad");
  if (rc) return rc;
  int T = kd * 9;
  int per_cta = T * 64 * a.NP;
  wgrad_reduce_kernel<<<(per_cta + 255) / 256, 256, 0, st>>>(a.partial, grad_w, grid, T, a.NP, Cout_real, Cin_real, a.bias_partial, grad_b,
                                                             accumulate);
  return check_launch("conv3d_tc_wgrad_reduce");
}
