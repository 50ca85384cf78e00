// Conv3d k=3 s=1 p=1 as an implicit GEMM on the Hopper tensor cores (wgmma.mma_async, accumulators in registers) —
// the one-MMA-per-tap engine behind reference voxelmorph/torch/networks.py:299-304 (ConvBlock) and :211,257 (flow head),
// kept as the tested baseline of the kw-stacked kernels (tc.conv_fwd).  Forward and dgrad share this kernel
// (dgrad = same convolution with swapped channel roles and flipped taps, see vxm_conv3d_tc_pack).
//
// Formulation (per output d-slice of a 16 x 8 (h x w) tile):
//     D[128 voxels x N=Cout] += A_tap[128 voxels x 16 ch] * W_tap[N x 16 ch]        27 taps x Cin/16 K-steps
//   * activations are bf16, channels-last (NDHWC); a halo'd slab of each input slice, (16+2) x (8+2) voxels,
//     is staged in shared memory as [Cin/8][180 rows][8 ch] = the wgmma "K-major, no swizzle" canonical
//     layout (core matrix = 8 voxels x 16 B).  In that layout a tap shift (kh, kw) is just a start-address
//     offset of (kh*10 + kw) * 16 bytes, so all 9 in-plane taps read the SAME staged slab, and the 3 kd taps
//     read the 3 resident slabs of a ring that slides along D: every input voxel is fetched from L2/HBM ~1.4x, not 27x.
//   * weights: bf16, pre-packed per (tap, K-step) into the canonical K-major layout; the whole filter bank
//     stays resident in shared memory, loaded once per CTA with bulk-TMA copies (cp.async.bulk + mbarrier tx).
//   * warp-specialised persistent CTA: warps 4-7 stage slabs with zero-filling cp.async (padding, nearest-x2
//     upsample and the channel concat with the skip tensor are all address arithmetic in the loader — the
//     48/64-channel concat tensor of networks.py:138 is never materialised); warpgroup 0 issues the wgmma chain of a
//     tile (two m64 halves), then drains its registers (one voxel's Cout channels per thread after a shared-memory
//     transpose), adds bias, applies LeakyReLU (or the dgrad mask) and writes 16-byte bf16 NDHWC vectors.
//     Pipeline: slab ring full/empty mbarriers (loader <-> MMA warpgroup).
#include <stdlib.h>

#include "tc_common.cuh"

namespace vxm {
namespace tc {

constexpr int TH = 16, TW = 8;
constexpr int SW = TW + 2, SH = TH + 2;
constexpr int ROWS = SH * SW;     // 180 voxels per channel-chunk plane
constexpr int PLANE = ROWS * 16;  // bytes
constexpr int MAXSLOT = 8, KMAX = 12;
constexpr int NLOADER = 128, NTHREADS = 256;   // warps 0-3: MMA + epilogue warpgroup, warps 4-7: loader

struct ConvTcArgs {
  const __nv_bfloat16* xa;    // bf16 NDHWC source A (B,Da,Ha,Wa,Ca); half resolution when up == 1
  const __nv_bfloat16* xb;    // bf16 NDHWC source B (B,D,H,W,Cb) or null
  const float* xf[4];         // planar fp32 sources (each (B,1,D,H,W)-like planes), nplanar of them, when Ca == 0
  long long xf_bstride[4];    // batch stride of each planar source in floats
  int nplanar;
  const __nv_bfloat16* wpk;   // packed weights
  const float* bias;
  void* out;
  void* out2;                 // optional second bf16 NDHWC output: channels [csplit, Cout) go there (dgrad of a concat layer)
  int csplit;
  const __nv_bfloat16* mask;  // optional bf16 NDHWC (B,D,H,W,Cout): out *= (mask < 0 ? slope : 1), no activation
  int B, D, H, W;
  int Ca, Cb, up, upd;
  int Cout, NP, KD, out_mode;
  float slope;
  int tiles_h, tiles_w, dchunk, nchunks, nitems, nslot;
  uint32_t wbytes;
};

template <int KD, int NK16, int NP>
__global__ void __launch_bounds__(NTHREADS, 1) conv_tc_kernel(const ConvTcArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const bool planar = a.nplanar > 0;
  // "half-K" inputs (8 real channels: the planar fp32 sources, or an 8-channel bf16 tensor): one staged plane;
  // the second 16-byte K chunk of the single K step reads a shared all-zero plane
  const bool halfk = planar || (a.Ca + a.Cb == 8);
  const int Cin = NK16 * 16;
  const int nc8 = halfk ? 1 : Cin / 8;
  const uint32_t slab_bytes = (uint32_t)nc8 * PLANE;
  uint8_t* s_w = smem;
  uint8_t* s_slab = smem + ((a.wbytes + 127u) & ~127u);
  const int NSLOT = a.nslot;
  uint8_t* s_zero = s_slab + NSLOT * slab_bytes;   // one all-zero plane (only used in planar mode)
  float* s_stage = reinterpret_cast<float*>(s_zero + PLANE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stage + ACC_STAGE_FLOATS);
  uint64_t* full = bars;
  uint64_t* empty = bars + MAXSLOT;
  uint64_t* wbar = empty + MAXSLOT;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < NSLOT; ++i) { mbar_init(&full[i], NLOADER); mbar_init(&empty[i], 4); }   // one arrival per MMA warp
    mbar_init(wbar, 1);
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < PLANE / 16; i += NTHREADS) reinterpret_cast<uint4*>(s_zero)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  if (threadIdx.x == 0) {  // weights: bulk TMA copies, one mbarrier transaction
    mbar_expect_tx(wbar, a.wbytes);
    for (uint32_t off = 0; off < a.wbytes; off += 16384u) {
      uint32_t n = a.wbytes - off < 16384u ? a.wbytes - off : 16384u;
      bulk_g2s(s_w + off, reinterpret_cast<const uint8_t*>(a.wpk) + off, n, wbar);
    }
  }

  const int HW_tiles = a.tiles_h * a.tiles_w;

  if (warp >= 4) {
    // ================================ LOADER (128 threads) ================================
    // Runs ahead of the tensor core by (nslot - 3) slabs.  cp.async completion is reported straight to the
    // slab's "full" mbarrier (cp.async.mbarrier.arrive.noinc), so issuing slab s+1 never waits for slab s.
    const int lt = threadIdx.x - 4 * 32;
    uint32_t cnt = 0;
    const int Da = a.upd ? a.D >> 1 : a.D, Ha = a.up ? a.H >> 1 : a.H, Wa = a.up ? a.W >> 1 : a.W;
    const int nca8 = a.Ca >> 3;
    const int nchunk = nc8 * ROWS;
    for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
      const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
      const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
      const int h0 = ht * TH, w0 = wt * TW, d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, a.D);
      const int s_begin = KD == 3 ? d0 - 1 : d0, s_end = KD == 3 ? d1 + 1 : d1;
      // per-item address table of this thread's 16-byte chunks: (source offset within a slice | source select), smem offset
      int soff[KMAX];
      uint32_t doff[KMAX];
      if (!planar) {
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
          const int id = lt + k * NLOADER;
          soff[k] = -1;
          doff[k] = 0;
          if (id < nchunk) {
            const int c8 = id % nc8, row = id / nc8;
            const int r = row / SW, c = row - r * SW;
            const int h = h0 - 1 + r, w = w0 - 1 + c;
            doff[k] = (uint32_t)c8 * PLANE + (uint32_t)row * 16u;
            if (h >= 0 && h < a.H && w >= 0 && w < a.W) {
              if (c8 < nca8) soff[k] = (((a.up ? h >> 1 : h) * Wa + (a.up ? w >> 1 : w)) * a.Ca + c8 * 8) << 1;
              else soff[k] = (((h * a.W + w) * a.Cb + (c8 - nca8) * 8) << 1) | 1;
            }
          }
        }
      }
      for (int ds = s_begin; ds < s_end; ++ds) {
        const int slot = cnt % NSLOT;
        mbar_wait(&empty[slot], ((cnt / NSLOT) & 1) ^ 1);
        uint8_t* slab = s_slab + (size_t)slot * slab_bytes;
        const bool dok = ds >= 0 && ds < a.D;
        if (!planar) {
          const __nv_bfloat16* baseA = a.xa ? a.xa + (((size_t)b * Da + (dok ? (a.upd ? ds >> 1 : ds) : 0)) * Ha * Wa) * a.Ca : nullptr;
          const __nv_bfloat16* baseB = a.xb ? a.xb + (((size_t)b * a.D + (dok ? ds : 0)) * a.H * a.W) * a.Cb : nullptr;
          const __nv_bfloat16* dummy = a.xa ? a.xa : a.xb;
#pragma unroll
          for (int k = 0; k < KMAX; ++k) {
            if (lt + k * NLOADER < nchunk) {
              const bool ok = dok && soff[k] >= 0;
              const __nv_bfloat16* src = ok ? ((soff[k] & 1) ? baseB : baseA) + (soff[k] >> 1) : dummy;
              cp_async16(slab + doff[k], src, ok ? 16u : 0u);
            }
          }
          cp_async_arrive_noinc(&full[slot]);
        } else {
          // planar fp32 sources -> channels 0..nplanar-1 of the first 16-byte chunk (rest zero)
          for (int row = lt; row < ROWS; row += NLOADER) {
            const int r = row / SW, c = row - r * SW;
            const int h = h0 - 1 + r, w = w0 - 1 + c;
            const bool ok = dok && h >= 0 && h < a.H && w >= 0 && w < a.W;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            if (ok) {
              const size_t off = ((size_t)ds * a.H + h) * a.W + w;
              for (int p = 0; p < a.nplanar; ++p) v[p] = __ldg(a.xf[p] + (size_t)b * a.xf_bstride[p] + off);
            }
            uint4 q = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), 0u, 0u);
            *reinterpret_cast<uint4*>(slab + row * 16) = q;
          }
          fence_proxy_async();   // generic-proxy stores -> visible to the tensor core (async proxy)
          mbar_arrive(&full[slot]);
        }
        ++cnt;
      }
    }
  } else {
    // ================================ MMA + EPILOGUE (warpgroup 0) ================================
    // The warpgroup issues the wgmma chain of a tile (two m64 halves: tile rows 0-63 / 64-127), releases the oldest
    // slab of the window once the chain has completed, then drains its accumulators: one voxel's Cout channels per
    // thread, bias, LeakyReLU (or the dgrad mask), 16-byte bf16 NDHWC vectors.
    const uint32_t slab_u32 = smem_u32(s_slab), w_u32 = smem_u32(s_w);
    const uint32_t a_lbo = halfk ? (smem_u32(s_zero) - slab_u32) : (uint32_t)PLANE;
    constexpr uint32_t b_tile16 = (uint32_t)NP * 32u / 16u;
    constexpr uint32_t half16 = 8u * SW;          // rows 64-127: 8 groups of 8 rows further, in 16-byte units
    mbar_wait(wbar, 0);
    const uint64_t bdesc0 = make_desc_kmajor_noswz(w_u32, (uint32_t)NP * 16u, 128u);
    uint32_t cnt_base = 0;
    const int row = warp * 32 + lane;
    const int rh = row >> 3, rw = row & 7;
    const size_t HW = (size_t)a.H * a.W;
    for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
      const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
      const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
      const int h = ht * TH + rh, w = wt * TW + rw, d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, a.D);
      const int nd = d1 - d0;
      const bool inside = h < a.H && w < a.W;
      for (int j = 0; j < nd; ++j) {
        const int d = d0 + j;
        if (KD == 3) {
          if (j == 0) {
            for (int q = 0; q < 2; ++q) { uint32_t c = cnt_base + q; mbar_wait(&full[c % NSLOT], (c / NSLOT) & 1); }
          }
          uint32_t c = cnt_base + j + 2;
          mbar_wait(&full[c % NSLOT], (c / NSLOT) & 1);
        } else {
          uint32_t c = cnt_base + j;
          mbar_wait(&full[c % NSLOT], (c / NSLOT) & 1);
        }
        uint64_t adesc_kd[KD];
#pragma unroll
        for (int kd = 0; kd < KD; ++kd) {
          const uint32_t sl = (cnt_base + j + kd) % NSLOT;
          // planar mode: the second K chunk (channels 8..15) reads the shared all-zero plane
          adesc_kd[kd] = make_desc_kmajor_noswz(slab_u32 + sl * slab_bytes, halfk ? (a_lbo - sl * slab_bytes) : a_lbo, (uint32_t)SW * 16u);
        }
        float acc0[NP / 2], acc1[NP / 2];
        wg_fence();
#pragma unroll
        for (int kd = 0; kd < KD; ++kd) {
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) {
#pragma unroll
              for (int k = 0; k < NK16; ++k) {
                const int tap = (kd * 3 + kh) * 3 + kw;
                // start-address field is in 16-byte units: tap shift (kh*SW + kw) rows, K step = 2 planes
                const uint64_t adesc = adesc_kd[kd] + (uint64_t)(kh * SW + kw + k * (2 * PLANE / 16));
                const uint64_t bdesc = bdesc0 + (uint64_t)((tap * NK16 + k) * b_tile16);
                const uint32_t accum = (kd | kh | kw | k) ? 1u : 0u;
                Wgmma<NP, 0, 0>::mma(acc0, adesc, bdesc, accum);
                Wgmma<NP, 0, 0>::mma(acc1, adesc + half16, bdesc, accum);
              }
            }
          }
        }
        wg_commit();
        wg_wait<0>();
        if (lane == 0) mbar_arrive(&empty[(cnt_base + j) % NSLOT]);   // oldest slab of the window is no longer needed
        uint32_t r[NP];
        acc_row16(acc0, acc1, 0, s_stage, 1, r);
        if constexpr (NP > 16) acc_row16(acc0, acc1, 16, s_stage, 1, r + 16);
        if constexpr (NP > 32) acc_row16(acc0, acc1, 32, s_stage, 1, r + 32);
        if constexpr (NP > 48) acc_row16(acc0, acc1, 48, s_stage, 1, r + 48);
        if (!inside) continue;
        const size_t vox = (((size_t)b * a.D + d) * a.H + h) * a.W + w;
        if (a.out_mode == 0) {
          const int c1 = a.out2 ? a.csplit : a.Cout;          // channels [0,c1) -> out, [c1,Cout) -> out2
          __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(a.out) + vox * c1;
          __nv_bfloat16* o2 = a.out2 ? reinterpret_cast<__nv_bfloat16*>(a.out2) + vox * (a.Cout - c1) - c1 : nullptr;
          const __nv_bfloat16* mk = a.mask ? a.mask + vox * a.Cout : nullptr;
#pragma unroll
          for (int c0 = 0; c0 < NP; c0 += 8) {
            if (c0 < a.Cout) {
              float v[8];
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                float x = __uint_as_float(r[c0 + e]);
                if (a.bias) x += __ldg(a.bias + c0 + e);
                v[e] = x;
              }
              if (mk) {
                uint4 m4 = *reinterpret_cast<const uint4*>(mk + c0);
                const __nv_bfloat16* mb = reinterpret_cast<const __nv_bfloat16*>(&m4);
#pragma unroll
                for (int e = 0; e < 8; ++e) if (__bfloat162float(mb[e]) < 0.f) v[e] *= a.slope;
              } else if (a.slope >= 0.f) {
#pragma unroll
                for (int e = 0; e < 8; ++e) v[e] = v[e] >= 0.f ? v[e] : v[e] * a.slope;
              }
              uint4 q = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
              *reinterpret_cast<uint4*>((c0 < c1 ? o : o2) + c0) = q;
            }
          }
        } else {
          float* o = reinterpret_cast<float*>(a.out);
#pragma unroll
          for (int c = 0; c < NP; ++c) {
            if (c < a.Cout) {
              float x = __uint_as_float(r[c]);
              if (a.bias) x += __ldg(a.bias + c);
              if (a.slope >= 0.f) x = x >= 0.f ? x : x * a.slope;
              o[(((size_t)b * a.Cout + c) * a.D + d) * HW + (size_t)h * a.W + w] = x;
            }
          }
        }
      }
      if (KD == 3) {
        if (lane == 0) {
          mbar_arrive(&empty[(cnt_base + nd) % NSLOT]);
          mbar_arrive(&empty[(cnt_base + nd + 1) % NSLOT]);
        }
        cnt_base += nd + 2;
      } else {
        cnt_base += nd;
      }
    }
  }
}

// Weight packing: fp32 (Cout, Cin, KD, 3, 3) -> bf16 [tap][k16][2][NP][8]  (canonical K-major, no swizzle).
// transposed == 1 packs the dgrad operator: input channels = Cout, outputs = Cin, taps flipped.
__global__ void pack_weights_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int Cout, int Cin, int T,
                                    int NP, int K16, int transposed) {
  const int total = T * K16 * 2 * NP * 8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int e = i & 7, n = (i >> 3) % NP, kc = (i / (8 * NP)) & 1, k16 = (i / (16 * NP)) % K16, tap = i / (16 * NP * K16);
    int ci = k16 * 16 + kc * 8 + e;
    float v = 0.f;
    if (!transposed) {
      if (n < Cout && ci < Cin) v = w[((size_t)n * Cin + ci) * T + tap];
    } else {
      if (n < Cin && ci < Cout) v = w[((size_t)ci * Cin + n) * T + (T - 1 - tap)];
    }
    out[i] = __float2bfloat16_rn(v);
  }
}

}  // namespace tc
}  // namespace vxm

using namespace vxm;
using namespace vxm::tc;

extern "C" size_t vxm_conv3d_tc_packed_bytes(int cin_eff, int np, int kd) {
  int k16 = (cin_eff + 15) / 16;
  return (size_t)kd * 9 * k16 * 2 * np * 8 * sizeof(__nv_bfloat16);
}

extern "C" int vxm_conv3d_tc_pack(const float* w, void* wpk, int Cout, int Cin, int kd, int np, int transposed, void* stream) {
  VXM_REQUIRE(w && wpk && Cout > 0 && Cin > 0 && (kd == 1 || kd == 3) && np % 16 == 0 && np <= 64, "conv3d_tc_pack: bad argument");
  int cin_eff = transposed ? Cout : Cin, nout = transposed ? Cin : Cout;
  VXM_REQUIRE(nout <= np, "conv3d_tc_pack: %d output channels do not fit N=%d", nout, np);
  int K16 = (cin_eff + 15) / 16, T = kd * 9;
  int total = T * K16 * 2 * np * 8;
  pack_weights_kernel<<<(total + 255) / 256, 256, 0, as_stream(stream)>>>(w, (__nv_bfloat16*)wpk, Cout, Cin, T, np, K16, transposed);
  return check_launch("conv3d_tc_pack");
}

extern "C" int vxm_conv3d_tc_fwd(const void* xa, const void* xb, const float* const* xf, const long long* xf_bstride, int nplanar,
                                 const void* wpk, const float* bias, void* out, const void* mask, int B, int D, int H, int W,
                                 int Ca, int Cb, int up, int Cout, int np, int kd, int out_mode, float slope, void* out2, int csplit,
                                 void* stream) {
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0 && wpk && out, "conv3d_tc_fwd: bad argument");
  VXM_REQUIRE(kd == 1 || kd == 3, "conv3d_tc_fwd: kd must be 1 or 3");
  VXM_REQUIRE(np == 16 || np == 32 || np == 48 || np == 64, "conv3d_tc_fwd: N must be 16, 32, 48 or 64");
  VXM_REQUIRE(Cout > 0 && Cout <= np && (out_mode == 1 || Cout % 8 == 0), "conv3d_tc_fwd: unsupported Cout %d", Cout);
  ConvTcArgs a{};
  int Cin;
  if (nplanar > 0) {
    VXM_REQUIRE(nplanar <= 4 && xf && xf_bstride, "conv3d_tc_fwd: at most 4 planar fp32 sources");
    for (int i = 0; i < nplanar; ++i) { a.xf[i] = xf[i]; a.xf_bstride[i] = xf_bstride[i]; }
    a.nplanar = nplanar;
    Cin = 16;
  } else {
    VXM_REQUIRE(xa || xb, "conv3d_tc_fwd: no input");
    VXM_REQUIRE(Ca % 8 == 0 && Cb % 8 == 0 && ((Ca + Cb) % 16 == 0 || Ca + Cb == 8) && Ca + Cb >= 8 && Ca + Cb <= 64,
                "conv3d_tc_fwd: channel counts (%d,%d) unsupported", Ca, Cb);
    VXM_REQUIRE((Ca == 0 || xa) && (Cb == 0 || xb), "conv3d_tc_fwd: missing source tensor");
    VXM_REQUIRE(!up || (H % 2 == 0 && W % 2 == 0 && (kd == 1 || D % 2 == 0)), "conv3d_tc_fwd: upsampled source needs even sizes");
    Cin = Ca + Cb == 8 ? 16 : Ca + Cb;
  }
  a.xa = (const __nv_bfloat16*)xa; a.xb = (const __nv_bfloat16*)xb; a.wpk = (const __nv_bfloat16*)wpk; a.bias = bias;
  a.out = out; a.mask = (const __nv_bfloat16*)mask;
  a.out2 = out2; a.csplit = csplit;
  VXM_REQUIRE(!out2 || (out_mode == 0 && csplit > 0 && csplit < Cout && csplit % 8 == 0 && !mask), "conv3d_tc_fwd: bad output split");
  a.B = B; a.D = D; a.H = H; a.W = W; a.Ca = Ca; a.Cb = Cb; a.up = up; a.upd = (up && kd == 3) ? 1 : 0;
  a.Cout = Cout; a.NP = np; a.KD = kd; a.out_mode = out_mode; a.slope = slope;
  a.tiles_h = (H + TH - 1) / TH; a.tiles_w = (W + TW - 1) / TW;
  int nsm = sm_count();
  int dchunk = D;
  auto items = [&](int dc) { return (long long)B * a.tiles_h * a.tiles_w * ((D + dc - 1) / dc); };
  while (items(dchunk) < 4LL * nsm && dchunk > 8) dchunk = (dchunk + 1) / 2;
  a.dchunk = dchunk; a.nchunks = (D + dchunk - 1) / dchunk;
  long long ni = items(dchunk);
  VXM_REQUIRE(ni < (1LL << 31), "conv3d_tc_fwd: too many tiles");
  a.nitems = (int)ni;
  a.wbytes = (uint32_t)vxm_conv3d_tc_packed_bytes(Cin, np, kd);   // Cin is rounded up to the K step (16)
  int nc8 = (nplanar > 0 || Ca + Cb == 8) ? 1 : Cin / 8;
  VXM_REQUIRE(nc8 * ROWS <= KMAX * NLOADER, "conv3d_tc_fwd: slab too large for the loader table");
  size_t fixed = ((a.wbytes + 127u) & ~127u) + PLANE + ACC_STAGE_FLOATS * sizeof(float) + 256;
  int nslot = (int)((227 * 1024 - fixed) / ((size_t)nc8 * PLANE));
  if (nslot > MAXSLOT) nslot = MAXSLOT;
  VXM_REQUIRE(nslot >= 4, "conv3d_tc_fwd: not enough shared memory for the slab ring");
  a.nslot = nslot;
  size_t smem = fixed + (size_t)nslot * nc8 * PLANE;
  int grid = a.nitems < nsm ? a.nitems : nsm;
  int nk16 = Cin / 16;
  cudaStream_t st = as_stream(stream);
#define VXM_TC_LAUNCH(KD_, NK_, NP_)                                                                                   \
  do {                                                                                                                 \
    VXM_CUDA(cudaFuncSetAttribute(conv_tc_kernel<KD_, NK_, NP_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    conv_tc_kernel<KD_, NK_, NP_><<<grid, NTHREADS, smem, st>>>(a);                                                     \
  } while (0)
#define VXM_TC_NK(KD_, NP_)                                                    \
  switch (nk16) {                                                              \
    case 1: VXM_TC_LAUNCH(KD_, 1, NP_); break;                                 \
    case 2: VXM_TC_LAUNCH(KD_, 2, NP_); break;                                 \
    case 3: VXM_TC_LAUNCH(KD_, 3, NP_); break;                                 \
    default: VXM_TC_LAUNCH(KD_, 4, NP_); break;                                \
  }
  if (kd == 3) { if (np == 16) { VXM_TC_NK(3, 16) } else if (np == 32) { VXM_TC_NK(3, 32) } else if (np == 48) { VXM_TC_NK(3, 48) } else { VXM_TC_NK(3, 64) } }
  else { if (np == 16) { VXM_TC_NK(1, 16) } else if (np == 32) { VXM_TC_NK(1, 32) } else if (np == 48) { VXM_TC_NK(1, 48) } else { VXM_TC_NK(1, 64) } }
  return check_launch("conv3d_tc_fwd");
}
