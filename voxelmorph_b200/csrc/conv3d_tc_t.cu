// Conv3d k=3 on the Hopper tensor cores (wgmma), "kw-stacked" formulation with SWIZZLE_NONE operands
// (reference voxelmorph/torch/networks.py:299-304, :211,257; forward and dgrad).
//
// conv3d_tc.cu issues one 128 x Cout x 16 MMA per (tap, 16 channels) and re-reads its activation operand 27 times.
// Here the three kw taps are stacked along the MMA N dimension:
//     D[128 voxels][(kw, co) : N = 3*Cout] += X_(kd,kh)[128 voxels][16 ch] * Wt[(kw,co)][16 ch]
//   * the K loop runs over (kd, kh, Cin/16) only: 9*Cin/16 MMAs of N = 96 (48) per tile instead of 27*Cin/16 of N = 32
//     (16): the activation operand is read 9 times instead of 27 (layers wider than 32 output channels run in passes of
//     16 channels, one wgmma per kw, to keep the accumulators within the register budget);
//   * the 128 M rows are 4 (h) x 32 (w') voxels of one d-slice; the slab [Cin/8][6 x 32 rows][8 ch] has a row pitch of
//     32 voxels, so a (kd, kh) tap is a whole-row (512-byte) shift of the A operand start address;
//   * after the accumulators are transposed to one voxel per thread, each epilogue warp owns one 32-voxel row and the
//     kw shift is a warp shuffle: out[w'][co] = D[w'-1][(0,co)] + D[w'][(1,co)] + D[w'+1][(2,co)]; lanes 0 and 31 are
//     halo (30 useful outputs per row);
//   * two MMA + epilogue warpgroups take alternate tiles; everything else (persistent warp-specialised CTA, cp.async
//     loader with fused upsample / concat / zero padding, bulk-TMA weight load, slab ring sliding along D) is as in
//     conv3d_tc.cu.
#include "tc_common.cuh"

namespace vxm {
namespace tct {

using namespace vxm::tc;

constexpr int HT = 4, WT = 32, WUSE = 30;
constexpr int SROWS = (HT + 2) * WT;   // 192 voxels per slab plane
constexpr int TPLANE = SROWS * 16;     // 3072 bytes
constexpr int MAXSLOT = 8, KMAX = 12;
constexpr int NLOADER = 128, NTHREADS = 384;   // warps 0-3 / 4-7: MMA + epilogue groups 0 / 1, warps 8-11: loader

struct ConvTArgs {
  const __nv_bfloat16* xa; const __nv_bfloat16* xb;
  const __nv_bfloat16* wpk; const float* bias;
  void* out; const __nv_bfloat16* mask;
  void* out2; int csplit;   // optional second bf16 output: channels [csplit, Cout) (single-pass dgrad of a concat layer)
  int B, D, H, W, Ca, Cb, up, upd, Cout, out_mode;
  float slope;
  int tiles_h, tiles_w, dchunk, nchunks, nitems, nslot;
  uint32_t wbytes;
};

template <int KD, int NK16, int COUT>
__global__ void __launch_bounds__(NTHREADS, 1) conv_tct_kernel(const ConvTArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const bool halfk = (a.Ca + a.Cb == 8);
  const int nc8 = halfk ? 1 : NK16 * 2;
  const uint32_t slab_bytes = (uint32_t)nc8 * TPLANE;
  const int NSLOT = a.nslot;
  uint8_t* s_w = smem;
  uint8_t* s_slab = smem + ((a.wbytes + 127u) & ~127u);
  uint8_t* s_zero = s_slab + NSLOT * slab_bytes;
  float* s_stage = reinterpret_cast<float*>(s_zero + TPLANE);   // one accumulator read-out buffer per group
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stage + 2 * ACC_STAGE_FLOATS);
  uint64_t* full = bars;
  uint64_t* empty = bars + MAXSLOT;
  uint64_t* wbar = empty + MAXSLOT;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    // empty: one arrival per warp of both groups (each group releases every slab once, see below)
    for (int i = 0; i < NSLOT; ++i) { mbar_init(&full[i], NLOADER); mbar_init(&empty[i], 8); }
    mbar_init(wbar, 1);
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < TPLANE / 16; i += NTHREADS) reinterpret_cast<uint4*>(s_zero)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  if (threadIdx.x == 0) {
    mbar_expect_tx(wbar, a.wbytes);
    for (uint32_t off = 0; off < a.wbytes; off += 16384u) {
      uint32_t n = a.wbytes - off < 16384u ? a.wbytes - off : 16384u;
      bulk_g2s(s_w + off, reinterpret_cast<const uint8_t*>(a.wpk) + off, n, wbar);
    }
  }
  const int HW_tiles = a.tiles_h * a.tiles_w;

  if (warp >= 8) {
    // ================================ LOADER (128 threads) ================================
    setmaxnreg_dec<64>();
    const int lt = threadIdx.x - 8 * 32;
    uint32_t cnt = 0;
    const int Da = a.upd ? a.D >> 1 : a.D, Ha = a.up ? a.H >> 1 : a.H, Wa = a.up ? a.W >> 1 : a.W;
    const int nca8 = a.Ca >> 3;
    const int nchunk = nc8 * SROWS;
    for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
      const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
      const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
      const int h0 = ht * HT, w0 = wt * WUSE, d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, a.D);
      const int s_begin = KD == 3 ? d0 - 1 : d0, s_end = KD == 3 ? d1 + 1 : d1;
      int soff[KMAX];
      uint32_t doff[KMAX];
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        const int id = lt + k * NLOADER;
        soff[k] = -1;
        doff[k] = 0;
        if (id < nchunk) {
          const int c8 = id % nc8, row = id / nc8;
          const int r = row >> 5, c = row & 31;
          const int h = h0 - 1 + r, w = w0 - 1 + c;
          doff[k] = (uint32_t)c8 * TPLANE + (uint32_t)row * 16u;
          if (h >= 0 && h < a.H && w >= 0 && w < a.W) {
            if (c8 < nca8) soff[k] = (((a.up ? h >> 1 : h) * Wa + (a.up ? w >> 1 : w)) * a.Ca + c8 * 8) << 1;
            else soff[k] = (((h * a.W + w) * a.Cb + (c8 - nca8) * 8) << 1) | 1;
          }
        }
      }
      for (int ds = s_begin; ds < s_end; ++ds) {
        const int slot = cnt % NSLOT;
        mbar_wait(&empty[slot], ((cnt / NSLOT) & 1) ^ 1);
        uint8_t* slab = s_slab + (size_t)slot * slab_bytes;
        const bool dok = ds >= 0 && ds < a.D;
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
        ++cnt;
      }
    }
  } else {
    // ================================ MMA + EPILOGUE (2 warpgroups; warp = tile row hh, lane = w') ==================
    // Group g issues and drains the tiles with (tile counter & 1) == g, so the tensor core works on one group's tile
    // while the other group runs its epilogue (global-memory latencies of mask prefetch and stores).
    // Slab release: every group walks ALL slabs in order (waiting for each one's full phase) and arrives once on each
    // slab's empty barrier after its last MMA reading it has completed, so a slot is refilled only after both groups
    // are past it and no barrier phase can alias.
    setmaxnreg_inc<216>();
    const int grp = warp >> 2;
    const int wq = warp & 3;
    float* stage = s_stage + grp * ACC_STAGE_FLOATS;
    const int nbar = 1 + grp;
    // MMA N per wgmma: the three kw taps stacked (N = 3 * COUT) up to COUT = 32; wider layers run in passes of 16
    // output channels with one wgmma per kw (the accumulators of a pass stay within the register budget)
    constexpr bool STACK = COUT <= 32;
    constexpr int CW = STACK ? COUT : 16;            // output channels per pass
    constexpr int NPASS = COUT / CW;
    constexpr int NA = STACK ? 3 * COUT : CW;        // N of one wgmma
    constexpr int NW = STACK ? 1 : 3;                // wgmmas per K step and tile half
    const uint32_t slab_u32 = smem_u32(s_slab), w_u32 = smem_u32(s_w);
    const uint32_t a_lbo0 = halfk ? (smem_u32(s_zero) - slab_u32) : (uint32_t)TPLANE;
    constexpr uint32_t NN = 3 * COUT;
    constexpr uint32_t b_step16 = NN * 32u / 16u;
    constexpr uint32_t half16 = 2u * WT;             // rows 64-127: two slab rows further, in 16-byte units
    mbar_wait(wbar, 0);
    const uint64_t bdesc0 = make_desc_kmajor_noswz(w_u32, NN * 16u, 128u);
    uint32_t cnt_base = 0, tcnt = 0, wcur = 0;
    auto observe = [&](uint32_t upto) {              // wait for every slab up to global index `upto`, in order
      for (; wcur <= upto; ++wcur) mbar_wait(&full[wcur % NSLOT], (wcur / NSLOT) & 1);
    };
    const size_t HWp = (size_t)a.H * a.W;
    auto bias_at = [&](int c) -> float { return a.bias ? __ldg(a.bias + c) : 0.f; };
    for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
      const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
      const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
      const int h = ht * HT + wq, w = wt * WUSE - 1 + lane, d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, a.D);
      const int nd = d1 - d0;
      const bool valid = lane >= 1 && lane <= WUSE && h < a.H && w < a.W;
      for (int j = 0; j < nd; ++j, ++tcnt) {
        const int d = d0 + j;
        observe(cnt_base + (uint32_t)j + (KD == 3 ? 2u : 0u));
        if ((int)(tcnt & 1) == grp) {
          const size_t vox = (((size_t)b * a.D + d) * a.H + h) * a.W + w;
          // prefetch the LeakyReLU-derivative mask of this voxel before the MMAs
          uint4 mreg[COUT / 8];
          if (a.mask && valid) {
#pragma unroll
            for (int q = 0; q < COUT / 8; ++q)
              if (q * 8 < a.Cout) mreg[q] = __ldg(reinterpret_cast<const uint4*>(a.mask + vox * a.Cout) + q);
          }
          uint64_t adesc_kd[KD];
#pragma unroll
          for (int kd = 0; kd < KD; ++kd) {
            const uint32_t sl = (cnt_base + j + kd) % NSLOT;
            adesc_kd[kd] = make_desc_kmajor_noswz(slab_u32 + sl * slab_bytes, halfk ? (a_lbo0 - sl * slab_bytes) : a_lbo0, 128u);
          }
          const int c1 = a.out2 ? a.csplit : a.Cout;          // channels [0,c1) -> out, [c1,Cout) -> out2
#pragma unroll
          for (int pass = 0; pass < NPASS; ++pass) {
            float acc[2][NW][NA / 2];
            wg_fence();
#pragma unroll
            for (int kd = 0; kd < KD; ++kd) {
#pragma unroll
              for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
                for (int k = 0; k < NK16; ++k) {
                  const int step = (kd * 3 + kh) * NK16 + k;
                  const uint64_t adesc = adesc_kd[kd] + (uint64_t)(kh * WT + k * (2 * TPLANE / 16));   // 16-byte units
                  const uint64_t bdesc = bdesc0 + (uint64_t)(step * b_step16);
#pragma unroll
                  for (int g = 0; g < NW; ++g) {
                    // non-stacked: rows kw * COUT + pass * 16 of the packed weights (8-row groups 128 bytes apart)
                    const uint64_t bd = STACK ? bdesc : bdesc + (uint64_t)(((g * COUT + pass * CW) / 8) * 8);
#pragma unroll
                    for (int hf = 0; hf < 2; ++hf) Wgmma<NA, 0, 0>::mma(acc[hf][g], adesc + hf * half16, bd, step ? 1u : 0u);
                  }
                }
              }
            }
            wg_commit();
            wg_wait<0>();
            // 16 output channels at a time: the kw = 0, 1, 2 partial sums, shuffle-combined across lanes, stored
#pragma unroll
            for (int cc = 0; cc < CW; cc += 16) {
              const int c0 = pass * CW + cc;
              // one 16-column read-out at a time (register budget): out[w'] = P0[w'-1] + P1[w'] + P2[w'+1]
              uint32_t r[16];
              float v[16];
              acc_row16(acc[0][0], acc[1][0], STACK ? cc : 0, stage, nbar, r);
#pragma unroll
              for (int c = 0; c < 16; ++c) v[c] = __shfl_up_sync(0xffffffffu, __uint_as_float(r[c]), 1);
              acc_row16(acc[0][NW > 1 ? 1 : 0], acc[1][NW > 1 ? 1 : 0], STACK ? COUT + cc : 0, stage, nbar, r);
#pragma unroll
              for (int c = 0; c < 16; ++c) v[c] += __uint_as_float(r[c]);
              acc_row16(acc[0][NW - 1], acc[1][NW - 1], STACK ? 2 * COUT + cc : 0, stage, nbar, r);
#pragma unroll
              for (int c = 0; c < 16; ++c) v[c] += __shfl_down_sync(0xffffffffu, __uint_as_float(r[c]), 1);
              if (valid && c0 < a.Cout) {
                if (a.out_mode == 0) {
#pragma unroll
                  for (int q = 0; q < 16; q += 8) {
                    if (c0 + q < a.Cout) {
                      float x[8];
#pragma unroll
                      for (int e = 0; e < 8; ++e) x[e] = v[q + e] + bias_at(c0 + q + e);
                      if (a.mask) {
                        const uint4 m4 = mreg[(c0 + q) / 8];
                        const __nv_bfloat16* mb = reinterpret_cast<const __nv_bfloat16*>(&m4);
#pragma unroll
                        for (int e = 0; e < 8; ++e) if (__bfloat162float(mb[e]) < 0.f) x[e] *= a.slope;
                      } else if (a.slope >= 0.f) {
#pragma unroll
                        for (int e = 0; e < 8; ++e) x[e] = x[e] >= 0.f ? x[e] : x[e] * a.slope;
                      }
                      // a split never falls inside a group of 8 channels (csplit % 8 == 0)
                      const int cg = c0 + q;
                      __nv_bfloat16* oo = cg < c1 ? reinterpret_cast<__nv_bfloat16*>(a.out) + vox * c1 + cg
                                                  : reinterpret_cast<__nv_bfloat16*>(a.out2) + vox * (a.Cout - c1) + (cg - c1);
                      *reinterpret_cast<uint4*>(oo) = make_uint4(pack_bf16x2(x[0], x[1]), pack_bf16x2(x[2], x[3]), pack_bf16x2(x[4], x[5]), pack_bf16x2(x[6], x[7]));
                    }
                  }
                } else {
                  float* o = reinterpret_cast<float*>(a.out);
#pragma unroll
                  for (int c = 0; c < 16; ++c) {
                    if (c0 + c < a.Cout) {
                      float x = v[c] + bias_at(c0 + c);
                      if (a.slope >= 0.f) x = x >= 0.f ? x : x * a.slope;
                      o[(((size_t)b * a.Cout + c0 + c) * a.D + d) * HWp + (size_t)h * a.W + w] = x;
                    }
                  }
                }
              }
            }
          }
        }
        if (lane == 0) mbar_arrive(&empty[(cnt_base + j) % NSLOT]);   // this group no longer reads slab j
      }
      if (KD == 3) {
        observe(cnt_base + (uint32_t)nd + 1u);
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

// fp32 (Cout, Cin, KD, 3, 3) -> bf16 [step = (kd*3+kh)*K16 + k16][2][N rows = kw*COUT + co][8]
__global__ void pack_weights_t_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int Cout, int Cin, int KD, int COUT,
                                      int M, int K16, int transposed) {
  const int T = KD * 9;
  const int total = KD * 3 * K16 * 2 * M * 8;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int e = i & 7, r = (i >> 3) % M, kc = (i / (8 * M)) & 1, k16 = (i / (16 * M)) % K16, st = i / (16 * M * K16);
    const int kd = st / 3, kh = st % 3, g = r / COUT, co = r % COUT;
    const int ci = k16 * 16 + kc * 8 + e;
    float v = 0.f;
    if (g < 3) {
      const int tap = (kd * 3 + kh) * 3 + g;
      if (!transposed) {
        if (co < Cout && ci < Cin) v = w[((size_t)co * Cin + ci) * T + tap];
      } else {
        if (co < Cin && ci < Cout) v = w[((size_t)ci * Cin + co) * T + (T - 1 - tap)];
      }
    }
    out[i] = __float2bfloat16_rn(v);
  }
}

}  // namespace tct
}  // namespace vxm

using namespace vxm;
using namespace vxm::tct;

static int tct_m(int coutp) { return 3 * coutp; }   // rows of the packed weight operand = MMA N

extern "C" size_t vxm_conv3d_tct_packed_bytes(int cin_eff, int coutp, int kd) {
  int k16 = (cin_eff + 15) / 16;
  return (size_t)kd * 3 * k16 * 2 * tct_m(coutp) * 8 * sizeof(__nv_bfloat16);
}

extern "C" int vxm_conv3d_tct_pack(const float* w, void* wpk, int Cout, int Cin, int kd, int coutp, int transposed, void* stream) {
  VXM_REQUIRE(w && wpk && Cout > 0 && Cin > 0 && (kd == 1 || kd == 3) && (coutp == 16 || coutp == 32 || coutp == 48 || coutp == 64), "conv3d_tct_pack: bad argument");
  int cin_eff = transposed ? Cout : Cin, nout = transposed ? Cin : Cout;
  VXM_REQUIRE(nout <= coutp, "conv3d_tct_pack: %d output channels do not fit %d", nout, coutp);
  int K16 = (cin_eff + 15) / 16, M = tct_m(coutp);
  int total = kd * 3 * K16 * 2 * M * 8;
  pack_weights_t_kernel<<<(total + 255) / 256, 256, 0, as_stream(stream)>>>(w, (__nv_bfloat16*)wpk, Cout, Cin, kd, coutp, M, K16, transposed);
  return check_launch("conv3d_tct_pack");
}

extern "C" int vxm_conv3d_tct_supported(int Ca, int Cb, int Cout) {
  int cin = Ca + Cb;
  return (Cout <= 64) && (cin == 8 || cin == 16 || cin == 32 || cin == 48 || cin == 64) && Ca % 8 == 0 && Cb % 8 == 0;
}

extern "C" int vxm_conv3d_tct_fwd(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, const void* mask,
                                  int B, int D, int H, int W, int Ca, int Cb, int up, int Cout, int coutp, int kd, int out_mode,
                                  float slope, void* out2, int csplit, void* stream) {
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0 && wpk && out, "conv3d_tct_fwd: bad argument");
  VXM_REQUIRE(kd == 1 || kd == 3, "conv3d_tct_fwd: kd must be 1 or 3");
  VXM_REQUIRE(coutp == 16 || coutp == 32 || coutp == 48 || coutp == 64, "conv3d_tct_fwd: padded Cout must be 16, 32, 48 or 64");
  VXM_REQUIRE(!out2 || (out_mode == 0 && csplit > 0 && csplit < Cout && csplit % 8 == 0 && !mask), "conv3d_tct_fwd: bad output split");
  VXM_REQUIRE(Cout > 0 && Cout <= coutp && (out_mode == 1 || Cout % 8 == 0), "conv3d_tct_fwd: unsupported Cout %d", Cout);
  VXM_REQUIRE(vxm_conv3d_tct_supported(Ca, Cb, Cout), "conv3d_tct_fwd: channel counts (%d,%d)->%d unsupported", Ca, Cb, Cout);
  VXM_REQUIRE((Ca == 0 || xa) && (Cb == 0 || xb), "conv3d_tct_fwd: missing source tensor");
  VXM_REQUIRE(!up || (H % 2 == 0 && W % 2 == 0 && (kd == 1 || D % 2 == 0)), "conv3d_tct_fwd: upsampled source needs even sizes");
  ConvTArgs a{};
  const int cin = Ca + Cb;
  const int nk16 = cin == 8 ? 1 : cin / 16;
  a.xa = (const __nv_bfloat16*)xa; a.xb = (const __nv_bfloat16*)xb; a.wpk = (const __nv_bfloat16*)wpk; a.bias = bias;
  a.out = out; a.mask = (const __nv_bfloat16*)mask; a.out2 = out2; a.csplit = csplit;
  a.B = B; a.D = D; a.H = H; a.W = W; a.Ca = Ca; a.Cb = Cb; a.up = up; a.upd = (up && kd == 3) ? 1 : 0;
  a.Cout = Cout; a.out_mode = out_mode; a.slope = slope;
  a.tiles_h = (H + HT - 1) / HT; a.tiles_w = (W + WUSE - 1) / WUSE;
  int nsm = sm_count();
  int dchunk = D;
  auto items = [&](int dc) { return (long long)B * a.tiles_h * a.tiles_w * ((D + dc - 1) / dc); };
  while (items(dchunk) < 4LL * nsm && dchunk > 8) dchunk = (dchunk + 1) / 2;
  a.dchunk = dchunk; a.nchunks = (D + dchunk - 1) / dchunk;
  a.nitems = (int)items(dchunk);
  a.wbytes = (uint32_t)vxm_conv3d_tct_packed_bytes(nk16 * 16, coutp, kd);
  const int nc8 = cin == 8 ? 1 : cin / 8;
  VXM_REQUIRE(nc8 * SROWS <= KMAX * NLOADER, "conv3d_tct_fwd: slab too large for the loader table");
  size_t fixed = ((a.wbytes + 127u) & ~127u) + TPLANE + 2 * ACC_STAGE_FLOATS * sizeof(float) + 512;
  int nslot = (int)((227 * 1024 - fixed) / ((size_t)nc8 * TPLANE));
  if (nslot > MAXSLOT) nslot = MAXSLOT;
  VXM_REQUIRE(nslot >= 4, "conv3d_tct_fwd: not enough shared memory for the slab ring");
  a.nslot = nslot;
  size_t smem = fixed + (size_t)nslot * nc8 * TPLANE;
  int grid = a.nitems < nsm ? a.nitems : nsm;
  cudaStream_t st = as_stream(stream);
#define VXM_TCT_LAUNCH(KD_, NK_, CO_)                                                                                   \
  do {                                                                                                                  \
    VXM_CUDA(cudaFuncSetAttribute(conv_tct_kernel<KD_, NK_, CO_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    conv_tct_kernel<KD_, NK_, CO_><<<grid, NTHREADS, smem, st>>>(a);                                                     \
  } while (0)
#define VXM_TCT_NK(KD_, CO_)                                \
  switch (nk16) {                                           \
    case 1: VXM_TCT_LAUNCH(KD_, 1, CO_); break;             \
    case 2: VXM_TCT_LAUNCH(KD_, 2, CO_); break;             \
    case 3: VXM_TCT_LAUNCH(KD_, 3, CO_); break;             \
    default: VXM_TCT_LAUNCH(KD_, 4, CO_); break;            \
  }
  if (kd == 3) { if (coutp == 16) { VXM_TCT_NK(3, 16) } else if (coutp == 32) { VXM_TCT_NK(3, 32) } else if (coutp == 48) { VXM_TCT_NK(3, 48) } else { VXM_TCT_NK(3, 64) } }
  else { if (coutp == 16) { VXM_TCT_NK(1, 16) } else if (coutp == 32) { VXM_TCT_NK(1, 32) } else if (coutp == 48) { VXM_TCT_NK(1, 48) } else { VXM_TCT_NK(1, 64) } }
  return check_launch("conv3d_tct_fwd");
}
