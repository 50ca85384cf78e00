// Conv3d k=3 on the Hopper tensor cores (wgmma), "kw-stacked" formulation with 128/64/32-byte SWIZZLED K-major operands.
//
// Same algorithm as conv3d_tc_t.cu (N = 3*Cout stacks the kw taps, K loop over (kd, kh, Cin/16), kw shift by warp
// shuffle in the epilogue), but the shared-memory operands use the wgmma swizzled canonical layouts instead of
// SWIZZLE_NONE: every slab row is one voxel with all channels of a channel group contiguous (32 / 64 / 128 bytes)
// and the 16-byte chunks of a row are XOR-swizzled with the row index (Swizzle<B,4,3>), which the cp.async loader
// applies to its destination addresses and the weight packer applies on the host side of the operand.  The input
// channels are split into at most two groups of 16 / 32 / 64 channels (48 = 32 + 16), each with its own slab region.
// A (kd, kh) tap shifts the A operand by whole 32-voxel rows (a multiple of the 8-row swizzle period), so the start
// address stays pattern-aligned and the descriptor base offset is 0.
#include <stdlib.h>
#include <string.h>

#include "tc_common.cuh"

namespace vxm {
namespace tcs {

using namespace vxm::tc;

constexpr int WT = 32, WUSE = 30;      // tile: HT (4 or 8) rows x 32 columns (30 written), slab = (HT + 2) x 32 voxel rows
constexpr int MAXSLOT = 16;
constexpr int NLOADER = 128, NTHREADS = 384, NGRP = 2;   // warps 0-3 / 4-7: MMA + epilogue groups 0 / 1, warps 8-11: loader

struct ConvSArgs {
  const __nv_bfloat16* xa; const __nv_bfloat16* xb;
  const __nv_bfloat16* wpk; const float* bias;
  void* out; const __nv_bfloat16* mask;
  void* out2; int csplit;   // optional second bf16 output: channels [csplit, Cout) (single-pass dgrad of a concat layer)
  // split-precision (bf16x3) passes: `acc_in` (fp32 channels-last, COUT channels per voxel) is added to the tile before the
  // epilogue; out_mode 2 stores the raw fp32 sums back in that layout (no bias / activation), out_mode 3 applies bias +
  // activation and stores the result as a bf16 (hi, lo) pair: hi -> out, lo = bf16(x - hi) -> out_lo
  int B, D, H, W, Ca, Cb, up, upd, Cout, out_mode;
  float slope;
  int tiles_h, tiles_w, dchunk, nchunks, nitems, nslot;
  uint32_t wbytes;
  const float* acc_in; void* out_lo;
  // TMA tile staging of the A operand: bit g of tma_mask = channel group g of every slab arrives as ONE tiled tensor copy
  // (cp.async.bulk.tensor.5d, box {G channels, 32 columns, HT + 2 rows}) of tensor map tm[g], starting at channel tc0[g];
  // zero padding is the copy's out-of-bounds fill.  Groups read through the nearest-neighbour upsampler (decoder concat
  // layers), the 64-channel group that interleaves two sources and the 8-plane image input stay on the cp.async loader.
  int tma_mask, tc0[2];
  // channel pitch of out / out_lo / mask in the OP kernels: one block of output channels of a wider tensor (the caller
  // offsets the pointers to the block's first channel); acc_in and the out_mode 2 sums stay dense (COUT per voxel)
  int opitch;
  alignas(64) CUtensorMap tm[2];
};

// byte offset inside a swizzled K-major tile whose rows are `width` bytes (32, 64 or 128): Swizzle<log2(width/16),4,3>
__host__ __device__ inline uint32_t swz(uint32_t off, uint32_t width) {
  return off ^ (((off >> 7) & (width / 16 - 1)) << 4);
}
__device__ __forceinline__ uint64_t make_desc_kmajor_swz(uint32_t saddr, uint32_t width) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;                                   // LBO: unused for K inside one swizzle atom
  d |= (uint64_t)(((8u * width) >> 4) & 0x3FFF) << 32;      // SBO: 8 rows
  return d | desc_swizzle(width);
}

__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// HT = 8: one slab step feeds TWO 4-row accumulators (one per epilogue group), halving the per-step issue / barrier
// overhead that bounds the thin layers and cutting the halo re-reads from 1.5x to 1.25x.
// ACC: the split-precision epilogue (acc_in / out_mode 2, 3) is compiled in; the plain kernels (ACC = false) keep the
// round-1 epilogue — with the extra live registers the 32-channel variants spilled and lost up to 1.8x.
// EPI: epilogue specialisation.  0 = generic run-time epilogue; 1 = forward (bias + LeakyReLU with
// 0 <= slope <= 1, bf16 channels-last, all COUT channels real); 2 = dgrad (LeakyReLU derivative from the saved activation);
// 3 = raw sums with an optional channel split at a multiple of 16 (single-pass dgrad of a concat layer); 4 = fp32 planar
// (B, Cout, D, H, W) output of the first a.Cout channels, optional bias, LeakyReLU iff slope >= 0 (the flow head, the
// image dgrad).  1, 2 and 4 exist for KD = 1 as well (kd-folded layers, 2-D models), for up to 32 outputs.
// OP: the bf16 outputs and the mask are one channel block of a wider tensor (pitch a.opitch, no out2); the channel-blocked
// execution of the layers whose weights do not fit shared memory in one piece (64 -> 64, 128 -> 64, ...).
// PD: polyphase forms of a layer that reads a nearest-x2 upsampled source (3-D, EPI != 0).  Along each axis the upsampled
// data has one value per pair of fine positions, so two of the three taps always read the same coarse voxel:
//   1 = forward: channel group 0 is the upsampled source.  An even output slice 2c reads slabs (2c - 1, 2c) with the merged
//       weights (W0, W1 + W2), an odd one 2c + 1 reads slabs (2c + 1, 2c + 2) with (W0 + W1, W2): 2 kd steps instead of 3
//       for that group.  Group 1 (the skip source) keeps its 3 kd steps.  The ring and the loader do not change.
//   2 = coarse dgrad (EPI 2, G1 = 0, HT 8): the gradient w.r.t. the coarse source itself.  The same algebra holds along d
//       and h: coarse slice c reads the 4 fine gradient slabs 2c - 1 .. 2c + 2 and coarse row q of a tile the 4 fine slab
//       rows 2q .. 2q + 3, with the transposed taps (T0, T0 + T1, T1 + T2, T2) along each of the two axes: 16 (kd, kh)
//       steps per coarse (d, h), against 2 x 2 x 9 over the fine ones.  The slab rows are staged parity-major (even rows
//       first), so that the rows 2q + k of the coarse rows q, q + 1 of an m64 block are adjacent; an 8-row tile is ONE
//       128-row event of 4 coarse rows, and the ring window advances by 2 slabs per coarse slice.  w stays fine (kw stacked
//       in N, as everywhere): the epilogue adds the w' pairs (2c, 2c + 1) across lanes, applies the LeakyReLU derivative of
//       the coarse activation (a.mask) and stores the coarse gradient.  Staged by cp.async only (no TMA box permutes rows).
template <int KD, int G0, int G1, int COUT, int HT, bool ACC, int EPI, bool OP = false, int PD = 0>
__global__ void __launch_bounds__(NTHREADS, 1) conv_tcs_kernel(const __grid_constant__ ConvSArgs a) {
  static_assert(PD == 0 || (KD == 3 && EPI != 0 && !ACC && !OP), "polyphase forms: 3-D, specialised epilogue");
  static_assert(PD != 1 || G1 > 0, "the polyphase forward merges channel group 0 and keeps group 1");
  static_assert(PD != 2 || (G1 == 0 && COUT == 32 && HT == 8 && EPI == 2), "the coarse dgrad: 32 -> 32 channels, 8-row tiles");
  static_assert(EPI != 4 || (PD == 0 && !ACC && !OP && COUT <= 32), "the fp32 planar epilogue drains in the fragment layout");
  static_assert(KD == 3 || EPI == 0 || (EPI != 3 && COUT <= 32), "KD = 1: fragment-layout epilogues 1, 2, 4 only");
  constexpr int SROWS = (HT + 2) * WT;
  constexpr int NH = PD == 2 ? 1 : HT / 4;                // tile events per slab step (PD 2: 4 coarse rows = 128 rows)
  constexpr int NEVEN = (HT + 3) / 2;                     // PD 2: even slab rows, staged first
  constexpr int W0 = G0 * 2, W1 = G1 * 2;                 // row bytes of the two channel groups
  constexpr int NC8 = (G0 + G1) / 8;                      // 16-byte chunks per voxel
  constexpr uint32_t SLAB0 = SROWS * W0, SLAB1 = SROWS * W1;
  constexpr int NN = 3 * COUT;   // (kw, co) columns of the packed weights
  extern __shared__ __align__(1024) uint8_t smem[];
  const bool halfk = (a.Ca + a.Cb == 8);                  // 8 real channels in a 16-channel group: chunk 1 is zero-filled
  constexpr uint32_t slab_bytes = SLAB0 + SLAB1;
  const int NSLOT = a.nslot;
  uint8_t* s_w = smem;
  uint8_t* s_slab = smem + ((a.wbytes + 1023u) & ~1023u);
  // one accumulator read-out (or seam exchange) buffer per group
  float* s_stage = reinterpret_cast<float*>(s_slab + NSLOT * slab_bytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stage + NGRP * ACC_STAGE_FLOATS);
  uint64_t* full = bars;
  uint64_t* empty = bars + MAXSLOT;
  uint64_t* wbar = empty + MAXSLOT;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const bool tma0 = a.tma_mask & 1, tma1 = (a.tma_mask & 2) != 0;
  const bool all_tma = tma0 && (G1 == 0 || tma1);        // no cp.async traffic at all: one producer thread
  if (threadIdx.x == 0) {
    // empty: one arrival per warp of every group (each group releases every slab once, see below)
    for (int i = 0; i < NSLOT; ++i) { mbar_init(&full[i], all_tma ? 1 : NLOADER); mbar_init(&empty[i], 4 * NGRP); }
    mbar_init(wbar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (threadIdx.x == 0) {
    mbar_expect_tx(wbar, a.wbytes);
    for (uint32_t off = 0; off < a.wbytes; off += 16384u) {
      uint32_t n = a.wbytes - off < 16384u ? a.wbytes - off : 16384u;
      bulk_g2s(s_w + off, reinterpret_cast<const uint8_t*>(a.wpk) + off, n, wbar);
    }
  }
  const int HW_tiles = a.tiles_h * a.tiles_w;
  const int Dout = PD == 2 ? a.D >> 1 : a.D;              // output slices (a.D: slices of the slab source)

  if (warp >= 8) {
    // ================================ LOADER (128 threads) ================================
    const int lt = threadIdx.x - 8 * 32;
    uint32_t slot = 0, lphase = 1;   // producer side: the first lap passes on the fresh barriers
    const int Da = a.upd ? a.D >> 1 : a.D, Ha = a.up ? a.H >> 1 : a.H, Wa = a.up ? a.W >> 1 : a.W;
    const int nca8 = a.Ca >> 3;
    constexpr int nchunk = NC8 * SROWS;
    constexpr int KMAX = (nchunk + NLOADER - 1) / NLOADER;
    if (lt == 0) {
      if (tma0) tma_prefetch_desc(&a.tm[0]);
      if (tma1) tma_prefetch_desc(&a.tm[1]);
    }
    const uint32_t tma_bytes = (tma0 ? SLAB0 : 0u) + (tma1 ? SLAB1 : 0u);
    for (int item = blockIdx.x; item < a.nitems && !(all_tma && lt != 0); item += gridDim.x) {
      const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
      const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
      const int h0 = ht * HT, w0 = wt * WUSE, d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, Dout);
      const int s_begin = PD == 2 ? 2 * d0 - 1 : (KD == 3 ? d0 - 1 : d0), s_end = PD == 2 ? 2 * d1 + 1 : (KD == 3 ? d1 + 1 : d1);
      int soff[KMAX];
      uint32_t doff[KMAX];
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        const int id = lt + k * NLOADER;
        soff[k] = -1;
        doff[k] = 0;
        if (id < nchunk) {
          const int c8 = id % NC8, row = id / NC8;
          const int r = row >> 5, c = row & 31;
          const int h = h0 - 1 + r, w = w0 - 1 + c;
          const int srow = PD == 2 ? ((r & 1) ? NEVEN + (r >> 1) : (r >> 1)) * WT + c : row;   // parity-major rows (PD 2)
          doff[k] = c8 < G0 / 8 ? swz((uint32_t)srow * W0 + (uint32_t)c8 * 16u, W0)
                                : SLAB0 + swz((uint32_t)row * W1 + (uint32_t)(c8 - G0 / 8) * 16u, W1 ? W1 : 32);
          if (c8 < G0 / 8 ? tma0 : tma1) soff[k] = -2;      // this chunk's group arrives by tensor copy
          else if (h >= 0 && h < a.H && w >= 0 && w < a.W && !(halfk && c8 > 0)) {
            if (c8 < nca8) soff[k] = (((a.up ? h >> 1 : h) * Wa + (a.up ? w >> 1 : w)) * a.Ca + c8 * 8) << 1;
            else soff[k] = (((h * a.W + w) * a.Cb + (c8 - nca8) * 8) << 1) | 1;
          }
        }
      }
      for (int ds = s_begin; ds < s_end; ++ds) {
        mbar_wait(&empty[slot], lphase);
        uint8_t* slab = s_slab + (size_t)slot * slab_bytes;
        const bool dok = ds >= 0 && ds < a.D;
        const __nv_bfloat16* baseA = a.xa ? a.xa + (((size_t)b * Da + (dok ? (a.upd ? ds >> 1 : ds) : 0)) * Ha * Wa) * a.Ca : nullptr;
        const __nv_bfloat16* baseB = a.xb ? a.xb + (((size_t)b * a.D + (dok ? ds : 0)) * a.H * a.W) * a.Cb : nullptr;
        const __nv_bfloat16* dummy = a.xa ? a.xa : a.xb;
        if (lt == 0 && tma_bytes) {
          if (all_tma) mbar_expect_tx(&full[slot], tma_bytes);
          else mbar_expect_tx_noarrive(&full[slot], tma_bytes);
          if (tma0) tma_load_5d(slab, &a.tm[0], a.tc0[0], w0 - 1, h0 - 1, ds, b, &full[slot]);
          if (tma1) tma_load_5d(slab + SLAB0, &a.tm[1], a.tc0[1], w0 - 1, h0 - 1, ds, b, &full[slot]);
        }
        if (!all_tma) {
#pragma unroll
          for (int k = 0; k < KMAX; ++k) {
            if (lt + k * NLOADER < nchunk && soff[k] != -2) {
              const bool ok = dok && soff[k] >= 0;
              const __nv_bfloat16* src = ok ? ((soff[k] & 1) ? baseB : baseA) + (soff[k] >> 1) : dummy;
              cp_async16(slab + doff[k], src, ok ? 16u : 0u);
            }
          }
          cp_async_arrive_noinc(&full[slot]);
        }
        if (++slot == (uint32_t)NSLOT) { slot = 0; lphase ^= 1; }
      }
    }
  } else {
    // ================================ MMA + EPILOGUE (2 warpgroups; warp = tile row hh, lane = w') ==================
    // Tile event e (one per 4-row tile half, counted over the CTA's lifetime) belongs to group e % 2: the group issues
    // its wgmma chain and drains the accumulators, so the tensor core works on one group's tile while the other runs its
    // epilogue.  With 8-row tiles group g always takes half g of every slab step.
    // Slab release: every group walks ALL slabs in order (waiting for each one's full phase) and arrives once on each
    // slab's empty barrier after its last MMA reading it has completed, so a slot is refilled only after both groups
    // are past it and no barrier phase can alias.
    const int grp = warp >> 2;
    const int wq = warp & 3;
    float* stage = s_stage + grp * ACC_STAGE_FLOATS;
    const int nbar = 1 + grp;
    // Every wgmma stacks the three kw taps (N = 3 * COUT).  Up to COUT = 32 one chain covers the 128-row tile half in
    // two m64 accumulators and thread t drains row t.  Wider layers run one chain per m64 half (`sub`: tile rows
    // 2 sub, 2 sub + 1) so that its single accumulator stays at 72 / 96 floats per thread; all 128 threads drain it, two
    // per voxel row, the warp pair wq >> 1 taking every other 16-channel chunk.
    constexpr int NSUB = NN > 96 ? 2 : 1;            // chains per tile half
    constexpr int NF = 2 / NSUB;                     // m64 accumulators per chain
    constexpr int NCH = NSUB == 1 ? COUT / 16 : (COUT + 31) / 32;   // 16-channel chunks per thread and chain
    const int trow0 = NSUB == 1 ? wq : (wq & 1);     // tile row of this thread in sub-tile `sub`: trow0 + 2 * sub
    auto chan = [&](int i) { return NSUB == 1 ? 16 * i : 32 * i + 16 * (wq >> 1); };   // first channel of chunk i
    const uint32_t slab_u32 = smem_u32(s_slab), w_u32 = smem_u32(s_w);
    constexpr uint32_t WSTEP = (uint32_t)NN * (W0 + W1);          // bytes of packed weights per (kd, kh) step
    mbar_wait(wbar, 0);
    const uint64_t bdesc0 = make_desc_kmajor_swz(w_u32, W0);
    const uint64_t bdesc1 = make_desc_kmajor_swz(w_u32 + NN * W0, W1 ? W1 : 32);
    uint32_t cnt_base = 0, ecnt = 0, wcur = 0;
    auto observe = [&](uint32_t upto) {              // wait for every slab up to global index `upto`, in order
      for (; wcur <= upto; ++wcur) mbar_wait(&full[wcur % NSLOT], (wcur / NSLOT) & 1);
    };
    // wgmma chain of sub-tile `sub` of tile half hb of the step whose kd window starts at ring slot `hslot`; `par`: parity
    // of the output slice (PD 1)
    constexpr int NKD = PD == 2 ? 4 : KD;            // slabs of the kd window
    // (issues and commits the chain; the caller waits for it)
    auto mma = [&](uint32_t hslot, int hb, int sub, float (&acc)[NF][NN / 2], int par) {
      uint64_t adesc0_kd[NKD], adesc1_kd[NKD];
      uint32_t sl = hslot;
#pragma unroll
      for (int kd = 0; kd < NKD; ++kd) {
        adesc0_kd[kd] = make_desc_kmajor_swz(slab_u32 + sl * slab_bytes, W0);
        adesc1_kd[kd] = make_desc_kmajor_swz(slab_u32 + sl * slab_bytes + SLAB0, W1 ? W1 : 32);
        if (++sl == (uint32_t)NSLOT) sl = 0;
      }
      wg_fence();
#pragma unroll
      for (int kd = 0; kd < NKD; ++kd) {
#pragma unroll
        for (int kh = 0; kh < (PD == 2 ? 4 : 3); ++kh) {
          const int st = kd * (PD == 2 ? 4 : 3) + kh;
#pragma unroll
          for (int k = 0; k < (G0 + G1) / 16; ++k) {  // start-address field is in 16-byte units: kh rows, 32 B per K step
            const bool g0 = k < G0 / 16;
            if (PD == 1 && g0 && kd == 2) continue;    // the upsampled group has 2 kd steps (see PD)
            const int kk = g0 ? k : k - G0 / 16;
            const uint32_t wr = g0 ? W0 : W1;
            uint64_t abase = g0 ? adesc0_kd[kd] : adesc1_kd[kd];
            uint32_t wst = st * WSTEP;
            if (PD == 1 && g0 && par) {                // odd slice: slabs (d, d + 1), tiles (W0 + W1 after the 9 steps, W2)
              abase = adesc0_kd[kd + 1 < NKD ? kd + 1 : kd];
              wst = kd == 0 ? 9 * WSTEP + kh * NN * W0 : (6 + kh) * WSTEP;
            }
            // first slab row of tap kh: row hb * 4 + kh; PD 2: row 2q + kh of coarse row q = 0 in the parity-major order
            const int r0 = PD == 2 ? ((kh & 1) ? NEVEN : 0) + (kh >> 1) : hb * 4 + kh;
            const uint64_t adesc = abase + (uint64_t)((r0 * WT * wr + kk * 32) >> 4);
            const uint64_t bdesc = (g0 ? bdesc0 : bdesc1) + (uint64_t)((wst + kk * 32) >> 4);
#pragma unroll
            for (int f = 0; f < NF; ++f)                // m64 half sub + f of the tile half: two (PD 2: coarse) rows per half
              Wgmma<NN, 0, 0>::mma(acc[f], adesc + (uint64_t)(((sub + f) * 2 * WT * wr) >> 4), bdesc, (st | k) ? 1u : 0u);
          }
        }
      }
      wg_commit();
    };
    // columns [c, c + 16) of the chain's accumulators in row form (see chan for the 16 this thread receives)
    auto readout = [&](float (&acc)[NF][NN / 2], int c, uint32_t (&r)[16]) {
      if constexpr (NSUB == 1) acc_row16(acc[0], acc[NF - 1], c, stage, nbar, r);
      else acc_half_row16(acc[0], c, COUT - (c % COUT) < 32 ? 16 : 32, stage, nbar, r);
    };
    // v[c] = out[w'][chan(i) + c] = P0[w'-1] + P1[w'] + P2[w'+1] (kw partial sums, shuffled across lanes)
    auto combine = [&](float (&acc)[NF][NN / 2], int i, float (&v)[16]) {
      const int cb = NSUB == 1 ? 16 * i : 32 * i;
      uint32_t r[16];
      readout(acc, cb, r);
#pragma unroll
      for (int c = 0; c < 16; ++c) v[c] = __shfl_up_sync(0xffffffffu, __uint_as_float(r[c]), 1);
      readout(acc, COUT + cb, r);
#pragma unroll
      for (int c = 0; c < 16; ++c) v[c] += __uint_as_float(r[c]);
      readout(acc, 2 * COUT + cb, r);
#pragma unroll
      for (int c = 0; c < 16; ++c) v[c] += __shfl_down_sync(0xffffffffu, __uint_as_float(r[c]), 1);
    };
    auto release = [&](int nd) {                     // end of an item: the last two slabs of a 3-D window
      if (KD == 3) {
        const uint32_t last = PD == 2 ? 2u * nd : (uint32_t)nd;
        observe(cnt_base + last + 1u);
        if (lane == 0) {
          mbar_arrive(&empty[(cnt_base + last) % NSLOT]);
          mbar_arrive(&empty[(cnt_base + last + 1) % NSLOT]);
        }
        cnt_base += last + 2;
      } else {
        cnt_base += nd;
      }
    };
    if constexpr (EPI != 0) {
      // Drain in the wgmma fragment layout: thread (warp wq, lane = 4 q + p) of the group holds, in m64 accumulator
      // `blk` = sub + f of a tile half, tile row 2 blk + (wq >> 1) and the columns w' = 16 (wq & 1) + q + 8 i (i = 0, 1),
      // channels 8 jj + 2 p + {0, 1} of each kw partial sum P0 | P1 | P2.  The kw neighbours w' -/+ 1 are lane -/+ 4
      // (lane -/+ 28 and the other i at the q = 0 / 7 seam); only the 15 | 16 seam between the two warps of a slab row
      // crosses warps: warp 2k publishes P0 of w' = 15, warp 2k + 1 P2 of w' = 16 in the group's exchange buffer, one
      // warp-pair barrier per chain.  The buffer alternates between two halves, so a write never overtakes the other
      // warp's last read.  The 48 / 64-output chains and the coarse dgrad (PD 2) keep the row read-out (see ROWS).
      const float slope = a.slope;
      const int c1 = (EPI == 3 && a.out2) ? a.csplit : COUT;       // channels [0, c1) -> out, [c1, COUT) -> out2
      const int Ho = PD == 2 ? a.H >> 1 : a.H, Wo = PD == 2 ? a.W >> 1 : a.W;   // output rows, columns
      const size_t HWp = (size_t)Ho * Wo;
      const int q = lane >> 2, p = lane & 3, half = wq & 1, pair = wq >> 1;
      const int xbar = 3 + 2 * grp + pair;                      // named barrier of this warp pair
      // Row read-out instead: the 48 / 64-output chains (in the fragment form their bias / mask loads spill next to the
      // 72 / 96 accumulator floats) and the coarse dgrad (its 32-channel mask, prefetched before the chain, spills there)
      constexpr bool ROWS = NSUB > 1 || PD == 2;
      constexpr int XPAIR = NF * 2 * COUT;                       // floats per warp pair and buffer half: P0 of 15, P2 of 16
      static_assert(2 * 2 * XPAIR <= ACC_STAGE_FLOATS, "seam exchange fits the stage buffer");
      uint32_t xpar = 0;
      // Ordered hand-off of the tensor pipe (fragment drain): group g issues the chain of its tile event e only after the
      // other group has issued event e - 1 (named barrier 7 + g, 256 threads: the waiting group's bar.sync and the other
      // group's bar.arrive right after its wg_commit).  Issued in event order, the chains complete in event order, so one
      // group drains while the other's chain is on the tensor pipe instead of both draining at once.  Group 1 opens the
      // first turn; a group arrives after event e only if event e + 1 exists, so every barrier phase gets exactly one
      // arrival and one sync (the next arrival on a barrier needs a turn that only its completion grants).
      constexpr bool ORD = !ROWS;
      [[maybe_unused]] uint32_t nev = 0;                         // tile events of this CTA
      if constexpr (ORD) {
        for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
          const int d0 = ((item / HW_tiles) % a.nchunks) * a.dchunk;
          nev += (uint32_t)(min(d0 + a.dchunk, Dout) - d0) * NH;
        }
        if (grp == 1) named_bar_arrive(7, 256);                 // (event 0 exists: every CTA has an item)
      }
      for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
        const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
        const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
        const int d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, Dout);
        const int nd = d1 - d0;
        // column i of block blk of tile half hb: voxel vbase + (4 hb + 2 blk) Wo + 8 i, written iff bit 4 hb + 2 blk + i of okm
        const int wp = 16 * half + q, w = wt * WUSE - 1 + wp;
        const int hbase = ht * HT + pair;
        uint32_t okm = 0;
#pragma unroll
        for (int hb = 0; hb < NH; ++hb)
#pragma unroll
          for (int blk = 0; blk < 2; ++blk)
#pragma unroll
            for (int i = 0; i < 2; ++i)
              if (wp + 8 * i >= 1 && wp + 8 * i <= WUSE && w + 8 * i < a.W && hbase + 4 * hb + 2 * blk < Ho)
                okm |= 1u << (4 * hb + 2 * blk + i);
        size_t vbase = (((size_t)b * Dout + d0) * Ho + hbase) * Wo + (size_t)(long long)w;
        // EPI 4: channel c of voxel v (channels-last index) sits at v + (b (Cout - 1) + c) D H W in the planar output
        [[maybe_unused]] const size_t DHWp = (size_t)Dout * HWp, pbase = (size_t)b * (a.Cout - 1) * DHWp;
        for (int j = 0; j < nd; ++j) {
          const uint32_t js = PD == 2 ? 2u * j : (uint32_t)j;   // ring index of the window's first slab
          observe(cnt_base + js + (PD == 2 ? 3u : (KD == 3 ? 2u : 0u)));
          const uint32_t hslot = (cnt_base + js) % NSLOT;
#pragma unroll
          for (int hb = 0; hb < NH; ++hb) {
            if ((int)(ecnt++ % NGRP) != grp) continue;
            auto vox_of = [&](int blk, int i) { return vbase + (size_t)((4 * hb + 2 * blk) * Wo + 8 * i); };
#pragma unroll
            for (int sub = 0; sub < NSUB; ++sub) {
              // the saved activations (EPI 2) of this thread's columns in accumulator f: loaded before the chain where
              // they fit beside it (16 outputs), else at the start of f's drain
              [[maybe_unused]] uint32_t mreg[EPI == 2 && !ROWS ? NF : 1][2][COUT / 8];
              auto load_mask = [&](int f) {
                if constexpr (EPI == 2 && !ROWS) {
#pragma unroll
                  for (int i = 0; i < 2; ++i)
                    if (okm >> (4 * hb + 2 * f + i) & 1u) {
                      const uint32_t* mp = reinterpret_cast<const uint32_t*>(a.mask + vox_of(f, i) * (OP ? a.opitch : COUT) + 2 * p);
#pragma unroll
                      for (int jj = 0; jj < COUT / 8; ++jj) mreg[f][i][jj] = __ldg(mp + 4 * jj);
                    }
                }
              };
              if constexpr (COUT == 16) {
#pragma unroll
                for (int f = 0; f < NF; ++f) load_mask(f);
              }
              // ROWS: thread t of the group drains voxel row t of the tile half (48 / 64 outputs: of its m64 sub-tile, two
              // threads per row, the warp pair wq >> 1 taking every other 16-channel chunk); PD 2: the odd lanes (even w)
              // hold the sums of their w' pairs and store coarse column w / 2
              const int rh = PD == 2 ? ht * (HT / 2) + trow0 : ht * HT + hb * 4 + trow0 + 2 * sub, rw = wt * WUSE - 1 + lane;
              const bool rvalid = lane >= 1 && lane <= WUSE && rw < a.W && rh < Ho && (PD != 2 || (lane & 1));
              const size_t rvox = (((size_t)b * Dout + d0 + j) * Ho + rh) * Wo + (PD == 2 ? rw >> 1 : rw);
              [[maybe_unused]] uint32_t mrow[PD == 2 ? NCH : 1][8];
              if constexpr (PD == 2) {
#pragma unroll
                for (int i = 0; i < NCH; ++i)
                  if (rvalid) ld_global_nc_v8(a.mask + rvox * COUT + chan(i), mrow[i]);
              }
              float acc[NF][NN / 2];
              [[maybe_unused]] const uint32_t e = ecnt - 1;      // this tile event
              if constexpr (ORD) named_bar(7 + grp, 256);        // event e - 1 is issued
              mma(hslot, hb, sub, acc, (d0 + j) & 1);
              if (ORD && e + 1 < nev) named_bar_arrive(8 - grp, 256);   // event e + 1 may issue
              wg_wait<0>();
              if constexpr (ROWS) {
                const bool valid = rvalid;
                const size_t vox = rvox;
#pragma unroll
                for (int i = 0; i < NCH; ++i) {
                  const int c0 = chan(i);
                  float v[16];
                  combine(acc, i, v);
                  if (c0 >= COUT) continue;                      // (48 channels: the second warp pair has one chunk less)
                  if constexpr (PD == 2) {                       // coarse column: the sum of the w' pair (w, w + 1)
#pragma unroll
                    for (int c = 0; c < 16; ++c) v[c] += __shfl_down_sync(0xffffffffu, v[c], 1);
                  }
                  if constexpr (EPI == 1) {
#pragma unroll
                    for (int c = 0; c < 16; ++c) {
                      const float x = v[c] + (a.bias ? __ldg(a.bias + c0 + c) : 0.f);
                      v[c] = fmaxf(x, x * slope);
                    }
                  } else if constexpr (EPI == 2) {
                    uint32_t mreg[8];
                    if constexpr (PD == 2) {
#pragma unroll
                      for (int e = 0; e < 8; ++e) mreg[e] = mrow[i][e];
                    } else if (valid) {
                      ld_global_nc_v8(a.mask + vox * (OP ? a.opitch : COUT) + c0, mreg);
                    }
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                      if (mreg[e] & 0x8000u) v[2 * e] *= slope;
                      if (mreg[e] & 0x80000000u) v[2 * e + 1] *= slope;
                    }
                  }
                  if (valid) {
                    __nv_bfloat16* dst = (EPI == 3 && c0 >= c1) ? reinterpret_cast<__nv_bfloat16*>(a.out2) + vox * (COUT - c1) + (c0 - c1)
                                                                : reinterpret_cast<__nv_bfloat16*>(a.out) + vox * (OP ? a.opitch : c1) + c0;
                    st_global_v8(dst, pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]),
                                 pack_bf16x2(v[8], v[9]), pack_bf16x2(v[10], v[11]), pack_bf16x2(v[12], v[13]), pack_bf16x2(v[14], v[15]));
                  }
                }
                continue;
              }
              float* xb = stage + xpar * (2 * XPAIR) + pair * XPAIR;
              xpar ^= 1u;
              if (half == 0 ? q == 7 : q == 0) {                 // publish the seam rows (one 8-byte store per channel pair)
#pragma unroll
                for (int f = 0; f < NF; ++f)
#pragma unroll
                  for (int jj = 0; jj < COUT / 8; ++jj) {
                    float2* xs = reinterpret_cast<float2*>(xb + f * 2 * COUT + 8 * jj + 2 * p);
                    const int k0 = 4 * jj + 2, k2 = 4 * (COUT / 4 + jj);       // P0 of row q + 8, P2 of row q
                    if (half == 0) xs[0] = make_float2(acc[f][k0], acc[f][k0 + 1]);        // P0 of w' = 15
                    else xs[COUT / 2] = make_float2(acc[f][k2], acc[f][k2 + 1]);           // P2 of w' = 16
                  }
              }
              named_bar(xbar, 64);
#pragma unroll
              for (int f = 0; f < NF; ++f) {
                const int blk = sub + f;
                if constexpr (COUT != 16) load_mask(f);
#pragma unroll
                for (int jj = 0; jj < COUT / 8; ++jj) {
                  if (EPI == 4 && 8 * jj >= a.Cout) break;       // (uniform) no real channel from here on
                  const int c0 = 8 * jj + 2 * p;
                  float v[2][2];                                 // [i][e]: channel c0 + e of column w' + 8 i
#pragma unroll
                  for (int e = 0; e < 2; ++e) {
                    const float* xs = xb + f * 2 * COUT + c0 + e;
                    const int k0 = 4 * jj + e, k1 = 4 * (COUT / 8 + jj) + e, k2 = 4 * (COUT / 4 + jj) + e;
                    // P0[w' - 1], P2[w' + 1] from the lanes 4 below / above (the sender picks the other i at the seam)
                    const float a1 = __shfl_sync(0xffffffffu, q == 7 ? acc[f][k0] : acc[f][k0 + 2], (lane + 28) & 31);
                    const float a0 = __shfl_sync(0xffffffffu, acc[f][k0], (lane + 28) & 31);
                    const float b0 = __shfl_sync(0xffffffffu, q == 0 ? acc[f][k2 + 2] : acc[f][k2], (lane + 4) & 31);
                    const float b1 = __shfl_sync(0xffffffffu, acc[f][k2 + 2], (lane + 4) & 31);
                    float x0 = q == 0 ? xs[0] : a0;
                    x0 += acc[f][k1];
                    x0 += b0;
                    float x1 = a1;
                    x1 += acc[f][k1 + 2];
                    x1 += q == 7 ? xs[COUT] : b1;
                    v[0][e] = x0;
                    v[1][e] = x1;
                  }
#pragma unroll
                  for (int i = 0; i < 2; ++i) {
                    if constexpr (EPI == 1) {
#pragma unroll
                      for (int e = 0; e < 2; ++e) {
                        const float x = v[i][e] + (a.bias ? __ldg(a.bias + c0 + e) : 0.f);
                        v[i][e] = fmaxf(x, x * slope);           // LeakyReLU for 0 <= slope <= 1
                      }
                    } else if constexpr (EPI == 2 && KD == 3) {  // sign bits of the saved bf16 activations
                      const uint32_t mw = mreg[f][i][jj];
                      if (mw & 0x8000u) v[i][0] *= slope;
                      if (mw & 0x80000000u) v[i][1] *= slope;
                    } else if constexpr (EPI == 2) {
                      // KD = 1 keeps the generic epilogue's arithmetic: + 0 (no bias), then the derivative where the saved
                      // bf16 activation compares below zero (a saved -0.0 or NaN does not)
                      const uint32_t mw = mreg[f][i][jj];
                      v[i][0] += 0.f;
                      v[i][1] += 0.f;
                      if (__uint_as_float(mw << 16) < 0.f) v[i][0] *= slope;
                      if (__uint_as_float(mw & 0xffff0000u) < 0.f) v[i][1] *= slope;
                    } else if constexpr (EPI == 4) {
#pragma unroll
                      for (int e = 0; e < 2; ++e) {
                        float x = v[i][e] + (a.bias && c0 + e < a.Cout ? __ldg(a.bias + c0 + e) : 0.f);
                        if (slope >= 0.f) x = x >= 0.f ? x : x * slope;
                        v[i][e] = x;
                      }
                    }
                    if constexpr (EPI == 4) {
                      if (okm >> (4 * hb + 2 * blk + i) & 1u) {
                        float* o = reinterpret_cast<float*>(a.out) + vox_of(blk, i) + pbase + (size_t)c0 * DHWp;
                        if (c0 < a.Cout) o[0] = v[i][0];
                        if (c0 + 1 < a.Cout) o[DHWp] = v[i][1];
                      }
                    } else if (okm >> (4 * hb + 2 * blk + i) & 1u) {
                      const size_t vox = vox_of(blk, i);
                      __nv_bfloat16* dst = (EPI == 3 && c0 >= c1) ? reinterpret_cast<__nv_bfloat16*>(a.out2) + vox * (COUT - c1) + (c0 - c1)
                                                                  : reinterpret_cast<__nv_bfloat16*>(a.out) + vox * (OP ? a.opitch : c1) + c0;
                      *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(v[i][0], v[i][1]);
                    }
                  }
                }
              }
            }
          }
          vbase += HWp;
          if (lane == 0) {                               // this group no longer reads slab js (PD 2: nor js + 1)
            mbar_arrive(&empty[hslot]);
            if (PD == 2) mbar_arrive(&empty[(hslot + 1) % NSLOT]);
          }
        }
        release(nd);
      }
    } else {
    const size_t HWp = (size_t)a.H * a.W;
    auto bias_at = [&](int c) -> float { return a.bias ? __ldg(a.bias + c) : 0.f; };
    for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
      const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
      const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
      const int w = wt * WUSE - 1 + lane, d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, a.D);
      const int nd = d1 - d0;
      for (int j = 0; j < nd; ++j) {
        const int d = d0 + j;
        observe(cnt_base + (uint32_t)j + (KD == 3 ? 2u : 0u));
        const uint32_t hslot = (cnt_base + j) % NSLOT;
#pragma unroll
        for (int hb = 0; hb < NH; ++hb) {
        if ((int)(ecnt++ % NGRP) != grp) continue;
#pragma unroll
        for (int sub = 0; sub < NSUB; ++sub) {
        const int h = ht * HT + hb * 4 + trow0 + 2 * sub;
        const bool valid = lane >= 1 && lane <= WUSE && h < a.H && w < a.W;
        const size_t vox = (((size_t)b * a.D + d) * a.H + h) * a.W + w;
        // prefetch the LeakyReLU-derivative mask of this voxel before the MMAs (one chain per m64 half: read after the
        // combine instead, the prefetch would spill next to the wider accumulator)
        constexpr bool PREF = NSUB == 1;
        [[maybe_unused]] uint4 mreg[PREF ? NCH : 1][2];
        if (PREF && a.mask && valid) {
#pragma unroll
          for (int i = 0; i < NCH; ++i)
#pragma unroll
            for (int q = 0; q < 2; ++q)
              if (chan(i) + 8 * q < a.Cout)
                mreg[i][q] = __ldg(reinterpret_cast<const uint4*>(a.mask + vox * (OP ? a.opitch : a.Cout) + chan(i)) + q);
        }
        const int c1 = a.out2 ? a.csplit : a.Cout;          // channels [0,c1) -> out, [c1,Cout) -> out2
        float acc[NF][NN / 2];
        mma(hslot, hb, sub, acc, 0);
        wg_wait<0>();
        // 16 output channels at a time: the kw = 0, 1, 2 partial sums, shuffle-combined across lanes, stored
#pragma unroll
        for (int i = 0; i < NCH; ++i) {
          const int c0 = chan(i);
          [[maybe_unused]] float4 ain[ACC ? 4 : 1];
          if constexpr (ACC && !OP && PREF) {     // (otherwise read after the combine, the prefetch would spill)
            if (a.acc_in && valid && c0 < COUT) {      // partial sums of the earlier split-precision passes
              const float4* ap = reinterpret_cast<const float4*>(a.acc_in + vox * COUT + c0);
#pragma unroll
              for (int q = 0; q < 4; ++q) ain[q] = __ldg(ap + q);
            }
          }
          float v[16];
          combine(acc, i, v);
          if (NSUB > 1 && c0 >= COUT) continue;            // (48 channels: the second warp pair has one chunk less)
          bool handled = false;
          if constexpr (ACC) {
            if (a.acc_in && valid) {
              if constexpr (OP || !PREF) {
                const float4* ap = reinterpret_cast<const float4*>(a.acc_in + vox * COUT + c0);
#pragma unroll
                for (int q = 0; q < 4; ++q) ain[q] = __ldg(ap + q);
              }
#pragma unroll
              for (int q = 0; q < 4; ++q) { v[4 * q] += ain[q].x; v[4 * q + 1] += ain[q].y; v[4 * q + 2] += ain[q].z; v[4 * q + 3] += ain[q].w; }
            }
            if (a.out_mode == 2) {
              handled = true;
              if (valid) {
                float4* op = reinterpret_cast<float4*>(reinterpret_cast<float*>(a.out) + vox * COUT + c0);
#pragma unroll
                for (int q = 0; q < 4; ++q) op[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
              }
            } else if (a.out_mode == 3) {
              handled = true;
              if (valid && c0 < a.Cout) {
#pragma unroll
                for (int q = 0; q < 16; q += 8) {
                  if (c0 + q < a.Cout) {
                    uint32_t hi[4], lo[4];
#pragma unroll
                    for (int e = 0; e < 8; e += 2) {
                      float x0 = v[q + e] + bias_at(c0 + q + e), x1 = v[q + e + 1] + bias_at(c0 + q + e + 1);
                      if (a.slope >= 0.f) { x0 = x0 >= 0.f ? x0 : x0 * a.slope; x1 = x1 >= 0.f ? x1 : x1 * a.slope; }
                      const __nv_bfloat16 h0 = __float2bfloat16_rn(x0), h1 = __float2bfloat16_rn(x1);
                      hi[e >> 1] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
                      lo[e >> 1] = pack_bf16x2(x0 - __bfloat162float(h0), x1 - __bfloat162float(h1));
                    }
                    const size_t o = vox * (OP ? a.opitch : a.Cout) + c0 + q;
                    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(a.out) + o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(a.out_lo) + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                  }
                }
              }
            }
          }
          if (!handled && valid && c0 < a.Cout) {
            if (a.out_mode == 0) {
#pragma unroll
              for (int q = 0; q < 16; q += 8) {
                if (c0 + q < a.Cout) {
                  float x[8];
#pragma unroll
                  for (int e = 0; e < 8; ++e) x[e] = v[q + e] + bias_at(c0 + q + e);
                  if (a.mask) {
                    uint4 m4;
                    if constexpr (PREF) m4 = mreg[i][q / 8];
                    else m4 = __ldg(reinterpret_cast<const uint4*>(a.mask + vox * (OP ? a.opitch : a.Cout) + c0) + q / 8);
                    const __nv_bfloat16* mb = reinterpret_cast<const __nv_bfloat16*>(&m4);
#pragma unroll
                    for (int e = 0; e < 8; ++e) if (__bfloat162float(mb[e]) < 0.f) x[e] *= a.slope;
                  } else if (a.slope >= 0.f) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) x[e] = x[e] >= 0.f ? x[e] : x[e] * a.slope;
                  }
                  // a split never falls inside a group of 8 channels (csplit % 8 == 0)
                  const int cg = c0 + q;
                  __nv_bfloat16* oo = cg < c1 ? reinterpret_cast<__nv_bfloat16*>(a.out) + vox * (OP ? a.opitch : c1) + cg
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
        if (lane == 0) mbar_arrive(&empty[hslot]);    // this group no longer reads slab j
      }
      release(nd);
    }
    }
  }
}

// fp32 (Cout, Cin, KD, 3, 3) -> bf16, per (kd,kh) step two swizzled K-major tiles [N rows = kw*COUT + co][G0 ch] and [N][G1 ch]
__global__ void pack_weights_s_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int Cout, int Cin, int KD, int COUT,
                                      int NN, int G0, int G1, int transposed) {
  const int T = KD * 9;
  const int CG = G0 + G1;
  const int total = KD * 3 * NN * CG;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int ci = i % CG, n = (i / CG) % NN, st = i / (CG * NN);
    const int kd = st / 3, kh = st % 3, g = n / COUT, co = n % COUT;
    const int tap = (kd * 3 + kh) * 3 + g;
    float v = 0.f;
    if (!transposed) {
      if (co < Cout && ci < Cin) v = w[((size_t)co * Cin + ci) * T + tap];
    } else {
      if (co < Cin && ci < Cout) v = w[((size_t)ci * Cin + co) * T + (T - 1 - tap)];
    }
    // destination: step tile = [group 0: NN x G0][group 1: NN x G1], bytes swizzled inside each group tile
    const uint32_t W0 = G0 * 2, W1 = G1 * 2;
    uint32_t off;
    if (ci < G0) off = swz((uint32_t)n * W0 + (uint32_t)ci * 2u, W0);
    else off = (uint32_t)NN * W0 + swz((uint32_t)n * W1 + (uint32_t)(ci - G0) * 2u, W1);
    out[((size_t)st * NN * (W0 + W1) + off) / 2] = __float2bfloat16_rn(v);
  }
}

// All packed operands of a model in ONE launch (23 pack launches per training step otherwise: forward + transposed copy
// of every layer, a few kilobytes each).  `descs` lives in device memory; element ranges are consecutive.
struct PackDesc {
  const float* w;
  __nv_bfloat16* out;
  int Cout, Cin, KD, COUT, NN, G0, G1, transposed;
  int begin, count;      // global element range [begin, begin + count)
  // fold > 0: `w` is a 3-D (Cout, Cin, 3, 3, 3) weight whose kd taps are folded into the input channels of a 2-D operand
  // (KD = 1 here): operand input channel kd * fold + c <-> (tap kd, real channel c), fold = real channel count of the
  // operand's input side (Cin forward, Cout transposed)
  int fold;
  // channel block of an unfolded operand: operand output channels [n0, n0 + nb), input channels [k0, k0 + kb) (in the
  // operand's own orientation: transposed swaps the weight's Cout and Cin)
  int n0, nb, k0, kb;
  // polyphase operand (conv_tcs_kernel PD): 1 = forward, group 0 (the upsampled source) holds W1 + W2 in its kd = 1
  // tiles and 3 more group-0 tiles (one per kh) after the 9 steps hold W0 + W1; 2 = coarse dgrad, 4 x 4 (kd, kh) steps
  // (step kd * 4 + kh) of transposed taps T0, T0 + T1, T1 + T2, T2 along both axes.  Merged taps are summed in fp32 (kd
  // outer, kh inner) and rounded to bf16 once.
  int poly;
};
__global__ void pack_weights_multi_kernel(const PackDesc* __restrict__ descs, int ndesc, int total) {
  for (int gi = blockIdx.x * blockDim.x + threadIdx.x; gi < total; gi += gridDim.x * blockDim.x) {
    int lo = 0, hi = ndesc - 1;
    while (lo < hi) {                         // last descriptor whose begin <= gi
      const int mid = (lo + hi + 1) >> 1;
      if (descs[mid].begin <= gi) lo = mid; else hi = mid - 1;
    }
    const PackDesc d = descs[lo];
    const int i = gi - d.begin;
    const int T = d.KD * 9, CG = d.G0 + d.G1;
    const int base = d.KD * 3 * d.NN * CG;               // elements of the (kd, kh) step tiles
    const bool extra = d.poly == 1 && i >= base;          // the W0 + W1 group-0 tiles of a polyphase forward operand
    const int ie = i - base;
    const int ci = extra ? ie % d.G0 : i % CG, n = extra ? (ie / d.G0) % d.NN : (i / CG) % d.NN;
    const int st = extra ? ie / (d.G0 * d.NN) : i / (CG * d.NN);
    const int kd = extra ? 0 : (d.poly == 2 ? st >> 2 : st / 3), kh = extra ? st : (d.poly == 2 ? st & 3 : st % 3);
    const int g = n / d.COUT, co = n % d.COUT;
    const int tap = (kd * 3 + kh) * 3 + g;
    float v = 0.f;
    if (d.poly) {
      if (co < d.nb && ci < d.kb) {
        int t0 = kd, t1 = kd, u0 = kh, u1 = kh;            // the kd and kh taps merged into this tile
        if (d.poly == 1 && ci < d.G0) t1 = extra ? 1 : (kd == 1 ? 2 : kd);
        if (d.poly == 2) {                                 // 4 merged taps along d and along h: T0, T0 + T1, T1 + T2, T2
          t0 = kd > 0 ? kd - 1 : 0; t1 = kd < 2 ? kd : 2;
          u0 = kh > 0 ? kh - 1 : 0; u1 = kh < 2 ? kh : 2;
        }
        for (int t = t0; t <= t1; ++t)
          for (int u = u0; u <= u1; ++u) {
            const int tp = (t * 3 + u) * 3 + g;
            v += !d.transposed ? d.w[((size_t)(d.n0 + co) * d.Cin + d.k0 + ci) * 27 + tp]
                               : d.w[((size_t)(d.k0 + ci) * d.Cin + d.n0 + co) * 27 + (26 - tp)];
          }
      }
    } else if (d.fold) {
      const int fk = ci / d.fold, c = ci % d.fold;              // folded kd tap, real input channel of the operand
      const int tap3 = (fk * 3 + kh) * 3 + g;
      if (fk < 3) {
        if (!d.transposed) { if (co < d.Cout) v = d.w[((size_t)co * d.Cin + c) * 27 + tap3]; }
        else if (co < d.Cin) v = d.w[((size_t)c * d.Cin + co) * 27 + (26 - tap3)];
      }
    } else if (co < d.nb && ci < d.kb) {
      if (!d.transposed) v = d.w[((size_t)(d.n0 + co) * d.Cin + d.k0 + ci) * T + tap];
      else v = d.w[((size_t)(d.k0 + ci) * d.Cin + d.n0 + co) * T + (T - 1 - tap)];
    }
    const uint32_t W0 = d.G0 * 2, W1 = d.G1 * 2;
    uint32_t off;
    if (extra) off = (uint32_t)base * 2u + (uint32_t)(st * d.NN) * W0 + swz((uint32_t)n * W0 + (uint32_t)ci * 2u, W0);
    else if (ci < d.G0) off = (uint32_t)(st * d.NN) * (W0 + W1) + swz((uint32_t)n * W0 + (uint32_t)ci * 2u, W0);
    else off = (uint32_t)(st * d.NN) * (W0 + W1) + (uint32_t)d.NN * W0 + swz((uint32_t)n * W1 + (uint32_t)(ci - d.G0) * 2u, W1);
    d.out[off / 2] = __float2bfloat16_rn(v);
  }
}

// channel grouping of a convolution input of `cin` channels (8 counts as a zero-padded 16)
static void groups_of(int cin, int* g0, int* g1) {
  if (cin == 8 || cin == 16) { *g0 = 16; *g1 = 0; }
  else if (cin == 32) { *g0 = 32; *g1 = 0; }
  else if (cin == 48) { *g0 = 32; *g1 = 16; }
  else { *g0 = 64; *g1 = 0; }
}

// Which channel groups of the slab can be staged by tiled tensor copies: a group whose channels all come from one source
// tensor that is read at its own resolution.  VXM_B200_TMA=0 keeps every group on the cp.async loader (A/B switch).
static int plan_tma(ConvSArgs& a, int g0, int g1, int HTv) {
  a.tma_mask = 0;
  a.tc0[0] = a.tc0[1] = 0;
  const char* e = getenv("VXM_B200_TMA");
  if (e && e[0] == '0') return 0;
  const int lo[2] = {0, g0}, hi[2] = {g0, g0 + g1};
  for (int g = 0; g < 2; ++g) {
    if (hi[g] == lo[g]) continue;
    const void* base = nullptr;
    int C = 0, c0 = 0;
    if (a.xa && hi[g] <= a.Ca && !a.up) { base = a.xa; C = a.Ca; c0 = lo[g]; }
    else if (a.xb && lo[g] >= a.Ca && hi[g] <= a.Ca + a.Cb) { base = a.xb; C = a.Cb; c0 = lo[g] - a.Ca; }
    if (!base) continue;
    if (tc::make_act_tmap(&a.tm[g], base, a.B, a.D, a.H, a.W, C, hi[g] - lo[g], WT, HTv + 2) != 0) return -1;
    a.tma_mask |= 1 << g;
    a.tc0[g] = c0;
  }
  return 0;
}

}  // namespace tcs
}  // namespace vxm

using namespace vxm;
using namespace vxm::tcs;

extern "C" size_t vxm_conv3d_tcs_packed_bytes(int cin_eff, int coutp, int kd) {
  int g0, g1;
  groups_of(cin_eff <= 8 ? 8 : (cin_eff <= 16 ? 16 : (cin_eff <= 32 ? 32 : (cin_eff <= 48 ? 48 : 64))), &g0, &g1);
  return (size_t)kd * 3 * (3 * coutp) * (g0 + g1) * sizeof(__nv_bfloat16);
}

extern "C" int vxm_conv3d_tcs_pack(const float* w, void* wpk, int Cout, int Cin, int kd, int coutp, int transposed, void* stream) {
  VXM_REQUIRE(w && wpk && Cout > 0 && Cin > 0 && (kd == 1 || kd == 3) && (coutp == 16 || coutp == 32 || coutp == 48 || coutp == 64), "conv3d_tcs_pack: bad argument");
  int cin_eff = transposed ? Cout : Cin, nout = transposed ? Cin : Cout;
  VXM_REQUIRE(nout <= coutp, "conv3d_tcs_pack: %d output channels do not fit %d", nout, coutp);
  VXM_REQUIRE(cin_eff <= 64, "conv3d_tcs_pack: at most 64 input channels");
  int g0, g1;
  groups_of(cin_eff <= 8 ? 8 : (cin_eff <= 16 ? 16 : (cin_eff <= 32 ? 32 : (cin_eff <= 48 ? 48 : 64))), &g0, &g1);
  int NN = 3 * coutp;
  int total = kd * 3 * NN * (g0 + g1);
  pack_weights_s_kernel<<<(total + 255) / 256, 256, 0, as_stream(stream)>>>(w, (__nv_bfloat16*)wpk, Cout, Cin, kd, coutp, NN, g0, g1, transposed);
  return check_launch("conv3d_tcs_pack");
}

extern "C" size_t vxm_conv3d_tcs_pack_desc_bytes(void) { return sizeof(PackDesc); }

// Fill one host-side descriptor (the caller uploads the array once and keeps it while the pointers stay valid).
extern "C" int vxm_conv3d_tcs_pack_desc_blk(void* desc_host, const float* w, void* wpk, int Cout, int Cin, int kd, int coutp, int transposed,
                                            int n0, int nb, int k0, int kb, int begin) {
  VXM_REQUIRE(desc_host && w && wpk && Cout > 0 && Cin > 0 && (kd == 1 || kd == 3) && (coutp == 16 || coutp == 32 || coutp == 48 || coutp == 64),
              "conv3d_tcs_pack_desc: bad argument");
  const int cin_eff = transposed ? Cout : Cin, nout = transposed ? Cin : Cout;
  VXM_REQUIRE(n0 >= 0 && nb > 0 && n0 + nb <= nout && k0 >= 0 && kb > 0 && k0 + kb <= cin_eff, "conv3d_tcs_pack_desc: block out of range");
  VXM_REQUIRE(nb <= coutp && kb <= 64, "conv3d_tcs_pack_desc: channel counts do not fit");
  int g0, g1;
  groups_of(kb <= 8 ? 8 : (kb <= 16 ? 16 : (kb <= 32 ? 32 : (kb <= 48 ? 48 : 64))), &g0, &g1);
  PackDesc d;
  d.w = w; d.out = (__nv_bfloat16*)wpk; d.Cout = Cout; d.Cin = Cin; d.KD = kd; d.COUT = coutp; d.NN = 3 * coutp; d.G0 = g0; d.G1 = g1;
  d.transposed = transposed; d.begin = begin; d.count = kd * 3 * d.NN * (g0 + g1); d.fold = 0;
  d.n0 = n0; d.nb = nb; d.k0 = k0; d.kb = kb; d.poly = 0;
  memcpy(desc_host, &d, sizeof(d));
  return d.count;      // elements of this operand (>= 0), so the caller can chain `begin`
}

extern "C" int vxm_conv3d_tcs_pack_desc(void* desc_host, const float* w, void* wpk, int Cout, int Cin, int kd, int coutp, int transposed,
                                        int begin) {
  VXM_REQUIRE(Cout > 0 && Cin > 0, "conv3d_tcs_pack_desc: bad argument");
  return vxm_conv3d_tcs_pack_desc_blk(desc_host, w, wpk, Cout, Cin, kd, coutp, transposed, 0, transposed ? Cin : Cout, 0,
                                      transposed ? Cout : Cin, begin);
}

// Descriptor of a kd-folded 2-D operand of the 3-D weight w (Cout, Cin, 3, 3, 3): the operand has 3 * (Cin | Cout if
// transposed) input channels (padded to 8 / 16) and kd = 1; packed size = vxm_conv3d_tcs_packed_bytes(3 * that, coutp, 1).
extern "C" int vxm_conv3d_tcs_pack_desc_fold(void* desc_host, const float* w, void* wpk, int Cout, int Cin, int coutp, int transposed, int begin) {
  VXM_REQUIRE(desc_host && w && wpk && Cout > 0 && Cin > 0 && (coutp == 16 || coutp == 32), "conv3d_tcs_pack_desc_fold: bad argument");
  const int real_in = transposed ? Cout : Cin, nout = transposed ? Cin : Cout;
  VXM_REQUIRE(3 * real_in <= 16 && nout <= coutp, "conv3d_tcs_pack_desc_fold: %d x 3 input channels / %d outputs do not fit", real_in, nout);
  int g0, g1;
  groups_of(3 * real_in <= 8 ? 8 : 16, &g0, &g1);
  PackDesc d;
  d.w = w; d.out = (__nv_bfloat16*)wpk; d.Cout = Cout; d.Cin = Cin; d.KD = 1; d.COUT = coutp; d.NN = 3 * coutp; d.G0 = g0; d.G1 = g1;
  d.transposed = transposed; d.begin = begin; d.count = 3 * d.NN * (g0 + g1); d.fold = real_in;
  d.n0 = d.nb = d.k0 = d.kb = 0; d.poly = 0;
  memcpy(desc_host, &d, sizeof(d));
  return d.count;
}

// Polyphase operands of a 3-D concat layer whose first Ca input channels are a nearest-x2 upsampled source
// (conv_tcs_kernel PD): mode 1 = forward ((Ca = 32) + (Cb = 16) -> Cout = 32), mode 2 = coarse dgrad (the Cout = 32
// gradient channels -> the Ca = 32 channels of the coarse source).
static int poly_geometry(int mode, int Cout, int Cin, int Ca, int* g0, int* g1, int* kd, int* coutp) {
  if (mode == 1 && Ca == 32 && Cin == 48 && Cout == 32) { *g0 = 32; *g1 = 16; *kd = 3; *coutp = 32; return 1; }
  if (mode == 2 && Ca == 32 && Cin > Ca && Cout == 32) { *g0 = 32; *g1 = 0; *kd = 4; *coutp = 32; return 1; }
  return 0;
}

static size_t poly_bytes(int mode) {
  const size_t NN = 3 * 32;
  return (mode == 1 ? 9 * NN * (32 + 16) + 3 * NN * 32 : 16 * NN * 32) * sizeof(__nv_bfloat16);
}

extern "C" size_t vxm_conv3d_tcs_poly_packed_bytes(int mode, int Cout, int Cin, int Ca) {
  int g0, g1, kd, coutp;
  return poly_geometry(mode, Cout, Cin, Ca, &g0, &g1, &kd, &coutp) ? poly_bytes(mode) : 0;
}

extern "C" int vxm_conv3d_tcs_pack_desc_poly(void* desc_host, const float* w, void* wpk, int Cout, int Cin, int Ca, int mode, int begin) {
  int g0, g1, kd, coutp;
  VXM_REQUIRE(desc_host && w && wpk && poly_geometry(mode, Cout, Cin, Ca, &g0, &g1, &kd, &coutp),
              "conv3d_tcs_pack_desc_poly: no polyphase operand for mode %d, (%d of %d) -> %d", mode, Ca, Cin, Cout);
  PackDesc d;
  d.w = w; d.out = (__nv_bfloat16*)wpk; d.Cout = Cout; d.Cin = Cin; d.KD = kd; d.COUT = coutp; d.NN = 3 * coutp; d.G0 = g0; d.G1 = g1;
  d.transposed = mode == 2; d.begin = begin; d.fold = 0; d.poly = mode;
  d.n0 = 0; d.nb = mode == 1 ? Cout : Ca; d.k0 = 0; d.kb = mode == 1 ? Cin : Cout;
  d.count = (int)(vxm_conv3d_tcs_poly_packed_bytes(mode, Cout, Cin, Ca) / sizeof(__nv_bfloat16));
  memcpy(desc_host, &d, sizeof(d));
  return d.count;
}

extern "C" int vxm_conv3d_tcs_pack_multi(const void* descs_dev, int ndesc, int total, void* stream) {
  VXM_REQUIRE(descs_dev && ndesc > 0 && total > 0, "conv3d_tcs_pack_multi: bad argument");
  const int blocks = (total + 255) / 256, cap = sm_count() * 8;
  pack_weights_multi_kernel<<<blocks < cap ? blocks : cap, 256, 0, as_stream(stream)>>>((const PackDesc*)descs_dev, ndesc, total);
  return check_launch("conv3d_tcs_pack_multi");
}

extern "C" int vxm_conv3d_tcs_supported(int Ca, int Cb, int Cout) {
  int cin = Ca + Cb;
  bool split_ok = cin != 48 || (Ca == 32 && Cb == 16) || Cb == 0 || Ca == 0;   // 48 = 32 + 16 channel groups
  return (Cout <= 64) && (cin == 8 || cin == 16 || cin == 32 || cin == 48 || cin == 64) && Ca % 8 == 0 && Cb % 8 == 0 && split_ok;
}

static int conv_tcs_launch(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, const void* mask,
                           int B, int D, int H, int W, int Ca, int Cb, int up, int Cout, int coutp, int kd, int out_mode,
                           float slope, void* out2, int csplit, const float* acc_in, void* out_lo, int opitch, int poly,
                           void* stream);

// Polyphase launches (conv_tcs_kernel PD, operands from vxm_conv3d_tcs_pack_desc_poly).  mode 1: forward of a
// (32 upsampled + 16) -> 32 concat layer, bias + LeakyReLU, bf16 (B, D, H, W, 32) out; xa is the coarse source, (D, H, W)
// the fine grid.  mode 2: xa = the 32-channel gradient (B, D, H, W, 32) of a layer whose first 32 input channels are an
// upsampled source, mask = that source (B, D / 2, H / 2, W / 2, 32), its LeakyReLU activation; out = the gradient w.r.t.
// it, (B, D / 2, H / 2, W / 2, 32), times the LeakyReLU derivative (slope).
extern "C" int vxm_conv3d_tcs_poly(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, const void* mask, int B,
                                   int D, int H, int W, int Ca, int Cb, int Cout, int mode, float slope, void* stream) {
  VXM_REQUIRE(mode == 1 || mode == 2, "conv3d_tcs_poly: mode must be 1 (forward) or 2 (coarse dgrad)");
  return conv_tcs_launch(xa, xb, wpk, bias, out, mask, B, D, H, W, Ca, Cb, mode == 1 ? 1 : 0, Cout, 32, 3, 0, slope, nullptr, 0,
                         nullptr, nullptr, 0, mode, stream);
}

// shared memory of one launch outside the slab ring: packed weights, accumulator read-out buffers, barriers
static size_t fixed_smem(uint32_t wbytes) { return ((wbytes + 1023u) & ~1023u) + NGRP * ACC_STAGE_FLOATS * sizeof(float) + 1024 + 512; }

extern "C" int vxm_conv3d_tcs_fits(int cin, int coutp, int kd) {
  int g0, g1;
  groups_of(cin <= 8 ? 8 : (cin <= 16 ? 16 : (cin <= 32 ? 32 : (cin <= 48 ? 48 : 64))), &g0, &g1);
  const size_t slab4 = (size_t)6 * WT * (g0 + g1) * 2;
  return fixed_smem((uint32_t)vxm_conv3d_tcs_packed_bytes(cin, coutp, kd)) + 4 * slab4 <= 227 * 1024;
}

extern "C" int vxm_conv3d_tcs_fwd(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, const void* mask,
                                  int B, int D, int H, int W, int Ca, int Cb, int up, int Cout, int coutp, int kd, int out_mode,
                                  float slope, void* out2, int csplit, void* stream) {
  VXM_REQUIRE(out_mode == 0 || out_mode == 1, "conv3d_tcs_fwd: out_mode must be 0 (bf16 channels-last) or 1 (fp32 planar)");
  return conv_tcs_launch(xa, xb, wpk, bias, out, mask, B, D, H, W, Ca, Cb, up, Cout, coutp, kd, out_mode, slope, out2, csplit,
                         nullptr, nullptr, 0, 0, stream);
}

extern "C" int vxm_conv3d_tcs_fwd_blk(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, void* out_lo,
                                      const void* mask, const float* acc_in, int B, int D, int H, int W, int Ca, int Cb, int up, int Cout,
                                      int coutp, int kd, int out_mode, float slope, int opitch, void* stream) {
  VXM_REQUIRE(out_mode == 0 || out_mode == 2 || out_mode == 3, "conv3d_tcs_fwd_blk: out_mode must be 0 (bf16), 2 (fp32 partial sums) or 3 (bf16 hi/lo pair)");
  VXM_REQUIRE(out_mode != 3 || out_lo, "conv3d_tcs_fwd_blk: out_mode 3 needs out_lo");
  VXM_REQUIRE(opitch == 0 || (opitch >= Cout && opitch % 8 == 0 && out_mode != 2), "conv3d_tcs_fwd_blk: bad output pitch %d", opitch);
  return conv_tcs_launch(xa, xb, wpk, bias, out, mask, B, D, H, W, Ca, Cb, up, Cout, coutp, kd, out_mode, slope, nullptr, 0,
                         acc_in, out_lo, opitch == Cout ? 0 : opitch, 0, stream);
}

extern "C" int vxm_conv3d_tcs_fwd_acc(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, void* out_lo,
                                      const float* acc_in, int B, int D, int H, int W, int Ca, int Cb, int up, int Cout, int coutp,
                                      int kd, int out_mode, float slope, void* stream) {
  VXM_REQUIRE(out_mode >= 1 && out_mode <= 3, "conv3d_tcs_fwd_acc: out_mode must be 1 (fp32 planar), 2 (fp32 partial sums) or 3 (bf16 hi/lo pair)");
  VXM_REQUIRE(out_mode != 3 || out_lo, "conv3d_tcs_fwd_acc: out_mode 3 needs out_lo");
  return conv_tcs_launch(xa, xb, wpk, bias, out, nullptr, B, D, H, W, Ca, Cb, up, Cout, coutp, kd, out_mode, slope, nullptr, 0,
                         acc_in, out_lo, 0, 0, stream);
}

static int conv_tcs_launch(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, const void* mask,
                           int B, int D, int H, int W, int Ca, int Cb, int up, int Cout, int coutp, int kd, int out_mode,
                           float slope, void* out2, int csplit, const float* acc_in, void* out_lo, int opitch, int poly,
                           void* stream) {
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0 && wpk && out, "conv3d_tcs_fwd: bad argument");
  VXM_REQUIRE(kd == 1 || kd == 3, "conv3d_tcs_fwd: kd must be 1 or 3");
  VXM_REQUIRE(coutp == 16 || coutp == 32 || coutp == 48 || coutp == 64, "conv3d_tcs_fwd: padded Cout must be 16, 32, 48 or 64");
  VXM_REQUIRE(!out2 || (out_mode == 0 && csplit > 0 && csplit < Cout && csplit % 8 == 0 && !mask), "conv3d_tcs_fwd: bad output split");
  VXM_REQUIRE(Cout > 0 && Cout <= coutp && (out_mode == 1 || out_mode == 2 || Cout % 8 == 0), "conv3d_tcs_fwd: unsupported Cout %d", Cout);
  VXM_REQUIRE(vxm_conv3d_tcs_supported(Ca, Cb, Cout), "conv3d_tcs_fwd: channel counts (%d,%d)->%d unsupported", Ca, Cb, Cout);
  VXM_REQUIRE((Ca == 0 || xa) && (Cb == 0 || xb), "conv3d_tcs_fwd: missing source tensor");
  VXM_REQUIRE(!up || (H % 2 == 0 && W % 2 == 0 && (kd == 1 || D % 2 == 0)), "conv3d_tcs_fwd: upsampled source needs even sizes");
  VXM_REQUIRE(poly == 0 || (kd == 3 && coutp == 32 && Cout == 32 && out_mode == 0 && !out2 && !acc_in && !opitch &&
                            (poly == 1 ? up && Ca == 32 && Cb == 16 && bias && !mask && slope >= 0.f && slope <= 1.f
                                       : !up && Ca == 32 && Cb == 0 && !bias && mask && D % 2 == 0 && H % 2 == 0 && W % 2 == 0)),
              "conv3d_tcs_poly: no polyphase mode %d kernel for (%d,%d)->%d", poly, Ca, Cb, Cout);
  ConvSArgs a{};
  const int cin = Ca + Cb;
  int g0, g1;
  groups_of(cin, &g0, &g1);
  a.xa = (const __nv_bfloat16*)xa; a.xb = (const __nv_bfloat16*)xb; a.wpk = (const __nv_bfloat16*)wpk; a.bias = bias;
  a.out = out; a.mask = (const __nv_bfloat16*)mask; a.out2 = out2; a.csplit = csplit;
  a.acc_in = acc_in; a.out_lo = out_lo;
  a.B = B; a.D = D; a.H = H; a.W = W; a.Ca = Ca; a.Cb = Cb; a.up = up; a.upd = (up && kd == 3) ? 1 : 0;
  a.Cout = Cout; a.out_mode = out_mode; a.slope = slope; a.opitch = opitch;
  // the channel-blocked launches: 32-channel blocks of a 3-D layer, K groups of 64 or 32 + 16 channels (see tc.conv_blocks)
  VXM_REQUIRE(!opitch || (!out2 && out_mode != 1 && kd == 3 && coutp == 32 && ((g0 == 64 && g1 == 0) || (g0 == 32 && g1 == 16))),
              "conv3d_tcs_fwd: no blocked kernel for (%d,%d)->%d/%d, kd %d", Ca, Cb, Cout, coutp, kd);
  a.wbytes = (uint32_t)(poly ? poly_bytes(poly) : vxm_conv3d_tcs_packed_bytes(cin, coutp, kd));
  const size_t fixed = fixed_smem(a.wbytes);
  // tile height: 8 rows (two tile halves per slab step, one per MMA warpgroup) when the ring still holds >= 5 slabs
  int HTv = 4;
  {
    const size_t slab8 = (size_t)10 * WT * (g0 + g1) * 2;
    const int ns8 = (int)((227 * 1024 - fixed) / slab8);
    if (g0 <= 32 && coutp <= 32 && ns8 >= (kd == 3 ? 5 : 3) && H > 4 && !opitch) HTv = 8;
    if (poly) HTv = poly == 2 ? 8 : 4;               // the polyphase kernels exist at one tile height each
  }
  a.tiles_h = (H + HTv - 1) / HTv; a.tiles_w = (W + WUSE - 1) / WUSE;
  int nsm = conv_ctas();
  // depth chunking: balance the persistent CTAs (waves of nsm items) against the 2 halo slabs every chunk re-loads
  const long long tiles = (long long)B * a.tiles_h * a.tiles_w;
  // (the coarse dgrad: output slices of 2 fine slabs each, so the halo weighs half as much)
  const int Do = poly == 2 ? D / 2 : D;
  a.dchunk = depth_chunk(Do, tiles, nsm, poly == 2 ? 1.25 : (kd == 3 ? 2.5 : 0.5), 40);
  a.nchunks = (Do + a.dchunk - 1) / a.dchunk;
  a.nitems = (int)(tiles * a.nchunks);
  const size_t slab = (size_t)(HTv + 2) * WT * (g0 + g1) * 2;
  int nslot = (int)((227 * 1024 - fixed) / slab);
  // ring depth: the slabs of up to 13 steps ahead (16-channel layers) hide the L2 / HBM latency of the tensor copies
  if (nslot > MAXSLOT) nslot = MAXSLOT;
  VXM_REQUIRE(nslot >= 4, "conv3d_tcs_fwd: not enough shared memory for the slab ring");
  a.nslot = nslot;
  size_t smem = fixed + (size_t)nslot * slab;
  int grid = a.nitems < nsm ? a.nitems : nsm;
  cudaStream_t st = as_stream(stream);
  if (poly != 2 && plan_tma(a, g0, g1, HTv) != 0) return VXM_ERR_CUDA;   // (the coarse dgrad permutes its slab rows)
  const bool acc_epi = acc_in != nullptr || out_mode >= 2;
  // epilogue specialisation: bf16 channels-last output with every padded channel real (EPI 1-3; KD = 1: 1 and 2, up to
  // 32 outputs), or the fp32 planar output (EPI 4, up to 32 padded outputs, one 16- or 32-channel input group)
  int epi = 0;
  {
    const char* e = getenv("VXM_B200_TCS_EPI");       // "0": generic epilogue everywhere (A/B switch)
    const bool spec = !acc_epi && !(e && e[0] == '0');
    const bool plain = spec && out_mode == 0 && Cout == coutp && (kd == 3 || coutp <= 32);
    if (plain && !out2 && !mask && slope >= 0.f && slope <= 1.f) epi = 1;
    else if (plain && !out2 && mask && !bias) epi = 2;
    else if (plain && kd == 3 && !mask && !bias && slope < 0.f && (!out2 || csplit % 16 == 0)) epi = 3;
    else if (spec && out_mode == 1 && !out2 && coutp <= 32 && g0 <= 32 && g1 == 0) epi = 4;
    if (poly) epi = poly;               // the polyphase forms exist with their specialised epilogue only
  }
#define VXM_TCS_LAUNCH_E(KD_, G0_, G1_, CO_, HT_, ACC_, E_, ...)                                                                  \
  do {                                                                                                                            \
    VXM_CUDA(cudaFuncSetAttribute(conv_tcs_kernel<KD_, G0_, G1_, CO_, HT_, ACC_, E_, ##__VA_ARGS__>,                              \
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                                       \
    conv_tcs_kernel<KD_, G0_, G1_, CO_, HT_, ACC_, E_, ##__VA_ARGS__><<<grid, NTHREADS, smem, st>>>(a);                           \
  } while (0)
#define VXM_TCS_LAUNCH_OP(G0_, G1_)                                                                                               \
  do {                                                                                                                            \
    if (acc_epi) VXM_TCS_LAUNCH_E(3, G0_, G1_, 32, 4, true, 0, true);                                                             \
    else if (epi == 1) VXM_TCS_LAUNCH_E(3, G0_, G1_, 32, 4, false, 1, true);                                                      \
    else if (epi == 2) VXM_TCS_LAUNCH_E(3, G0_, G1_, 32, 4, false, 2, true);                                                      \
    else if (epi == 3) VXM_TCS_LAUNCH_E(3, G0_, G1_, 32, 4, false, 3, true);                                                      \
    else VXM_TCS_LAUNCH_E(3, G0_, G1_, 32, 4, false, 0, true);                                                                    \
  } while (0)
// which specialised instantiations exist (the others' dead branches name the generic one): EPI 1 / 2 with KD = 1 up to 32
// outputs, EPI 4 up to 32 outputs over one 16- or 32-channel group
#define VXM_TCS_KD1(KD_, CO_) ((KD_) == 3 || (CO_) <= 32)
#define VXM_TCS_PL(G0_, G1_, CO_) ((CO_) <= 32 && (G0_) <= 32 && (G1_) == 0)
#define VXM_TCS_LAUNCH(KD_, G0_, G1_, CO_, HT_)                                                                                   \
  do {                                                                                                                            \
    if (acc_epi) VXM_TCS_LAUNCH_E(KD_, G0_, G1_, CO_, HT_, true, 0);                                                              \
    else if (VXM_TCS_KD1(KD_, CO_) && epi == 1) VXM_TCS_LAUNCH_E(KD_, G0_, G1_, CO_, HT_, false, VXM_TCS_KD1(KD_, CO_) ? 1 : 0);  \
    else if (VXM_TCS_KD1(KD_, CO_) && epi == 2) VXM_TCS_LAUNCH_E(KD_, G0_, G1_, CO_, HT_, false, VXM_TCS_KD1(KD_, CO_) ? 2 : 0);  \
    else if (KD_ == 3 && epi == 3) VXM_TCS_LAUNCH_E(3, G0_, G1_, CO_, HT_, false, 3);                                             \
    else if (VXM_TCS_PL(G0_, G1_, CO_) && epi == 4) VXM_TCS_LAUNCH_E(KD_, G0_, G1_, CO_, HT_, false, VXM_TCS_PL(G0_, G1_, CO_) ? 4 : 0); \
    else VXM_TCS_LAUNCH_E(KD_, G0_, G1_, CO_, HT_, false, 0);                                                                     \
  } while (0)
#define VXM_TCS_G8(KD_, CO_)                                                  \
  do {                                                                        \
    if (g0 == 16) VXM_TCS_LAUNCH(KD_, 16, 0, CO_, 8);                         \
    else if (g0 == 32 && g1 == 0) VXM_TCS_LAUNCH(KD_, 32, 0, CO_, 8);         \
    else VXM_TCS_LAUNCH(KD_, 32, 16, CO_, 8);                                 \
  } while (0)
#define VXM_TCS_G(KD_, CO_)                                                   \
  do {                                                                        \
    if (g0 == 16) VXM_TCS_LAUNCH(KD_, 16, 0, CO_, 4);                         \
    else if (g0 == 32 && g1 == 0) VXM_TCS_LAUNCH(KD_, 32, 0, CO_, 4);         \
    else if (g0 == 32) VXM_TCS_LAUNCH(KD_, 32, 16, CO_, 4);                   \
    else VXM_TCS_LAUNCH(KD_, 64, 0, CO_, 4);                                  \
  } while (0)
  if (poly) {
    if (poly == 1) VXM_TCS_LAUNCH_E(3, 32, 16, 32, 4, false, 1, false, 1);
    else VXM_TCS_LAUNCH_E(3, 32, 0, 32, 8, false, 2, false, 2);
  } else if (opitch) {
    if (g0 == 64) VXM_TCS_LAUNCH_OP(64, 0); else VXM_TCS_LAUNCH_OP(32, 16);
  } else if (HTv == 8) {
    if (kd == 3) { if (coutp == 16) VXM_TCS_G8(3, 16); else VXM_TCS_G8(3, 32); }
    else { if (coutp == 16) VXM_TCS_G8(1, 16); else VXM_TCS_G8(1, 32); }
  } else if (kd == 3) { if (coutp == 16) VXM_TCS_G(3, 16); else if (coutp == 32) VXM_TCS_G(3, 32); else if (coutp == 48) VXM_TCS_G(3, 48); else VXM_TCS_G(3, 64); }
  else { if (coutp == 16) VXM_TCS_G(1, 16); else if (coutp == 32) VXM_TCS_G(1, 32); else if (coutp == 48) VXM_TCS_G(1, 48); else VXM_TCS_G(1, 64); }
  return check_launch("conv3d_tcs_fwd");
}
