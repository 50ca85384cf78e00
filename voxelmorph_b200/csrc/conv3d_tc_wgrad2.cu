// Weight gradient of the k=3 convolution on the Hopper tensor cores (wgmma), "kw-stacked Toeplitz" formulation:
//     gw[kd][kh][kw][ci][co] = sum_{b,v} x[b, v + (kd,kh,kw) - 1, ci] * gz[b, v, co]
// (autograd of nn.Conv3d at reference voxelmorph/torch/networks.py:299,211; gz = grad wrt the conv output).
//
// Both operands are staged exactly like the forward kernel's A operand (conv3d_tc_s.cu): one shared-memory row per
// voxel, the channels of the row contiguous (32 or 64 bytes) and XOR-swizzled, rows of a 32-voxel-wide (h, w) tile
// in linear order.  Read "MN-major" (MN = channels, K = voxels) the same bytes are a valid wgmma operand, and a
// one-voxel shift of the window is a one-row shift of the start address.  One MMA then covers 16 voxels (K) and
//   M = (kd, ci) : the x slabs of input slices d-1, d, d+1 are adjacent in the ring, so the three kd taps are three
//                  MN atoms one slab apart (leading byte offset = slab pitch);
//   N = (kw, co) : the three kw taps are three MN atoms ONE ROW apart (leading byte offset = one row): the B operand
//                  is a Toeplitz view of the single gz slab, nothing is copied;
//   kh           : three accumulators, the A window start moves by one 32-voxel tile row.
// 24 MMAs per (tile, slice) instead of 72-216 in conv3d_tc_wgrad.cu, each with N = 48 or 96 instead of 16 or 32.
// The x slab keeps its halo columns, the gz slab has ZERO halo columns (and zero pad rows before and after), so the
// products that pair a voxel with a neighbour across the tile-row wrap vanish.
// All 3 (kh) x [M x 3*GOUT] fp32 accumulators stay in the registers of two MMA warpgroups for the CTA's whole lifetime
// (M = 128: one m64 half each; M = 64: kh 0-1 / kh 2); each CTA writes ONE partial
// [27][G][GOUT]; wgrad2_reduce_multi_kernel sums the partials in fixed order (deterministic).  The first MMA warpgroup also
// folds the bias gradient (sum of gz) out of the staged gz rows while its wgmma chain runs.
#include <stdlib.h>

#include <type_traits>

#include "tc_common.cuh"

namespace vxm {
namespace tcw {

using namespace vxm::tc;

constexpr int TH = 4, TWR = 32, TUSE = 30;
constexpr int XROWS = (TH + 2) * TWR;                       // 192 voxel rows per x slab
constexpr int GPAD = 16, GROWS = TH * TWR, GSROWS = GROWS + 2 * GPAD;   // gz slab: 16 zero rows, 128 rows, 16 zero rows
constexpr int MAXSLOT = 8, NGS = 4;
constexpr int NLOADER = 128, NTHREADS = 384;   // warps 0-3 / 4-7: MMA warpgroups (0-3 also sum the bias), 8-11: loader

struct Wgrad2Args {
  const __nv_bfloat16* x; int Cx, up, upd;   // (B, Dx, Hx, Wx, Cx) bf16, Cx in {8,16,32}; up: nearest x2 (H, W), upd: also D
  const __nv_bfloat16* gz; int Cg;           // (B, D, H, W, Cg) bf16, Cg in {8,16,32}
  float* partial;                            // [grid][T][G][GOUT]
  float* bias_partial;                       // [grid][GOUT] or null
  int B, D, H, W;
  int tiles_h, tiles_w, dchunk, nchunks, nitems, nslot;
  int xpitch, gpitch;   // channels per voxel of the x / gz tensors (> Cx / Cg: a channel slice of a wider tensor)
};

__host__ __device__ inline uint32_t swz(uint32_t off, uint32_t width) { return off ^ (((off >> 7) & (width / 16 - 1)) << 4); }

// MN-major swizzled operand: rows of WIDTH bytes (one voxel, WIDTH/2 channels = one MN atom), 8-row K groups contiguous
// (SBO = 8 * WIDTH), MN atoms `lbo_bytes` apart.  cute make_umma_desc<Major::MN>: LBO = atom stride, SBO = K-group stride.
template <int WIDTH>
__device__ __forceinline__ uint64_t make_desc_mn_swz(uint32_t saddr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)(((8u * WIDTH) >> 4) & 0x3FFF) << 32;
  return d | desc_swizzle(WIDTH);    // base offset 0: the swizzle is a function of the absolute address
}

// KHM ("kh in M", KD == 1 only): the three kh taps become three MN atoms of the A operand ONE TILE ROW (32 voxel rows) apart —
// the same Toeplitz trick the B operand plays for kw — so a (tile, slice) costs 8 MMAs with one accumulator instead of 24
// with three.  Used for the layers whose kd taps are folded into the channels of one operand (first layer: 2 image planes
// x 3 slices; flow head: 3 flow-gradient planes x 3 slices), i.e. exactly the layers that otherwise pad 2 or 3 real
// channels to 16.
template <int KD, int G, int GOUT, bool KHM = false>
__global__ void __launch_bounds__(NTHREADS, 1) wgrad2_kernel(const Wgrad2Args a) {
  static_assert(!KHM || (KD == 1 && G == 16), "kh-in-M needs a 2-D operand with 16-channel rows");
  constexpr int WA = 2 * G, WG = 2 * GOUT;                  // row bytes
  constexpr uint32_t XSLAB = XROWS * WA, GSLAB = GSROWS * WG;
  constexpr int MM = (KD * G > 64) ? 128 : 64;              // KHM: M = (kh, ci) = 48 -> 64
  constexpr int NN = 3 * GOUT;
  constexpr int NMIRROR = KD == 3 ? 2 : 0, NPADSLAB = KD == 3 ? 1 : 0;
  constexpr int T = KD * 9;
  constexpr int KX = XROWS * (G / 8) / NLOADER, KG = GROWS * (GOUT / 8) / NLOADER;
  static_assert(XROWS * (G / 8) % NLOADER == 0 && GROWS * (GOUT / 8) % NLOADER == 0, "loader tables");
  // Accumulators (fp32, registers): MM = 128 -> warpgroup g owns rows 64g..64g+63 of all three kh accumulators;
  // MM = 64 -> warpgroup 0 owns kh = 0, 1 and warpgroup 1 kh = 2; KHM -> warpgroup 0 owns the single accumulator.
  constexpr int NPART = KHM ? 1 : 2;                          // warpgroups that issue MMAs
  constexpr int NKH = KHM ? 1 : (MM == 128 ? 3 : 2);          // accumulators per warpgroup

  extern __shared__ __align__(1024) uint8_t smem[];
  const int NS = a.nslot;
  uint8_t* s_x = smem;
  uint8_t* s_g = s_x + (size_t)(NS + NMIRROR + NPADSLAB) * XSLAB;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_g + NGS * GSLAB);
  uint64_t* xfull = bars;
  uint64_t* xempty = bars + MAXSLOT;
  uint64_t* gfull = bars + 2 * MAXSLOT;
  uint64_t* gempty = gfull + NGS;
  float* s_bsum = reinterpret_cast<float*>(bars) + 128;     // [128 rows][GOUT + 1]: bias sums (after 512 bytes of barriers)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // the gz slabs' pad rows (and everything else there) start as zeros; the loader only ever writes rows GPAD..GPAD+127
  for (uint32_t i = threadIdx.x * 16u; i < NGS * GSLAB; i += NTHREADS * 16u) *reinterpret_cast<uint4*>(s_g + i) = make_uint4(0u, 0u, 0u, 0u);
  if (NPADSLAB)   // the M atom past the kd window reads one more slab: keep it finite
    for (uint32_t i = threadIdx.x * 16u; i < XSLAB; i += NTHREADS * 16u)
      *reinterpret_cast<uint4*>(s_x + (size_t)(NS + NMIRROR) * XSLAB + i) = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async();
  if (threadIdx.x == 0) {
    // one arrival per warp of every MMA warpgroup, after its last MMA reading the slab has completed
    for (int i = 0; i < NS; ++i) { mbar_init(&xfull[i], NLOADER); mbar_init(&xempty[i], 4 * NPART); }
    for (int i = 0; i < NGS; ++i) { mbar_init(&gfull[i], NLOADER); mbar_init(&gempty[i], 4 * NPART); }
    fence_barrier_init();
  }
  __syncthreads();
  const int HW_tiles = a.tiles_h * a.tiles_w;
  const bool has_work = blockIdx.x < a.nitems;

  if (warp >= 8) {
    // ================================ LOADER (128 threads) ================================
    setmaxnreg_dec<64>();
    const int lt = threadIdx.x - 8 * 32;
    uint32_t xslot = 0, xphase = 1, gslot = 0, gphase = 1;    // producer side: first lap passes on the fresh barriers
    const int Dx = a.upd ? a.D >> 1 : a.D, Hx = a.up ? a.H >> 1 : a.H, Wx = a.up ? a.W >> 1 : a.W;
    const int ncx = a.Cx >> 3, ncg = a.Cg >> 3;
    for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
      const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
      const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
      const int h0 = ht * TH, w0 = wt * TUSE, d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, a.D);
      const int s_begin = KD == 3 ? d0 - 1 : d0, s_end = KD == 3 ? d1 + 1 : d1;
      int soff[KX];
      uint32_t doff[KX];
#pragma unroll
      for (int k = 0; k < KX; ++k) {
        const int id = lt + k * NLOADER;
        const int c8 = id % (G / 8), row = id / (G / 8);
        const int h = h0 - 1 + (row >> 5), w = w0 - 1 + (row & 31);
        doff[k] = swz((uint32_t)row * WA + (uint32_t)c8 * 16u, WA);
        soff[k] = -1;
        if (h >= 0 && h < a.H && w >= 0 && w < a.W && c8 < ncx) soff[k] = ((a.up ? h >> 1 : h) * Wx + (a.up ? w >> 1 : w)) * a.xpitch + c8 * 8;
      }
      int goff[KG];
      uint32_t gdoff[KG];
#pragma unroll
      for (int k = 0; k < KG; ++k) {
        const int id = lt + k * NLOADER;
        const int c8 = id % (GOUT / 8), row = id / (GOUT / 8);
        const int jj = row & 31, h = h0 + (row >> 5), w = w0 - 1 + jj;
        gdoff[k] = swz((uint32_t)(GPAD + row) * WG + (uint32_t)c8 * 16u, WG);
        goff[k] = -1;
        if (jj >= 1 && jj <= TUSE && h < a.H && w < a.W && c8 < ncg) goff[k] = (h * a.W + w) * a.gpitch + c8 * 8;
      }
      for (int ds = s_begin; ds < s_end; ++ds) {
        // ---- x slab of input slice ds ----
        mbar_wait(&xempty[xslot], xphase);
        uint8_t* slab = s_x + (size_t)xslot * XSLAB;
        const bool dok = ds >= 0 && ds < a.D;
        const __nv_bfloat16* base = a.x + (((size_t)b * Dx + (dok ? (a.upd ? ds >> 1 : ds) : 0)) * Hx * Wx) * a.xpitch;
#pragma unroll
        for (int k = 0; k < KX; ++k) {
          const bool ok = dok && soff[k] >= 0;
          const __nv_bfloat16* src = ok ? base + soff[k] : a.x;
          cp_async16(slab + doff[k], src, ok ? 16u : 0u);
          if (NMIRROR && xslot < (uint32_t)NMIRROR) cp_async16(slab + (size_t)NS * XSLAB + doff[k], src, ok ? 16u : 0u);
        }
        cp_async_arrive_noinc(&xfull[xslot]);
        if (++xslot == (uint32_t)NS) { xslot = 0; xphase ^= 1; }
        // ---- gz slab of OUTPUT slice dg (the slice whose kd window this x slab completes) ----
        const int dg = KD == 3 ? ds - 1 : ds;
        if (dg >= d0 && dg < d1) {
          mbar_wait(&gempty[gslot], gphase);
          uint8_t* gt = s_g + (size_t)gslot * GSLAB;
          const __nv_bfloat16* baseG = a.gz + (((size_t)b * a.D + dg) * a.H * a.W) * a.gpitch;
#pragma unroll
          for (int k = 0; k < KG; ++k) {
            const bool ok = goff[k] >= 0;
            cp_async16(gt + gdoff[k], ok ? baseG + goff[k] : a.gz, ok ? 16u : 0u);
          }
          cp_async_arrive_noinc(&gfull[gslot]);
          if (++gslot == NGS) { gslot = 0; gphase ^= 1; }
        }
      }
    }
  } else {
    // ================================ MMA WARPGROUPS ================================
    setmaxnreg_inc<216>();
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    float acc[NKH][NN / 2];
    // warpgroup 0 also folds the bias gradient out of the staged gz slabs: thread t owns gz slab row t and its row of
    // s_bsum (shared memory, not registers: the accumulators of the widest layer need them all)
    float* bsum = s_bsum + t * (GOUT + 1);
    if (wg == 0)
#pragma unroll
      for (int c = 0; c < GOUT; ++c) bsum[c] = 0.f;
    const bool do_bias = wg == 0 && a.bias_partial;
    uint32_t roff[GOUT / 8];
#pragma unroll
    for (int c8 = 0; c8 < GOUT / 8; ++c8) roff[c8] = swz((uint32_t)(GPAD + t) * WG + (uint32_t)c8 * 16u, WG);
    if (has_work && wg < NPART) {
      const uint32_t x_u32 = smem_u32(s_x), g_u32 = smem_u32(s_g);
      uint32_t wslot = 0, wphase = 0;   // next x slab to wait for
      uint32_t hslot = 0;               // head of the kd window
      uint32_t gs = 0, gph = 0;
      uint32_t acc0 = 0;                // 0 only for the very first (tile, slice) of this CTA
      // MM = 128: rows 64-127 (warpgroup 1) are M atoms 2 and 3 of the kd window, two atom strides further
      const uint32_t m_off = (MM == 128 && wg == 1) ? 2u * XSLAB : 0u;
      for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
        const int ch = (item / HW_tiles) % a.nchunks;
        const int nd = min(ch * a.dchunk + a.dchunk, a.D) - ch * a.dchunk;
        for (int j = 0; j < nd; ++j) {
          const int nwait = (KD == 3 && j == 0) ? 3 : 1;
          for (int q = 0; q < nwait; ++q) {
            mbar_wait(&xfull[wslot], wphase);
            if (++wslot == (uint32_t)NS) { wslot = 0; wphase ^= 1; }
          }
          mbar_wait(&gfull[gs], gph);
          const uint32_t a_start = x_u32 + hslot * XSLAB + m_off;
          const uint32_t b_start = g_u32 + gs * GSLAB + (uint32_t)(GPAD - 1) * WG;
          const uint64_t adesc0 = make_desc_mn_swz<WA>(a_start, KHM ? (uint32_t)(TWR * WA) : (KD == 3 ? XSLAB : 0u));
          const uint64_t bdesc0 = make_desc_mn_swz<WG>(b_start, (uint32_t)WG);
          // one straight-line wgmma chain per warpgroup role (no warpgroup-divergent branch inside a chain): NK
          // accumulators for the consecutive kh taps kh0 .. kh0 + NK - 1
          auto chain = [&](auto nk, int kh0) {
            constexpr int NK = decltype(nk)::value;
            wg_fence();
#pragma unroll
            for (int s = 0; s < NK; ++s) {
#pragma unroll
              for (int i = 0; i < GROWS / 16; ++i) {
                const uint64_t adesc = adesc0 + (uint64_t)((((kh0 + s) * TWR + 16 * i) * WA) >> 4);
                const uint64_t bdesc = bdesc0 + (uint64_t)((16 * i * WG) >> 4);
                Wgmma<NN, 1, 1>::mma(acc[s], adesc, bdesc, i == 0 ? acc0 : 1u);
              }
            }
            wg_commit();
          };
          if (MM == 128 || KHM || wg == 0) chain(std::integral_constant<int, NKH>{}, 0);
          else chain(std::integral_constant<int, 1>{}, 2);    // warpgroup 1 of an M = 64 layer: kh = 2
          if (do_bias) {
            const uint8_t* gt = s_g + (size_t)gs * GSLAB;
#pragma unroll
            for (int c8 = 0; c8 < GOUT / 8; ++c8) {
              const uint4 q = *reinterpret_cast<const uint4*>(gt + roff[c8]);
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
            mbar_arrive(&xempty[hslot]);
            mbar_arrive(&gempty[gs]);
          }
          acc0 = 1u;
          if (++hslot == (uint32_t)NS) hslot = 0;
          if (++gs == NGS) { gs = 0; gph ^= 1; }
        }
        if (KD == 3) {
          if (lane == 0) {
            mbar_arrive(&xempty[hslot]);
            mbar_arrive(&xempty[hslot + 1 == (uint32_t)NS ? 0 : hslot + 1]);
          }
          hslot = hslot + 2 >= (uint32_t)NS ? hslot + 2 - NS : hslot + 2;
        }
      }
    }
    float* part = a.partial + (size_t)blockIdx.x * T * G * GOUT;
    if (!has_work) {
      if (wg == 0)
        for (int i = t; i < T * G * GOUT; i += 128) part[i] = 0.f;
    } else if (wg < NPART) {
      // fragment (row m, column n) of accumulator s: m = (kd, ci) (KHM: (kh, ci)), n = q * GOUT + co with kw = 2 - q
      const int w4 = t >> 5, qr = lane >> 2, pc = lane & 3;
#pragma unroll
      for (int s = 0; s < NKH; ++s) {
        const int kh = KHM ? 0 : (MM == 128 ? s : (wg == 0 ? s : 2));
        if (MM != 128 && !KHM && wg == 1 && s > 0) break;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int m = (MM == 128 ? 64 * wg : 0) + 16 * w4 + 8 * i + qr;
          const int kd = KHM ? 0 : m / G, ci = m % G, khm = KHM ? m / G : kh;
          if (kd >= KD || khm >= 3) continue;
#pragma unroll
          for (int jn = 0; jn < NN / 8; ++jn) {
            const int n = 8 * jn + 2 * pc, q = n / GOUT, co = n % GOUT;
            const int tap = (kd * 3 + khm) * 3 + (2 - q);
            *reinterpret_cast<float2*>(part + ((size_t)tap * G + ci) * GOUT + co) = make_float2(acc[s][4 * jn + 2 * i], acc[s][4 * jn + 2 * i + 1]);
          }
        }
      }
    }
    if (wg == 0 && a.bias_partial) {
      // bias partial of this CTA: fixed-order reduction over the 128 rows
      named_bar(1, 128);
      if (t < GOUT) {
        float sum = 0.f;
        for (int r2 = 0; r2 < 128; ++r2) sum += s_bsum[r2 * (GOUT + 1) + t];
        a.bias_partial[(size_t)blockIdx.x * GOUT + t] = sum;
      }
    }
  }
}

// ---- weight gradient of a nearest-x2 upsampled 32-channel source, on the coarse voxels ---------------------------------
// With u = up(x) and tap offset t in {-1, 0, +1} per axis,
//     gw[t][ci][co] = sum_v u[v + t][ci] gz[v][co] = sum_c x[c + s(t)][ci] G_a(t)[c][co],
// where per axis t = 0 -> (E, s = 0), t = +1 -> (O, s = 0), t = -1 -> (O, s = -1), E[c] = g[2c] + g[2c+1] and
// O[c] = g[2c-1] + g[2c] (c = 0 .. Dc; fine voxels outside the volume are zero, as is x[-1] and x[Dc]).  So 8 coarse
// pair-summed gradients G_{ad ah aw} (a = O or E per axis) replace the fine gz: a quarter of the fine form's K.
// The loader warpgroup streams the fine gz slices through a 3-slice shared-memory ring (cp.async; slice 2s+1 serves
// coarse slices s and s+1), forms G from it (fp32 sums), splits each value into bf16 hi + lo (G = hi + lo to ~2^-17
// relative, so the result differs from the fine form by fp32 re-association only) and writes 16 swizzled slabs per
// coarse slice; the x slabs are coarse, staged as in wgrad2_kernel.  MMA warpgroup k owns the depth tap kd = k
// ((O, -1), (E, 0), (O, 0)) and three accumulators, one per kh ((O, -1), (E, 0), (O, 0): the A window one tile row
// lower for s = 0).  Each is m64n64: M = (sw, ci) is a Toeplitz view of the x slab (two M atoms one row apart: x[w-1],
// x[w]), N = (aw, co) the O and E slabs; (sw = -1, E) is padding, so 3/4 of the MMA work is useful.  hi and lo are two
// MMAs into the same accumulator.  Per coarse voxel: 2 x 36864 MACs instead of the fine form's 8 x 27648 (1/3).
constexpr int PTH = 2, PTU = 31;                                 // coarse tile: 2 rows x 31 columns (+1 zero column)
constexpr int PXROWS = (PTH + 1) * TWR, PXR = PXROWS + 8;        // x slab: rows h0-1 .. h0+PTH-1, + 8 zero rows
// G slab: rows h0 .. h0+PTH-1.  The MMAs read one row past a slab: row 0 of the next slab (or of the zero tail after
// the last), which is always zero (column w0 - 1 belongs to the previous tile).
constexpr int PGROWS = PTH * TWR;
constexpr uint32_t PXSLAB = PXR * 64, PGSLAB = PGROWS * 64, PGSTAGE = 16 * PGSLAB;
// fine gz slice of a tile: rows 2h0-1 .. 2(h0+PTH)-1, columns 2w0-3 .. 2(w0+PTU)-1, 32 channels (16-byte chunks, unswizzled)
constexpr int PFROWS = 2 * PTH + 1, PFCOLS = 2 * TWR + 1, PFCHUNKS = PFROWS * PFCOLS * 4;
constexpr uint32_t PFSLICE = PFCHUNKS * 16;
constexpr int PNGS = 2, PNSLOT = 4, PMAXSLOT = 8, PNTHREADS = 512;   // warps 0-11: MMA warpgroups (kd = 0, 1, 2), 12-15: loader
constexpr size_t PSMEM = (size_t)PNGS * PGSTAGE + 512 + (size_t)PNSLOT * PXSLAB + 3 * PFSLICE + 512 + 128 * 8 * sizeof(float);

struct Wgrad2PolyArgs {
  const __nv_bfloat16* x; int xpitch;        // coarse (B, Dc, Hc, Wc, xpitch), channels [0, 32) used
  const __nv_bfloat16* gz; int Cg, gpitch;   // fine (B, D, H, W, gpitch), channels [0, Cg) used, Cg <= 32
  float* partial;                            // [grid][27][32][32]
  float* bias_partial;                       // [grid][32] or null
  int B, D, H, W, Dc, Hc, Wc;
  int tiles_h, tiles_w, dchunk, nchunks, nitems, nslot;
};

// G slab of (hi/lo, ad, ah, aw), index 0 = O, 1 = E per axis
__host__ __device__ constexpr int poly_slab(int hl, int ad, int ah, int aw) { return ((hl * 2 + ad) * 2 + ah) * 2 + aw; }

__global__ void __launch_bounds__(PNTHREADS, 1) wgrad2_poly_kernel(const Wgrad2PolyArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int NS = a.nslot;
  uint8_t* s_g = smem;
  uint8_t* s_x = s_g + PNGS * PGSTAGE + 512;                  // after the G stages' zero tail
  uint8_t* s_f = s_x + (size_t)NS * PXSLAB;                   // fine gz ring: slice f in slot f mod 3
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_f + 3 * PFSLICE);
  uint64_t* xfull = bars;
  uint64_t* xempty = bars + PMAXSLOT;
  uint64_t* gfull = bars + 2 * PMAXSLOT;
  uint64_t* gempty = gfull + PNGS;
  float* s_bsum = reinterpret_cast<float*>(bars) + 128;       // [128 loader threads][8]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // zero rows past every slab (never written by the loader) start as zeros
  for (uint32_t i = threadIdx.x * 16u; i < (uint32_t)(PNGS * PGSTAGE + 512 + NS * PXSLAB); i += PNTHREADS * 16u)
    *reinterpret_cast<uint4*>(smem + i) = make_uint4(0u, 0u, 0u, 0u);
  fence_proxy_async();
  if (threadIdx.x == 0) {
    for (int i = 0; i < NS; ++i) { mbar_init(&xfull[i], 128); mbar_init(&xempty[i], 12); }
    for (int i = 0; i < PNGS; ++i) { mbar_init(&gfull[i], 128); mbar_init(&gempty[i], 12); }
    fence_barrier_init();
  }
  __syncthreads();
  const int HW_tiles = a.tiles_h * a.tiles_w;
  const bool has_work = blockIdx.x < a.nitems;

  if (warp >= 12) {
    // ================================ LOADER (128 threads) ================================
    const int lt = threadIdx.x - 12 * 32;
    const int c8 = lt & 3;                      // this thread's 8 channels, for every unit it handles
    uint32_t xslot = 0, xphase = 1, gslot = 0, gphase = 1;
    float* bsum = s_bsum + lt * 8;              // this thread's bias sums (shared memory: the loader has no registers to spare)
#pragma unroll
    for (int e = 0; e < 8; ++e) bsum[e] = 0.f;
    const bool cok = c8 * 8 < a.Cg;
    for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
      const int wt = item % a.tiles_w, ht = (item / a.tiles_w) % a.tiles_h;
      const int ch = (item / HW_tiles) % a.nchunks, b = item / (HW_tiles * a.nchunks);
      const int h0 = ht * PTH, w0 = wt * PTU, d0 = ch * a.dchunk, d1 = min(d0 + a.dchunk, a.Dc + 1);
      constexpr int KX = PXROWS * 4 / 128;
      int soff[KX];
      uint32_t doff[KX];
#pragma unroll
      for (int k = 0; k < KX; ++k) {
        const int row = (lt + k * 128) >> 2;
        const int h = h0 - 1 + row / TWR, w = w0 - 1 + row % TWR;
        doff[k] = swz((uint32_t)row * 64u + (uint32_t)c8 * 16u, 64);
        soff[k] = (h >= 0 && h < a.Hc && w >= 0 && w < a.Wc) ? (h * a.Wc + w) * a.xpitch + c8 * 8 : -1;
      }
      // fine slice f into its ring slot (one cp.async group per call, empty when not needed)
      auto load_fine = [&](int f, bool need) {
        if (need) {
          uint8_t* dst = s_f + (size_t)((f + 3) % 3) * PFSLICE;
          const bool fok = f >= 0 && f < a.D;
          for (int idx = lt; idx < PFCHUNKS; idx += 128) {
            const int r = idx / (PFCOLS * 4), rem = idx - r * (PFCOLS * 4), col = rem >> 2, cc = rem & 3;
            const int fh = 2 * h0 - 1 + r, fw = 2 * w0 - 3 + col;
            const bool ok = fok && fh >= 0 && fh < a.H && fw >= 0 && fw < a.W && cc * 8 < a.Cg;
            cp_async16(dst + (size_t)idx * 16, ok ? a.gz + ((((size_t)b * a.D + f) * a.H + fh) * a.W + fw) * a.gpitch + cc * 8 : a.gz,
                       ok ? 16u : 0u);
          }
        }
        cp_async_commit();
      };
      load_fine(2 * d0 - 1, true);
      load_fine(2 * d0, true);
      load_fine(2 * d0 + 1, true);
      for (int s = d0 - 1; s < d1; ++s) {
        // ---- coarse x slab of slice s ----
        mbar_wait(&xempty[xslot], xphase);
        uint8_t* slab = s_x + (size_t)xslot * PXSLAB;
        const bool dok = s >= 0 && s < a.Dc;
        const __nv_bfloat16* base = a.x + ((size_t)b * a.Dc + (dok ? s : 0)) * a.Hc * a.Wc * a.xpitch;
#pragma unroll
        for (int k = 0; k < KX; ++k) {
          const bool ok = dok && soff[k] >= 0;
          cp_async16(slab + doff[k], ok ? base + soff[k] : a.x, ok ? 16u : 0u);
        }
        cp_async_arrive_noinc(&xfull[xslot]);
        if (++xslot == (uint32_t)NS) { xslot = 0; xphase ^= 1; }
        if (s < d0) continue;
        // ---- the 16 G slabs of coarse slice s ----
        mbar_wait(&gempty[gslot], gphase);
        uint8_t* st = s_g + (size_t)gslot * PGSTAGE;
        // one depth parity per pass (ad = 0: O, fine slices 2s-1, 2s; ad = 1: E, 2s, 2s+1): 32 live sums.  Before a
        // pass, all but the most recent fine load group have landed: the pass's two slices (the newest is the next one)
#pragma unroll 1
        for (int ad = 0; ad < 2; ++ad) {
          cp_async_wait<1>();
          named_bar(1, 128);
#pragma unroll 1
          for (int u = lt >> 2; u < PGROWS; u += 32) {
            const int i = u / TWR, j = u % TWR;
            float g[2][2][8];                   // [ah][aw][channel], fp32 pair sums
#pragma unroll
            for (int q = 0; q < 32; ++q) (&g[0][0][0])[q] = 0.f;
            if (j > 0 && cok) {
#pragma unroll
              for (int kd = 0; kd < 2; ++kd) {
                const int fd = 2 * s - 1 + ad + kd;
                if (fd < 0 || fd >= a.D) continue;
                const uint8_t* fs = s_f + (size_t)((fd + 3) % 3) * PFSLICE;
#pragma unroll
                for (int kh = 0; kh < 3; ++kh) {
                  float f[3][8];
#pragma unroll
                  for (int kw = 0; kw < 3; ++kw) {
                    const uint4 q = *reinterpret_cast<const uint4*>(fs + (size_t)((((2 * i + kh) * PFCOLS) + 2 * j + kw) * 4 + c8) * 16);
                    const __nv_bfloat162* hq = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                      const float2 v = __bfloat1622float2(hq[e]);
                      f[kw][2 * e] = v.x; f[kw][2 * e + 1] = v.y;
                    }
                  }
                  // fine tap k of an axis feeds O (k = 0, 1) and E (k = 1, 2)
#pragma unroll
                  for (int ah = 0; ah < 2; ++ah) {
                    if (ah == 0 ? kh == 2 : kh == 0) continue;
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                      g[ah][0][e] += f[0][e] + f[1][e];
                      g[ah][1][e] += f[1][e] + f[2][e];
                    }
                  }
                }
              }
              if (ad == 1)
#pragma unroll
                for (int e = 0; e < 8; ++e) bsum[e] += g[1][1][e];   // every fine voxel lies in exactly one E box
            }
            const uint32_t roff = swz((uint32_t)u * 64u + (uint32_t)c8 * 16u, 64);
#pragma unroll
            for (int ah = 0; ah < 2; ++ah)
#pragma unroll
              for (int aw = 0; aw < 2; ++aw) {
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float v0 = g[ah][aw][2 * e], v1 = g[ah][aw][2 * e + 1];
                  const __nv_bfloat162 h2 = __floats2bfloat162_rn(v0, v1);
                  const float2 hf = __bfloat1622float2(h2);
                  hi[e] = *reinterpret_cast<const uint32_t*>(&h2);
                  lo[e] = pack_bf16x2(v0 - hf.x, v1 - hf.y);
                }
                *reinterpret_cast<uint4*>(st + (size_t)poly_slab(0, ad, ah, aw) * PGSLAB + roff) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                *reinterpret_cast<uint4*>(st + (size_t)poly_slab(1, ad, ah, aw) * PGSLAB + roff) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
              }
          }
          // every loader thread is done with slice 2s-1+ad: its slot takes slice 2s+2+ad (needed by slice s+1)
          named_bar(1, 128);
          load_fine(2 * s + 2 + ad, s + 1 < d1);
        }
        fence_proxy_async();                    // generic-proxy stores -> the wgmma (async proxy) reads
        mbar_arrive(&gfull[gslot]);
        if (++gslot == PNGS) { gslot = 0; gphase ^= 1; }
      }
    }
    if (a.bias_partial) {
      // bias partial of this CTA: fixed-order reduction over the 32 loader threads of each channel group
      named_bar(1, 128);
      if (lt < 32) {
        float sum = 0.f;
        for (int r = 0; r < 32; ++r) sum += s_bsum[(4 * r + (lt >> 3)) * 8 + (lt & 7)];
        a.bias_partial[(size_t)blockIdx.x * 32 + lt] = has_work ? sum : 0.f;
      }
    }
  } else {
    // ================================ MMA WARPGROUPS ================================
    const int wg = warp >> 2;                   // = kd: (O, -1), (E, 0), (O, 0)
    const int t = threadIdx.x & 127;
    const int ad = wg == 1 ? 1 : 0;
    float acc[3][32];
    if (has_work) {
      const uint32_t x_u32 = smem_u32(s_x), g_u32 = smem_u32(s_g);
      uint32_t wslot = 0, wphase = 0, hslot = 0, gs = 0, gph = 0, acc0 = 0;
      for (int item = blockIdx.x; item < a.nitems; item += gridDim.x) {
        const int ch = (item / HW_tiles) % a.nchunks;
        const int nd = min(ch * a.dchunk + a.dchunk, a.Dc + 1) - ch * a.dchunk;
        for (int j = 0; j < nd; ++j) {
          for (int q = 0; q < (j == 0 ? 2 : 1); ++q) {
            mbar_wait(&xfull[wslot], wphase);
            if (++wslot == (uint32_t)NS) { wslot = 0; wphase ^= 1; }
          }
          mbar_wait(&gfull[gs], gph);
          const uint32_t cur = hslot + 1 == (uint32_t)NS ? 0 : hslot + 1;   // slab of slice s; hslot: slice s - 1
          const uint32_t a_base = x_u32 + (wg == 0 ? hslot : cur) * PXSLAB;
          const uint32_t b_base = g_u32 + gs * PGSTAGE + 64u;                // G row k + 1 pairs with x rows k, k + 1
          wg_fence();
#pragma unroll
          for (int s3 = 0; s3 < 3; ++s3) {      // kh: (O, -1), (E, 0), (O, 0)
            const int ah = s3 == 1 ? 1 : 0;
            const uint64_t adesc0 = make_desc_mn_swz<64>(a_base + (s3 == 0 ? 0u : (uint32_t)TWR * 64u), 64u);
#pragma unroll
            for (int i = 0; i < PGROWS / 16; ++i)
#pragma unroll
              for (int hl = 0; hl < 2; ++hl) {
                const uint64_t adesc = adesc0 + (uint64_t)((16 * i * 64) >> 4);
                const uint64_t bdesc = make_desc_mn_swz<64>(b_base + (uint32_t)poly_slab(hl, ad, ah, 0) * PGSLAB + 16u * i * 64u, PGSLAB);
                Wgmma<64, 1, 1>::mma(acc[s3], adesc, bdesc, (i == 0 && hl == 0) ? acc0 : 1u);
              }
          }
          wg_commit();
          wg_wait<0>();
          if (lane == 0) {
            mbar_arrive(&xempty[hslot]);
            mbar_arrive(&gempty[gs]);
          }
          acc0 = 1u;
          hslot = cur;
          if (++gs == PNGS) { gs = 0; gph ^= 1; }
        }
        if (lane == 0) mbar_arrive(&xempty[hslot]);
        if (++hslot == (uint32_t)NS) hslot = 0;
      }
    }
    float* part = a.partial + (size_t)blockIdx.x * 27 * 32 * 32;
    if (!has_work) {
      for (int i = threadIdx.x; i < 27 * 32 * 32; i += 384) part[i] = 0.f;
    } else {
      // fragment (row m, column n): m = (sw, ci), n = (aw, co); kw = 0 for (sw = -1, O), 2 for (0, O), 1 for (0, E)
      const int w4 = t >> 5, qr = lane >> 2, pc = lane & 3;
#pragma unroll
      for (int s3 = 0; s3 < 3; ++s3)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int m = 16 * w4 + 8 * i + qr, sw = m >> 5, ci = m & 31;
#pragma unroll
          for (int jn = 0; jn < 8; ++jn) {
            const int n = 8 * jn + 2 * pc, aw = n >> 5, co = n & 31;
            if (sw == 0 && aw == 1) continue;
            const int kw = aw == 1 ? 1 : (sw == 0 ? 0 : 2);
            const int tap = (wg * 3 + s3) * 3 + kw;
            *reinterpret_cast<float2*>(part + ((size_t)tap * 32 + ci) * 32 + co) = make_float2(acc[s3][4 * jn + 2 * i], acc[s3][4 * jn + 2 * i + 1]);
          }
        }
    }
  }
}

// gw[co_off + co][ci_off + ci][tap] (+)= sum_cta partial[cta][tap][ci][co] for every pending reduction of a backward pass,
// in ONE launch (16 reduce launches per training step otherwise); fixed order -> deterministic.  Block = 64 elements x 4
// quarters of the CTA range: threads follow the partial layout (co fastest) so the reads coalesce, and the four quarter
// sums (combined in fixed order through shared memory) keep 4x more loads in flight than one serial loop.  The
// descriptors travel by value in the kernel parameters (no device table to keep alive or re-upload inside a captured graph).
constexpr int MAXRED = 40;
struct ReduceBatch {
  ReduceDesc d[MAXRED];
  int n, total_blocks;
};
__global__ void __launch_bounds__(256) wgrad2_reduce_multi_kernel(const ReduceBatch rb) {
  __shared__ float sh[4][64];
  int k = 0;
  for (int i = 1; i < rb.n; ++i)
    if ((int)blockIdx.x >= rb.d[i].blk_begin) k = i;
  const ReduceDesc& r = rb.d[k];
  const int blk = blockIdx.x - r.blk_begin;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  if (r.gb && blk == 0 && threadIdx.x < r.Cout) {
    float acc = r.accumulate ? r.gb[threadIdx.x] : 0.f;
    for (int c = 0; c < r.ncta; ++c) acc += r.bias_partial[(size_t)c * r.GOUT + threadIdx.x];
    r.gb[threadIdx.x] = acc;
  }
  const int per_cta = r.T * r.G * r.GOUT;
  const int j = blk * 64 + tx;
  const int q = (r.ncta + 3) / 4, c0 = ty * q, c1 = min(c0 + q, r.ncta);
  float acc = 0.f;
  if (j < per_cta)
    for (int c = c0; c < c1; ++c) acc += r.partial[(size_t)c * per_cta + j];
  sh[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && j < per_cta) {
    const int co = j % r.GOUT, ci = (j / r.GOUT) % r.G, tap = j / (r.GOUT * r.G);
    if (co < r.Cout && ci < r.ci_cnt) {
      const float tot = ((sh[0][tx] + sh[1][tx]) + sh[2][tx]) + sh[3][tx];
      float* dst = r.gw + ((size_t)(r.co_off + co) * r.Cin_total + r.ci_off + ci) * r.T + tap;
      *dst = (r.accumulate ? *dst : 0.f) + tot;
    }
  }
}

}  // namespace tcw
}  // namespace vxm

using namespace vxm;
using namespace vxm::tcw;

namespace vxm {
namespace tcw {

static bool chan_ok(int c) { return c == 8 || c == 16 || c == 32; }

bool wgrad2_supported(int Ca, int Cb, int Cg) {
  return (Ca == 0 || chan_ok(Ca)) && (Cb == 0 || chan_ok(Cb)) && Ca + Cb > 0 && chan_ok(Cg);
}

// Partials of `grid` CTAs of T x G x GOUT floats at `partial` (bias partials at `bias_partial`): record their reduction.
static void wgrad2_record(float* partial, float* bias_partial, int grid, int T, int G, int GOUT, float* grad_w, float* grad_b, int Cout_real,
                          int Cin_total, int ci_off, int ci_cnt, int accumulate, ReduceDesc* desc, int co_off) {
  const int per_cta = T * G * GOUT;
  desc->partial = partial; desc->gw = grad_w; desc->bias_partial = bias_partial; desc->gb = grad_b;
  desc->ncta = grid; desc->T = T; desc->G = G; desc->GOUT = GOUT; desc->Cout = Cout_real; desc->Cin_total = Cin_total;
  desc->ci_off = ci_off; desc->ci_cnt = ci_cnt; desc->accumulate = accumulate; desc->blk_begin = (per_cta + 63) / 64;   // block count, turned into an offset by wgrad2_reduce
  desc->co_off = co_off;
}

// The coarse form (wgrad2_poly_kernel) serves every 3-D launch whose source is a 32-channel nearest-x2 upsampled slice
// against a 32-channel gz slice, on even fine extents; VXM_B200_POLYPHASE=0 keeps the fine kernel (A/B switch).
static bool wgrad2_poly_ok(int Cx, int up, int Cg, int kd, int D, int H, int W) {
  const char* e = getenv("VXM_B200_POLYPHASE");
  if (e && e[0] == '0' && e[1] == 0) return false;
  return up && kd == 3 && Cx == 32 && Cg == 32 && D % 2 == 0 && H % 2 == 0 && W % 2 == 0;
}

static int wgrad2_poly_launch(const void* x, int x_pitch, const void* gz, int Cg, int g_pitch, float* grad_w, float* grad_b, void* work, int B,
                              int D, int H, int W, int Cout_real, int Cin_total, int ci_off, int ci_cnt, int accumulate, cudaStream_t st,
                              ReduceDesc* desc, size_t* work_used, int co_off) {
  Wgrad2PolyArgs a{};
  a.x = (const __nv_bfloat16*)x; a.xpitch = x_pitch;
  a.gz = (const __nv_bfloat16*)gz; a.Cg = Cg; a.gpitch = g_pitch;
  a.B = B; a.D = D; a.H = H; a.W = W; a.Dc = D / 2; a.Hc = H / 2; a.Wc = W / 2;
  // G has Dc + 1 (Hc + 1, Wc + 1) coarse positions per axis: O[Dc] pairs the last fine voxel with the zero past it
  a.tiles_h = (a.Hc + PTH) / PTH; a.tiles_w = (a.Wc + PTU) / PTU;
  const int nsm = conv_ctas();
  const long long tiles = (long long)B * a.tiles_h * a.tiles_w;
  a.dchunk = depth_chunk(a.Dc + 1, tiles, nsm, 0.5, 32);
  a.nchunks = (a.Dc + a.dchunk) / a.dchunk;
  a.nitems = (int)(tiles * a.nchunks);
  int grid = a.nitems < nsm ? a.nitems : nsm;
  if (grid > 256) grid = 256;
  // this launch owns exactly [work, work + *work_used): partials, then bias partials
  a.partial = (float*)work;
  const size_t npart = (size_t)grid * 27 * 32 * 32;
  a.bias_partial = grad_b ? (float*)work + npart : nullptr;
  *work_used = (npart + (grad_b ? (size_t)grid * 32 : 0)) * sizeof(float);
  *work_used = (*work_used + 255) & ~(size_t)255;
  a.nslot = PNSLOT;
  const size_t smem = PSMEM;
  VXM_CUDA(cudaFuncSetAttribute(wgrad2_poly_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  wgrad2_poly_kernel<<<grid, PNTHREADS, smem, st>>>(a);
  int rc = check_launch("conv3d_tc_wgrad2_poly");
  if (rc) return rc;
  wgrad2_record(a.partial, a.bias_partial, grid, 27, 32, 32, grad_w, grad_b, Cout_real, Cin_total, ci_off, ci_cnt, accumulate, desc, co_off);
  return VXM_OK;
}

// one source tensor (C channels, optionally nearest-x2 upsampled) against gz; weights [ci_off, ci_off + ci_cnt) of Cin_total
int wgrad2_launch(const void* x, int Cx, int up, const void* gz, int Cg, float* grad_w, float* grad_b, void* work, int B, int D, int H, int W,
                  int kd, int Cout_real, int Cin_total, int ci_off, int ci_cnt, int accumulate, cudaStream_t st, ReduceDesc* desc,
                  size_t* work_used, bool khm, int x_pitch, int g_pitch, int co_off) {
  if (!khm && wgrad2_poly_ok(Cx, up, Cg, kd, D, H, W))
    return wgrad2_poly_launch(x, x_pitch ? x_pitch : Cx, gz, Cg, g_pitch ? g_pitch : Cg, grad_w, grad_b, work, B, D, H, W, Cout_real, Cin_total,
                              ci_off, ci_cnt, accumulate, st, desc, work_used, co_off);
  Wgrad2Args a{};
  a.x = (const __nv_bfloat16*)x; a.Cx = Cx; a.up = up; a.upd = (up && kd == 3) ? 1 : 0;
  a.gz = (const __nv_bfloat16*)gz; a.Cg = Cg;
  a.xpitch = x_pitch ? x_pitch : Cx; a.gpitch = g_pitch ? g_pitch : Cg;
  a.B = B; a.D = D; a.H = H; a.W = W;
  a.tiles_h = (H + TH - 1) / TH; a.tiles_w = (W + TUSE - 1) / TUSE;
  const int G = Cx <= 16 ? 16 : 32, GOUT = Cg <= 16 ? 16 : 32;
  const int nsm = conv_ctas();
  // depth chunking: balance the persistent CTAs (waves of nsm items) against the 2 halo slabs every chunk re-loads
  const long long tiles = (long long)B * a.tiles_h * a.tiles_w;
  a.dchunk = depth_chunk(D, tiles, nsm, kd == 3 ? 2.5 : 0.5, 32);
  a.nchunks = (D + a.dchunk - 1) / a.dchunk;
  a.nitems = (int)(tiles * a.nchunks);
  int grid = a.nitems < nsm ? a.nitems : nsm;
  if (grid > 256) grid = 256;
  // this launch owns exactly [work, work + *work_used): partials, then bias partials
  a.partial = (float*)work;
  const size_t npart = (size_t)grid * kd * 9 * G * GOUT;
  a.bias_partial = grad_b ? (float*)work + npart : nullptr;
  *work_used = (npart + (grad_b ? (size_t)grid * GOUT : 0)) * sizeof(float);
  *work_used = (*work_used + 255) & ~(size_t)255;
  const size_t xslab = (size_t)XROWS * 2 * G, gslab = (size_t)GSROWS * 2 * GOUT;
  const int extra = kd == 3 ? 3 : 0;
  int nslot = (int)((200 * 1024 - NGS * gslab - 512) / xslab) - extra;
  if (nslot > MAXSLOT) nslot = MAXSLOT;
  VXM_REQUIRE(nslot >= 4, "conv3d_tc_wgrad: not enough shared memory for the slab ring");
  a.nslot = nslot;
  const size_t smem = (size_t)(nslot + extra) * xslab + NGS * gslab + 512 + 128 * (GOUT + 1) * sizeof(float);   // + bias rows
#define VXM_W2_LAUNCH(KD_, G_, GO_)                                                                                          \
  do {                                                                                                                       \
    VXM_CUDA(cudaFuncSetAttribute(wgrad2_kernel<KD_, G_, GO_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));     \
    wgrad2_kernel<KD_, G_, GO_><<<grid, NTHREADS, smem, st>>>(a);                                                             \
  } while (0)
#define VXM_W2_G(KD_)                                                                                                        \
  do {                                                                                                                       \
    if (G == 16 && GOUT == 16) VXM_W2_LAUNCH(KD_, 16, 16); else if (G == 16) VXM_W2_LAUNCH(KD_, 16, 32);                     \
    else if (GOUT == 16) VXM_W2_LAUNCH(KD_, 32, 16); else VXM_W2_LAUNCH(KD_, 32, 32);                                        \
  } while (0)
  if (khm) {
    VXM_REQUIRE(kd == 1 && G == 16 && GOUT == 16 && !up, "conv3d_tc_wgrad2 (kh in M): needs kd = 1 and at most 16 channels on both sides");
    VXM_CUDA(cudaFuncSetAttribute(wgrad2_kernel<1, 16, 16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    wgrad2_kernel<1, 16, 16, true><<<grid, NTHREADS, smem, st>>>(a);
  } else if (kd == 3) VXM_W2_G(3); else VXM_W2_G(1);
  int rc = check_launch("conv3d_tc_wgrad2");
  if (rc) return rc;
  wgrad2_record(a.partial, a.bias_partial, grid, kd * 9, G, GOUT, grad_w, grad_b, Cout_real, Cin_total, ci_off, ci_cnt, accumulate, desc,
                co_off);
  return VXM_OK;
}

// Every recorded reduction d[0 .. n), 0 < n <= MAXRED, in one launch on `st`
int wgrad2_reduce(const ReduceDesc* d, int n, cudaStream_t st) {
  ReduceBatch rb;
  int blocks = 0;
  for (int i = 0; i < n; ++i) {
    rb.d[i] = d[i];
    const int nb = d[i].blk_begin;      // wgrad2_record stored the block count here
    rb.d[i].blk_begin = blocks;
    blocks += nb;
  }
  rb.n = n; rb.total_blocks = blocks;
  wgrad2_reduce_multi_kernel<<<blocks, 256, 0, st>>>(rb);
  return check_launch("conv3d_tc_wgrad2_reduce_multi");
}

}  // namespace tcw
}  // namespace vxm

// ---- deferred reduction API -------------------------------------------------------------------------------------------
// vxm_conv3d_tc_wgrad2_partial launches the weight-gradient kernel(s) of one layer into caller-provided workspace and
// appends the pending reductions to a HOST descriptor buffer; vxm_conv3d_tc_wgrad2_flush then runs every pending
// reduction of the backward pass in one launch (fixed summation order -> deterministic, as before).
extern "C" size_t vxm_conv3d_tc_wgrad2_desc_bytes(void) { return sizeof(ReduceDesc); }
extern "C" int vxm_conv3d_tc_wgrad2_max_pending(void) { return MAXRED; }
extern "C" size_t vxm_conv3d_tc_wgrad2_partial_bytes(int kd) {
  // upper bound for one layer (two sources): 2 x 256 CTAs x 27 x 32 x 32 floats + bias partials
  return 2 * ((size_t)256 * kd * 9 * 32 * 32 + 256 * 32) * sizeof(float) + 1024;
}

static bool chan_ok64(int c) { return chan_ok(c) || c == 64; }

// A 64-channel x source or gz runs as 32-channel slices of both operands (every kernel launch one of the existing
// <= 32 x 32 instantiations), each slice pair with its own pending reduction into its block of grad_w.  Workspace per
// layer: at most vxm_conv3d_tc_wgrad2_partial_bytes(kd) per two slice pairs.
extern "C" int vxm_conv3d_tc_wgrad2_partial(const void* xa, const void* xb, const void* gz, float* grad_w, float* grad_b, void* work,
                                            size_t work_bytes, size_t* work_used, void* descs_host, int* ndesc, int B, int D, int H, int W,
                                            int Ca, int Cb, int up, int Cin_real, int Cg, int Cout_real, int kd, int accumulate, void* stream) {
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0 && grad_w && work && work_used && descs_host && ndesc && gz, "conv3d_tc_wgrad2_partial: bad argument");
  VXM_REQUIRE(kd == 1 || kd == 3, "conv3d_tc_wgrad2_partial: kd must be 1 or 3");
  VXM_REQUIRE((Ca == 0 || chan_ok64(Ca)) && (Cb == 0 || chan_ok64(Cb)) && Ca + Cb > 0 && chan_ok64(Cg),
              "conv3d_tc_wgrad2_partial: channel counts (%d,%d | %d) unsupported", Ca, Cb, Cg);
  VXM_REQUIRE((Ca == 0 || xa) && (Cb == 0 || xb), "conv3d_tc_wgrad2_partial: missing source tensor");
  const int nsub = ((Ca + 31) / 32 + (Cb + 31) / 32) * ((Cg + 31) / 32);
  VXM_REQUIRE(*ndesc + (nsub > 2 ? nsub : 2) <= MAXRED, "conv3d_tc_wgrad2_partial: too many pending reductions (flush first)");
  VXM_REQUIRE(Cout_real > 0 && Cout_real <= Cg, "conv3d_tc_wgrad2_partial: Cout_real out of range");
  ReduceDesc* d = (ReduceDesc*)descs_host;
  cudaStream_t st = as_stream(stream);
  size_t total = 0;
  char* wp = (char*)work;
  const void* src[2] = {xa, xb};
  const int C[2] = {Ca, Cb}, ci0[2] = {0, Ca}, sup[2] = {up, 0};
  for (int s = 0; s < 2; ++s) {
    for (int xs = 0; xs < C[s] && ci0[s] + xs < Cin_real; xs += 32) {
      const int cx = C[s] - xs < 32 ? C[s] - xs : 32;
      const int cnt = Cin_real - ci0[s] - xs < cx ? Cin_real - ci0[s] - xs : cx;
      for (int gs = 0; gs < Cg && gs < Cout_real; gs += 32) {
        const int cg = Cg - gs < 32 ? Cg - gs : 32;
        const int cout = Cout_real - gs < cg ? Cout_real - gs : cg;
        // the bias gradient (sum of gz) is taken once per gz slice, with the first x slice
        float* gb = (grad_b && ci0[s] + xs == 0) ? grad_b + gs : nullptr;
        size_t used = 0;
        int rc = wgrad2_launch((const __nv_bfloat16*)src[s] + xs, cx, sup[s], (const __nv_bfloat16*)gz + gs, cg, grad_w, gb, wp, B, D, H, W,
                               kd, cout, Cin_real, ci0[s] + xs, cnt, accumulate, st, &d[*ndesc], &used, false, C[s], Cg, gs);
        if (rc) return rc;
        VXM_REQUIRE(total + used <= work_bytes, "conv3d_tc_wgrad2_partial: workspace too small");
        ++*ndesc; wp += used; total += used;
      }
    }
  }
  *work_used = total;
  return VXM_OK;
}

// Weight gradient of a kd-folded layer (see vxm_planar_fold_kd_bf16): x (B, D, H, W, Cx <= 16) against gz (B, D, H, W, Cg <= 16) as a
// 2-D problem per slice with the kh taps stacked in M.  grad_w receives the 2-D layout (Cout_real, Cin_real, 1, 3, 3).
extern "C" int vxm_conv3d_tc_wgrad2_partial_khm(const void* x, const void* gz, float* grad_w, float* grad_b, void* work, size_t work_bytes,
                                                size_t* work_used, void* descs_host, int* ndesc, int B, int D, int H, int W, int Cx,
                                                int Cin_real, int Cg, int Cout_real, int accumulate, void* stream) {
  VXM_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0 && x && gz && grad_w && work && work_used && descs_host && ndesc, "conv3d_tc_wgrad2_partial_khm: bad argument");
  VXM_REQUIRE((Cx == 8 || Cx == 16) && (Cg == 8 || Cg == 16), "conv3d_tc_wgrad2_partial_khm: channel counts (%d | %d) unsupported", Cx, Cg);
  VXM_REQUIRE(Cin_real > 0 && Cin_real <= Cx && Cout_real > 0 && Cout_real <= Cg, "conv3d_tc_wgrad2_partial_khm: real channel counts out of range");
  VXM_REQUIRE(*ndesc + 1 <= MAXRED, "conv3d_tc_wgrad2_partial_khm: too many pending reductions (flush first)");
  ReduceDesc* d = (ReduceDesc*)descs_host;
  size_t used = 0;
  int rc = wgrad2_launch(x, Cx, 0, gz, Cg, grad_w, grad_b, work, B, D, H, W, 1, Cout_real, Cin_real, 0, Cin_real, accumulate, as_stream(stream),
                         &d[*ndesc], &used, true, 0, 0, 0);
  if (rc) return rc;
  VXM_REQUIRE(used <= work_bytes, "conv3d_tc_wgrad2_partial_khm: workspace too small");
  ++*ndesc;
  *work_used = used;
  return VXM_OK;
}

extern "C" int vxm_conv3d_tc_wgrad2_flush(const void* descs_host, int ndesc, void* stream) {
  VXM_REQUIRE(descs_host && ndesc > 0 && ndesc <= MAXRED, "conv3d_tc_wgrad2_flush: bad argument");
  return wgrad2_reduce((const ReduceDesc*)descs_host, ndesc, as_stream(stream));
}
