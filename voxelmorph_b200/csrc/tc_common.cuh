// Thin PTX wrappers for the sm_90a tensor-core path: mbarrier, cp.async, bulk (TMA) copies, wgmma and its
// shared-memory descriptor encoders.
#pragma once
#include <cuda.h>        // CUtensorMap (types only: the encoder is resolved at run time, libcuda is not linked)
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace vxm {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- mbarrier ----------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (the launch fails with an error) instead of hanging the GPU.  No printf here: a
// function call in a kernel that issues wgmma makes ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// one lane of a converged warp (keeps the surrounding control flow warp-uniform, so descriptors stay in uniform registers)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- proxies / fences ---------
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- cp.async (LDGSTS) --------
// 16-byte copy, zero-filled when src_bytes == 0 (padding / out-of-volume voxels)
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst_smem)), "l"(src), "r"(src_bytes) : "memory");
}
// the mbarrier receives one (pre-counted) arrival once all cp.async issued so far by this thread have landed
__device__ __forceinline__ void cp_async_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------- bulk copy (TMA, 1-D) -----
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---------------------------------------------------------------- tiled tensor copy (TMA, 5-D) ------
// A bf16 channels-last activation (B, D, H, W, C) is described to the TMA unit as the 5-D tensor {C, W, H, D, B}; one
// copy moves a box {G channels, 32 columns, rows, 1 slice, 1 batch item} into shared memory with the 32 / 64 / 128-byte
// swizzle the wgmma K-major operand layouts use (row = voxel, channels contiguous).  Coordinates may lie outside the
// tensor (negative, or >= the extent): those elements arrive as zeros, which is exactly the convolution's zero padding.
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst_smem, const void* tmap, int c0, int c1, int c2, int c3, int c4, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
      ::"r"(smem_u32(dst_smem)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(smem_u32(bar))
      : "memory");
}
// raises the barrier's pending transaction count without arriving (the caller arrives separately)
__device__ __forceinline__ void mbar_expect_tx_noarrive(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

// Host side: encode the tensor map of a bf16 (B, D, H, W, C) activation with box {boxC, boxW, boxH, 1, 1}.  boxC * 2 bytes
// is the shared-memory row width (32 / 64 / 128) and selects the swizzle mode.  Returns 0, or -1 with vxm_last_error set.
int make_act_tmap(CUtensorMap* out, const void* base, int B, int D, int H, int W, int C, int boxC, int boxW, int boxH);

// ---------------------------------------------------------------- wgmma (warpgroup MMA) ------
// The four warps of a warpgroup issue wgmma.mma_async together; the accumulators live in their registers (m64nNk16
// fragment layout, see Wgmma in wgmma.cuh).  A 128-row tile is two m64 halves, rows 0-63 in d0 and 64-127 in d1.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// register budget moved between warpgroups (every warp of the warpgroup executes it): producers give registers up,
// MMA warpgroups take them.  ptxas still compiles every role within the __launch_bounds__ budget (168 registers at 384
// threads), so this only pays where the producer needs few registers: it is used by the kernels whose spill counts
// (-Xptxas -v) it lowers (conv_tct_kernel, wgrad2_kernel) and left out where it raises them.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void named_bar(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// Accumulator read-out in row form: thread t of the warpgroup (t = threadIdx.x % 128) receives row t, columns
// [c0, c0 + 16) of the 128 x N accumulator held as two m64 fragments d0 / d1 (c0: a multiple of 16 known at compile time
// after unrolling, so the fragments stay in registers).  The fragments pass through `stage` (ACC_STAGE_FLOATS floats of
// shared memory per warpgroup); `bar` is a named barrier owned by the warpgroup.
constexpr int ACC_STAGE_LD = 17;                     // padded row: conflict-free row reads
constexpr int ACC_STAGE_FLOATS = 128 * ACC_STAGE_LD;
__device__ __forceinline__ void acc_row16(const float* d0, const float* d1, int c0, float* stage, int bar, uint32_t* r) {
  const int t = threadIdx.x & 127, w = t >> 5, q = (t & 31) >> 2, p = t & 3;
  named_bar(bar, 128);                                // the previous read-out of `stage` is complete
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float* d = h ? d1 : d0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float* srow = stage + (64 * h + 16 * w + 8 * i + q) * ACC_STAGE_LD + 2 * p;
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int j = c0 / 8 + jj;
        srow[8 * jj] = d[4 * j + 2 * i];
        srow[8 * jj + 1] = d[4 * j + 2 * i + 1];
      }
    }
  }
  named_bar(bar, 128);
  const float* mine = stage + t * ACC_STAGE_LD;
#pragma unroll
  for (int k = 0; k < 16; ++k) r[k] = __float_as_uint(mine[k]);
}

// Read-out of ONE m64 fragment d with two threads per row: `ncol` (16 or 32) columns [c0, c0 + ncol) pass through
// `stage`, and thread t of the warpgroup receives row (t & 31) + 32 * ((t >> 5) & 1), columns [c0 + 16 * (t >> 6), +16)
// (with ncol = 16, threads t >= 64 receive nothing meaningful).  c0 and ncol are compile-time after unrolling.
constexpr int ACC_HALF_LD = 33;                      // padded 32-column row: conflict-free row reads
static_assert(64 * ACC_HALF_LD <= ACC_STAGE_FLOATS, "half read-out fits the stage buffer");
__device__ __forceinline__ void acc_half_row16(const float* d, int c0, int ncol, float* stage, int bar, uint32_t* r) {
  const int t = threadIdx.x & 127, w = t >> 5, q = (t & 31) >> 2, p = t & 3;
  named_bar(bar, 128);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float* srow = stage + (16 * w + 8 * i + q) * ACC_HALF_LD + 2 * p;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      if (8 * jj < ncol) {
        const int j = c0 / 8 + jj;
        srow[8 * jj] = d[4 * j + 2 * i];
        srow[8 * jj + 1] = d[4 * j + 2 * i + 1];
      }
    }
  }
  named_bar(bar, 128);
  const float* mine = stage + ((t & 31) + 32 * ((t >> 5) & 1)) * ACC_HALF_LD + 16 * (t >> 6);
#pragma unroll
  for (int k = 0; k < 16; ++k) r[k] = __float_as_uint(mine[k]);
}

// ---------------------------------------------------------------- descriptors ---------------
// wgmma shared-memory matrix descriptor (sm_90): start address, LBO, SBO in 16-byte units; bits 62-63 = swizzle
// (0 none, 1 = 128 B, 2 = 64 B, 3 = 32 B).
// K-major, SWIZZLE_NONE: core matrix = 8 rows x 16 B, rows 16 B apart; LBO = byte distance between the two 16-byte
// K chunks of one MMA (K = 16 bf16), SBO = byte distance between consecutive 8-row groups.
__device__ __forceinline__ uint64_t make_desc_kmajor_noswz(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;                // base_offset 0, layout_type 0 (SWIZZLE_NONE)
}
// MN-major, SWIZZLE_NONE: core matrix = 8 (K) x 8 (MN, 16 B contiguous); the 8 K-rows are 16 B apart.
// SBO = stride between 8-element MN chunks, LBO = stride between 8-row K groups.
__device__ __forceinline__ uint64_t make_desc_mnmajor_noswz(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return make_desc_kmajor_noswz(saddr, lbo_bytes, sbo_bytes);
}
// swizzle field of a `width`-byte swizzled row (32, 64 or 128)
__host__ __device__ constexpr uint64_t desc_swizzle(uint32_t width) {
  return (uint64_t)(width == 128 ? 1 : (width == 64 ? 2 : 3)) << 62;
}

// A lane's 16 bf16 channels (32 bytes, one sector) as two adjacent 128-bit accesses (the widest global access on sm_90).
// `p` must be 32-byte aligned.
__device__ __forceinline__ void st_global_v8(void* p, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3, uint32_t r4, uint32_t r5, uint32_t r6,
                                             uint32_t r7) {
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = make_uint4(r0, r1, r2, r3);
  q[1] = make_uint4(r4, r5, r6, r7);
}
__device__ __forceinline__ void ld_global_nc_v8(const void* p, uint32_t (&r)[8]) {
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(p)), b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
  r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// Depth chunking of a persistent launch over `tiles` (b, h, w) tiles and D slices: balance the CTAs' waves of nsm items
// against the `halo` slabs every chunk re-loads, over 1 .. max_chunks chunks.  Returns the chunk depth.
inline int depth_chunk(int D, long long tiles, int nsm, double halo, int max_chunks) {
  int best_nch = 1;
  double best_cost = 1e300;
  for (int nch = 1; nch <= max_chunks && nch <= D; ++nch) {
    const int dc = (D + nch - 1) / nch;
    const long long items = tiles * ((D + dc - 1) / dc);
    const long long waves = (items + nsm - 1) / nsm;
    const double cost = (double)waves * (dc + halo);
    if (cost < best_cost - 1e-9) { best_cost = cost; best_nch = nch; }
  }
  return (D + best_nch - 1) / best_nch;
}

}  // namespace tc

namespace tcw {
// One pending reduction of the Toeplitz weight gradient (conv3d_tc_wgrad2.cu): `ncta` per-CTA partials of T x G x GOUT
// floats at `partial` (and GOUT bias partials each at `bias_partial`), summed in fixed order into gw / gb.
struct ReduceDesc {
  const float* partial; float* gw; const float* bias_partial; float* gb;
  int ncta, T, G, GOUT, Cout, Cin_total, ci_off, ci_cnt, accumulate, blk_begin;
  int co_off;            // first output channel of a gz slice (gw rows co_off .. co_off + Cout - 1; gb already offset)
};
}  // namespace tcw
}  // namespace vxm
