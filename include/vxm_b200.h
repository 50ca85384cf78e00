/*
 * vxm_b200 — C ABI of the H100-native (sm_90a) VxmDense registration path.
 *
 * Drop-in boundary.  The reference (voxelmorph/voxelmorph, torch backend) has no FFI
 * layer of its own: its hot path bottoms out in PyTorch operators (F.grid_sample,
 * F.interpolate, nn.Conv3d, F.conv3d, torch.optim.Adam).  Each entry point below
 * replaces one of those call sites; the reference file:line it stands in for is cited
 * on the declaration.  The host side that binds them (ctypes) is
 * voxelmorph_b200/_lib.py; INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *  - plain pointers and sizes only: every pointer is a DEVICE pointer owned by the caller
 *    (PyTorch caching allocator); the library allocates nothing persistent;
 *  - tensors are contiguous, float32, batch-major "NCDHW" (B, C, D, H, W) unless a
 *    declaration says otherwise; a 2-D problem is passed with D == 1 and nd == 2
 *    (flows then carry 2 channels: H, W);
 *  - all work is enqueued on `stream` (a cudaStream_t passed as void*); no implicit
 *    synchronisation; the current CUDA device is the caller's;
 *  - return value 0 on success, negative on error; vxm_last_error() gives the text
 *    (thread local).  Nothing throws or aborts;
 *  - `*_workspace_bytes` functions are pure host arithmetic (no CUDA calls).
 */
#ifndef VXM_B200_H
#define VXM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VXM_OK 0
#define VXM_ERR_ARG (-1)
#define VXM_ERR_CUDA (-2)
#define VXM_ERR_UNSUPPORTED (-3)

/* interpolation mode of the resampler (reference SpatialTransformer(mode=...), layers.py:11-14) */
#define VXM_MODE_LINEAR 0
#define VXM_MODE_NEAREST 1
/* how `loc / (S-1)` of layers.py:37 is rounded: a true fp32 division (torch CPU) or a
 * multiply by fl(1/(S-1)) (what torch's CUDA `tensor / python_scalar` computes). */
#define VXM_ARITH_TRUE_DIV 0
#define VXM_ARITH_RECIPROCAL 1
/* linear mode only: coord = (p + flow) * (Ssrc-1)/(S-1) without replaying the reference's fp32 round trip; results
 * agree with the exact modes to a few 1e-6 of the value range (north_star tolerance for floating point: 1e-4) and the
 * kernels are memory bound instead of instruction bound.  The nearest mode always replays the exact arithmetic. */
#define VXM_ARITH_FAST 2

const char* vxm_last_error(void);
/* library / build identification ("vxm_b200 <version> sm_90a") */
const char* vxm_version(void);
/* number of kernel launches issued through this library by the calling process so far */
uint64_t vxm_launch_count(void);

/* ---- SpatialTransformer: reference voxelmorph/torch/layers.py:30-48 (F.grid_sample :48) ----
 * out[b,c,p] = sample(src[b,c], p + flow[b,:,p]); zeros padding; align_corners=True.
 * src: (B,C,Ds,Hs,Ws)  flow: (B,nd,D,H,W)  out: (B,C,D,H,W).  The reference always uses
 * (Ds,Hs,Ws) == (D,H,W); distinct sizes follow grid_sample's semantics. */
int vxm_warp_fwd(const float* src, const float* flow, float* out,
                 int B, int C, int Ds, int Hs, int Ws, int D, int H, int W, int nd,
                 int mode, int arith, void* stream);
/* backward of the above.  grad_src (B,C,Ds,Hs,Ws) is ACCUMULATED into (caller zero-fills) and
 * may be NULL; grad_flow (B,nd,D,H,W) is overwritten and may be NULL. */
int vxm_warp_bwd(const float* grad_out, const float* src, const float* flow,
                 float* grad_src, float* grad_flow,
                 int B, int C, int Ds, int Hs, int Ws, int D, int H, int W, int nd,
                 int mode, int arith, void* stream);

/* ---- VecInt: reference voxelmorph/torch/layers.py:51-68 (scaling and squaring) ----
 * vel, out: (B,nd,D,H,W).  All nsteps squarings run in one cooperative launch.
 * If `states` is non-NULL it receives the nsteps intermediate fields v_0..v_{n-1}
 * (nsteps * B*nd*D*H*W floats) needed by the backward; otherwise `work` must hold
 * vxm_vecint_workspace_bytes() bytes of scratch. */
size_t vxm_vecint_workspace_bytes(int B, int D, int H, int W, int nd, int nsteps);
int vxm_vecint_fwd(const float* vel, float* out, float* states, void* work,
                   int B, int D, int H, int W, int nd, int nsteps, int arith, void* stream);
/* grad_vel (B,nd,D,H,W) overwritten.  `states` as written by the forward; `work` holds
 * 2 * B*nd*D*H*W floats of scratch. */
int vxm_vecint_bwd(const float* grad_out, const float* states, float* grad_vel, void* work,
                   int B, int D, int H, int W, int nd, int nsteps, int arith, void* stream);
/* arith == VXM_ARITH_FAST (3-D, nsteps >= 1): the launch keeps the field in an interleaved float4 (z,y,x,0) layout.
 * `states` then holds vxm_vecint_fast_states_bytes() bytes (nsteps float4 fields), `work`
 * vxm_vecint_fast_work_bytes(backward) bytes (2 float4 fields forward without states, 3 backward). */
size_t vxm_vecint_fast_states_bytes(int B, int D, int H, int W, int nsteps);
size_t vxm_vecint_fast_work_bytes(int B, int D, int H, int W, int backward);
/* measurement aid: a cooperative launch (512 threads per CTA, `ctas_per_sm` CTAs per SM or the occupancy limit when 0)
 * that executes `nsync` grid-wide synchronisations and nothing else */
int vxm_debug_gridsync(int nsync, int ctas_per_sm, void* stream);

/* ---- ResizeTransform: reference voxelmorph/torch/layers.py:85-97 (F.interpolate :88,:94) ----
 * out = post * lerp(pre * x) with align_corners=True linear interpolation.
 * x: (B,C,Di,Hi,Wi)  out: (B,C,Do,Ho,Wo). */
int vxm_resize_fwd(const float* x, float* out, int B, int C, int Di, int Hi, int Wi,
                   int Do, int Ho, int Wo, float pre, float post, void* stream);
/* adjoint (deterministic gather form).  grad_x overwritten. */
int vxm_resize_bwd(const float* grad_out, float* grad_x, int B, int C, int Di, int Hi, int Wi,
                   int Do, int Ho, int Wo, float pre, float post, void* stream);

/* ---- NCC: reference voxelmorph/torch/losses.py:15-67 (5 x F.conv3d with a ones filter) ----
 * I = y_true, J = y_pred: (B,1,D,H,W).  win = (wd,wh,ww) odd window (1 along D for 2-D).
 * loss[0] = -mean(cc).  `work`: vxm_reduce_workspace_bytes().  If `saved` is non-NULL the
 * forward stores 4 fields (4 * B*D*H*W floats) that the backward consumes. */
int vxm_ncc_fwd(const float* I, const float* J, float* loss, float* saved, void* work,
                int B, int D, int H, int W, int wd, int wh, int ww, void* stream);
/* grad_J = grad_loss[0] * d(-mean cc)/dJ.  grad_loss is a device scalar. */
int vxm_ncc_bwd(const float* I, const float* J, const float* saved, const float* grad_loss,
                float* grad_J, int B, int D, int H, int W, int wd, int wh, int ww, void* stream);
/* NCC differentiated w.r.t. either image.  `which`: bit 0 = y_true (I), bit 1 = y_pred (J); 1, 2 or 3.
 * vxm_ncc_fwd2 stores 3 fields per voxel (which = 1 or 2; which = 2 is vxm_ncc_fwd itself) or 5 (which = 3) in `saved`
 * (that many * B*D*H*W floats); vxm_ncc_bwd2 takes them with the same `which` and writes grad_I and / or grad_J
 * (= grad_loss[0] * d(-mean cc)/dI, dJ; the pointer of a gradient that is not asked for is ignored).  which = 3 is
 * one launch for both gradients. */
int vxm_ncc_fwd2(const float* I, const float* J, float* loss, float* saved, void* work, int which,
                 int B, int D, int H, int W, int wd, int wh, int ww, void* stream);
int vxm_ncc_bwd2(const float* I, const float* J, const float* saved, const float* grad_loss, float* grad_I,
                 float* grad_J, int which, int B, int D, int H, int W, int wd, int wh, int ww, void* stream);

/* ---- Jacobian determinant of x -> x + disp(x): reference voxelmorph/py/utils.py:473-516 (numpy, np.gradient) ----
 * disp: (B,nd,D,H,W) displacement in voxels (the layout VxmDense(registration=True) returns).  det (B,D,H,W), may be NULL;
 * folds (one uint64, may be NULL) receives the number of voxels with det <= 0. */
int vxm_jacdet(const float* disp, float* det, unsigned long long* folds, int B, int D, int H, int W, int nd, void* stream);

/* ---- Grad: reference voxelmorph/torch/losses.py:102-135 ----
 * y: (B,nd,D,H,W) (any channel count C).  penalty 1 = l1, 2 = l2.  loss[0] = mult * mean_b mean_axes mean |dy|^p */
size_t vxm_reduce_workspace_bytes(void);
int vxm_gradloss_fwd(const float* y, float* loss, void* work, int B, int C, int D, int H, int W,
                     int nd, int penalty, float mult, void* stream);
int vxm_gradloss_bwd(const float* y, const float* grad_loss, float* grad_y, int B, int C, int D,
                     int H, int W, int nd, int penalty, float mult, void* stream);

/* ---- MSE: reference voxelmorph/torch/losses.py:75-76 ---- */
int vxm_mse_fwd(const float* y_true, const float* y_pred, float* loss, void* work, size_t n,
                void* stream);
int vxm_mse_bwd(const float* y_true, const float* y_pred, const float* grad_loss,
                float* grad_pred, size_t n, void* stream);
/* MSE(image_sigma) of reference voxelmorph/tf/losses.py:112-134: loss[0] = scale * mean (y_true - y_pred)^2 with
 * scale = 1 / image_sigma^2 (vxm_mse_fwd / _bwd are these with scale 1) */
int vxm_mse_scaled_fwd(const float* y_true, const float* y_pred, float* loss, void* work, size_t n, double scale,
                       void* stream);
int vxm_mse_scaled_bwd(const float* y_true, const float* y_pred, const float* grad_loss, float* grad_pred, size_t n,
                       double scale, void* stream);

/* ---- KL(prior_lambda) of probabilistic VoxelMorph: reference voxelmorph/tf/losses.py:247-349 ----
 * params: flow_params (B, 2 nd, D, H, W) (D == 1 for nd == 2), channels [0, nd) the mean mu, [nd, 2 nd) l = log sigma^2.
 * deg(v) = number of in-volume axial neighbours of v (the conv of ones with _adj_filt, SAME zero padding):
 *   loss[0] = 0.5 nd (mean_{B,V,nd}(lambda deg e^l - l) + lambda 0.5 / nd sum_axes mean (mu_{x + e_axis} - mu_x)^2),
 * each mean over that axis's own difference tensor; an axis of size 1 contributes nothing.  Deterministic reduction
 * through the reduce workspace.  The backward writes the (B, 2 nd, D, H, W) gradient (pointwise in l, the 2 nd-point
 * Laplacian of mu). */
int vxm_kl_fwd(const float* params, float* loss, void* work, int B, int D, int H, int W, int nd, float prior_lambda,
               void* stream);
int vxm_kl_bwd(const float* params, const float* grad_loss, float* grad_params, int B, int D, int H, int W, int nd,
               float prior_lambda, void* stream);

/* ---- Dice: reference voxelmorph/torch/losses.py:84-90 ----
 * y_true, y_pred: (B,L,V) with V = D*H*W.  `work`: vxm_dice_workspace_bytes(B*L).
 * `sums` (2*B*L floats: top, bottom(unclamped)) is written for the backward. */
size_t vxm_dice_workspace_bytes(int BL);
int vxm_dice_fwd(const float* y_true, const float* y_pred, float* loss, float* sums, void* work,
                 int BL, size_t V, void* stream);
/* grad_pred = grad_loss[0] * d loss / d y_pred.  The loss is symmetric in its two arguments, so the gradient w.r.t.
 * y_true is the same call with y_pred in the place of y_true. */
int vxm_dice_bwd(const float* y_true, const float* sums, const float* grad_loss, float* grad_pred,
                 int BL, size_t V, void* stream);

/* ---- Conv3d k=3 s=1 p=1 (+bias, +LeakyReLU 0.2): reference voxelmorph/torch/networks.py:299-304
 * (ConvBlock), :211,:257 (flow head, no activation).  fp32 "parity" engine, NCDHW.
 * x: (B,Cin,D,H,W)  w: (Cout,Cin,kd,3,3) with kd = 3 (3-D) or 1 (2-D)  y: (B,Cout,D,H,W).
 * leaky_slope < 0 disables the activation. */
int vxm_conv3d_fwd_f32(const float* x, const float* w, const float* bias, float* y,
                       int B, int Cin, int Cout, int D, int H, int W, int kd,
                       float leaky_slope, void* stream);
/* grad_y is the gradient w.r.t. the ACTIVATED output y; y (saved forward output) supplies the
 * LeakyReLU mask (y < 0).  grad_x may be NULL (first layer).  grad_w / grad_b are ACCUMULATED
 * into (caller zero-fills once per step).  work: vxm_conv3d_bwd_workspace_bytes(). */
size_t vxm_conv3d_bwd_workspace_bytes(int B, int Cin, int Cout, int D, int H, int W, int kd);
int vxm_conv3d_bwd_f32(const float* grad_y, const float* y, const float* x, const float* w,
                       float* grad_x, float* grad_w, float* grad_b, void* work,
                       int B, int Cin, int Cout, int D, int H, int W, int kd,
                       float leaky_slope, void* stream);

/* ---- Conv3d k=3 on the tensor cores (wgmma, bf16 operands, fp32 register accumulation), channels-last ----
 * The throughput engine for reference networks.py:299-304 / :211,257; forward and dgrad share one kernel.
 * Activations are bf16 NDHWC (B,D,H,W,C).  Weights are pre-packed by vxm_conv3d_tc_pack into the wgmma
 * canonical K-major layout [tap][K/16][2][N][8] (bf16); `transposed` = 1 packs the dgrad operator
 * (channel roles swapped, taps flipped).  np = MMA N (16 or 32) >= number of output channels. */
size_t vxm_conv3d_tc_packed_bytes(int cin_eff, int np, int kd);
int vxm_conv3d_tc_pack(const float* w, void* wpk, int Cout, int Cin, int kd, int np, int transposed,
                       void* stream);
/* Input = channel concat of [xa (Ca ch; at HALF resolution and nearest-upsampled x2 on the fly when up=1),
 * xb (Cb ch)], both bf16 NDHWC; or, when nplanar > 0, `nplanar` (<= 4) planar fp32 volumes xf[i]
 * ((B,D,H,W) each, batch stride xf_bstride[i] floats) converted on load (first layer: source/target images;
 * flow-head dgrad: the 3 flow-gradient planes).  out_mode 0: bf16 NDHWC (B,D,H,W,Cout), Cout % 8 == 0;
 * out_mode 1: fp32 NCDHW.  Epilogue: + bias (may be NULL), then LeakyReLU(slope) if slope >= 0; if `mask`
 * (bf16 NDHWC, same shape as out) is given the activation is replaced by  out *= (mask < 0 ? slope : 1)
 * (LeakyReLU derivative of the layer below, for dgrad). */
int vxm_conv3d_tc_fwd(const void* xa, const void* xb, const float* const* xf, const long long* xf_bstride,
                      int nplanar, const void* wpk, const float* bias, void* out, const void* mask,
                      int B, int D, int H, int W, int Ca, int Cb, int up, int Cout, int np, int kd,
                      int out_mode, float slope, void* out2, int csplit, void* stream);
/* out2 != NULL (bf16 outputs only): channels [0,csplit) go to `out` (B,D,H,W,csplit) and [csplit,Cout) to `out2`
 * (B,D,H,W,Cout-csplit) — the single-pass dgrad of a layer whose input was a channel concat; np may then be 48 or 64. */
/* "kw-stacked" variant of the tensor-core convolution (Cin in {8,16,32,48,64}, Cout <= 64): the three kw taps are
 * stacked along the MMA N dimension (N = 3*coutp), the K loop runs over (kd,kh,Cin/16) only and the kw shift is a warp
 * shuffle in the epilogue — the activation operand is read 9x instead of 27x.  Same inputs / outputs / epilogue options
 * as vxm_conv3d_tc_fwd (no planar sources); weights are packed by vxm_conv3d_tct_pack (coutp in {16,32,48,64}). */
size_t vxm_conv3d_tct_packed_bytes(int cin_eff, int coutp, int kd);
int vxm_conv3d_tct_pack(const float* w, void* wpk, int Cout, int Cin, int kd, int coutp, int transposed, void* stream);
int vxm_conv3d_tct_supported(int Ca, int Cb, int Cout);
int vxm_conv3d_tct_fwd(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, const void* mask,
                       int B, int D, int H, int W, int Ca, int Cb, int up, int Cout, int coutp, int kd, int out_mode,
                       float slope, void* out2, int csplit, void* stream);
/* Swizzled-operand variant of the kw-stacked kernel (128/64/32-byte swizzled K-major shared-memory layouts): same
 * arguments and semantics as vxm_conv3d_tct_*; weights are packed by vxm_conv3d_tcs_pack. */
size_t vxm_conv3d_tcs_packed_bytes(int cin_eff, int coutp, int kd);
int vxm_conv3d_tcs_pack(const float* w, void* wpk, int Cout, int Cin, int kd, int coutp, int transposed, void* stream);
int vxm_conv3d_tcs_supported(int Ca, int Cb, int Cout);
/* every packed operand of a model in ONE launch: the caller fills an array of descriptors on the host
 * (vxm_conv3d_tcs_pack_desc_bytes() bytes each; vxm_conv3d_tcs_pack_desc returns the operand's element count so that
 * `begin` can be chained), uploads it once and calls vxm_conv3d_tcs_pack_multi with the summed element count. */
size_t vxm_conv3d_tcs_pack_desc_bytes(void);
int vxm_conv3d_tcs_pack_desc(void* desc_host, const float* w, void* wpk, int Cout, int Cin, int kd, int coutp, int transposed,
                             int begin);
/* descriptor of a kd-folded 2-D operand of the 3-D weight w (Cout, Cin, 3, 3, 3): operand input channel kd * r + c is tap kd of
 * real channel c, r = Cin (Cout when transposed), 3 r <= 16; packed size = vxm_conv3d_tcs_packed_bytes(3 r, coutp, 1) */
/* descriptor of one channel block of an operand: operand output channels [n0, n0 + nb), input channels [k0, k0 + kb) (the
 * operand's orientation: transposed swaps Cout and Cin); packed size = vxm_conv3d_tcs_packed_bytes(kb, coutp, kd) */
int vxm_conv3d_tcs_pack_desc_blk(void* desc_host, const float* w, void* wpk, int Cout, int Cin, int kd, int coutp, int transposed,
                                 int n0, int nb, int k0, int kb, int begin);
int vxm_conv3d_tcs_pack_desc_fold(void* desc_host, const float* w, void* wpk, int Cout, int Cin, int coutp, int transposed, int begin);
int vxm_conv3d_tcs_pack_multi(const void* descs_dev, int ndesc, int total, void* stream);
int vxm_conv3d_tcs_fwd(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, const void* mask,
                       int B, int D, int H, int W, int Ca, int Cb, int up, int Cout, int coutp, int kd, int out_mode,
                       float slope, void* out2, int csplit, void* stream);
/* Split-precision ("bf16x3") passes of the same kernel — the in-tolerance tensor-core mode (reference layer:
 * voxelmorph/torch/networks.py:290-305 in fp32).  Every operand is a bf16 pair hi + lo (16 mantissa bits); a layer is
 * three launches that accumulate  x_lo*w_hi + x_hi*w_lo + x_hi*w_hi  in fp32:
 *   out_mode 2: out (fp32, channels-last, `coutp` channels per voxel) = acc_in + conv   (no bias / activation; acc_in may
 *               be NULL or alias out);
 *   out_mode 3: x = act(acc_in + conv + bias) stored as the bf16 pair out (hi), out_lo (lo = bf16(x - hi));
 *   out_mode 1: fp32 planar out = acc_in + conv + bias (the flow head).
 * acc_in has `coutp` channels per voxel. */
int vxm_conv3d_tcs_fwd_acc(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, void* out_lo,
                           const float* acc_in, int B, int D, int H, int W, int Ca, int Cb, int up, int Cout, int coutp,
                           int kd, int out_mode, float slope, void* stream);
/* 1 when one launch of the kernel has the shared memory for a (cin -> coutp, kd) operand; wider layers run in channel blocks. */
int vxm_conv3d_tcs_fits(int cin, int coutp, int kd);
/* One channel block of a layer too wide for one launch.  out_mode 0: bf16 act(acc_in + conv + bias) (acc_in may be NULL;
 * mask: LeakyReLU derivative from the saved activation, as vxm_conv3d_tcs_fwd); 2 and 3: as vxm_conv3d_tcs_fwd_acc.
 * opitch: channels per voxel of out / out_lo / mask when the block is part of a wider tensor (the pointers are offset to
 * the block's first channel; 0 = dense).  acc_in and the out_mode 2 output are dense with `coutp` channels. */
int vxm_conv3d_tcs_fwd_blk(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, void* out_lo,
                           const void* mask, const float* acc_in, int B, int D, int H, int W, int Ca, int Cb, int up, int Cout,
                           int coutp, int kd, int out_mode, float slope, int opitch, void* stream);
/* Polyphase launches of a 3-D concat layer whose first Ca = 32 input channels are a nearest-x2 upsampled source (the taps
 * that read the same coarse voxel merged into one).  mode 1: forward of (32 upsampled + 16) -> 32 with bias + LeakyReLU
 * (xa coarse, xb and out at the fine (D, H, W); kd taps merged).  mode 2: coarse dgrad (kd and kh taps merged): xa = the
 * layer's 32-channel output gradient (B, D, H, W, 32), mask = the coarse source (B, D / 2, H / 2, W / 2, 32), a LeakyReLU
 * activation of negative slope `slope`; out = the gradient w.r.t. its pre-activation, same shape.  Operands:
 * vxm_conv3d_tcs_pack_desc_poly (same mode; Cout, Cin: the weight's, Ca: the upsampled channels),
 * vxm_conv3d_tcs_poly_packed_bytes bytes (0: no such operand). */
size_t vxm_conv3d_tcs_poly_packed_bytes(int mode, int Cout, int Cin, int Ca);
int vxm_conv3d_tcs_pack_desc_poly(void* desc_host, const float* w, void* wpk, int Cout, int Cin, int Ca, int mode, int begin);
int vxm_conv3d_tcs_poly(const void* xa, const void* xb, const void* wpk, const float* bias, void* out, const void* mask, int B, int D,
                        int H, int W, int Ca, int Cb, int Cout, int mode, float slope, void* stream);
/* Weight (and bias) gradient on tensor cores.  x sources as in vxm_conv3d_tc_fwd (the layer's forward input);
 * gz = gradient w.r.t. the convolution output (already multiplied by the activation derivative): bf16 NDHWC with
 * Cg in {8,16,32} channels, or nplanar_g (<= 4) planar fp32 volumes (flow head).  grad_w: fp32
 * (Cout_real, Cin_real, kd, 3, 3); grad_b: fp32 (Cout_real), may be NULL.  accumulate = 0 overwrites them, 1 adds to
 * them (gradient buffers zeroed once per step).  work: vxm_conv3d_tc_wgrad_workspace_bytes(kd). */
size_t vxm_conv3d_tc_wgrad_workspace_bytes(int kd);
int vxm_conv3d_tc_wgrad(const void* xa, const void* xb, const float* const* xf, const long long* xf_bstride,
                        int nplanar_x, const void* gz, const float* const* gf, const long long* gf_bstride,
                        int nplanar_g, float* grad_w, float* grad_b, void* work, int B, int D, int H, int W,
                        int Ca, int Cb, int up, int Cin_real, int Cg, int Cout_real, int kd, int accumulate, void* stream);
/* Deferred reduction of the weight gradient (channels-last bf16 sources only): `_partial` launches the wgmma kernel(s) of
 * one layer into caller-provided workspace (`work_used` bytes of it are then owned by this layer until the flush) and
 * appends the pending reductions to a HOST array of descriptors (vxm_conv3d_tc_wgrad2_desc_bytes() each, at most
 * vxm_conv3d_tc_wgrad2_max_pending()); `_flush` reduces every pending layer in ONE launch, in a fixed order
 * (deterministic).  Arguments as vxm_conv3d_tc_wgrad, except that Ca, Cb and Cg may also be 64: such a layer runs as
 * 32-channel slices of both operands, one pending reduction per slice pair. */
size_t vxm_conv3d_tc_wgrad2_desc_bytes(void);
int vxm_conv3d_tc_wgrad2_max_pending(void);
size_t vxm_conv3d_tc_wgrad2_partial_bytes(int kd);
int vxm_conv3d_tc_wgrad2_partial(const void* xa, const void* xb, const void* gz, float* grad_w, float* grad_b, void* work,
                                 size_t work_bytes, size_t* work_used, void* descs_host, int* ndesc, int B, int D, int H, int W,
                                 int Ca, int Cb, int up, int Cin_real, int Cg, int Cout_real, int kd, int accumulate, void* stream);
int vxm_conv3d_tc_wgrad2_flush(const void* descs_host, int ndesc, void* stream);
/* Weight gradient of a "kd-folded" layer (vxm_planar_fold_kd_bf16): x (B,D,H,W,Cx) against gz (B,D,H,W,Cg), Cx, Cg in {8,16}, as
 * a 2-D problem per slice with the kh taps stacked in the MMA's M; grad_w has the 2-D layout (Cout_real, Cin_real, 1, 3, 3).
 * Deferred like vxm_conv3d_tc_wgrad2_partial (one pending reduction). */
int vxm_conv3d_tc_wgrad2_partial_khm(const void* x, const void* gz, float* grad_w, float* grad_b, void* work, size_t work_bytes,
                                     size_t* work_used, void* descs_host, int* ndesc, int B, int D, int H, int W, int Cx,
                                     int Cin_real, int Cg, int Cout_real, int accumulate, void* stream);
/* ---- channels-last bf16 glue of the tensor-core U-Net engine (reference networks.py:126-138 and its autograd) ----
 * All tensors bf16 (B,D,H,W,C), C % 8 == 0.  (Dc,Hc,Wc) are the COARSE dims; the fine tensor is (fd*Dc, 2Hc, 2Wc)
 * with fd = 2 for nd == 3 and 1 for nd == 2. */
int vxm_pool2_ndhwc_bf16(const void* x_fine, void* y_coarse, int B, int Dc, int Hc, int Wc, int C, int nd, void* stream);
/* out_coarse = (sum over the 2^nd children of g_fine) * (act_coarse < 0 ? slope : 1); act_coarse may be NULL */
int vxm_sumpool_mask_ndhwc_bf16(const void* g_fine, const void* act_coarse, void* out_coarse, int B, int Dc, int Hc,
                                int Wc, int C, int nd, float slope, void* stream);
/* out_fine = (g_skip_fine + [child is the first max of e_fine in its window] * g_pool_coarse) * (e_fine < 0 ? slope : 1);
 * g_skip or g_pool may be NULL (not both) */
int vxm_unpool_combine_ndhwc_bf16(const void* e_fine, const void* g_skip_fine, const void* g_pool_coarse, void* out_fine,
                                  int B, int Dc, int Hc, int Wc, int C, int nd, float slope, void* stream);
/* out (B,V,8) bf16 <- up to 8 planar fp32 volumes (channel c = planes[c], batch stride bstrides[c] floats); unused
 * channels are zero.  Feeds the fp32 images / the fp32 flow gradient to the tensor-core kernels. */
int vxm_planar_to_ndhwc8_bf16(const float* const* planes, const long long* bstrides, int nplanes, void* out, int B,
                              size_t V, void* stream);
/* kd folded into the channels: out (B,D,HW,cout) bf16, cout in {8,16}, channel kd * nplanes + p = planes[p] at slice d + kd - 1
 * (zero outside the volume), kd = 0..2; 3 * nplanes <= cout.  A 3-D convolution with so few real input channels then runs as a
 * 2-D one over the folded tensor (reference layers: the first ConvBlock, networks.py:122-130, and the flow head's autograd). */
int vxm_planar_fold_kd_bf16(const float* const* planes, const long long* bstrides, int nplanes, void* out, int B, int D,
                            size_t HW, int cout, void* stream);
/* split-precision variants: out_hi = bf16(x), out_lo = bf16(x - out_hi); MaxPool(2) of a (hi, lo) pair tensor (the
 * maximum is taken on hi + lo, the winning child's pair is copied) */
int vxm_planar_to_ndhwc8_split_bf16(const float* const* planes, const long long* bstrides, int nplanes, void* out_hi,
                                    void* out_lo, int B, size_t V, void* stream);
int vxm_pool2_split_ndhwc_bf16(const void* x_hi, const void* x_lo, void* y_hi, void* y_lo, int B, int Dc, int Hc, int Wc,
                               int C, int nd, void* stream);
/* vxm_unpool_combine_ndhwc_bf16 after a split-precision pool: the pool gradient goes to the first child with the largest
 * e_hi + e_lo (the child vxm_pool2_split_ndhwc_bf16 copied); the LeakyReLU derivative reads e_hi < 0 */
int vxm_unpool_combine_split_ndhwc_bf16(const void* e_hi, const void* e_lo, const void* g_skip_fine, const void* g_pool_coarse,
                                        void* out_fine, int B, int Dc, int Hc, int Wc, int C, int nd, float slope, void* stream);

/* ---- MaxPool(2) / nearest Upsample(2) + concat: reference networks.py:83-85,130,137-138 ----
 * pool factor is 2 on H, W and on D when D > 1 (nd == 3).  idx (uint8, same shape as y) stores the
 * argmax within the window for the backward. */
int vxm_maxpool2_fwd(const float* x, float* y, uint8_t* idx, int B, int C, int D, int H, int W,
                     int nd, void* stream);
int vxm_maxpool2_bwd(const float* grad_y, const uint8_t* idx, float* grad_x, int B, int C, int D,
                     int H, int W, int nd, void* stream);
/* out (B, Ca+Cb, 2D,2H,2W) = cat(upsample2(a (B,Ca,D,H,W)), skip (B,Cb,2D,2H,2W)); skip may be NULL (Cb=0) */
int vxm_upcat_fwd(const float* a, const float* skip, float* out, int B, int Ca, int Cb, int D,
                  int H, int W, int nd, void* stream);
/* grad_a overwritten (sum over the 2^nd children), grad_skip overwritten (may be NULL) */
int vxm_upcat_bwd(const float* grad_out, float* grad_a, float* grad_skip, int B, int Ca, int Cb,
                  int D, int H, int W, int nd, void* stream);

/* ---- Adam on one flat buffer: reference scripts/torch/train.py:161,220 (torch.optim.Adam) ----
 * p, g, m, v: n floats.  grad_scale multiplies g first (1/world_size after an allreduce-sum). */
int vxm_adam_step(float* p, const float* g, float* m, float* v, size_t n, int step, float lr,
                  float beta1, float beta2, float eps, float weight_decay, float grad_scale,
                  void* stream);

/* Same update with the step count kept on the device (incremented by the call): safe to capture in a CUDA graph. */
int vxm_adam_step_dev(float* p, const float* g, float* m, float* v, size_t n, int* step_counter, float lr,
                      float beta1, float beta2, float eps, float weight_decay, float grad_scale, void* stream);

/* ---- MeanStream(cap): the capped running mean TemplateCreation keeps of its inverse flow (reference
 * voxelmorph/tf/networks.py:761-853, neurite's MeanStream) ----
 * x (B, n) fp32 (n = nd * voxels, 2-D or 3-D alike), mean (n) and count (1) fp32 device state:
 *   S = sum_b x_b, n' = count + B, alpha = B / min(n', cap), m' = mean (1 - alpha) + (S / B) alpha,
 *   out (n) = min(1, n' / cap) m'; commit = 1 (training) also writes mean <- m', count <- n' (0: state untouched).
 * saved (1 float) receives min(1, n' / cap) alpha / B for the backward; work is the reduce workspace
 * (vxm_reduce_workspace_bytes: only its ticket counter is used).  count is read and written on the device only. */
int vxm_mean_stream_fwd(const float* x, float* mean, float* count, float* out, float* saved, void* work, int B, size_t n,
                        float cap, int commit, void* stream);
/* grad_x_b = saved[0] * sum_b' grad_out_b' for every b (sum in b' order); grad_out's batch stride is n, or 0 for a
 * gradient that is itself broadcast over the batch */
int vxm_mean_stream_bwd(const float* grad_out, const float* saved, float* grad_x, int B, size_t n, size_t gout_bstride,
                        void* stream);

/* ---- SampleNormalLogVar of probabilistic VoxelMorph (reference voxelmorph/tf/networks.py:155-165) ----
 * params: flow_params (B, 2 nd, V) fp32 (mu = channels [0, nd), logvar = [nd, 2 nd)); z (B, nd, V) fp32:
 *   z = mu + exp(logvar / 2) eps,  eps ~ N(0, 1) from Philox4x32-10 keyed by state[0] (the seed): element
 *   i = (b nd + c) V + v takes word i mod 4 of the block with counter (lo32(i / 4), hi32(i / 4), lo32(call), hi32(call)),
 *   Box-Muller on the word pairs (0, 1), (2, 3) with u1 = ((w0 >> 8) + 1) 2^-24, u2 = (w1 >> 8) 2^-24:
 *   eps0 = sqrt(-2 log u1) cos(2 pi u2), eps1 = sqrt(-2 log u1) sin(2 pi u2).
 * state (2 int64, device) = (seed, call): the forward writes call to ticket (1 int64, device) and commits call + 1 (work:
 * the reduce workspace, whose ticket counter orders the commit); no host read.  The backward regenerates eps from
 * (state[0], *ticket): grad_params[mu] = grad_z, grad_params[logvar] = grad_z eps exp(logvar / 2) / 2. */
int vxm_sample_normal_logvar_fwd(const float* params, float* z, long long* state, long long* ticket, void* work, int B,
                                 int nd, size_t V, void* stream);
int vxm_sample_normal_logvar_bwd(const float* grad_z, const float* params, const long long* state, const long long* ticket,
                                 float* grad_params, int B, int nd, size_t V, void* stream);

/* ---- Phenotype decoder of ConditionalTemplateCreation (reference voxelmorph/tf/networks.py:856-983): Dense(V F, 'elu')
 * and neurite's conv_dec with no levels (one 1x1 convolution F -> F, bias, linear) as one launch each way ----
 * pheno (B, P), W (P, F, V), bias (F, V), like_w (F, F, [1, 1, 1]) (output channel g, input channel f), like_b (F),
 * out (B, F, V), all fp32 device memory owned by the caller; V = prod(vol) (2-D and 3-D alike), 1 <= P <= 16,
 * 1 <= F <= 32:
 *   pre[b,f,v] = bias[f,v] + sum_p pheno[b,p] W[p,f,v],  h = pre > 0 ? pre : expm1(pre),
 *   out[b,g,v] = like_b[g] + sum_f like_w[g,f] h[b,f,v]            (out overwritten)
 * The backward recomputes pre and h (no activation is stored) and gives, with g_pre = (like_w^T grad_out) (h < 0 ? h + 1 : 1):
 *   grad_W[p,f,v] = sum_b pheno[b,p] g_pre[b,f,v],  grad_bias[f,v] = sum_b g_pre[b,f,v],
 *   grad_like_w[g,f] = sum_{b,v} grad_out[b,g,v] h[b,f,v],  grad_like_b[g] = sum_{b,v} grad_out[b,g,v];
 * accumulate = 1 adds them to the four gradient buffers, 0 overwrites them (a batch larger than the kernel's register
 * chunk, 64 / F entries rounded down to 1, 2 or 4, is added to grad_W and grad_bias one chunk at a time).  No gradient is
 * formed for pheno.  Sums run in a fixed order: results are bit-reproducible.  work:
 * vxm_pheno_decoder_workspace_bytes(F) bytes, zero before its first use; the call leaves it reusable. */
size_t vxm_pheno_decoder_workspace_bytes(int F);
int vxm_pheno_decoder_fwd(const float* pheno, const float* W, const float* bias, const float* like_w, const float* like_b,
                          float* out, int B, int P, int F, size_t V, void* stream);
int vxm_pheno_decoder_bwd(const float* grad_out, const float* pheno, const float* W, const float* bias, const float* like_w,
                          float* grad_W, float* grad_bias, float* grad_like_w, float* grad_like_b, void* work, int B, int P,
                          int F, size_t V, int accumulate, void* stream);

/* ---- HyperMorph (reference voxelmorph/tf/networks.py:1192-1231): the hypernetwork and the U-Net weights it generates ----
 * Hypernetwork: hyp (P), nb_layers Dense layers of U units with ReLU, weights in torch.nn.Linear's (out, in) layout:
 * weights[0] (U, P), weights[l > 0] (U, U), biases[l] (U).  `weights`, `biases`, `grad_weights` and `grad_biases` are
 * HOST arrays of nb_layers device pointers.  1 <= P <= 16, 1 <= U <= 256, 1 <= nb_layers <= 8.
 *   pre (nb_layers, U): every layer's pre-activation (kept for the backward),  h (U) = relu(pre[nb_layers - 1])
 * The backward turns grad_h (U) into the gradient of every weight and bias (TF's ReluGrad: pre > 0); none for hyp.
 * Generated weights: A (U, N) row-major, a (N), W (N), all fp32 device memory:
 *   W[j] = a[j] + sum_k h[k] A[k,j]                                                         (W overwritten)
 *   grad_A[k,j] = h[k] grad_W[j],  grad_a[j] = grad_W[j],  grad_h[k] = sum_j A[k,j] grad_W[j]  (grad_h overwritten)
 * accumulate = 1 adds the parameter gradients to their buffers (a rounded product, then a rounded sum: what autograd's
 * accumulation computes), 0 overwrites them.  Sums run in a fixed order: results are bit-reproducible.  work:
 * vxm_hyper_workspace_bytes(U, N) bytes of scratch (no initial value needed); 0 for sizes the kernels refuse. */
size_t vxm_hyper_workspace_bytes(int U, size_t N);
int vxm_hyper_mlp_fwd(const float* hyp, const float* const* weights, const float* const* biases, float* pre, float* h,
                      int P, int U, int nb_layers, void* stream);
int vxm_hyper_mlp_bwd(const float* grad_h, const float* hyp, const float* const* weights, const float* pre,
                      float* const* grad_weights, float* const* grad_biases, int P, int U, int nb_layers, int accumulate,
                      void* stream);
int vxm_hyper_weights_fwd(const float* h, const float* A, const float* a, float* W, int U, size_t N, void* stream);
int vxm_hyper_weights_bwd(const float* h, const float* A, const float* grad_W, float* grad_A, float* grad_a,
                          float* grad_h, void* work, int U, size_t N, int accumulate, void* stream);

/* ---- MutualInformation: reference voxelmorph/tf/losses.py:352-367 (neurite's soft-binned MI, `volumes` form) ----
 * y_true = x, y_pred = y: (N, V) fp32 each (single-channel volumes).  2 <= nbins = B <= 64.  centers: B device floats
 * used for both tensors, or NULL for c_b = lo + (hi - lo) b / (B - 1) with lo, hi the min and max of that tensor over
 * all N V elements.  For each tensor t~ = clip(t, min_clip, max_clip), w_vb = softmax_b(-alpha (t~_v - c_b)^2); per item,
 * with eps = 1e-7:  P = sum_v wx_v wy_v^T,  pxy = P / (sum P + eps),  px = sx / (sum sx + eps), sx = sum_v wx_v (py
 * likewise),  MI_n = sum pxy log(pxy / (px py^T + eps) + eps);  loss[0] = -mean_n MI_n.
 * The backward writes grad_loss[0] * dloss/dy_true and/or dloss/dy_pred (a NULL output is not computed): the exact
 * derivative, clip gradients passed where min_clip <= t <= max_clip, and with data-driven centres the min/max path
 * split equally among the voxels tied at the min and at the max.  work: vxm_mi_workspace_bytes(N, V, nbins) bytes (no
 * initial value needed), written by the forward and read by the backward of the same inputs.  reduce_work
 * (vxm_reduce_workspace_bytes, zeroed once) is used only with data-driven centres.  Sums run in a fixed order and
 * there is no host synchronisation: results are bit-reproducible and the calls can be captured in a CUDA graph. */
size_t vxm_mi_workspace_bytes(int N, size_t V, int nbins);
int vxm_mi_fwd(const float* y_true, const float* y_pred, const float* centers, float* loss, void* work, void* reduce_work,
               int N, size_t V, int nbins, float alpha, float min_clip, float max_clip, void* stream);
int vxm_mi_bwd(const float* y_true, const float* y_pred, const float* centers, const float* grad_loss, float* grad_true,
               float* grad_pred, void* work, int N, size_t V, int nbins, float alpha, float min_clip, float max_clip,
               void* stream);

/* ---- Surface points: reference voxelmorph/tf/utils/utils.py:465-499 (point_spatial_transformer) and 71-88
 * (value_at_location), as VxmDenseSemiSupervisedPointCloud uses them (voxelmorph/tf/networks.py:391-486) ----
 * Sampling is neurite's interpn(..., 'linear', fill_value=None): per axis of size n at x, c = clip(x, 0, n-1),
 * i0 = clip(floor x, 0, n-1), i1 = clip(i0+1, 0, n-1), weight i1 - c on i0 and 1 - (i1 - c) on i1, weights multiplied
 * across axes; outside the volume the border value, and d/dx = 0 there (the clip passes its gradient for 0 <= x <= n-1).
 * points: (B, N, nd+1), the spatial coordinates in the flow's axis order (3-D: D, H, W; 2-D: H, W), the last column a
 * label index.  flow: (B, nd, D, H, W).  Point warp: out (B, N, nd+1), out = p + r * interp(flow, p), label column
 * copied.  Its backward ADDS to grad_flow (B, nd, D, H, W) the flow gradient of grad_out (B, N, nd+1; label column
 * ignored): pairs sorted by voxel (CUB radix sort) and summed per voxel in point order in fp64, no float atomics and no
 * host synchronisation, so it is bit-reproducible and graph-capturable.  work: vxm_point_warp_workspace_bytes(...)
 * bytes, O(B N 2^nd), no initial value (the size query asks CUB for its scratch size, which reads the current
 * device; 0 for sizes the kernels refuse: B * D * H * W must stay below 2^32, B * N * 2^nd below 2^31).
 * Distance lookup: sdt (B, L, D, H, W), points (B, N, nd+1) with the label index interpolated (and clamped) as an
 * (nd+1)-th axis; out (B, N) = |interp(sdt, q)|.  Backward: grad_points (B, N, nd+1) = grad_out * sign(v) * d interp/dq
 * over the spatial columns (sign(0) = 0), 0 in the label column (overwritten). */
size_t vxm_point_warp_workspace_bytes(int B, int N, int D, int H, int W, int nd);
int vxm_point_warp_fwd(const float* points, const float* flow, float* out, int B, int N, int D, int H, int W, int nd,
                       float r, void* stream);
int vxm_point_warp_bwd(const float* points, const float* grad_out, float* grad_flow, void* work, size_t work_bytes,
                       int B, int N, int D, int H, int W, int nd, float r, void* stream);
int vxm_value_at_fwd(const float* sdt, const float* points, float* out, int B, int N, int L, int D, int H, int W,
                     int nd, void* stream);
int vxm_value_at_bwd(const float* sdt, const float* points, const float* grad_out, float* grad_points, int B, int N,
                     int L, int D, int H, int W, int nd, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VXM_B200_H */
