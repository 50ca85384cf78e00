"""SpatialTransformer / VecInt / ResizeTransform with the reference's surface
(reference voxelmorph/torch/layers.py) over the sm_90a kernels of libvxm_b200.so.

Same class names, constructor arguments, forward signatures and error behaviour as the
reference; the arithmetic runs in hand-written CUDA kernels reached through the C ABI
(include/vxm_b200.h).  There is no CPU path.
"""
import math
import os

import torch
import torch.nn as nn

from . import _lib

MODE_LINEAR, MODE_NEAREST = 0, 1
ARITH_TRUE_DIV, ARITH_RECIPROCAL, ARITH_FAST = 0, 1, 2


def default_arith():
    """How `loc / (S-1)` (reference layers.py:37) is rounded.  'cpu' (default) replays torch's CPU
    true division — the oracle this repo is bit-exact against; 'cuda' replays torch's CUDA
    multiply-by-reciprocal."""
    return ARITH_RECIPROCAL if os.environ.get("VXM_B200_NEAREST_ARITH", "cpu") == "cuda" else ARITH_TRUE_DIV


def linear_arith():
    """Coordinate arithmetic of the LINEAR resampler (SpatialTransformer 'bilinear', VecInt).  Default 'fast':
    coord = (p + flow) * (Ssrc-1)/(S-1) — the reference's map without its fp32 normalise / un-normalise round trip;
    agrees with the replayed arithmetic to a few 1e-6 of the value range (north_star asks 1e-4) and lets the kernels run
    memory bound.  VXM_B200_LINEAR_ARITH=exact replays torch's arithmetic op for op (bit-identical to the torch CPU
    reference on every input tried), like the nearest mode always does."""
    return default_arith() if os.environ.get("VXM_B200_LINEAR_ARITH", "fast") == "exact" else ARITH_FAST


def _dims(t):
    """(B, C, D, H, W, nd) of a (B,C,[D,]H,W) tensor; 2-D is carried as D == 1."""
    if t.dim() == 5:
        B, C, D, H, W = t.shape
        return B, C, D, H, W, 3
    if t.dim() == 4:
        B, C, H, W = t.shape
        return B, C, 1, H, W, 2
    raise _lib.VxmError("voxelmorph_b200: expected a (B,C,H,W) or (B,C,D,H,W) tensor, got shape %s" % (tuple(t.shape),))


class _WarpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, src, flow, mode, arith):
        _lib.require_cuda(src, flow, what="SpatialTransformer")
        src, flow = _lib.contig(src), _lib.contig(flow)
        B, C, Ds, Hs, Ws, nd = _dims(src)
        Bf, Cf, D, H, W, ndf = _dims(flow)
        if nd != ndf or Cf != nd or Bf != B:
            raise _lib.VxmError("SpatialTransformer: src %s and flow %s are inconsistent"
                                % (tuple(src.shape), tuple(flow.shape)))
        out = torch.empty((B, C) + tuple(flow.shape[2:]), dtype=torch.float32, device=src.device)
        lib = _lib.load()
        _lib.check(lib.vxm_warp_fwd(_lib.ptr(src), _lib.ptr(flow), _lib.ptr(out), B, C, Ds, Hs, Ws, D, H, W, nd,
                                    mode, arith, _lib.stream_ptr()), "vxm_warp_fwd")
        ctx.save_for_backward(src, flow)
        ctx.cfg = (mode, arith)
        return out

    @staticmethod
    def backward(ctx, gout):
        src, flow = ctx.saved_tensors
        mode, arith = ctx.cfg
        gout = _lib.contig(gout)
        B, C, Ds, Hs, Ws, nd = _dims(src)
        _, _, D, H, W, _ = _dims(flow)
        need_src, need_flow = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        gsrc = torch.zeros_like(src) if need_src else None
        gflow = None
        if need_flow:
            gflow = torch.zeros_like(flow) if mode == MODE_NEAREST else torch.empty_like(flow)
        if need_src or (need_flow and mode == MODE_LINEAR):
            lib = _lib.load()
            _lib.check(lib.vxm_warp_bwd(_lib.ptr(gout), _lib.ptr(src), _lib.ptr(flow), _lib.ptr(gsrc),
                                        _lib.ptr(gflow) if mode == MODE_LINEAR else None,
                                        B, C, Ds, Hs, Ws, D, H, W, nd, mode, arith, _lib.stream_ptr()),
                       "vxm_warp_bwd")
        return gsrc, gflow, None, None


class SpatialTransformer(nn.Module):
    """N-D spatial transformer (reference layers.py:6-48).

    `size` is kept for signature compatibility; no identity-grid buffer is materialised (the
    reference registers an 82.6 MB `grid` buffer per instance at 160x192x224) — checkpoints
    never contain it (modelio drops `*.grid`), so state_dict compatibility is unaffected.
    """

    def __init__(self, size, mode='bilinear'):
        super().__init__()
        self.mode = mode
        self.size = tuple(int(s) for s in size)

    def forward(self, src, flow):
        if self.mode == 'bilinear':
            m = MODE_LINEAR
        elif self.mode == 'nearest':
            m = MODE_NEAREST
        else:
            # F.grid_sample raises for anything but bilinear / nearest / bicubic; bicubic is 4-D only
            raise ValueError("nn.functional.grid_sample(): expected mode to be 'bilinear' or 'nearest', "
                             "but got: '%s'" % self.mode)
        return _WarpFn.apply(src, flow, m, linear_arith() if m == MODE_LINEAR else default_arith())


class _VecIntFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vec, nsteps, arith):
        _lib.require_cuda(vec, what="VecInt")
        vec = _lib.contig(vec)
        B, C, D, H, W, nd = _dims(vec)
        if C != nd:
            raise _lib.VxmError("VecInt: expected %d flow channels, got %d" % (nd, C))
        lib = _lib.load()
        out = torch.empty_like(vec)
        need_grad = ctx.needs_input_grad[0]
        if arith == ARITH_FAST and (nd != 3 or nsteps < 1 or min(D, H, W) < 2):
            arith = default_arith()      # the float4 fast path is 3-D only
        states = work = None
        if nsteps > 0:
            if arith == ARITH_FAST:
                if need_grad:
                    states = torch.empty(int(lib.vxm_vecint_fast_states_bytes(B, D, H, W, nsteps)), dtype=torch.uint8, device=vec.device)
                else:
                    work = torch.empty(int(lib.vxm_vecint_fast_work_bytes(B, D, H, W, 0)), dtype=torch.uint8, device=vec.device)
            elif need_grad:
                states = torch.empty((nsteps,) + tuple(vec.shape), dtype=torch.float32, device=vec.device)
            else:
                work = torch.empty_like(vec)
        _lib.check(lib.vxm_vecint_fwd(_lib.ptr(vec), _lib.ptr(out), _lib.ptr(states), _lib.ptr(work), B, D, H, W, nd,
                                      nsteps, arith, _lib.stream_ptr()), "vxm_vecint_fwd")
        ctx.states = states
        ctx.cfg = (nsteps, arith, (B, D, H, W, nd))
        return out

    @staticmethod
    def backward(ctx, gout):
        nsteps, arith, (B, D, H, W, nd) = ctx.cfg
        gout = _lib.contig(gout)
        gvel = torch.empty_like(gout)
        lib = _lib.load()
        work = None
        if nsteps > 0:
            if arith == ARITH_FAST:
                work = torch.empty(int(lib.vxm_vecint_fast_work_bytes(B, D, H, W, 1)), dtype=torch.uint8, device=gout.device)
            else:
                work = torch.empty((2,) + tuple(gout.shape), dtype=torch.float32, device=gout.device)
        _lib.check(lib.vxm_vecint_bwd(_lib.ptr(gout), _lib.ptr(ctx.states), _lib.ptr(gvel), _lib.ptr(work), B, D, H, W,
                                      nd, nsteps, arith, _lib.stream_ptr()), "vxm_vecint_bwd")
        return gvel, None, None


class VecInt(nn.Module):
    """Integrates a vector field via scaling and squaring (reference layers.py:51-68), all
    `nsteps` squarings fused into one cooperative kernel launch."""

    def __init__(self, inshape, nsteps):
        super().__init__()
        assert nsteps >= 0, 'nsteps should be >= 0, found: %d' % nsteps
        self.nsteps = nsteps
        self.scale = 1.0 / (2 ** self.nsteps)
        self.transformer = SpatialTransformer(inshape)

    def forward(self, vec):
        return _VecIntFn.apply(vec, self.nsteps, linear_arith())


class _ResizeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, out_spatial, pre, post):
        _lib.require_cuda(x, what="ResizeTransform")
        x = _lib.contig(x)
        B, C, Di, Hi, Wi, nd = _dims(x)
        if nd == 3:
            Do, Ho, Wo = out_spatial
        else:
            Do, (Ho, Wo) = 1, out_spatial
        out = torch.empty((B, C) + tuple(out_spatial), dtype=torch.float32, device=x.device)
        lib = _lib.load()
        _lib.check(lib.vxm_resize_fwd(_lib.ptr(x), _lib.ptr(out), B, C, Di, Hi, Wi, Do, Ho, Wo, pre, post,
                                      _lib.stream_ptr()), "vxm_resize_fwd")
        ctx.cfg = (B, C, Di, Hi, Wi, Do, Ho, Wo, pre, post, tuple(x.shape))
        return out

    @staticmethod
    def backward(ctx, gout):
        B, C, Di, Hi, Wi, Do, Ho, Wo, pre, post, xshape = ctx.cfg
        gout = _lib.contig(gout)
        gx = torch.empty(xshape, dtype=torch.float32, device=gout.device)
        lib = _lib.load()
        _lib.check(lib.vxm_resize_bwd(_lib.ptr(gout), _lib.ptr(gx), B, C, Di, Hi, Wi, Do, Ho, Wo, pre, post,
                                      _lib.stream_ptr()), "vxm_resize_bwd")
        return gx, None, None, None


class ResizeTransform(nn.Module):
    """Resize a transform: resize the vector field *and* rescale it (reference layers.py:71-97)."""

    def __init__(self, vel_resize, ndims):
        super().__init__()
        self.factor = 1.0 / vel_resize
        self.mode = 'linear'
        if ndims == 2:
            self.mode = 'bi' + self.mode
        elif ndims == 3:
            self.mode = 'tri' + self.mode

    def forward(self, x):
        if self.factor == 1:
            return x  # layers.py:96: "don't do anything if resize is 1"
        nd = x.dim() - 2
        if (nd == 2 and self.mode != 'bilinear') or (nd == 3 and self.mode != 'trilinear') or nd not in (2, 3):
            raise NotImplementedError("Got %dD input, but interpolation mode '%s' needs a matching dimensionality"
                                      % (x.dim(), self.mode))
        # F.interpolate(scale_factor=...) output size: floor(in * scale)
        out_spatial = tuple(int(math.floor(float(s) * self.factor)) for s in x.shape[2:])
        if self.factor < 1:   # resize first, then rescale (layers.py:86-89)
            return _ResizeFn.apply(x, out_spatial, 1.0, float(self.factor))
        return _ResizeFn.apply(x, out_spatial, float(self.factor), 1.0)  # layers.py:91-94


class _MeanStreamFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mean, count, cap, commit):
        _lib.require_cuda(x, mean, count, what="MeanStream")
        x = _lib.contig(x)
        B, n = x.shape[0], mean.numel()
        if tuple(x.shape[1:]) != tuple(mean.shape) or not mean.is_contiguous() or count.numel() != 1:
            raise _lib.VxmError("MeanStream: input %s does not match the state %s" % (tuple(x.shape), tuple(mean.shape)))
        out = torch.empty_like(mean)
        saved = torch.empty(1, dtype=torch.float32, device=x.device)
        _lib.check(_lib.load().vxm_mean_stream_fwd(_lib.ptr(x), _lib.ptr(mean), _lib.ptr(count), _lib.ptr(out), _lib.ptr(saved),
                                                   _lib.ptr(_lib.reduce_workspace(x.device)), B, n, float(cap), int(commit),
                                                   _lib.stream_ptr()), "vxm_mean_stream_fwd")
        ctx.saved = saved
        ctx.cfg = (B, n)
        # one copy of the output, broadcast over the batch (stride 0)
        return out.unsqueeze(0).expand((B,) + tuple(mean.shape))

    @staticmethod
    def backward(ctx, gout):
        B, n = ctx.cfg
        if B > 1 and gout.stride(0) == 0 and gout[0].is_contiguous():
            bstride = 0
        else:
            gout, bstride = _lib.contig(gout), n
        gx = torch.empty(gout.shape, dtype=torch.float32, device=gout.device)
        _lib.check(_lib.load().vxm_mean_stream_bwd(_lib.ptr(gout), _lib.ptr(ctx.saved), _lib.ptr(gx), B, n, bstride,
                                                   _lib.stream_ptr()), "vxm_mean_stream_bwd")
        return gx, None, None, None, None


class MeanStream(nn.Module):
    """Capped running mean of its input over the batches seen in training (neurite's MeanStream, which the reference's
    TemplateCreation wraps around the inverse flow, voxelmorph/tf/networks.py:761-853).

    State: buffers `mean` (`shape`, the input's shape without the batch axis) and `count` (1,), zero at first.  For x
    (B, *shape): n' = count + B, alpha = B / min(n', cap), m' = mean (1 - alpha) + mean_b(x) alpha, and the output is
    min(1, n' / cap) m' for every batch entry (one tensor expanded over B).  In training mode the call commits
    mean <- m' and count <- n' on the device; in eval mode the output is still computed from the batch, nothing is
    committed (Keras skips `add_update` outside training).  The gradient reaches x only: d out / d x_b =
    min(1, n' / cap) alpha / B."""

    def __init__(self, shape, cap=100):
        super().__init__()
        self.cap = float(cap)
        self.register_buffer("mean", torch.zeros(tuple(int(s) for s in shape), dtype=torch.float32))
        self.register_buffer("count", torch.zeros(1, dtype=torch.float32))

    def forward(self, x):
        return _MeanStreamFn.apply(x, self.mean, self.count, self.cap, self.training)


class _SampleNormalLogVarFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, params, state):
        _lib.require_cuda(params, what="SampleNormalLogVar")
        params = _lib.contig(params)
        B, C, D, H, W, nd = _dims(params)
        if C != 2 * nd:
            raise _lib.VxmError("SampleNormalLogVar: expected 2 * %d channels (mean, log variance), got %d" % (nd, C))
        if not state.is_cuda or state.dtype != torch.int64 or state.numel() != 2 or not state.is_contiguous():
            raise _lib.VxmError("SampleNormalLogVar: the noise state must be a contiguous (seed, call) int64 CUDA tensor")
        z = torch.empty((B, nd) + tuple(params.shape[2:]), dtype=torch.float32, device=params.device)
        ticket = torch.empty(1, dtype=torch.int64, device=params.device)
        _lib.check(_lib.load().vxm_sample_normal_logvar_fwd(_lib.ptr(params), _lib.ptr(z), _lib.ptr(state), _lib.ptr(ticket),
                                                            _lib.ptr(_lib.reduce_workspace(params.device)), B, nd, D * H * W,
                                                            _lib.stream_ptr()), "vxm_sample_normal_logvar_fwd")
        ctx.save_for_backward(params)
        ctx.state, ctx.ticket = state, ticket
        return z

    @staticmethod
    def backward(ctx, gz):
        (params,) = ctx.saved_tensors
        B, C, D, H, W, nd = _dims(params)
        gz = _lib.contig(gz)
        gp = torch.empty_like(params)
        _lib.check(_lib.load().vxm_sample_normal_logvar_bwd(_lib.ptr(gz), _lib.ptr(params), _lib.ptr(ctx.state), _lib.ptr(ctx.ticket),
                                                            _lib.ptr(gp), B, nd, D * H * W, _lib.stream_ptr()),
                   "vxm_sample_normal_logvar_bwd")
        return gp, None


def sample_normal_logvar(params, state):
    """z = mu + exp(logvar / 2) eps with eps ~ N(0, 1) (neurite's SampleNormalLogVar, which the reference's probabilistic
    VxmDense draws its field with, voxelmorph/tf/networks.py:155-165), for params (B, 2 nd, *vol) = cat(mu, logvar).

    eps comes from a counter-based generator (Philox4x32-10, include/vxm_b200.h) keyed by state = (seed, call), an int64
    device tensor: each call draws the stream of the current `call` and advances it by one on the device, and its backward
    regenerates that same eps instead of storing it."""
    return _SampleNormalLogVarFn.apply(params, state)


_pd_ws = {}


def _pheno_decoder_workspace(device, F):
    """Per (device, stream, F) scratch of the decoder backward: zeroed once, the kernel leaves its ticket counter zero."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream, int(F))
    ws = _pd_ws.get(key)
    if ws is None:
        ws = torch.zeros(int(_lib.load().vxm_pheno_decoder_workspace_bytes(int(F))), dtype=torch.uint8, device=device)
        _pd_ws[key] = ws
    return ws


def _flat_grad(p):
    """p's .grad when it is a contiguous view of FusedAdam's flat gradient buffer (optim.FlatParams marks them)."""
    return p.grad if getattr(p, "_vxm_flat_grad", False) and p.grad is not None and p.grad.is_contiguous() else None


class _PhenoDecoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pheno, weight, bias, like_weight, like_bias):
        _lib.require_cuda(pheno, weight, bias, like_weight, like_bias, what="PhenoDecoder")
        pheno = _lib.contig(pheno)
        P, F = weight.shape[0], weight.shape[1]
        vol = tuple(weight.shape[2:])
        if pheno.dim() != 2 or pheno.shape[1] != P or tuple(bias.shape) != (F,) + vol \
                or like_weight.numel() != F * F or like_weight.shape[0] != F or tuple(like_bias.shape) != (F,):
            raise _lib.VxmError("PhenoDecoder: pheno %s does not match weight %s, bias %s, like_weight %s, like_bias %s"
                                % (tuple(pheno.shape), tuple(weight.shape), tuple(bias.shape), tuple(like_weight.shape),
                                   tuple(like_bias.shape)))
        if not (weight.is_contiguous() and bias.is_contiguous() and like_weight.is_contiguous()):
            raise _lib.VxmError("PhenoDecoder: the parameters must be contiguous")
        B, V = pheno.shape[0], bias[0].numel()
        out = torch.empty((B, F) + vol, dtype=torch.float32, device=pheno.device)
        _lib.check(_lib.load().vxm_pheno_decoder_fwd(_lib.ptr(pheno), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(like_weight),
                                                     _lib.ptr(like_bias), _lib.ptr(out), B, P, F, V, _lib.stream_ptr()),
                   "vxm_pheno_decoder_fwd")
        ctx.save_for_backward(pheno, weight, bias, like_weight, like_bias)
        ctx.cfg = (B, P, F, V)
        return out

    @staticmethod
    def backward(ctx, gout):
        pheno, weight, bias, like_weight, like_bias = ctx.saved_tensors
        B, P, F, V = ctx.cfg
        gout = _lib.contig(gout)
        params = (weight, bias, like_weight, like_bias)
        flat = [_flat_grad(p) for p in params]
        # like the tensor-core engine's weight gradients: straight into FusedAdam's flat buffer when every parameter has
        # its view there, and autograd then receives none; otherwise fresh tensors for autograd to accumulate
        accumulate = all(g is not None for g in flat)
        outs = flat if accumulate else [torch.empty_like(p) for p in params]
        _lib.check(_lib.load().vxm_pheno_decoder_bwd(_lib.ptr(gout), _lib.ptr(pheno), _lib.ptr(weight), _lib.ptr(bias),
                                                     _lib.ptr(like_weight), *[_lib.ptr(g) for g in outs],
                                                     _lib.ptr(_pheno_decoder_workspace(gout.device, F)), B, P, F, V,
                                                     int(accumulate), _lib.stream_ptr()), "vxm_pheno_decoder_bwd")
        if accumulate:
            return None, None, None, None, None
        return (None,) + tuple(outs)


class PhenoDecoder(nn.Module):
    """The phenotype decoder of ConditionalTemplateCreation (reference voxelmorph/tf/networks.py:905-915): a Dense layer
    from P subject attributes to a full-resolution F-channel image with ELU, then neurite's conv_dec with no levels, one
    1x1 convolution F -> F with bias and no activation.  For pheno (B, P):

        pre = bias + sum_p pheno[:, p] weight[p],  h = ELU(pre),  out = like_bias + like_weight * h  (1x1 convolution)

    out is (B, F, *inshape).  `weight` is stored (P, F, *inshape) and `bias` (F, *inshape), so the output is channels-first
    with no transpose.  A Keras Dense kernel (P, V F) and bias (V F,) (V = prod(inshape), F fastest, as Keras' Reshape to
    (*inshape, F) reads them) map onto it by reshaping to (P, *inshape, F) and (*inshape, F) and moving F to axis 1 and 0:
    see `from_keras`.  Initialisation is Keras': glorot-uniform kernels (the Dense's fans P and V F, the 1x1
    convolution's F and F), zero biases.

    Forward and backward are one kernel launch each (csrc/pheno_decoder.cu); no activation is kept, the backward recomputes
    it.  When every parameter's .grad is a view of FusedAdam's flat buffer the gradients are accumulated there directly.
    No gradient is formed for pheno.  Limits: 1 <= P <= 16, 1 <= F <= 32."""

    def __init__(self, P, F, inshape):
        super().__init__()
        inshape = tuple(int(s) for s in inshape)
        V = int(math.prod(inshape))
        nd = len(inshape)
        lim = math.sqrt(6.0 / (P + V * F))
        self.weight = nn.Parameter(torch.empty((P, F) + inshape).uniform_(-lim, lim))
        self.bias = nn.Parameter(torch.zeros((F,) + inshape))
        lim = math.sqrt(6.0 / (2 * F))
        self.like_weight = nn.Parameter(torch.empty((F, F) + (1,) * nd).uniform_(-lim, lim))
        self.like_bias = nn.Parameter(torch.zeros(F))

    @staticmethod
    def from_keras(kernel, bias, inshape):
        """(weight, bias) of this layout from a Keras Dense kernel (P, V F) and bias (V F,)."""
        kernel, bias = torch.as_tensor(kernel), torch.as_tensor(bias)
        inshape = tuple(inshape)
        w = kernel.reshape((kernel.shape[0],) + inshape + (-1,)).movedim(-1, 1)
        b = bias.reshape(inshape + (-1,)).movedim(-1, 0)
        return w.contiguous(), b.contiguous()

    def forward(self, pheno):
        return _PhenoDecoderFn.apply(pheno, self.weight, self.bias, self.like_weight, self.like_bias)


def _ptr_array(tensors):
    """A host array of device pointers (the hypernetwork entry points take one per layer)."""
    import ctypes
    arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
    return arr, ctypes.cast(arr, ctypes.c_void_p)


class _HyperWeightsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hyp, out, kernel, bias, *mlp):
        _lib.require_cuda(hyp, out, kernel, bias, *mlp, what="HyperWeights")
        U, N = kernel.shape
        L = len(mlp) // 2
        P = mlp[0].shape[1]
        if tuple(hyp.shape) != (1, P):
            raise _lib.VxmError("HyperWeights: hyp must have shape (1, %d) — one set of hyperparameters per step, shared by "
                                "every image of the batch; got %s" % (P, tuple(hyp.shape)))
        if not all(t.is_contiguous() for t in (out, kernel, bias) + mlp) or tuple(bias.shape) != (N,) \
                or tuple(out.shape) != (N,):
            raise _lib.VxmError("HyperWeights: the parameters must be contiguous, hyper_kernel (U, N), hyper_bias and the "
                                "generated buffer (N,)")
        hyp = _lib.contig(hyp)
        lib = _lib.load()
        pre = torch.empty((L, U), dtype=torch.float32, device=hyp.device)
        h = torch.empty(U, dtype=torch.float32, device=hyp.device)
        wa, wp = _ptr_array(mlp[0::2])
        ba, bp = _ptr_array(mlp[1::2])
        _lib.check(lib.vxm_hyper_mlp_fwd(_lib.ptr(hyp), wp, bp, _lib.ptr(pre), _lib.ptr(h), P, U, L, _lib.stream_ptr()),
                   "vxm_hyper_mlp_fwd")
        _lib.check(lib.vxm_hyper_weights_fwd(_lib.ptr(h), _lib.ptr(kernel), _lib.ptr(bias), _lib.ptr(out), U, N,
                                             _lib.stream_ptr()), "vxm_hyper_weights_fwd")
        # the U-Net's weights changed behind torch's version counters: the tensor-core engine's packed copies refresh
        from . import engine_bf16
        engine_bf16.bump_weights_epoch()
        ctx.save_for_backward(hyp, pre, h, kernel, bias, *mlp)
        ctx.cfg = (P, U, L, N)
        return out.detach()

    @staticmethod
    def backward(ctx, dW):
        hyp, pre, h, kernel, bias, *mlp = ctx.saved_tensors
        P, U, L, N = ctx.cfg
        dW = _lib.contig(dW)
        params = [kernel, bias] + mlp
        flat = [_flat_grad(p) for p in params]
        # as PhenoDecoder: straight into FusedAdam's flat buffer when every parameter has its view there (autograd then
        # receives none), otherwise fresh tensors for autograd to accumulate
        accumulate = all(g is not None for g in flat)
        outs = flat if accumulate else [torch.empty_like(p) for p in params]
        lib = _lib.load()
        dh = torch.empty(U, dtype=torch.float32, device=dW.device)
        work = torch.empty(int(lib.vxm_hyper_workspace_bytes(U, N)), dtype=torch.uint8, device=dW.device)
        _lib.check(lib.vxm_hyper_weights_bwd(_lib.ptr(h), _lib.ptr(kernel), _lib.ptr(dW), _lib.ptr(outs[0]), _lib.ptr(outs[1]),
                                             _lib.ptr(dh), _lib.ptr(work), U, N, int(accumulate), _lib.stream_ptr()),
                   "vxm_hyper_weights_bwd")
        wa, wp = _ptr_array(mlp[0::2])
        ga, gp = _ptr_array(outs[2::2])
        gba, gbp = _ptr_array(outs[3::2])
        _lib.check(lib.vxm_hyper_mlp_bwd(_lib.ptr(dh), _lib.ptr(hyp), wp, _lib.ptr(pre), gp, gbp, P, U, L, int(accumulate),
                                         _lib.stream_ptr()), "vxm_hyper_mlp_bwd")
        if accumulate:
            return (None,) * (4 + len(mlp))
        return (None, None) + tuple(outs)


def hyper_layout(shapes):
    """Offsets of the flat generated layout: [(weight offset, bias offset)] for convolutions of weight shapes `shapes`,
    each stored as [weight, bias] in the given (execution) order, and the total N."""
    offs, n = [], 0
    for s in shapes:
        k = int(math.prod(s))
        offs.append((n, n + k))
        n += k + int(s[0])
    return offs, n


class HyperWeights(nn.Module):
    """HyperMorph's hypernetwork and the weights it generates (Hoopes et al., IPMI 2021 / MELBA 2022; reference
    voxelmorph/tf/networks.py:1192-1231 with neurite's HyperConvFromDense).  For hyp (1, P):

        h = relu(Dense_{L-1}(... relu(Dense_0(hyp))))            hypernet.{i}: nn.Linear, U units each
        Wflat = hyper_bias + h @ hyper_kernel                      hyper_kernel (U, N), hyper_bias (N)

    `shapes` are the generated convolutions' weight shapes in the U-Net's execution order; Wflat holds each as
    [weight, bias] (hyper_layout), and `views(wflat)` returns them as (weight, bias) tensors.  Wflat is written by the
    device into one persistent buffer (`wflat`, not a checkpoint entry), so every step's weights sit at the same
    addresses: the tensor-core engine's packing descriptors and a captured CUDA graph stay valid.  Consequently the
    generated weights of a forward are valid until the next forward: run a backward before the next forward.

    Initialisation (the package's choice; neurite's HyperConvFromDense initialiser is not restated): the Dense layers as
    Keras initialises them, glorot-uniform kernels and zero biases; each convolution's block of hyper_kernel
    glorot-uniform over the fans (U, 27 Cin Cout) for its weight part and (U, Cout) for its bias part; hyper_bias zero.

    Forward and backward are two launches each (csrc/hyper.cu); when every parameter's .grad is a view of FusedAdam's
    flat buffer the gradients are accumulated there directly.  hyp receives no gradient.  Limits: 1 <= P <= 16,
    U <= 256, 1 <= nb_layers <= 8."""

    def __init__(self, shapes, nb_hyp_params=1, nb_hyp_layers=6, nb_hyp_units=128):
        super().__init__()
        P, L, U = int(nb_hyp_params), int(nb_hyp_layers), int(nb_hyp_units)
        if not (1 <= P <= 16 and 1 <= U <= 256 and 1 <= L <= 8):
            raise ValueError("HyperWeights: nb_hyp_params must be 1 to 16, nb_hyp_units 1 to 256 and nb_hyp_layers 1 to 8; "
                             "got %d, %d, %d" % (P, U, L))
        self.shapes = [tuple(int(d) for d in s) for s in shapes]
        self.offsets, N = hyper_layout(self.shapes)
        self.hypernet = nn.ModuleList()
        for i in range(L):
            lin = nn.Linear(P if i == 0 else U, U)
            lim = math.sqrt(6.0 / (lin.in_features + lin.out_features))
            with torch.no_grad():
                lin.weight.uniform_(-lim, lim)
                lin.bias.zero_()
            self.hypernet.append(lin)
        kernel = torch.empty(U, N)
        for s, (ow, ob) in zip(self.shapes, self.offsets):
            taps = int(math.prod(s[2:]))
            lim = math.sqrt(6.0 / (U + taps * s[0] * s[1]))
            kernel[:, ow:ob].uniform_(-lim, lim)
            lim = math.sqrt(6.0 / (U + s[0]))
            kernel[:, ob:ob + s[0]].uniform_(-lim, lim)
        self.hyper_kernel = nn.Parameter(kernel)
        self.hyper_bias = nn.Parameter(torch.zeros(N))
        self.register_buffer("wflat", torch.zeros(N), persistent=False)

    def forward(self, hyp):
        """Wflat (N,) for hyp (1, P), differentiable with respect to every parameter of this module."""
        mlp = [p for lin in self.hypernet for p in (lin.weight, lin.bias)]
        return _HyperWeightsFn.apply(hyp, self.wflat, self.hyper_kernel, self.hyper_bias, *mlp)

    def views(self, wflat):
        """[(weight, bias)] views of a flat layout, in the order of `shapes`."""
        return [(wflat[ow:ob].view(s), wflat[ob:ob + s[0]]) for s, (ow, ob) in zip(self.shapes, self.offsets)]


def _surface_dims(points, vol, what, vol_name):
    """(B, N, nd, C, D, H, W) of points (B, N, nd+1) and a (B, C, [D,] H, W) volume, or VxmError."""
    _lib.require_cuda(points, vol, what=what)
    if vol.dim() not in (4, 5):
        raise _lib.VxmError("%s: %s must be (B, C, H, W) or (B, C, D, H, W), got shape %s"
                            % (what, vol_name, tuple(vol.shape)))
    B, C, D, H, W, nd = _dims(vol)
    if points.dim() != 3 or points.shape[0] != B or points.shape[2] != nd + 1 or points.shape[1] < 1:
        raise _lib.VxmError("%s: points must be (B, N, nd + 1) = (%d, N, %d) for %s %s, got shape %s"
                            % (what, B, nd + 1, vol_name, tuple(vol.shape), tuple(points.shape)))
    return B, points.shape[1], nd, C, D, H, W


class _PointWarpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, flow, r):
        B, N, nd, C, D, H, W = _surface_dims(points, flow, "point_spatial_transformer", "flow")
        if C != nd:
            raise _lib.VxmError("point_spatial_transformer: flow must have %d channels, got %d" % (nd, C))
        points, flow = _lib.contig(points), _lib.contig(flow)
        out = torch.empty_like(points)
        _lib.check(_lib.load().vxm_point_warp_fwd(_lib.ptr(points), _lib.ptr(flow), _lib.ptr(out), B, N, D, H, W, nd,
                                                  r, _lib.stream_ptr()), "vxm_point_warp_fwd")
        ctx.save_for_backward(points)
        ctx.cfg = (B, N, D, H, W, nd, r, flow.shape)
        return out

    @staticmethod
    def backward(ctx, gout):
        if not ctx.needs_input_grad[1]:
            return None, None, None
        (points,) = ctx.saved_tensors
        B, N, D, H, W, nd, r, fshape = ctx.cfg
        lib = _lib.load()
        nbytes = int(lib.vxm_point_warp_workspace_bytes(B, N, D, H, W, nd))
        if nbytes == 0:
            raise _lib.VxmError("point_spatial_transformer: no workspace for B=%d, N=%d, volume %s: %s"
                                % (B, N, tuple(fshape[2:]), _lib.last_error()))
        work = torch.empty(nbytes, dtype=torch.uint8, device=points.device)
        gflow = torch.zeros(fshape, dtype=torch.float32, device=points.device)
        _lib.check(lib.vxm_point_warp_bwd(_lib.ptr(points), _lib.ptr(_lib.contig(gout)), _lib.ptr(gflow),
                                          _lib.ptr(work), nbytes, B, N, D, H, W, nd, r, _lib.stream_ptr()),
                   "vxm_point_warp_bwd")
        return None, gflow, None


class _ValueAtFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sdt, points):
        B, N, nd, L, D, H, W = _surface_dims(points, sdt, "value_at_location", "sdt")
        sdt, points = _lib.contig(sdt), _lib.contig(points)
        out = torch.empty((B, N, 1), dtype=torch.float32, device=sdt.device)
        _lib.check(_lib.load().vxm_value_at_fwd(_lib.ptr(sdt), _lib.ptr(points), _lib.ptr(out), B, N, L, D, H, W, nd,
                                                _lib.stream_ptr()), "vxm_value_at_fwd")
        ctx.save_for_backward(sdt, points)
        ctx.cfg = (B, N, L, D, H, W, nd)
        return out

    @staticmethod
    def backward(ctx, gout):
        if not ctx.needs_input_grad[1]:
            return None, None
        sdt, points = ctx.saved_tensors
        B, N, L, D, H, W, nd = ctx.cfg
        gpts = torch.empty_like(points)
        _lib.check(_lib.load().vxm_value_at_bwd(_lib.ptr(sdt), _lib.ptr(points), _lib.ptr(_lib.contig(gout)),
                                                _lib.ptr(gpts), B, N, L, D, H, W, nd, _lib.stream_ptr()),
                   "vxm_value_at_bwd")
        return None, gpts


def point_spatial_transformer(points, flow, sdt_vol_resize=1):
    """Move surface points with a displacement field (reference voxelmorph/tf/utils/utils.py:465-499).

    points (B, N, nd+1): spatial coordinates in the flow's axis order, the last column a label index (passed through);
    flow (B, nd, *S).  Returns p + r * interp(flow, p) with r = sdt_vol_resize and neurite's clamped linear interpn
    (a point outside the volume reads the border).  A field that moves image A onto B is defined on B's grid, so it
    moves points of B onto A.  Only `flow` is differentiated (deterministically, see include/vxm_b200.h); `points`
    must not require a gradient."""
    if points.requires_grad:
        raise _lib.VxmError("point_spatial_transformer: points must not require a gradient")
    return _PointWarpFn.apply(points, flow, float(sdt_vol_resize))


def value_at_location(sdt, points):
    """|sdt| at the points (reference voxelmorph/tf/utils/utils.py:71-88 with force_post_absolute_val): sdt
    (B, L, *S), points (B, N, nd+1) whose last column is the label channel, interpolated as an (nd+1)-th axis like the
    others.  Returns (B, N, 1).  Only `points` is differentiated (sign(v) times the spatial gradient, 0 for the label
    column); `sdt` must not require a gradient."""
    if sdt.requires_grad:
        raise _lib.VxmError("value_at_location: sdt must not require a gradient")
    return _ValueAtFn.apply(sdt, points)
