"""autograd wrappers of the U-Net kernels (conv k=3 + bias + LeakyReLU, MaxPool(2),
nearest-upsample(2) + concat) — the pieces reference voxelmorph/torch/networks.py reaches
through nn.ConvNd / nn.LeakyReLU / nn.MaxPoolNd / nn.Upsample / torch.cat.
"""
import os

import torch

from . import _lib
from .layers import _dims


_default_engine = "f32"


def set_default_engine(name):
    """Engine used when VXM_B200_CONV_ENGINE is not set ('f32' for `import voxelmorph_b200`, 'tc' through the
    `voxelmorph` drop-in package)."""
    global _default_engine
    if name not in ("f32", "bf16", "bf16x3", "tc"):
        raise ValueError("unknown convolution engine %r" % (name,))
    _default_engine = name


def conv_engine():
    """'f32'    — CUDA-core fp32 engine (FFMA; every U-Net shape);
    'bf16'   — wgmma implicit-GEMM engine, bf16 operands / fp32 accumulation (the throughput mode bench.py times);
    'bf16x3' — the same tensor-core kernels with every operand split into a bf16 hi + lo pair and three MMAs per tile
               (hi*hi + lo*hi + hi*lo): fp32-grade products, flow / moved image within 1e-4 of the reference;
    'tc'     — 'bf16x3' where the tensor-core engine supports the model, else 'f32'."""
    return os.environ.get("VXM_B200_CONV_ENGINE", _default_engine)


def resolve_engine(model):
    """Engine for one VxmDense forward: resolves 'tc' and falls back to f32 for shapes the tensor-core engine lacks."""
    e = conv_engine()
    if e == "tc":
        from . import engine_bf16
        return "bf16x3" if engine_bf16.supports(model) else "f32"
    return e


class _ConvK3Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, slope):
        _lib.require_cuda(x, weight, bias, what="conv3d")
        x, weight = _lib.contig(x), _lib.contig(weight)
        bias = _lib.contig(bias) if bias is not None else None
        B, Cin, D, H, W, nd = _dims(x)
        Cout = weight.shape[0]
        if weight.shape[1] != Cin or tuple(weight.shape[2:]) != (3,) * nd:
            raise _lib.VxmError("conv: weight %s does not match input %s (kernel must be 3^%d)"
                                % (tuple(weight.shape), tuple(x.shape), nd))
        kd = 3 if nd == 3 else 1
        y = torch.empty((B, Cout) + tuple(x.shape[2:]), dtype=torch.float32, device=x.device)
        lib = _lib.load()
        s = -1.0 if slope is None else float(slope)
        _lib.check(lib.vxm_conv3d_fwd_f32(_lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(y), B, Cin, Cout, D, H, W,
                                          kd, s, _lib.stream_ptr()), "vxm_conv3d_fwd_f32")
        ctx.save_for_backward(x, weight, y)
        ctx.cfg = (B, Cin, Cout, D, H, W, kd, s, bias is not None)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight, y = ctx.saved_tensors
        B, Cin, Cout, D, H, W, kd, s, has_bias = ctx.cfg
        gy = _lib.contig(gy)
        need_x, need_w, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2] and has_bias
        gx = torch.empty_like(x) if need_x else None
        gw = torch.zeros_like(weight) if (need_w or need_b) else None
        gb = torch.zeros(Cout, dtype=torch.float32, device=x.device) if need_b else None
        lib = _lib.load()
        work = None
        if gw is not None:
            work = torch.empty(int(lib.vxm_conv3d_bwd_workspace_bytes(B, Cin, Cout, D, H, W, kd)), dtype=torch.uint8,
                               device=x.device)
        _lib.check(lib.vxm_conv3d_bwd_f32(_lib.ptr(gy), _lib.ptr(y), _lib.ptr(x), _lib.ptr(weight), _lib.ptr(gx),
                                          _lib.ptr(gw), _lib.ptr(gb), _lib.ptr(work), B, Cin, Cout, D, H, W, kd, s,
                                          _lib.stream_ptr()), "vxm_conv3d_bwd_f32")
        return gx, (gw if need_w else None), gb, None


def conv_k3(x, weight, bias, leaky_slope=None):
    """y = LeakyReLU_slope(conv_{3^n, pad 1}(x, weight) + bias); slope None -> no activation."""
    return _ConvK3Fn.apply(x, weight, bias, leaky_slope)


class _MaxPool2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        _lib.require_cuda(x, what="maxpool")
        x = _lib.contig(x)
        B, C, D, H, W, nd = _dims(x)
        out_sp = tuple(s // 2 for s in x.shape[2:])
        y = torch.empty((B, C) + out_sp, dtype=torch.float32, device=x.device)
        idx = torch.empty((B, C) + out_sp, dtype=torch.uint8, device=x.device)
        lib = _lib.load()
        _lib.check(lib.vxm_maxpool2_fwd(_lib.ptr(x), _lib.ptr(y), _lib.ptr(idx), B, C, D, H, W, nd, _lib.stream_ptr()),
                   "vxm_maxpool2_fwd")
        ctx.save_for_backward(idx)
        ctx.cfg = (B, C, D, H, W, nd, tuple(x.shape))
        return y

    @staticmethod
    def backward(ctx, gy):
        (idx,) = ctx.saved_tensors
        B, C, D, H, W, nd, xshape = ctx.cfg
        gy = _lib.contig(gy)
        gx = torch.empty(xshape, dtype=torch.float32, device=gy.device)
        lib = _lib.load()
        _lib.check(lib.vxm_maxpool2_bwd(_lib.ptr(gy), _lib.ptr(idx), _lib.ptr(gx), B, C, D, H, W, nd, _lib.stream_ptr()),
                   "vxm_maxpool2_bwd")
        return gx


def maxpool2(x):
    return _MaxPool2Fn.apply(x)


class _UpCatFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, skip):
        _lib.require_cuda(a, skip, what="upsample+concat")
        a = _lib.contig(a)
        skip = _lib.contig(skip) if skip is not None else None
        B, Ca, D, H, W, nd = _dims(a)
        Cb = 0 if skip is None else skip.shape[1]
        out_sp = tuple(2 * s for s in a.shape[2:])
        if skip is not None and (tuple(skip.shape[2:]) != out_sp or skip.shape[0] != B):
            raise RuntimeError("Sizes of tensors must match except in dimension 1. Expected size %s but got size %s"
                               % (out_sp, tuple(skip.shape[2:])))
        out = torch.empty((B, Ca + Cb) + out_sp, dtype=torch.float32, device=a.device)
        lib = _lib.load()
        _lib.check(lib.vxm_upcat_fwd(_lib.ptr(a), _lib.ptr(skip), _lib.ptr(out), B, Ca, Cb, D, H, W, nd, _lib.stream_ptr()),
                   "vxm_upcat_fwd")
        ctx.cfg = (B, Ca, Cb, D, H, W, nd, tuple(a.shape), None if skip is None else tuple(skip.shape))
        return out

    @staticmethod
    def backward(ctx, go):
        B, Ca, Cb, D, H, W, nd, ashape, sshape = ctx.cfg
        go = _lib.contig(go)
        ga = torch.empty(ashape, dtype=torch.float32, device=go.device)
        gs = torch.empty(sshape, dtype=torch.float32, device=go.device) if sshape is not None else None
        lib = _lib.load()
        _lib.check(lib.vxm_upcat_bwd(_lib.ptr(go), _lib.ptr(ga), _lib.ptr(gs), B, Ca, Cb, D, H, W, nd, _lib.stream_ptr()),
                   "vxm_upcat_bwd")
        return ga, gs


def upsample2_cat(a, skip=None):
    """cat([nearest_upsample_x2(a), skip], dim=1) without materialising the upsampled tensor separately."""
    return _UpCatFn.apply(a, skip)


def upsample_free_cat(source, target):
    """cat([source, target], dim=1) (reference networks.py:253); device-side copy only."""
    _lib.require_cuda(source, target, what="VxmDense")
    return torch.cat([source, target], dim=1)
