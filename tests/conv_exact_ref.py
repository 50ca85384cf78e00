"""fp64 references of the tensor-core convolutions and of their epilogues, for the exact tests (test_gpu_conv_exact.py;
the helpers themselves are checked against fp64 autograd of F.conv3d in test_conv_exact_reference.py).

Tensors are channels-last (B, D, H, W, C), as the kernels hold them.  A layer input is a list of sources (x, up) whose
channels are concatenated, `up` marking a nearest x2 upsampled one, held at half resolution along the upsampled axes: d, h
and w of a 3-D layer (nd = 3), h and w of a 2-D one (nd = 2, tensors held as (B, 1, H, W, C), as the engine holds them).  Every
convolution is an explicit sum over its taps of shifted channel matmuls (no convolution algorithm is chosen for us),
computed in depth slabs so that the fp64 intermediates of a full-size layer stay small.  With operands that are small
multiples of one power of two, every fp64 sum here is exact whatever its order."""
import torch
import torch.nn.functional as F

SLAB = 8          # output slices per slab (even: a coarse slice never straddles two slabs)


def upsample2(x, nd=3):
    """nearest x2 of a (B, D, H, W, C) tensor along d, h and w (nd = 3) or h and w (nd = 2)"""
    x = x.repeat_interleave(2, 2).repeat_interleave(2, 3)
    return x.repeat_interleave(2, 1) if nd == 3 else x


def children_sum(y, nd=3):
    """(B, D, H, W, C) -> (B, D / 2, H / 2, W / 2, C) (nd = 3) or (B, D, H / 2, W / 2, C) (nd = 2): the sum over the 8 or 4
    fine children of every coarse voxel (the gradient through a nearest x2 upsampling)"""
    B, D, H, W, C = y.shape
    if nd == 2:
        return y.reshape(B, D, H // 2, 2, W // 2, 2, C).sum((3, 5))
    return y.reshape(B, D // 2, 2, H // 2, 2, W // 2, 2, C).sum((2, 4, 6))


def _slices(srcs, D, lo, hi, nd):
    """fp64 input slices lo .. hi - 1 of the concatenated sources, zero outside [0, D)"""
    a, b = max(lo, 0), min(hi, D)
    parts = []
    for x, up in srcs:
        if up and nd == 3:
            c0 = a // 2
            parts.append(upsample2(x[:, c0:(b + 1) // 2].double())[:, a - 2 * c0:b - 2 * c0])
        elif up:
            parts.append(upsample2(x[:, a:b].double(), 2))
        else:
            parts.append(x[:, a:b].double())
    return F.pad(torch.cat(parts, -1), (0, 0, 0, 0, 0, 0, a - lo, hi - b))


def _windows(srcs, D, d0, d1, kd, nd):
    """the padded input of output slices d0 .. d1 - 1 (one halo voxel around h and w, kd // 2 slices around d)"""
    assert nd == 3 or kd == 1
    return F.pad(_slices(srcs, D, d0 - kd // 2, d1 + kd // 2, nd), (0, 0, 1, 1, 1, 1))


def conv(srcs, w, D, finish=None, slab=SLAB, nd=3):
    """Cross-correlation with padding 1 (0 along d when kd = 1): y[v, co] = sum_tap sum_ci x[v + tap - 1, ci] w[co, ci, tap],
    w (Cout, Cin, kd, 3, 3).  D: output (= input) slices.  nd: which axes an `up` source is upsampled along (2: h and w,
    with kd = 1).  finish(y, d0, d1) is applied to every slab of output slices d0 .. d1 - 1 (fp64, (B, d1 - d0, H, W, Cout))
    and the list of its results returned; without it, the whole fp64 output."""
    w = w.double()
    kd = w.shape[2]
    out = []
    for d0 in range(0, D, slab):
        d1 = min(d0 + slab, D)
        x = _windows(srcs, D, d0, d1, kd, nd)
        H, W = x.shape[2] - 2, x.shape[3] - 2
        y = None
        for i in range(kd):
            for j in range(3):
                for k in range(3):
                    t = x[:, i:i + d1 - d0, j:j + H, k:k + W] @ w[:, :, i, j, k].t().to(x.device)
                    y = t if y is None else y.add_(t)
        out.append(y if finish is None else finish(y, d0, d1))
    return torch.cat(out, 1) if finish is None else out


def dgrad_weight(w):
    """the weight whose cross-correlation with the output gradient is the input gradient: (Cin, Cout, kd, 3, 3), taps flipped"""
    return w.transpose(0, 1).flip(2, 3, 4)


def wgrad(srcs, gz, kd=3, absolute=False, slab=SLAB, nd=3):
    """Weight and bias gradient of conv(srcs, w, nd=nd) against the output gradient gz (B, D, H, W, Cout): fp64
    (Cout, Cin, kd, 3, 3) and (Cout,).  absolute: the same sums over |x| and |gz|, which bound every partial sum of any
    summation order."""
    D, Cout = gz.shape[1], gz.shape[-1]
    gw, gb = None, None
    for d0 in range(0, D, slab):
        d1 = min(d0 + slab, D)
        x = _windows(srcs, D, d0, d1, kd, nd)
        g = gz[:, d0:d1].double()
        if absolute:
            x, g = x.abs(), g.abs()
        H, W, Cin = x.shape[2] - 2, x.shape[3] - 2, x.shape[-1]
        gf = g.reshape(-1, Cout)
        taps = torch.stack([x[:, i:i + d1 - d0, j:j + H, k:k + W].reshape(-1, Cin).t() @ gf
                            for i in range(kd) for j in range(3) for k in range(3)], -1)
        gw = taps if gw is None else gw.add_(taps)
        gb = gf.sum(0) if gb is None else gb.add_(gf.sum(0))
    return gw.view(Cin, Cout, kd, 3, 3).transpose(0, 1).contiguous(), gb


def epilogue(y, bias=None, slope=None, mask=None, bf16=True):
    """The convolution kernels' epilogue on an exact fp64 sum y (B, ..., C): fl32(y), + bias as an fp32 add, then in fp32
    either the LeakyReLU fmaxf(v, v * slope) or, given the saved activation `mask`, the LeakyReLU derivative
    (v * slope where mask < 0); then bf16 with round-to-nearest-even unless bf16 is False (the flow head's fp32 output)."""
    v = y.float()
    if bias is not None:
        v = v + bias.float().to(v.device)
    if slope is not None:
        s = torch.tensor(slope, dtype=torch.float32, device=v.device)
        v = torch.where(mask < 0, v * s, v) if mask is not None else torch.maximum(v, v * s)
    return v.to(torch.bfloat16) if bf16 else v
