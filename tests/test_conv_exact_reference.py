"""The fp64 references of the exact convolution tests (conv_exact_ref.py) against fp64 autograd of F.conv3d (F.conv2d for
2-D layers, held as (B, 1, H, W, C)), on small shapes with kd = 1 and 3, upsampled sources, concatenations and several
depth slabs; and their epilogue emulation against a direct per-element fp32 computation with an explicit
round-to-nearest-even to bf16."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_exact_ref as ref

CASES = [
    # (B, (D, H, W) or (H, W) for a 2-D layer, Ca, Cb, up, Cout, kd)
    (2, (6, 5, 7), 3, 0, False, 4, 3),
    (1, (8, 6, 4), 3, 2, True, 5, 3),          # upsampled source + skip
    (2, (7, 4, 6), 4, 3, False, 2, 3),          # concatenation, odd depth
    (1, (5, 6, 5), 3, 2, False, 4, 1),          # kd = 1 (the kd-folded layers)
    (2, (10, 6), 3, 2, True, 4, 1),             # 2-D: upsampled source (h and w only) + skip
    (3, (5, 7), 4, 0, False, 3, 1),             # 2-D, odd sizes
]


def _case(B, shape, Ca, Cb, up, Cout, kd, integer):
    g = torch.Generator().manual_seed(B * 100 + Ca * 10 + Cb + kd + 1000 * (len(shape) == 2))
    D, H, W = shape if len(shape) == 3 else (1,) + shape
    Dc = D if len(shape) == 2 else D // 2
    gen = (lambda s: torch.randint(-3, 4, s, generator=g).double()) if integer else (lambda s: torch.randn(s, generator=g, dtype=torch.float64))
    xa = gen((B, Dc, H // 2, W // 2, Ca) if up else (B, D, H, W, Ca))
    xb = gen((B, D, H, W, Cb)) if Cb else None
    w, b, gy = gen((Cout, Ca + Cb, kd, 3, 3)), gen((Cout,)), gen((B, D, H, W, Cout))
    return xa, xb, w, b, gy


def _autograd(xa, xb, w, b, gy, up, nd):
    xa, w, b = xa.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    xb = None if xb is None else xb.clone().requires_grad_(True)
    x = ref.upsample2(xa, nd) if up else xa
    if xb is not None:
        x = torch.cat([x, xb], -1)
    if nd == 2:
        y = F.conv2d(x[:, 0].permute(0, 3, 1, 2), w[:, :, 0], b, padding=1).permute(0, 2, 3, 1)[:, None]
    else:
        y = F.conv3d(x.permute(0, 4, 1, 2, 3), w, b, padding=(w.shape[2] // 2, 1, 1)).permute(0, 2, 3, 4, 1)
    (y * gy).sum().backward()
    return y.detach(), xa.grad, (None if xb is None else xb.grad), w.grad, b.grad


@pytest.mark.parametrize("integer", [True, False])
@pytest.mark.parametrize("slab", [2, 3, ref.SLAB])
@pytest.mark.parametrize("B,shape,Ca,Cb,up,Cout,kd", CASES)
def test_reference_helpers_match_autograd(B, shape, Ca, Cb, up, Cout, kd, slab, integer):
    nd = len(shape)
    xa, xb, w, b, gy = _case(B, shape, Ca, Cb, up, Cout, kd, integer)
    y, gxa, gxb, gw, gb = _autograd(xa, xb, w, b, gy, up, nd)
    srcs = [(xa, up)] + ([(xb, False)] if xb is not None else [])
    D = gy.shape[1]
    # integer operands: both sides exact, so equal; random ones: fp64 rounding in different orders
    same = torch.equal if integer else (lambda a, c: torch.allclose(a, c, rtol=1e-12, atol=1e-12))
    assert same(ref.conv(srcs, w, D, slab=slab, nd=nd) + b, y)
    # the finish hook sees every slab once, in order
    parts = ref.conv(srcs, w, D, finish=lambda t, d0, d1: (d0, d1, t), slab=slab, nd=nd)
    assert [(d0, d1) for d0, d1, _ in parts] == [(d, min(d + slab, D)) for d in range(0, D, slab)]
    assert same(torch.cat([t for _, _, t in parts], 1) + b, y)
    # dgrad: the transposed, flipped weight over the output gradient; the upsampled source's part summed over its children
    gx = ref.conv([(gy, False)], ref.dgrad_weight(w), D, slab=slab)
    assert same(ref.children_sum(gx[..., :Ca], nd) if up else gx[..., :Ca], gxa)
    if xb is not None:
        assert same(gx[..., Ca:], gxb)
    gw_r, gb_r = ref.wgrad(srcs, gy, kd, slab=slab, nd=nd)
    assert gw_r.shape == gw.shape and same(gw_r, gw) and same(gb_r, gb)
    # the absolute sums are the same sums over |x| and |gz|
    ga, gba = ref.wgrad([(xa.abs(), up)] + ([(xb.abs(), False)] if xb is not None else []), gy.abs(), kd, slab=slab, nd=nd)
    gw_a, gb_a = ref.wgrad(srcs, gy, kd, absolute=True, slab=slab, nd=nd)
    assert torch.equal(gw_a, ga) and torch.equal(gb_a, gba) and bool((gw_a >= gw_r.abs()).all())


def _bf16_rne(v):
    """float32 array -> the bf16 values (as float32) by round to nearest, ties to even, on the bit pattern (finite inputs)"""
    u = v.astype(np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32)


@pytest.mark.parametrize("mode", ["leaky", "mask", "raw"])
def test_epilogue_emulation_matches_direct_fp32(mode):
    g = torch.Generator().manual_seed(3)
    n, C = 4096, 8
    # sums of the exact tests (multiples of 2^-6), plus values whose products with the slope round in fp32 and bf16 ties
    y = torch.cat([torch.randint(-20000, 20001, (n // 2, C), generator=g).double() / 64,
                   torch.randn((n // 2, C), generator=g, dtype=torch.float64) * 100])
    y[:16] = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 2 ** -7 * 5, 0.0, -0.0, 255.5, -255.5] * 2, dtype=torch.float64)[:, None]
    bias = torch.randint(-8, 9, (C,), generator=g).float() / 64
    mask = torch.randint(-1, 2, (n, C), generator=g).to(torch.bfloat16)
    slope = 0.2
    kw = dict(leaky=dict(bias=bias, slope=slope), mask=dict(slope=slope, mask=mask), raw=dict())[mode]
    out = ref.epilogue(y, **kw).float().numpy()
    v = y.numpy().astype(np.float32)
    s = np.float32(slope)
    if mode == "leaky":
        v = v + bias.numpy()
        v = np.maximum(v, v * s)
    elif mode == "mask":
        v = np.where(mask.float().numpy() < 0, v * s, v)
    assert v.dtype == np.float32
    np.testing.assert_array_equal(out, _bf16_rne(v))
    if mode == "leaky":
        np.testing.assert_array_equal(ref.epilogue(y, bf16=False, **kw).numpy(), v)
