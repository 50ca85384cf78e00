"""Depth-axis index algebra of the polyphase concat layers (csrc/conv3d_tc_s.cu, conv_tcs_kernel PD), checked in fp64 on the CPU
against torch's own 3-D convolution.  Along d a nearest-x2 upsampled tensor has one value per slice pair, so:
- forward: an even output slice 2c is W0 x[c-1] + (W1 + W2) x[c], an odd one 2c+1 is (W0 + W1) x[c] + W2 x[c+1];
- dgrad: the gradient w.r.t. coarse slice c, summed over its two fine slices, is a stride-2 correlation of the fine
  output gradient at fine offsets -1, 0, +1, +2 from 2c with the transposed taps T0, T0 + T1, T1 + T2, T2."""
import torch
import torch.nn.functional as F


def up_d(x):
    return x.repeat_interleave(2, dim=2)


def poly_forward(x, w):
    """conv3d(up_d(x), w, padding=1) from the two merged kd taps of each output parity."""
    even = torch.stack([w[:, :, 0], w[:, :, 1] + w[:, :, 2]], dim=2)
    odd = torch.stack([w[:, :, 0] + w[:, :, 1], w[:, :, 2]], dim=2)
    ye = F.conv3d(F.pad(x, (0, 0, 0, 0, 1, 0)), even, padding=(0, 1, 1))      # slabs c - 1, c
    yo = F.conv3d(F.pad(x, (0, 0, 0, 0, 0, 1)), odd, padding=(0, 1, 1))       # slabs c, c + 1
    return torch.stack([ye, yo], dim=3).flatten(2, 3)


def poly_dgrad(g, w):
    """Gradient of conv3d(up_d(x), w, padding=1) w.r.t. x, from the fine output gradient g (4 merged transposed taps, stride 2)."""
    t = w.transpose(0, 1).flip(2, 3, 4)                   # conv_transpose3d(g, w) == conv3d(g, t)
    k = torch.stack([t[:, :, 0], t[:, :, 0] + t[:, :, 1], t[:, :, 1] + t[:, :, 2], t[:, :, 2]], dim=2)
    return F.conv3d(F.pad(g, (1, 1, 1, 1, 1, 1)), k, stride=(2, 1, 1))


def test_forward_phases_match_upsampled_convolution():
    g = torch.Generator().manual_seed(3)
    x = torch.randn((2, 5, 4, 6, 7), generator=g, dtype=torch.float64)
    w = torch.randn((3, 5, 3, 3, 3), generator=g, dtype=torch.float64)
    ref = F.conv3d(up_d(x), w, padding=1)
    assert torch.allclose(poly_forward(x, w), ref, rtol=0, atol=1e-12)


def test_coarse_depth_dgrad_matches_autograd():
    g = torch.Generator().manual_seed(4)
    x = torch.randn((2, 5, 4, 6, 7), generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn((3, 5, 3, 3, 3), generator=g, dtype=torch.float64)
    gy = torch.randn((2, 3, 8, 6, 7), generator=g, dtype=torch.float64)
    F.conv3d(up_d(x), w, padding=1).backward(gy)
    assert torch.allclose(poly_dgrad(gy, w), x.grad, rtol=0, atol=1e-12)
    # what the engine stores before the (h, w) sum: the fine-(h, w) gradient of the upsampled tensor summed over slice pairs
    gup = F.conv_transpose3d(gy, w, padding=1)
    assert torch.allclose(poly_dgrad(gy, w), gup.view(2, 5, 4, 2, 6, 7).sum(3), rtol=0, atol=1e-12)
