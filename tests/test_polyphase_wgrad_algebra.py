"""Coarse-voxel form of the weight gradient of a nearest-x2 upsampled source (csrc/conv3d_tc_wgrad2.cu,
wgrad2_poly_kernel), checked in fp64 on the CPU against torch's autograd of conv3d(up(x), w, padding=1).  Per axis, tap
index 0 (offset -1) pairs x[c - 1] with O[c] = g[2c - 1] + g[2c], index 1 pairs x[c] with E[c] = g[2c] + g[2c + 1] and
index 2 pairs x[c] with O[c], for coarse positions c = 0 .. Dc (fine voxels outside the volume, x[-1] and x[Dc] are zero);
the bias gradient is the sum of G_EEE."""
import pytest
import torch
import torch.nn.functional as F


def up(x):
    return x.repeat_interleave(2, 2).repeat_interleave(2, 3).repeat_interleave(2, 4)


def pair_sums(g, dim, kind):
    """E (kind 1) or O (kind 0) pair sums of g along `dim`: Dc + 1 coarse positions, the last E one zero"""
    pad = [0, 0] * (4 - dim)
    if kind == 1:
        return F.pad(g, pad + [0, 2]).unfold(dim, 2, 2).sum(-1)
    return F.pad(g, pad + [1, 1]).unfold(dim, 2, 2).sum(-1)


def coarse_wgrad(x, gz):
    """(gw (Cout, Cin, 3, 3, 3), gb (Cout,)) from the coarse x (B, Cin, Dc, Hc, Wc) and fine gz (B, Cout, 2Dc, 2Hc, 2Wc)"""
    B, Cin = x.shape[:2]
    Cout = gz.shape[1]
    # x on the Dc + 1 coarse positions of G, shifted by s in {-1, 0}: xs[s][c] = x[c + s]
    xp = F.pad(x, [1, 1, 1, 1, 1, 1])                     # xp[c + 1] = x[c], zero at -1 and Dc
    gw = torch.zeros((Cout, Cin, 3, 3, 3), dtype=x.dtype)
    kinds = {0: (0, -1), 1: (1, 0), 2: (0, 0)}            # tap index -> (O = 0 / E = 1, source shift)
    for td in range(3):
        for th in range(3):
            for tw in range(3):
                G = gz
                for dim, t in ((2, td), (3, th), (4, tw)):
                    G = pair_sums(G, dim, kinds[t][0])
                sd, sh, sw = kinds[td][1], kinds[th][1], kinds[tw][1]
                Dc1, Hc1, Wc1 = G.shape[2:]
                xs = xp[:, :, 1 + sd:1 + sd + Dc1, 1 + sh:1 + sh + Hc1, 1 + sw:1 + sw + Wc1]
                gw[:, :, td, th, tw] = torch.einsum("bcdhw,bodhw->oc", xs, G)
    geee = gz
    for dim in (2, 3, 4):
        geee = pair_sums(geee, dim, 1)
    return gw, geee.sum((0, 2, 3, 4))


@pytest.mark.parametrize("shape", [(3, 5, 7), (1, 3, 5), (2, 1, 3), (3, 2, 1), (1, 1, 1)])
def test_coarse_form_matches_autograd(shape):
    g = torch.Generator().manual_seed(sum(shape))
    B, Cin, Cout = 2, 5, 3
    x = torch.randn((B, Cin) + shape, generator=g, dtype=torch.float64)
    w = torch.randn((Cout, Cin, 3, 3, 3), generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.zeros(Cout, dtype=torch.float64, requires_grad=True)
    gz = torch.randn((B, Cout) + tuple(2 * s for s in shape), generator=g, dtype=torch.float64)
    F.conv3d(up(x), w, b, padding=1).backward(gz)
    gw, gb = coarse_wgrad(x, gz)
    torch.testing.assert_close(gw, w.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(gb, b.grad, rtol=1e-12, atol=1e-12)


def test_shift_convention_is_not_symmetric():
    """the index-0 and index-2 taps differ (x[c - 1] vs x[c] against the same O sums): swapping them must fail"""
    g = torch.Generator().manual_seed(1)
    x = torch.randn((1, 2, 3, 3, 3), generator=g, dtype=torch.float64)
    gz = torch.randn((1, 2, 6, 6, 6), generator=g, dtype=torch.float64)
    gw, _ = coarse_wgrad(x, gz)
    w = torch.zeros((2, 2, 3, 3, 3), dtype=torch.float64, requires_grad=True)
    F.conv3d(up(x), w, padding=1).backward(gz)
    assert not torch.allclose(gw.flip(2), w.grad)
    torch.testing.assert_close(gw, w.grad, rtol=1e-12, atol=1e-12)
