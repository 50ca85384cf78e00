"""The 48- and 64-output-channel tensor-core launches (one kw-stacked wgmma chain per 64-row half, drained by two
threads per voxel row): TMA / cp.async staging and the specialised / generic epilogues must stay bit-identical, and
the result must match torch's fp64 convolution on the same bf16-rounded operands (1e-2 of max|ref|: bf16 output)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    a = a.double()
    b = b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.fixture(scope="module")
def tc(cuda):
    import voxelmorph_b200 as v
    from voxelmorph_b200 import tc
    v._lib.load()
    return tc


@pytest.mark.parametrize("shape,Cin,Cout,mode", [
    ((9, 13, 35), 32, 64, "fwd"),      # both m64 halves at 96 accumulators, ragged sizes on every side
    ((9, 13, 35), 16, 48, "fwd"),      # 72 accumulators, the second warp pair drains one chunk less
    ((10, 20, 40), 32, 64, "dgrad"),   # mask (LeakyReLU derivative) epilogue
])
def test_wide_output_paths_agree_and_match_fp64(tc, cuda, monkeypatch, shape, Cin, Cout, mode):
    g = torch.Generator().manual_seed(91)
    x = torch.randn((2, Cin) + shape, generator=g).to(torch.bfloat16).float()
    xa = tc.to_ndhwc_bf16(x.to(cuda))
    if mode == "fwd":
        w = (torch.randn((Cout, Cin, 3, 3, 3), generator=g) * 0.1).to(torch.bfloat16).float()
        b = torch.randn(Cout, generator=g)
        wpk, cp = tc.pack_weights_t(w.to(cuda), variant="s")
        bd = b.to(cuda)
        run = lambda: tc.conv_fwd_t(xa, None, wpk, cp, bd, Cout, 3, slope=0.2)
        ref = F.leaky_relu(F.conv3d(x.double(), w.double(), b.double(), padding=1), 0.2)
    else:
        # dgrad of a Cout -> Cin layer: Cin gradient channels in, Cout out, times the LeakyReLU derivative of the mask
        w = (torch.randn((Cin, Cout, 3, 3, 3), generator=g) * 0.1).to(torch.bfloat16).float()
        m = torch.randn((2, Cout) + shape, generator=g).to(torch.bfloat16).float()
        wpk, cp = tc.pack_weights_t(w.to(cuda), transposed=True, variant="s")
        md = tc.to_ndhwc_bf16(m.to(cuda))
        run = lambda: tc.conv_fwd_t(xa, None, wpk, cp, None, Cout, 3, slope=0.2, mask=md)
        gin = F.conv_transpose3d(x.double(), w.double(), None, padding=1)
        ref = torch.where(m.double() < 0, gin * 0.2, gin)
    outs = {}
    for tma in ("1", "0"):
        for epi in ("1", "0"):
            monkeypatch.setenv("VXM_B200_TMA", tma)
            monkeypatch.setenv("VXM_B200_TCS_EPI", epi)
            outs[(tma, epi)] = tc.from_ndhwc(run()).float().cpu()
    torch.cuda.synchronize()
    base = outs[("0", "0")]
    assert torch.isfinite(base).all() and float(base.abs().max()) > 0
    for k, v in outs.items():
        assert torch.equal(v, base), k     # same MMAs in the same order, same fp32 epilogue arithmetic: bit-identical
    assert rel_err(base, ref) <= 1e-2
