"""GPU parity tests of the wgmma (bf16 operands, fp32 accumulation) convolution engine against the CPU
oracle evaluated on the SAME bf16-rounded operands (fp64 accumulation).  Tolerances: bf16-output paths 1e-2 of
max|ref| (output rounding is 2^-9 relative), fp32-output paths 1e-4."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    a = a.double()
    b = b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def bf(x):
    return x.to(torch.bfloat16).float()


@pytest.fixture(scope="module")
def tc(cuda):
    import voxelmorph_b200 as v
    from voxelmorph_b200 import tc
    v._lib.load()
    return tc


CASES = [
    # shape, Ca, Cb, up, Cout
    ((4, 16, 8), 16, 0, False, 16),
    ((20, 40, 24), 32, 0, False, 32),
    ((10, 12, 14), 32, 0, False, 32),     # ragged tiles (coarsest U-Net level shape)
    ((8, 32, 16), 32, 16, True, 32),      # nearest-x2 upsample + skip concat fused in the loader (48 -> 32)
    ((8, 16, 16), 32, 32, True, 32),      # 64 -> 32
    ((6, 16, 24), 32, 0, False, 16),
    ((1, 32, 24), 16, 0, False, 32),      # 2-D (kd = 1)
]


@pytest.mark.parametrize("shape,Ca,Cb,up,Cout", CASES)
def test_tc_conv_forward(tc, cuda, shape, Ca, Cb, up, Cout):
    g = torch.Generator().manual_seed(hash((shape, Ca, Cb)) % 1000)
    kd = 1 if shape[0] == 1 else 3
    D, H, W = shape
    ashape = ((D // 2 if kd == 3 else D), H // 2, W // 2) if up else shape
    xa = bf(torch.randn((2, Ca) + ashape, generator=g))
    xb = bf(torch.randn((2, Cb) + shape, generator=g)) if Cb else None
    w = bf(torch.randn((Cout, Ca + Cb, kd, 3, 3), generator=g) * 0.1)
    b = torch.randn(Cout, generator=g)
    xin = xa
    if up:
        xin = F.interpolate(xa, scale_factor=(2 if kd == 3 else 1, 2, 2), mode="nearest")
    if xb is not None:
        xin = torch.cat([xin, xb], dim=1)
    ref = F.leaky_relu(F.conv3d(xin.double(), w.double(), b.double(), padding=(kd // 2, 1, 1)), 0.2)
    wpk, NP = tc.pack_weights(w.to(cuda))
    out = tc.conv_fwd(tc.to_ndhwc_bf16(xa.to(cuda)), None if xb is None else tc.to_ndhwc_bf16(xb.to(cuda)), wpk, NP,
                      b.to(cuda), Cout, kd, up=up, slope=0.2)
    torch.cuda.synchronize()
    assert rel_err(tc.from_ndhwc(out).cpu(), ref) <= 1e-2


def test_tc_flow_head_fp32_out(tc, cuda):
    g = torch.Generator().manual_seed(5)
    x = bf(torch.randn((1, 16, 12, 20, 16), generator=g))
    w = bf(torch.randn((3, 16, 3, 3, 3), generator=g) * 0.05)
    b = torch.randn(3, generator=g) * 0.1
    ref = F.conv3d(x.double(), w.double(), b.double(), padding=1)
    wpk, NP = tc.pack_weights(w.to(cuda))
    out = tc.conv_fwd(tc.to_ndhwc_bf16(x.to(cuda)), None, wpk, NP, b.to(cuda), 3, 3, out_fp32_planar=True)
    assert rel_err(out.cpu(), ref) <= 1e-4


def test_tc_first_layer_planar_fp32_inputs(tc, cuda):
    g = torch.Generator().manual_seed(6)
    src, trg = torch.rand((2, 1, 8, 24, 16), generator=g), torch.rand((2, 1, 8, 24, 16), generator=g)
    w = bf(torch.randn((16, 2, 3, 3, 3), generator=g) * 0.2)
    b = torch.randn(16, generator=g) * 0.1
    ref = F.leaky_relu(F.conv3d(bf(torch.cat([src, trg], 1)).double(), w.double(), b.double(), padding=1), 0.2)
    wpk, NP = tc.pack_weights(w.to(cuda))
    out = tc.conv_fwd(None, None, wpk, NP, b.to(cuda), 16, 3, planar=[src.to(cuda), trg.to(cuda)], slope=0.2)
    assert rel_err(tc.from_ndhwc(out).cpu(), ref) <= 1e-2


def test_tc_dgrad_with_mask(tc, cuda):
    """dgrad = the same kernel on the transposed / flipped packed weights; the LeakyReLU derivative of the layer
    below is applied in the epilogue from its saved (bf16) activation."""
    g = torch.Generator().manual_seed(7)
    Cin, Cout, shape = 32, 16, (6, 16, 16)
    x = torch.randn((1, Cin) + shape, generator=g, dtype=torch.float64, requires_grad=True)
    w = bf(torch.randn((Cout, Cin, 3, 3, 3), generator=g) * 0.1)
    gy = bf(torch.randn((1, Cout) + shape, generator=g))
    F.conv3d(x, w.double(), None, padding=1).backward(gy.double())
    below = bf(torch.randn((1, Cin) + shape, generator=g))          # activation of the layer below (mask source)
    ref = x.grad * torch.where(below.double() < 0, 0.2, 1.0)
    wpk, NP = tc.pack_weights(w.to(cuda), transposed=True)
    out = tc.conv_fwd(tc.to_ndhwc_bf16(gy.to(cuda)), None, wpk, NP, None, Cin, 3, slope=0.2,
                      mask=tc.to_ndhwc_bf16(below.to(cuda)))
    assert rel_err(tc.from_ndhwc(out).cpu(), ref) <= 1e-2


@pytest.mark.parametrize("Cin,split", [(48, 32), (64, 32)])
def test_tc_dgrad_split_outputs(tc, cuda, Cin, split):
    """Single-pass dgrad of a concat layer: N = Cin (48 / 64) output channels written to two tensors."""
    g = torch.Generator().manual_seed(8)
    Cout, shape = 32, (6, 16, 24)
    x = torch.randn((1, Cin) + shape, generator=g, dtype=torch.float64, requires_grad=True)
    w = bf(torch.randn((Cout, Cin, 3, 3, 3), generator=g) * 0.1)
    gy = bf(torch.randn((1, Cout) + shape, generator=g))
    F.conv3d(x, w.double(), None, padding=1).backward(gy.double())
    wpk, NP = tc.pack_weights(w.to(cuda), transposed=True)
    assert NP == Cin
    oa, ob = tc.conv_fwd(tc.to_ndhwc_bf16(gy.to(cuda)), None, wpk, NP, None, Cin, 3, split=split)
    assert rel_err(tc.from_ndhwc(oa).cpu(), x.grad[:, :split]) <= 1e-2
    assert rel_err(tc.from_ndhwc(ob).cpu(), x.grad[:, split:]) <= 1e-2


WG_CASES = [
    # shape, Ca, Cb, up, Cout
    ((4, 16, 8), 16, 0, False, 16),
    ((12, 24, 20), 32, 0, False, 32),
    ((10, 12, 14), 32, 0, False, 32),
    ((8, 32, 16), 32, 16, True, 32),
    ((8, 16, 16), 32, 32, True, 32),
    ((6, 16, 24), 32, 0, False, 16),
    ((1, 32, 24), 16, 0, False, 32),
]


@pytest.mark.parametrize("shape,Ca,Cb,up,Cout", WG_CASES)
def test_tc_wgrad(tc, cuda, shape, Ca, Cb, up, Cout):
    g = torch.Generator().manual_seed(11)
    kd = 1 if shape[0] == 1 else 3
    D, H, W = shape
    ashape = ((D // 2 if kd == 3 else D), H // 2, W // 2) if up else shape
    xa = bf(torch.randn((2, Ca) + ashape, generator=g))
    xb = bf(torch.randn((2, Cb) + shape, generator=g)) if Cb else None
    gz = bf(torch.randn((2, Cout) + shape, generator=g))
    xin = xa
    if up:
        xin = F.interpolate(xa, scale_factor=(2 if kd == 3 else 1, 2, 2), mode="nearest")
    if xb is not None:
        xin = torch.cat([xin, xb], dim=1)
    w = torch.zeros((Cout, Ca + Cb, kd, 3, 3), dtype=torch.float64, requires_grad=True)
    b = torch.zeros(Cout, dtype=torch.float64, requires_grad=True)
    F.conv3d(xin.double(), w, b, padding=(kd // 2, 1, 1)).backward(gz.double())
    gw, gb = tc.conv_wgrad(tc.to_ndhwc_bf16(xa.to(cuda)), None if xb is None else tc.to_ndhwc_bf16(xb.to(cuda)),
                           tc.to_ndhwc_bf16(gz.to(cuda)), Ca + Cb, Cout, kd, up=up)
    assert rel_err(gw.cpu(), w.grad) <= 1e-4
    assert rel_err(gb.cpu(), b.grad) <= 1e-4


def test_tc_wgrad_planar_sources(tc, cuda):
    g = torch.Generator().manual_seed(12)
    shape = (8, 24, 16)
    src, trg = torch.rand((2, 1) + shape, generator=g), torch.rand((2, 1) + shape, generator=g)
    gz = bf(torch.randn((2, 16) + shape, generator=g))
    w = torch.zeros((16, 2, 3, 3, 3), dtype=torch.float64, requires_grad=True)
    F.conv3d(bf(torch.cat([src, trg], 1)).double(), w, None, padding=1).backward(gz.double())
    gw, _ = tc.conv_wgrad(None, None, tc.to_ndhwc_bf16(gz.to(cuda)), 2, 16, 3, planar_x=[src.to(cuda), trg.to(cuda)])
    assert rel_err(gw.cpu(), w.grad) <= 1e-4
    # flow head: planar fp32 gz (3 channels), bf16 x
    x = bf(torch.randn((2, 16) + shape, generator=g))
    gfl = torch.randn((2, 3) + shape, generator=g)
    w = torch.zeros((3, 16, 3, 3, 3), dtype=torch.float64, requires_grad=True)
    F.conv3d(x.double(), w, None, padding=1).backward(bf(gfl).double())
    planes = [gfl[:, i:i + 1].to(cuda) for i in range(3)]
    gfl_dev = gfl.to(cuda)
    planes = [gfl_dev[:, i:i + 1] for i in range(3)]
    gw, _ = tc.conv_wgrad(tc.to_ndhwc_bf16(x.to(cuda)), None, None, 16, 3, 3, planar_g=planes)
    assert rel_err(gw.cpu(), w.grad) <= 1e-4


T_CASES = [
    # shape, Ca, Cb, up, Cout
    ((4, 8, 32), 16, 0, False, 16),
    ((6, 12, 60), 32, 0, False, 32),      # two full w tiles
    ((10, 12, 14), 32, 0, False, 32),     # ragged (coarsest level)
    ((8, 32, 16), 32, 16, True, 32),      # 48 -> 32, fused upsample + concat
    ((6, 16, 24), 32, 0, False, 16),
    ((5, 20, 70), 8, 0, False, 16),       # half-K (8-channel) input
    ((1, 32, 44), 16, 0, False, 32),      # 2-D
    ((20, 40, 24), 16, 0, False, 32),     # d chunks
]


@pytest.fixture(params=["t", "s"])
def variant(request):
    return request.param


@pytest.mark.parametrize("shape,Ca,Cb,up,Cout", T_CASES)
def test_tct_conv_forward(tc, cuda, variant, shape, Ca, Cb, up, Cout):
    g = torch.Generator().manual_seed(21)
    kd = 1 if shape[0] == 1 else 3
    D, H, W = shape
    ashape = ((D // 2 if kd == 3 else D), H // 2, W // 2) if up else shape
    xa = bf(torch.randn((2, Ca) + ashape, generator=g))
    xb = bf(torch.randn((2, Cb) + shape, generator=g)) if Cb else None
    cin_real = 2 if Ca == 8 else Ca + Cb
    w = bf(torch.randn((Cout, cin_real, kd, 3, 3), generator=g) * 0.1)
    b = torch.randn(Cout, generator=g)
    xin = xa
    if up:
        xin = F.interpolate(xa, scale_factor=(2 if kd == 3 else 1, 2, 2), mode="nearest")
    if xb is not None:
        xin = torch.cat([xin, xb], dim=1)
    ref = F.leaky_relu(F.conv3d(xin[:, :cin_real].double(), w.double(), b.double(), padding=(kd // 2, 1, 1)), 0.2)
    wpk, cp = tc.pack_weights_t(w.to(cuda), variant=variant)
    out = tc.conv_fwd_t(tc.to_ndhwc_bf16(xa.to(cuda)), None if xb is None else tc.to_ndhwc_bf16(xb.to(cuda)), wpk, cp,
                        b.to(cuda), Cout, kd, up=up, slope=0.2)
    torch.cuda.synchronize()
    assert rel_err(tc.from_ndhwc(out).cpu(), ref) <= 1e-2


def test_tct_flow_head_and_masked_dgrad(tc, cuda, variant):
    g = torch.Generator().manual_seed(22)
    x = bf(torch.randn((1, 16, 6, 12, 40), generator=g))
    w = bf(torch.randn((3, 16, 3, 3, 3), generator=g) * 0.05)
    b = torch.randn(3, generator=g) * 0.1
    ref = F.conv3d(x.double(), w.double(), b.double(), padding=1)
    wpk, cp = tc.pack_weights_t(w.to(cuda), variant=variant)
    out = tc.conv_fwd_t(tc.to_ndhwc_bf16(x.to(cuda)), None, wpk, cp, b.to(cuda), 3, 3, out_fp32_planar=True)
    assert rel_err(out.cpu(), ref) <= 1e-4
    # dgrad with the LeakyReLU-derivative mask
    Cin, Cout, shape = 32, 16, (6, 16, 34)
    xx = torch.randn((1, Cin) + shape, generator=g, dtype=torch.float64, requires_grad=True)
    ww = bf(torch.randn((Cout, Cin, 3, 3, 3), generator=g) * 0.1)
    gy = bf(torch.randn((1, Cout) + shape, generator=g))
    F.conv3d(xx, ww.double(), None, padding=1).backward(gy.double())
    below = bf(torch.randn((1, Cin) + shape, generator=g))
    refg = xx.grad * torch.where(below.double() < 0, 0.2, 1.0)
    wpk, cp = tc.pack_weights_t(ww.to(cuda), transposed=True, variant=variant)
    og = tc.conv_fwd_t(tc.to_ndhwc_bf16(gy.to(cuda)), None, wpk, cp, None, Cin, 3, slope=0.2, mask=tc.to_ndhwc_bf16(below.to(cuda)))
    assert rel_err(tc.from_ndhwc(og).cpu(), refg) <= 1e-2


@pytest.mark.parametrize("Cin,split", [(48, 32), (64, 32)])
def test_tct_dgrad_split_outputs(tc, cuda, variant, Cin, split):
    g = torch.Generator().manual_seed(9)
    Cout, shape = 32, (6, 12, 40)
    x = torch.randn((1, Cin) + shape, generator=g, dtype=torch.float64, requires_grad=True)
    w = bf(torch.randn((Cout, Cin, 3, 3, 3), generator=g) * 0.1)
    gy = bf(torch.randn((1, Cout) + shape, generator=g))
    F.conv3d(x, w.double(), None, padding=1).backward(gy.double())
    wpk, cp = tc.pack_weights_t(w.to(cuda), transposed=True, variant=variant)
    assert cp[0] == Cin
    oa, ob = tc.conv_fwd_t(tc.to_ndhwc_bf16(gy.to(cuda)), None, wpk, cp, None, Cin, 3, split=split)
    assert rel_err(tc.from_ndhwc(oa).cpu(), x.grad[:, :split]) <= 1e-2
    assert rel_err(tc.from_ndhwc(ob).cpu(), x.grad[:, split:]) <= 1e-2


def test_tct_cin64(tc, cuda, variant):
    g = torch.Generator().manual_seed(10)
    shape = (8, 16, 32)
    xa = bf(torch.randn((1, 32, 4, 8, 16), generator=g))
    xb = bf(torch.randn((1, 32) + shape, generator=g))
    w = bf(torch.randn((32, 64, 3, 3, 3), generator=g) * 0.1)
    xin = torch.cat([F.interpolate(xa, scale_factor=2, mode="nearest"), xb], dim=1)
    ref = F.leaky_relu(F.conv3d(xin.double(), w.double(), None, padding=1), 0.2)
    wpk, cp = tc.pack_weights_t(w.to(cuda), variant=variant)
    out = tc.conv_fwd_t(tc.to_ndhwc_bf16(xa.to(cuda)), tc.to_ndhwc_bf16(xb.to(cuda)), wpk, cp, None, 32, 3, up=True, slope=0.2)
    assert rel_err(tc.from_ndhwc(out).cpu(), ref) <= 1e-2


# ---- TMA tile staging and the specialised epilogues are pure re-implementations: results must not change ----

@pytest.mark.parametrize("shape,Ca,Cb,up,Cout,mode", [
    ((12, 24, 70), 16, 0, False, 16, "fwd"),      # one channel group, tensor copy only (forward epilogue)
    ((12, 24, 70), 32, 16, True, 32, "fwd"),      # upsampled group on cp.async + skip group by tensor copy (conv_tcs)
    ((10, 20, 40), 16, 0, False, 32, "dgrad"),    # dgrad epilogue (mask)
    ((10, 20, 40), 32, 0, False, 48, "split"),    # raw + channel split epilogue
    ((9, 13, 35), 32, 0, False, 16, "fwd"),       # ragged sizes: out-of-bounds fill on every side
])
def test_tma_and_lean_epilogue_match_reference_paths(tc, cuda, monkeypatch, shape, Ca, Cb, up, Cout, mode):
    g = torch.Generator().manual_seed(77)
    D, H, W = shape
    ashape = (D // 2, H // 2, W // 2) if up else shape
    if up:
        shape = (ashape[0] * 2, ashape[1] * 2, ashape[2] * 2)
    xa = tc.to_ndhwc_bf16(torch.randn((2, Ca) + ashape, generator=g).to(cuda))
    xb = tc.to_ndhwc_bf16(torch.randn((2, Cb) + shape, generator=g).to(cuda)) if Cb else None
    if mode == "fwd":
        w = torch.randn((Cout, Ca + Cb, 3, 3, 3), generator=g).to(cuda) * 0.1
        b = torch.randn(Cout, generator=g).to(cuda)
        wpk, cp = tc.pack_weights_t(w, variant="s")
        run = lambda: tc.conv_fwd_t(xa, xb, wpk, cp, b, Cout, 3, up=up, slope=0.2)
    else:
        w = torch.randn((Ca, Cout, 3, 3, 3), generator=g).to(cuda) * 0.1       # dgrad of a Cout -> Ca layer: produces Cout channels
        wpk, cp = tc.pack_weights_t(w, transposed=True, variant="s")
        if mode == "dgrad":
            m = tc.to_ndhwc_bf16(torch.randn((2, Cout) + shape, generator=g).to(cuda))
            run = lambda: tc.conv_fwd_t(xa, None, wpk, cp, None, Cout, 3, slope=0.2, mask=m)
        else:
            run = lambda: torch.cat(tc.conv_fwd_t(xa, None, wpk, cp, None, Cout, 3, split=32), dim=-1)
    outs = {}
    for tma in ("1", "0"):
        for epi in ("1", "0"):
            monkeypatch.setenv("VXM_B200_TMA", tma)
            monkeypatch.setenv("VXM_B200_TCS_EPI", epi)
            outs[(tma, epi)] = run().float().cpu()
    torch.cuda.synchronize()
    ref = outs[("0", "0")]
    assert torch.isfinite(ref).all() and float(ref.abs().max()) > 0
    for k, v in outs.items():
        assert torch.equal(v, ref), k      # same MMAs in the same order, same fp32 epilogue arithmetic: bit-identical


# ---- kd folded into the channels (first convolution / flow head) ----

def _khm_wgrad(tc, x, gz, cin_real, cout_real, cuda):
    batch = tc.WgradBatch.get(cuda)
    batch.reset()
    gw = torch.empty((cout_real, cin_real, 1, 3, 3), dtype=torch.float32, device=cuda)
    gb = torch.empty(cout_real, dtype=torch.float32, device=cuda)
    batch.add_khm(x, gz, gw, gb, cin_real, cout_real)
    batch.flush()
    torch.cuda.synchronize()
    return gw.cpu(), gb.cpu()


@pytest.mark.parametrize("shape", [(6, 16, 34), (9, 13, 35)])
def test_kd_folded_first_layer(tc, cuda, shape):
    """Two image planes: fold -> 2-D convolution == the 3-D convolution; 2-D kh-in-M weight gradient == autograd."""
    g = torch.Generator().manual_seed(31)
    B, P, Cout = 2, 2, 16
    x = bf(torch.randn((B, P) + shape, generator=g))
    w = bf(torch.randn((Cout, P, 3, 3, 3), generator=g) * 0.2)
    b = torch.randn(Cout, generator=g) * 0.1
    xd = x.double().requires_grad_(False)
    wd = w.double().requires_grad_(True)
    pre = F.conv3d(xd, wd, b.double(), padding=1)
    ref = F.leaky_relu(pre, 0.2)
    planes = [x[:, i:i + 1].to(cuda).contiguous() for i in range(P)]
    x3 = tc.planar_fold_kd(planes, 8)
    assert tuple(x3.shape) == (B,) + shape + (8,)
    # the folded tensor itself: channel kd * P + p = plane p shifted by kd - 1 slices, zero outside
    xs = F.pad(x, (0, 0, 0, 0, 1, 1))
    for kd in range(3):
        for p in range(P):
            assert torch.equal(x3[..., kd * P + p].float().cpu(), xs[:, p, kd:kd + shape[0]])
    assert float(x3[..., 3 * P:].abs().max()) == 0.0
    wpk, cp = tc.pack_weights_fold(w.to(cuda))
    out = tc.conv_fwd_t(x3, None, wpk, cp, b.to(cuda), Cout, 1, slope=0.2)
    torch.cuda.synchronize()
    assert rel_err(tc.from_ndhwc(out).cpu(), ref) <= 1e-2
    # weight / bias gradient
    gy = bf(torch.randn((B, Cout) + shape, generator=g))
    pre.backward(gy.double())
    gw2, gb = _khm_wgrad(tc, x3, tc.to_ndhwc_bf16(gy.to(cuda)), 3 * P, Cout, cuda)
    gw = gw2.view(Cout, 3, P, 3, 3).permute(0, 2, 1, 3, 4)
    assert rel_err(gw, wd.grad) <= 2e-3
    assert rel_err(gb, gy.double().sum(dim=(0, 2, 3, 4))) <= 2e-3


@pytest.mark.parametrize("shape", [(6, 16, 34), (9, 13, 35)])
def test_kd_folded_flow_head_backward(tc, cuda, shape):
    """Flow head 16 -> 3: the flow gradient folded over kd gives the masked dgrad (2-D convolution) and the weight gradient."""
    g = torch.Generator().manual_seed(32)
    B, Cin, nd = 1, 16, 3
    x = bf(torch.randn((B, Cin) + shape, generator=g))
    w = bf(torch.randn((nd, Cin, 3, 3, 3), generator=g) * 0.1)
    gy = bf(torch.randn((B, nd) + shape, generator=g))          # bf16-exact flow gradient: both paths see the same operands
    xd = x.double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    F.conv3d(xd, wd, None, padding=1).backward(gy.double())
    below = x                                                     # the layer below is LeakyReLU(0.2): derivative from its output's sign
    refg = xd.grad * torch.where(below.double() < 0, 0.2, 1.0)
    planes = [gy[:, i:i + 1].to(cuda).float().contiguous() for i in range(nd)]
    g3 = tc.planar_fold_kd(planes, 16)
    wpk, cp = tc.pack_weights_fold(w.to(cuda), transposed=True)
    xn = tc.to_ndhwc_bf16(x.to(cuda))
    dg = tc.conv_fwd_t(g3, None, wpk, cp, None, Cin, 1, slope=0.2, mask=xn)
    torch.cuda.synchronize()
    assert rel_err(tc.from_ndhwc(dg).cpu(), refg) <= 1e-2
    gw2, gb2 = _khm_wgrad(tc, xn, g3, Cin, 3 * nd, cuda)
    gw = gw2.view(3, nd, Cin, 3, 3).flip(0).permute(1, 2, 0, 3, 4)
    assert rel_err(gw, wd.grad) <= 2e-3
    assert rel_err(gb2[nd:2 * nd], gy.double().sum(dim=(0, 2, 3, 4))) <= 2e-3
