"""The fragment-layout epilogues of the kd-folded layers, the 2-D layers and the fp32 planar outputs are pure
re-implementations of the generic epilogue, and the ordered hand-off of the tensor pipe between the two MMA warpgroups
changes no arithmetic: tensor copies on / off x specialised / generic epilogue (VXM_B200_TMA, VXM_B200_TCS_EPI) must be
torch.equal, under every persistent-grid cap (VXM_B200_CONV_CTAS: one item per CTA up to many, items ending on either
warpgroup), at ragged and full sizes, B = 1 and 2, 3-D and 2-D."""
import pytest
import torch

pytestmark = pytest.mark.gpu

FULL = (160, 192, 224)
CAPS = ("1", "2", "5", "13", None)


@pytest.fixture(scope="module")
def tc(cuda):
    import voxelmorph_b200 as v
    from voxelmorph_b200 import tc
    v._lib.load()
    return tc


def _ndhwc(tc, g, B, shape, c, cuda):
    return tc.to_ndhwc_bf16(torch.randn((B, c) + shape, generator=g, device=cuda))


def _launch(tc, kind, B, shape, cuda):
    """A launch of the given kind on seeded operands; `shape` is (D, H, W), D = 1 with kd = 1 for a 2-D layer."""
    g = torch.Generator(device=cuda).manual_seed(91)
    w = lambda co, ci, kd=3: torch.randn((co, ci, kd, 3, 3), generator=g, device=cuda) * 0.1
    if kind == "fold_fwd":                 # first convolution over kd-folded image planes (2 planes -> 6 of 8 channels)
        planes = [torch.randn((B, 1) + shape, generator=g, device=cuda) for _ in range(2)]
        x3 = tc.planar_fold_kd(planes, 8)
        pk, cp = tc.pack_weights_fold(w(16, 2))
        b = torch.randn(16, generator=g, device=cuda)
        return lambda: tc.conv_fwd_t(x3, None, pk, cp, b, 16, 1, slope=0.2)
    if kind == "fold_dgrad":               # flow-head dgrad over the kd-folded flow gradient (9 of 16 channels), masked
        planes = [torch.randn((B, 1) + shape, generator=g, device=cuda) for _ in range(3)]
        g3 = tc.planar_fold_kd(planes, 16)
        pk, cp = tc.pack_weights_fold(w(3, 16), transposed=True)
        m = _ndhwc(tc, g, B, shape, 16, cuda)
        # saved activations of -0.0: the generic epilogue does not apply the derivative there (bf16 < 0 is false)
        m.view(-1)[::7] = -0.0
        return lambda: tc.conv_fwd_t(g3, None, pk, cp, None, 16, 1, slope=0.2, mask=m)
    if kind.startswith("head"):            # flow head cin -> nout, fp32 planar, bias, no activation
        _, cin, nout, kd = kind.split("_")
        cin, nout, kd = int(cin), int(nout), int(kd)
        x = _ndhwc(tc, g, B, shape, cin, cuda)
        pk, cp = tc.pack_weights_t(w(nout, cin, kd), variant="s")
        b = torch.randn(nout, generator=g, device=cuda)
        return lambda: tc.conv_fwd_t(x, None, pk, cp, b, nout, kd, out_fp32_planar=True)
    if kind.startswith("imgdgrad"):        # first-layer image dgrad cg -> planes, fp32 planar, no bias
        _, cg, planes, kd = kind.split("_")
        cg, planes, kd = int(cg), int(planes), int(kd)
        gz = _ndhwc(tc, g, B, shape, cg, cuda)
        pk, cp = tc.pack_weights_t(w(cg, planes, kd), transposed=True, variant="s")
        return lambda: tc.conv_fwd_t(gz, None, pk, cp, None, planes, kd, out_fp32_planar=True)
    if kind.startswith("fwd2d"):           # 2-D forward, bias + LeakyReLU
        _, cin, cout = kind.split("_")
        cin, cout = int(cin), int(cout)
        x = _ndhwc(tc, g, B, shape, cin, cuda)
        pk, cp = tc.pack_weights_t(w(cout, cin, 1), variant="s")
        b = torch.randn(cout, generator=g, device=cuda)
        return lambda: tc.conv_fwd_t(x, None, pk, cp, b, cout, 1, slope=0.2)
    if kind.startswith("dgrad2d"):         # 2-D dgrad with the LeakyReLU-derivative mask
        _, cg, cin = kind.split("_")
        cg, cin = int(cg), int(cin)
        gz = _ndhwc(tc, g, B, shape, cg, cuda)
        pk, cp = tc.pack_weights_t(w(cg, cin, 1), transposed=True, variant="s")
        m = _ndhwc(tc, g, B, shape, cin, cuda)
        m.view(-1)[::5] = -0.0
        return lambda: tc.conv_fwd_t(gz, None, pk, cp, None, cin, 1, slope=0.2, mask=m)
    raise ValueError(kind)


CASES = [
    # kind, B, (D, H, W)
    ("fold_fwd", 1, (9, 13, 35)),
    ("fold_fwd", 2, (6, 16, 34)),
    ("fold_fwd", 1, FULL),
    ("fold_dgrad", 1, (9, 13, 35)),
    ("fold_dgrad", 2, (6, 16, 34)),
    ("fold_dgrad", 1, FULL),
    ("head_16_3_3", 1, (9, 13, 35)),
    ("head_16_3_3", 2, (6, 16, 34)),
    ("head_16_3_3", 1, FULL),
    ("head_16_6_3", 1, (9, 13, 35)),       # probabilistic head: mean and log-variance, 2 nd outputs
    ("head_16_6_3", 1, FULL),
    ("head_32_3_3", 1, (7, 10, 33)),       # a 32-channel last decoder layer
    ("head_16_2_1", 2, (1, 37, 70)),       # 2-D flow head
    ("head_16_4_1", 1, (1, 192, 224)),     # 2-D probabilistic head
    ("imgdgrad_16_2_3", 1, (9, 13, 35)),
    ("imgdgrad_16_2_3", 2, (6, 16, 34)),
    ("imgdgrad_16_2_3", 1, FULL),
    ("imgdgrad_16_2_1", 2, (1, 37, 70)),
    ("fwd2d_16_16", 2, (1, 37, 70)),
    ("fwd2d_32_32", 1, (1, 96, 112)),
    ("fwd2d_32_16", 1, (1, 192, 224)),
    ("fwd2d_64_32", 2, (1, 24, 28)),       # 4-row tiles
    ("fwd2d_48_32", 1, (1, 48, 56)),       # 32 + 16 channel groups
    ("dgrad2d_16_16", 2, (1, 37, 70)),
    ("dgrad2d_16_32", 1, (1, 96, 112)),
    ("dgrad2d_32_32", 1, (1, 192, 224)),
]


@pytest.mark.parametrize("kind,B,shape", CASES, ids=["%s-B%d-%s" % (k, b, "x".join(map(str, s))) for k, b, s in CASES])
def test_fragment_drain_matches_generic_epilogue(tc, cuda, monkeypatch, kind, B, shape):
    run = _launch(tc, kind, B, shape, cuda)
    outs = {}
    for cap in CAPS:
        if cap is None:
            monkeypatch.delenv("VXM_B200_CONV_CTAS", raising=False)
        else:
            monkeypatch.setenv("VXM_B200_CONV_CTAS", cap)
        for tma in ("1", "0"):
            for epi in ("1", "0"):
                monkeypatch.setenv("VXM_B200_TMA", tma)
                monkeypatch.setenv("VXM_B200_TCS_EPI", epi)
                outs[(cap, tma, epi)] = run().float().cpu()
    torch.cuda.synchronize()
    ref = outs[(None, "0", "0")]
    assert torch.isfinite(ref).all() and float(ref.abs().max()) > 0
    for k, v in outs.items():
        # same MMAs in the same order, same fp32 epilogue arithmetic: equal bit for bit
        assert torch.equal(v, ref) and torch.equal(torch.signbit(v), torch.signbit(ref)), k
