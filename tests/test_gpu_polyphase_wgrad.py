"""The coarse-voxel weight gradient of a 32-channel nearest-x2 upsampled source (wgrad2_poly_kernel) against fp64 and
against the fine kernel it replaces (VXM_B200_POLYPHASE=0).

- Ternary x and gz: every pair sum G is an integer with |G| <= 8 and every fp32 sum is exact, so the result equals the
  fp64 tap sums of conv_exact_ref.py at rem0's size (160x192x224), dec3's (80x96x112), B = 2 and ragged coarse shapes,
  under every persistent-grid cap (VXM_B200_CONV_CTAS), i.e. depth chunks starting on odd and even coarse slices.
- gz in {0, +-1, +-2^-8}: the pair sums need more than bf16's 8 bits, hi + lo holds them exactly, so the result still
  equals fp64 (without the lo pass it would not).
- Ordinary operands: equal to the fine kernel within fp32 re-association, and bit-identical between two runs."""
import pytest
import torch

import conv_exact_ref as ref

pytestmark = pytest.mark.gpu

CAPS = ["1", "2", "5", "13", None]


@pytest.fixture(scope="module")
def tc(cuda):
    import voxelmorph_b200 as vxm
    from voxelmorph_b200 import tc
    vxm._lib.load()
    return tc


def ternary(shape, g):
    nz = torch.randint(0, 2, shape, generator=g, device=g.device)
    return (nz * (2 * torch.randint(0, 2, shape, generator=g, device=g.device) - 1)).to(torch.bfloat16)


def run(tc, monkeypatch, xa, gz, cap=None, poly=True, batched=False):
    if cap is None:
        monkeypatch.delenv("VXM_B200_CONV_CTAS", raising=False)
    else:
        monkeypatch.setenv("VXM_B200_CONV_CTAS", cap)
    monkeypatch.setenv("VXM_B200_POLYPHASE", "1" if poly else "0")
    if batched:
        batch = tc.WgradBatch.get(gz.device)
        batch.reset()
        gw, gb = tc.conv_wgrad(xa, None, gz, 32, 32, 3, up=True, batch=batch)
        batch.flush()
    else:
        gw, gb = tc.conv_wgrad(xa, None, gz, 32, 32, 3, up=True)
    torch.cuda.synchronize()
    return gw.clone(), gb.clone()


# (B, coarse D, H, W): rem0 and dec3 of the default model, B = 2, ragged coarse extents
SHAPES = [(1, 80, 96, 112), (1, 40, 48, 56), (2, 7, 11, 33), (1, 9, 5, 31), (1, 3, 1, 2)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_exact_ternary(tc, cuda, monkeypatch, shape):
    g = torch.Generator(device=cuda).manual_seed(sum(shape))
    B, Dc, Hc, Wc = shape
    xa = ternary((B, Dc, Hc, Wc, 32), g)
    gz = ternary((B, 2 * Dc, 2 * Hc, 2 * Wc, 32), g)
    rw, rb = ref.wgrad([(xa, True)], gz, 3)
    aw, ab = ref.wgrad([(xa, True)], gz, 3, absolute=True)
    assert float(aw.max()) < 2 ** 24 and float(ab.max()) < 2 ** 24
    bad = {}
    for cap in CAPS:
        for batched in (False, True):
            gw, gb = run(tc, monkeypatch, xa, gz, cap, batched=batched)
            bad[(cap, batched)] = (int((gw.double() != rw).sum()), int((gb.double() != rb).sum()))
    print("\n[poly wgrad %s] mismatches (gw, gb) by (cap, batched): %s" % (shape, bad))
    assert all(v == (0, 0) for v in bad.values()), bad


def test_lo_pass(tc, cuda, monkeypatch):
    g = torch.Generator(device=cuda).manual_seed(3)
    B, Dc, Hc, Wc = 2, 7, 11, 33
    xa = ternary((B, Dc, Hc, Wc, 32), g)
    t = ternary((B, 2 * Dc, 2 * Hc, 2 * Wc, 32), g).float()
    small = torch.randint(0, 2, t.shape, generator=g, device=cuda).float()
    gz = (t * torch.where(small > 0, 2.0 ** -8, 1.0)).to(torch.bfloat16)
    rw, rb = ref.wgrad([(xa, True)], gz, 3)
    aw, _ = ref.wgrad([(xa, True)], gz, 3, absolute=True)
    assert float(aw.max()) * 2 ** 8 < 2 ** 24                 # multiples of 2^-8 below 2^24 units: exact in fp32
    # the pair sums really need the lo half: some are not bf16 numbers
    e = gz.float().unfold(1, 2, 2).sum(-1).unfold(2, 2, 2).sum(-1).unfold(3, 2, 2).sum(-1)
    assert not torch.equal(e, e.to(torch.bfloat16).float())
    for cap in ("5", None):
        gw, gb = run(tc, monkeypatch, xa, gz, cap)
        assert torch.equal(gw.double(), rw), cap
        assert torch.equal(gb.double(), rb), cap


@pytest.mark.parametrize("shape", [(1, 40, 48, 56), (2, 7, 11, 33)], ids=lambda s: "x".join(map(str, s)))
def test_ordinary_operands_vs_fine_kernel(tc, cuda, monkeypatch, shape):
    g = torch.Generator(device=cuda).manual_seed(11)
    B, Dc, Hc, Wc = shape
    xa = torch.randn((B, Dc, Hc, Wc, 32), generator=g, device=cuda).to(torch.bfloat16)
    gz = torch.randn((B, 2 * Dc, 2 * Hc, 2 * Wc, 32), generator=g, device=cuda).to(torch.bfloat16)
    pw, pb = run(tc, monkeypatch, xa, gz)
    pw2, pb2 = run(tc, monkeypatch, xa, gz)
    assert torch.equal(pw, pw2) and torch.equal(pb, pb2)         # fixed-order partials: deterministic
    fw, fb = run(tc, monkeypatch, xa, gz, poly=False)
    aw, ab = run(tc, monkeypatch, xa.abs(), gz.abs(), poly=False)  # sum of |terms|: the scale of re-association error
    err_w = float(((pw - fw).abs() / aw.clamp_min(1e-30)).max())
    err_b = float(((pb - fb).abs() / ab.clamp_min(1e-30)).max())
    print("\n[poly wgrad %s] max |poly - fine| / sum|terms|: gw %.2e gb %.2e" % (shape, err_w, err_b))
    assert err_w < 3e-5 and err_b < 3e-5
