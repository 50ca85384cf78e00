"""The polyphase concat-layer launches (csrc/conv3d_tc_s.cu, conv_tcs_kernel PD): the forward of a (32 upsampled + 16) -> 32
layer with the two kd taps that read the same coarse slice merged, and the coarse dgrad of the upsampled source (kd and kh
taps merged, w' pairs and the LeakyReLU derivative in the epilogue).  With weights and inputs quantised so that every merged
tap and every fp32 sum is exact, the bf16 results equal torch's fp64 result rounded to bf16.  With ordinary weights they
match fp64 on the merged weights rounded to bf16 as the packer rounds them.  TMA and cp.async staging of the forward agree
bit for bit.  The engine with the polyphase forms switched on tracks the engine with them off (VXM_B200_POLYPHASE=0), and
its graphed step matches its eager step."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SLOPE = 0.25          # exact in the epilogue, so that the quantised forward is exact up to the final bf16 rounding


def rel_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.fixture(scope="module")
def tc(cuda):
    import voxelmorph_b200 as v
    from voxelmorph_b200 import tc
    v._lib.load()
    return tc


def quant(shape, g, scale):
    """small integers times a power of two: bf16-exact, and so are their pairwise sums and the fp32 sums below"""
    return torch.randint(-8, 9, shape, generator=g).double() * scale


def bf(t):
    return t.to(torch.bfloat16).double()


def ref_forward(xc, xs, w, b, merged_bf16):
    """fp64 forward of the concat layer; merged_bf16: the upsampled group's merged kd taps rounded to bf16 as packed (w fp32)."""
    wa, wb = w[:, :32], w[:, 32:]
    q = bf if merged_bf16 else (lambda t: t.double())
    even = torch.stack([q(wa[:, :, 0]), q(wa[:, :, 1] + wa[:, :, 2])], 2)
    odd = torch.stack([q(wa[:, :, 0] + wa[:, :, 1]), q(wa[:, :, 2])], 2)
    xa = xc.repeat_interleave(2, 3).repeat_interleave(2, 4)          # (h, w) upsampled, d coarse
    ye = F.conv3d(F.pad(xa, (0, 0, 0, 0, 1, 0)), even, padding=(0, 1, 1))
    yo = F.conv3d(F.pad(xa, (0, 0, 0, 0, 0, 1)), odd, padding=(0, 1, 1))
    y = torch.stack([ye, yo], 3).flatten(2, 3) + F.conv3d(xs, q(wb), b.double(), padding=1)
    return F.leaky_relu(y, SLOPE)


def ref_dgrad_coarse(gz, w, act, merged_bf16):
    """fp64 gradient w.r.t. the coarse source's pre-activation: (B, 32, D / 2, H / 2, W / 2).  The packer sums the d taps
    in the outer loop and the h taps in the inner one."""
    t = w[:, :32].transpose(0, 1).flip(2, 3, 4)             # fp32, (32 source, 32 gradient, 3, 3, 3)
    kk = torch.zeros((32, 32, 4, 4, 3))
    for a in range(4):                                      # merged (T0, T0 + T1, T1 + T2, T2) along d and along h
        ta = [i for i in (a - 1, a) if 0 <= i <= 2]
        for b in range(4):
            ub = [i for i in (b - 1, b) if 0 <= i <= 2]
            acc = torch.zeros((32, 32, 3))
            for i in ta:
                for j in ub:
                    acc = acc + t[:, :, i, j]
            kk[:, :, a, b] = acc
    kk = bf(kk) if merged_bf16 else kk.double()
    g = F.conv3d(F.pad(gz, (1, 1, 1, 1, 1, 1)), kk, stride=(2, 2, 1))          # (B, 32, D / 2, H / 2, W), w fine
    g = g.view(*g.shape[:4], -1, 2).sum(-1)                                      # w' pairs
    return torch.where(act < 0, g * SLOPE, g)


SHAPES = [
    # 20 tiles of the forward on the H100's 132 SMs: depth chunks of 3 slices (chunks start on odd slices); the coarse dgrad
    # runs chunks of one coarse slice.  40 rows: 20 coarse rows, ragged for the dgrad's 8-row tiles
    (2, (18, 40, 30)),
    (2, (10, 20, 46)),      # two column tiles, the second ragged
    (1, (4, 6, 62)),        # fewer rows than one 8-row tile
]


@pytest.mark.parametrize("B,shape", SHAPES)
@pytest.mark.parametrize("quantised", [True, False])
def test_poly_forward_vs_fp64(tc, cuda, monkeypatch, B, shape, quantised):
    g = torch.Generator().manual_seed(11 + B)
    D, H, W = shape
    if quantised:
        xc, xs = quant((B, 32, D // 2, H // 2, W // 2), g, 1 / 16), quant((B, 16) + shape, g, 1 / 16)
        w, b = quant((32, 48, 3, 3, 3), g, 2.0 ** -6).float(), quant((32,), g, 2.0 ** -6).float()
    else:
        xc, xs = bf(torch.randn((B, 32, D // 2, H // 2, W // 2), generator=g)), bf(torch.randn((B, 16) + shape, generator=g))
        w, b = torch.randn((32, 48, 3, 3, 3), generator=g) * 0.05, torch.randn(32, generator=g) * 0.1
    wpk = tc.pack_weights_poly(w.to(cuda), 1, 32)
    xa_d, xs_d, b_d = tc.to_ndhwc_bf16(xc.float().to(cuda)), tc.to_ndhwc_bf16(xs.float().to(cuda)), b.to(cuda)
    outs = {}
    for tma in ("1", "0"):
        monkeypatch.setenv("VXM_B200_TMA", tma)
        outs[tma] = tc.from_ndhwc(tc.conv_fwd_poly(xa_d, xs_d, wpk, b_d, 32, SLOPE)).cpu()
    assert torch.equal(outs["1"], outs["0"])
    out = outs["1"]
    ref = ref_forward(xc, xs, w, b, merged_bf16=True)
    if quantised:
        assert ref_forward(xc, xs, w, b, merged_bf16=False).equal(ref)       # the merged taps are exact
        err = rel_err(out, bf(ref))                                          # exact fp32 sums: only the output rounding
        print("\n[poly fwd quantised %s] max rel diff to bf16(fp64): %.2e" % (shape, err))
        assert err <= 1e-5
    else:
        err = rel_err(out, ref)
        print("\n[poly fwd %s] max rel diff to fp64 (merged taps in bf16): %.2e" % (shape, err))
        assert err <= 5e-3                                                   # bf16 output rounding
    # the 27-tap path over the duplicated voxels computes the same function
    wpk_t, cp = tc.pack_weights_t(w.to(cuda), variant="s")
    old = tc.from_ndhwc(tc.conv_fwd_t(xa_d, xs_d, wpk_t, cp, b_d, 32, 3, up=True, slope=SLOPE)).cpu()
    assert rel_err(out, old) <= (1e-5 if quantised else 1e-2)


@pytest.mark.parametrize("B,shape", SHAPES)
@pytest.mark.parametrize("quantised", [True, False])
def test_poly_dgrad_vs_fp64(tc, cuda, B, shape, quantised):
    g = torch.Generator().manual_seed(23 + B)
    D, H, W = shape
    for cb in (16, 32):                                     # rem0 (32 + 16) and the decoder layers (32 + 32)
        if quantised:
            gz, w = quant((B, 32) + shape, g, 1 / 16), quant((32, 32 + cb, 3, 3, 3), g, 2.0 ** -6).float()
        else:
            gz, w = bf(torch.randn((B, 32) + shape, generator=g)), torch.randn((32, 32 + cb, 3, 3, 3), generator=g) * 0.05
        act = bf(torch.randn((B, 32, D // 2, H // 2, W // 2), generator=g))
        wpk = tc.pack_weights_poly(w.to(cuda), 2, 32)
        out = tc.from_ndhwc(tc.dgrad_poly(tc.to_ndhwc_bf16(gz.float().to(cuda)), wpk, tc.to_ndhwc_bf16(act.float().to(cuda)),
                                          SLOPE)).cpu()
        ref = ref_dgrad_coarse(gz, w, act, merged_bf16=True)
        if quantised:
            assert ref_dgrad_coarse(gz, w, act, merged_bf16=False).equal(ref)   # the merged taps are exact
            # the 27-tap gradient of the upsampled tensor, summed over the 8 children: the same function
            gup = F.conv_transpose3d(gz, w[:, :32].double(), padding=1).view(B, 32, D // 2, 2, H // 2, 2, W // 2, 2).sum((3, 5, 7))
            assert torch.where(act < 0, gup * SLOPE, gup).equal(ref)
            err = rel_err(out, bf(ref))
            print("\n[poly dgrad 32+%d quantised %s] max rel diff to bf16(fp64): %.2e" % (cb, shape, err))
            assert err <= 1e-5
        else:
            err = rel_err(out, ref)
            print("\n[poly dgrad 32+%d %s] max rel diff to fp64 (merged taps in bf16): %.2e" % (cb, shape, err))
            assert err <= 5e-3


def test_skip_part_dgrad_matches_split_dgrad(tc, cuda):
    """The skip part of the polyphase dgrad (a fine launch on the skip channels' block of the transposed weight) against the
    second output of the single split dgrad it replaces: the same products in the same order into fp32 (the kw-stacked N
    only sets how many output columns one wgmma computes), so the same bits."""
    g = torch.Generator().manual_seed(5)
    gz = torch.randn((2, 32, 10, 20, 46), generator=g)
    w = torch.randn((32, 48, 3, 3, 3), generator=g) * 0.05
    gz_d = tc.to_ndhwc_bf16(gz.to(cuda))
    packs = tc.pack_weights_blocks(w.to(cuda), True, (((2, 0, 32),), ((32, 16, 0, 0),)))
    wpk, coutp = packs[0, 0]
    skip = tc.conv_fwd_t(gz_d, None, wpk, (coutp, "s"), None, 16, 3)
    wpk_t, cp = tc.pack_weights_t(w.to(cuda), transposed=True, variant="s")
    _, old = tc.conv_fwd_t(gz_d, None, wpk_t, cp, None, 48, 3, split=32)
    assert torch.equal(skip, old)


def test_engine_polyphase_on_vs_off(cuda, monkeypatch):
    """The default 3-D model, switch on against switch off: forward, flow and every parameter gradient."""
    import voxelmorph_b200 as vxm
    from oracle import cases
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "bf16")
    shape = (32, 32, 48)
    s, t = cases.volume_pair(7, shape, sigma=1.5)
    S, T = torch.from_numpy(np.ascontiguousarray(s)).to(cuda), torch.from_numpy(np.ascontiguousarray(t)).to(cuda)
    res = {}
    for poly in ("1", "0"):
        monkeypatch.setenv("VXM_B200_POLYPHASE", poly)
        torch.manual_seed(3)
        model = vxm.networks.VxmDense(inshape=shape).to(cuda).train()
        with torch.no_grad():
            model.flow.weight.normal_(0, 2e-2)
        from voxelmorph_b200 import engine_bf16
        npoly = sum(1 for L in engine_bf16._walk(model) if isinstance(L, engine_bf16._Layer) and L.dgrad_skip is not None)
        assert npoly == (4 if poly == "1" else 0), npoly        # rem0 and dec1..dec3
        y, flow = model(S, T)
        loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
        loss.backward()
        torch.cuda.synchronize()
        res[poly] = (y.detach().cpu(), flow.detach().cpu(), float(loss),
                     {n: p.grad.detach().cpu().clone() for n, p in model.named_parameters() if p.grad is not None})
    y1, f1, l1, g1 = res["1"]
    y0, f0, l0, g0 = res["0"]
    e_y, e_flow, e_loss = rel_err(y1, y0), rel_err(f1, f0), abs(l1 - l0) / abs(l0)
    assert set(g1) == set(g0)
    errs = sorted(((rel_err(g1[n], g0[n]), n) for n in g0), reverse=True)
    print("\n[polyphase on vs off] moved %.2e flow %.2e loss %.2e | gradients: max %.2e (%s), median %.2e"
          % (e_y, e_flow, e_loss, errs[0][0], errs[0][1], float(np.median([e for e, _ in errs]))))
    assert e_flow <= 1e-2 and e_y <= 1e-2 and e_loss <= 1e-2
    assert errs[0][0] <= 1.5e-1 and np.median([e for e, _ in errs]) <= 5e-2


def test_graphed_step_refreshes_polyphase_operands(cuda, monkeypatch):
    """The captured step repacks the polyphase operands from the current parameters: after each replay, the forward and
    coarse-dgrad operands of every polyphase layer equal a fresh pack of the weights that replay ran with (the ones
    before its Adam update), bit for bit, and they change from replay to replay."""
    import voxelmorph_b200 as vxm
    from oracle import cases, ref_torch
    from test_oracle import full_cfg
    from voxelmorph_b200 import engine_bf16, tc
    from voxelmorph_b200.trainer import GraphedTrainStep
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "bf16")
    monkeypatch.setenv("VXM_B200_POLYPHASE", "1")
    kw = dict(inshape=(32, 32, 32))
    cfg = full_cfg(kw)
    s, t = cases.volume_pair(95, kw["inshape"], sigma=1.5)
    S, T = torch.from_numpy(np.ascontiguousarray(s)).to(cuda), torch.from_numpy(np.ascontiguousarray(t)).to(cuda)
    m = vxm.networks.VxmDense(**kw)
    m.load_state_dict(ref_torch.init_state_dict(cfg, seed=5, flow_std=2e-2), strict=False)
    m.to(cuda).train()
    step = GraphedTrainStep(m, vxm.optim.FusedAdam(m.parameters(), lr=1e-2), warmup=3).capture(S, T)
    plan = m.__dict__["_vxm_pack_plan"]
    layers = [L for L in plan.layers if L.dgrad_skip is not None]
    assert len(layers) == 4 and sum(1 for L in layers if L.fwd[0] == "poly") == 1      # rem0 forward; rem0, dec1..dec3 dgrad
    last = None
    for _ in range(3):
        before = [L.w.detach().clone() for L in layers]
        step(S, T)
        torch.cuda.synchronize()
        packs = []
        for L, w in zip(layers, before):
            for form, pk in ((L.fwd, L.pk_fwd), (L.dgrad, L.pk_dgrad)):
                if form[0] == "poly":
                    assert torch.equal(pk[0, 0][0], tc.pack_weights_poly(w, form[1], form[2])), (L.cout, L.ca, L.cb, form)
                    packs.append(pk[0, 0][0].clone())
        if last is not None:
            assert all(not torch.equal(a, b) for a, b in zip(packs, last))
        last = packs
