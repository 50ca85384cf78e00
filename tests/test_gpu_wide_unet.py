"""GPU tests of the channel-blocked tensor-core convolution: U-Nets with 64-channel layers and concatenations of up to 128
channels (the doubled VoxelMorph, `--enc 32 64 64 64 --dec 64 64 64 64 64 32 32`, and nb_unet_features=16,
nb_unet_levels=3, unet_feat_mult=2).  Kernel level against F.conv3d in fp64 on the same bf16-rounded operands (1e-2 of
max|ref| for bf16 outputs, 1e-4 for fp32 outputs, as tests/test_gpu_tc.py); model level as tests/test_gpu_bf16_engine.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cases, ref_torch

from test_oracle import full_cfg

pytestmark = pytest.mark.gpu

DOUBLED = [[32, 64, 64, 64], [64, 64, 64, 64, 64, 32, 32]]


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def bf(x):
    return x.to(torch.bfloat16).float()


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


@pytest.fixture(scope="module")
def tc(cuda):
    import voxelmorph_b200 as v
    from voxelmorph_b200 import tc
    v._lib.load()
    return tc


def _fwd(tc, xa, xb, w, b, cout, kd, up, slope=0.2):
    """Forward as the engine runs it: one launch where it fits, else channel blocks."""
    ca, cb = xa.shape[-1], 0 if xb is None else xb.shape[-1]
    blocks = tc.conv_blocks(ca, cb, cout, kd)
    if blocks is None:
        wpk, cp = tc.pack_weights_t(w, variant="s")
        return tc.conv_fwd_t(xa, xb, wpk, cp, b, cout, kd, up=up, slope=slope)
    return tc.conv_fwd_blocked(xa, xb, blocks, tc.pack_weights_blocks(w, False, blocks), b, cout, kd, up=up, slope=slope)


def _dgrad(tc, gz, w, kd, slope=None, mask=None, split=None):
    cin = w.shape[1]
    blocks = tc.conv_blocks(gz.shape[-1], 0, cin, kd, split)
    if blocks is None:
        wpk, cp = tc.pack_weights_t(w, transposed=True, variant="s")
        return tc.conv_fwd_t(gz, None, wpk, cp, None, cin, kd, slope=slope, mask=mask, split=split)
    return tc.conv_fwd_blocked(gz, None, blocks, tc.pack_weights_blocks(w, True, blocks), None, cin, kd, slope=slope, mask=mask, split=split)


def _inputs(g, shape, Ca, Cb, up, kd):
    D, H, W = shape
    ashape = ((D // 2 if kd == 3 else D), H // 2, W // 2) if up else shape
    xa = bf(torch.randn((2, Ca) + ashape, generator=g))
    xb = bf(torch.randn((2, Cb) + shape, generator=g)) if Cb else None
    xin = F.interpolate(xa, scale_factor=(2 if kd == 3 else 1, 2, 2), mode="nearest") if up else xa
    if xb is not None:
        xin = torch.cat([xin, xb], dim=1)
    return xa, xb, xin


FWD = [
    # shape, Ca, Cb, up, Cout
    ((8, 16, 40), 32, 0, False, 64),      # enc1: one launch, 64 outputs
    ((8, 16, 40), 64, 0, False, 64),      # enc2/3, dec0: two 32-channel output blocks
    ((10, 12, 14), 64, 0, False, 64),     # ragged tiles
    ((8, 16, 40), 64, 64, True, 64),      # dec1-3: K blocks per source (128 -> 64)
    ((10, 12, 14), 64, 64, True, 64),
    ((8, 16, 40), 64, 32, True, 64),      # rem0 (96 -> 64)
    ((8, 16, 40), 64, 32, True, 32),      # feat_mult = 2 decoder (96 -> 32)
    ((8, 16, 24), 32, 16, True, 64),      # 48 -> 64: K groups 32 + 16 in 32-channel output blocks
    ((1, 32, 40), 32, 0, False, 64),      # 2-D
    ((1, 32, 40), 64, 0, False, 64),
    ((1, 32, 40), 64, 64, True, 64),
    ((1, 32, 40), 64, 32, True, 64),
    ((1, 32, 40), 64, 32, True, 32),
]


@pytest.mark.parametrize("shape,Ca,Cb,up,Cout", FWD)
def test_wide_forward(tc, cuda, shape, Ca, Cb, up, Cout):
    g = torch.Generator().manual_seed(Ca * 7 + Cb * 3 + Cout + shape[0])
    kd = 1 if shape[0] == 1 else 3
    xa, xb, xin = _inputs(g, shape, Ca, Cb, up, kd)
    w = bf(torch.randn((Cout, Ca + Cb, kd, 3, 3), generator=g) * 0.05)
    b = torch.randn(Cout, generator=g)
    ref = F.leaky_relu(F.conv3d(xin.double(), w.double(), b.double(), padding=(kd // 2, 1, 1)), 0.2)
    out = _fwd(tc, tc.to_ndhwc_bf16(xa.to(cuda)), None if xb is None else tc.to_ndhwc_bf16(xb.to(cuda)), w.to(cuda), b.to(cuda),
               Cout, kd, up)
    assert rel(tc.from_ndhwc(out).cpu(), ref) <= 1e-2


@pytest.mark.parametrize("kd", [3, 1])
def test_wide_masked_dgrad(tc, cuda, kd):
    g = torch.Generator().manual_seed(21 + kd)
    shape = (6, 16, 40) if kd == 3 else (1, 24, 40)
    x = torch.randn((1, 64) + shape, generator=g, dtype=torch.float64, requires_grad=True)
    w = bf(torch.randn((64, 64, kd, 3, 3), generator=g) * 0.05)
    gy = bf(torch.randn((1, 64) + shape, generator=g))
    F.conv3d(x, w.double(), None, padding=(kd // 2, 1, 1)).backward(gy.double())
    below = bf(torch.randn((1, 64) + shape, generator=g))
    ref = x.grad * torch.where(below.double() < 0, 0.2, 1.0)
    out = _dgrad(tc, tc.to_ndhwc_bf16(gy.to(cuda)), w.to(cuda), kd, slope=0.2, mask=tc.to_ndhwc_bf16(below.to(cuda)))
    assert rel(tc.from_ndhwc(out).cpu(), ref) <= 1e-2


@pytest.mark.parametrize("kd,Cin,split,Cout", [(3, 128, 64, 64), (3, 96, 64, 64), (3, 96, 64, 32), (1, 128, 64, 64), (1, 96, 64, 64)])
def test_wide_split_dgrad(tc, cuda, kd, Cin, split, Cout):
    g = torch.Generator().manual_seed(Cin + Cout + kd)
    shape = (6, 16, 24) if kd == 3 else (1, 24, 40)
    x = torch.randn((1, Cin) + shape, generator=g, dtype=torch.float64, requires_grad=True)
    w = bf(torch.randn((Cout, Cin, kd, 3, 3), generator=g) * 0.05)
    gy = bf(torch.randn((1, Cout) + shape, generator=g))
    F.conv3d(x, w.double(), None, padding=(kd // 2, 1, 1)).backward(gy.double())
    oa, ob = _dgrad(tc, tc.to_ndhwc_bf16(gy.to(cuda)), w.to(cuda), kd, split=split)
    assert rel(tc.from_ndhwc(oa).cpu(), x.grad[:, :split]) <= 1e-2
    assert rel(tc.from_ndhwc(ob).cpu(), x.grad[:, split:]) <= 1e-2


WG = [
    # shape, Ca, Cb, up, Cout
    ((8, 16, 40), 32, 0, False, 64),
    ((8, 16, 40), 64, 0, False, 64),
    ((10, 12, 14), 64, 64, True, 64),
    ((8, 16, 40), 64, 32, True, 64),
    ((8, 16, 40), 64, 32, True, 32),
    ((8, 16, 40), 64, 0, False, 32),
    ((1, 32, 40), 64, 64, True, 64),
]


def _wgrad_ref(xin, gz, Cout, kd):
    w = torch.zeros((Cout, xin.shape[1], kd, 3, 3), dtype=torch.float64, requires_grad=True)
    b = torch.zeros(Cout, dtype=torch.float64, requires_grad=True)
    F.conv3d(xin.double(), w, b, padding=(kd // 2, 1, 1)).backward(gz.double())
    return w.grad, b.grad


@pytest.mark.parametrize("shape,Ca,Cb,up,Cout", WG)
def test_wide_wgrad(tc, cuda, shape, Ca, Cb, up, Cout):
    """Deferred weight gradient of 64-channel operands (32-channel slices), both into fresh tensors and accumulated into an
    existing gradient (the FusedAdam flat-gradient views)."""
    g = torch.Generator().manual_seed(31 + Ca + Cb + Cout)
    kd = 1 if shape[0] == 1 else 3
    xa, xb, xin = _inputs(g, shape, Ca, Cb, up, kd)
    gz = bf(torch.randn((2, Cout) + shape, generator=g))
    rw, rb = _wgrad_ref(xin, gz, Cout, kd)
    xa_d, xb_d, gz_d = tc.to_ndhwc_bf16(xa.to(cuda)), None if xb is None else tc.to_ndhwc_bf16(xb.to(cuda)), tc.to_ndhwc_bf16(gz.to(cuda))
    batch = tc.WgradBatch.get(cuda)
    batch.reset()
    gw, gb = tc.conv_wgrad(xa_d, xb_d, gz_d, Ca + Cb, Cout, kd, up=up, batch=batch)
    w0 = torch.randn((Cout, Ca + Cb, kd, 3, 3), generator=g)
    b0 = torch.randn(Cout, generator=g)
    ow, ob = w0.to(cuda), b0.to(cuda)
    tc.conv_wgrad(xa_d, xb_d, gz_d, Ca + Cb, Cout, kd, up=up, out_w=ow, out_b=ob, batch=batch)
    batch.flush()
    assert rel(gw.cpu(), rw) <= 1e-4 and rel(gb.cpu(), rb) <= 1e-4
    assert rel(ow.cpu() - w0, rw) <= 1e-4 and rel(ob.cpu() - b0, rb) <= 1e-4


def test_wide_wgrad_flushes_mid_pass(tc, cuda):
    """A workspace that holds one 128 x 64 layer's partials: the second layer's add flushes the first mid-pass."""
    g = torch.Generator().manual_seed(41)
    shape, kd = (8, 16, 24), 3
    layers = []
    for Ca, Cb, up, Cout in ((64, 64, True, 64), (64, 64, True, 64), (64, 0, False, 64), (64, 32, True, 32)):
        xa, xb, xin = _inputs(g, shape, Ca, Cb, up, kd)
        gz = bf(torch.randn((2, Cout) + shape, generator=g))
        layers.append((xa, xb, xin, gz, Ca + Cb, Cout, up))
    lib = tc._lib.load()

    class Small(tc.WgradBatch):
        WORK_BYTES = int(lib.vxm_conv3d_tc_wgrad2_partial_bytes(3)) * 4      # the bound of one 128 x 64 layer (8 slice pairs)

    batch = Small(cuda)
    flushes = []
    real_flush = batch.flush
    batch.flush = lambda: (flushes.append(batch.n.value), real_flush())
    outs = []
    for xa, xb, xin, gz, cin, cout, up in layers:
        outs.append(tc.conv_wgrad(tc.to_ndhwc_bf16(xa.to(cuda)), None if xb is None else tc.to_ndhwc_bf16(xb.to(cuda)),
                                  tc.to_ndhwc_bf16(gz.to(cuda)), cin, cout, kd, up=up, batch=batch))
    real_flush()
    assert any(n > 0 for n in flushes), flushes        # at least one flush with reductions pending, before the last add
    for (xa, xb, xin, gz, cin, cout, up), (gw, gb) in zip(layers, outs):
        rw, rb = _wgrad_ref(xin, gz, cout, kd)
        assert rel(gw.cpu(), rw) <= 1e-4 and rel(gb.cpu(), rb) <= 1e-4


@pytest.mark.parametrize("mode", ["fwd", "cat", "dgrad", "split"])
def test_wide_tma_and_lean_epilogue_match(tc, cuda, monkeypatch, mode):
    """The blocked launches give bit-identical results with and without TMA staging and the specialised epilogues."""
    g = torch.Generator().manual_seed(51)
    shape = (10, 20, 70)
    x = tc.to_ndhwc_bf16(torch.randn((2, 64) + shape, generator=g).to(cuda))
    xh = tc.to_ndhwc_bf16(torch.randn((2, 64) + (6, 10, 36), generator=g).to(cuda))
    xs = tc.to_ndhwc_bf16(torch.randn((2, 64) + (12, 20, 72), generator=g).to(cuda))
    if mode == "fwd":
        w, b = torch.randn((64, 64, 3, 3, 3), generator=g).to(cuda) * 0.05, torch.randn(64, generator=g).to(cuda)
        run = lambda: _fwd(tc, x, None, w, b, 64, 3, False)
    elif mode == "cat":
        w, b = torch.randn((64, 128, 3, 3, 3), generator=g).to(cuda) * 0.05, torch.randn(64, generator=g).to(cuda)
        run = lambda: _fwd(tc, xh, xs, w, b, 64, 3, True)
    elif mode == "dgrad":
        w = torch.randn((64, 64, 3, 3, 3), generator=g).to(cuda) * 0.05
        m = tc.to_ndhwc_bf16(torch.randn((2, 64) + shape, generator=g).to(cuda))
        run = lambda: _dgrad(tc, x, w, 3, slope=0.2, mask=m)
    else:
        w = torch.randn((64, 128, 3, 3, 3), generator=g).to(cuda) * 0.05
        run = lambda: torch.cat(_dgrad(tc, x, w, 3, split=64), dim=-1)
    outs = {}
    for tma in ("1", "0"):
        for epi in ("1", "0"):
            monkeypatch.setenv("VXM_B200_TMA", tma)
            monkeypatch.setenv("VXM_B200_TCS_EPI", epi)
            outs[(tma, epi)] = run().float().cpu()
    ref = outs[("0", "0")]
    assert torch.isfinite(ref).all() and float(ref.abs().max()) > 0
    for k, v in outs.items():
        assert torch.equal(v, ref), k


# ---- model level ------------------------------------------------------------------------------------------------------

WIDE_VARIANTS = {
    "doubled3d": dict(inshape=(32, 32, 48), nb_unet_features=DOUBLED),
    "featmult2_3d": dict(inshape=(32, 32, 48), nb_unet_features=16, nb_unet_levels=3, unet_feat_mult=2),
    "doubled2d": dict(inshape=(64, 64), nb_unet_features=DOUBLED),
    "doubled_bidir2d": dict(inshape=(32, 48), nb_unet_features=DOUBLED, bidir=True, int_steps=5),
    "doubled_halfres3d": dict(inshape=(16, 16, 32), nb_unet_features=DOUBLED, unet_half_res=True),
}


@pytest.fixture()
def vxm_env(cuda, monkeypatch):
    import voxelmorph_b200 as v
    v._lib.load()

    def use(engine):
        monkeypatch.setenv("VXM_B200_CONV_ENGINE", engine)
        return v
    yield use
    ref_torch.emulate_bf16(False)


@pytest.mark.parametrize("name", sorted(WIDE_VARIANTS))
def test_wide_bf16_forward_backward(vxm_env, cuda, name):
    vxm = vxm_env("bf16")
    kw = WIDE_VARIANTS[name]
    cfg = full_cfg(kw)
    model = vxm.networks.VxmDense(**kw)
    sd = ref_torch.init_state_dict(cfg, seed=77, flow_std=2e-2)
    model.load_state_dict(sd, strict=False)
    model.to(cuda).train()
    s, tr = cases.volume_pair(93, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    out = model(S, T)
    flow = out[-1]
    gen = torch.Generator().manual_seed(1)
    gflow = torch.randn(flow.shape, generator=gen)
    gy = torch.randn(out[0].shape, generator=gen)
    ((flow * gflow.to(cuda)).sum() + (out[0] * gy.to(cuda)).sum()).backward()
    ref_torch.emulate_bf16(True)
    sdc = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    outc = ref_torch.vxm_forward(sdc, cfg, t(s), t(tr))
    ((outc[-1] * gflow).sum() + (outc[0] * gy).sum()).backward()
    ref_torch.emulate_bf16(False)
    e_flow, e_moved = rel(flow.detach().cpu(), outc[-1].detach()), rel(out[0].detach().cpu(), outc[0].detach())
    errs = sorted(((rel(p.grad.cpu(), sdc[k].grad), k) for k, p in model.named_parameters()), reverse=True)
    print("\n[%s] vs bf16-emulating oracle: flow %.2e moved %.2e; worst gradients %s"
          % (name, e_flow, e_moved, ", ".join("%s %.2e" % (k, e) for e, k in errs[:3])))
    assert e_flow <= 1e-2 and e_moved <= 1e-2
    assert errs[0][0] <= 1.5e-1, (name, errs[:3])
    assert np.median([e for e, _ in errs]) <= 5e-2


@pytest.mark.parametrize("name", sorted(WIDE_VARIANTS))
def test_wide_bf16x3_within_reference_tolerance(vxm_env, cuda, name):
    vxm = vxm_env("bf16x3")
    kw = WIDE_VARIANTS[name]
    cfg = full_cfg(kw)
    model = vxm.networks.VxmDense(**kw)
    sd = ref_torch.init_state_dict(cfg, seed=1234, flow_std=2e-2)
    model.load_state_dict(sd, strict=False)
    model.to(cuda).eval()
    s, tr = cases.volume_pair(91, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    with torch.no_grad():
        out = model(S, T)
        ref = ref_torch.vxm_forward(sd, cfg, t(s), t(tr))
    errs = [rel(y.cpu(), r) for y, r in zip(out, ref)]
    print("\n[%s] bf16x3 vs fp32 oracle: %s" % (name, " ".join("%.2e" % e for e in errs)))
    assert max(errs) <= 1e-4, (name, errs)


def test_wide_bf16x3_matches_reference_golden(vxm_env, cuda, golden):
    """The doubled model on the bf16x3 engine against the unmodified reference's outputs (oracle/make_golden_wide.py)."""
    vxm = vxm_env("bf16x3")
    g = golden("wide")
    kw = dict(inshape=(16, 16, 32), nb_unet_features=DOUBLED)
    cfg = full_cfg(kw)
    model = vxm.networks.VxmDense(**kw)
    model.load_state_dict(ref_torch.init_state_dict(cfg, seed=1234, flow_std=2e-2), strict=False)
    model.to(cuda).eval()
    s, tr = cases.volume_pair(91, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    with torch.no_grad():
        out = model(S, T)
        reg = model(S, T, registration=True)
    for i, y in enumerate(out):
        assert rel(y.cpu(), t(g["train%d" % i])) <= 1e-4, i
    assert rel(reg[1].cpu(), t(g["reg_flow"])) <= 1e-4
    model.train()
    y, flow = model(S, T)
    loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
    loss.backward()
    assert abs(float(loss) - float(g["loss"])) <= 1e-4 * abs(float(g["loss"]))
    params = dict(model.named_parameters())
    for k in [k[5:] for k in g if k.startswith("grad/")]:
        assert rel(params[k].grad.cpu(), t(g["grad/" + k])) <= 5e-2, k     # backward on bf16 operands


def test_wide_graphed_train_step_matches_eager(vxm_env, cuda):
    vxm = vxm_env("bf16")
    from voxelmorph_b200.trainer import GraphedTrainStep
    kw = dict(inshape=(32, 32, 32), nb_unet_features=DOUBLED)
    cfg = full_cfg(kw)
    s, tr = cases.volume_pair(95, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)

    def make():
        m = vxm.networks.VxmDense(**kw)
        m.load_state_dict(ref_torch.init_state_dict(cfg, seed=5, flow_std=2e-2), strict=False)
        m.to(cuda).train()
        return m, vxm.optim.FusedAdam(m.parameters(), lr=1e-3)

    m1, o1 = make()
    eager = []
    for _ in range(3):
        o1.zero_grad()
        y, flow = m1(S, T)
        loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
        loss.backward()
        o1.step()
        eager.append(float(loss))
    m2, o2 = make()
    step = GraphedTrainStep(m2, o2, warmup=3).capture(S, T)
    graphed = [float(step(S, T)) for _ in range(3)]
    for i in range(3):
        assert abs(graphed[i] - eager[i]) <= 2e-3 * abs(eager[i]), (i, graphed, eager)
    assert int(o2.step_dev.item()) == 3


@pytest.mark.parametrize("engine", ["bf16", "bf16x3"])
def test_wide_multi_tile_step_vs_oracle(cuda, monkeypatch, engine):
    """The doubled model at a size with many tiles and depth chunks per layer: forward, loss and gradients vs the oracle."""
    import voxelmorph_b200 as vxm
    vxm._lib.load()
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", engine)
    kw = dict(inshape=(64, 96, 112), nb_unet_features=DOUBLED)
    cfg = full_cfg(kw)
    sd = ref_torch.init_state_dict(cfg, seed=1234, flow_std=1e-2)
    model = vxm.networks.VxmDense(**kw)
    model.load_state_dict(sd, strict=False)
    model.to(cuda).train()
    s, tr = cases.volume_pair(97, kw["inshape"], sigma=2.0)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    y, flow = model(S, T)
    loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
    loss.backward()
    torch.cuda.synchronize()
    sdc = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    yc, fc = ref_torch.vxm_forward(sdc, cfg, t(s), t(tr))
    lc = ref_torch.ncc_loss(t(tr), yc) + 0.01 * ref_torch.grad_loss(fc, "l2", 2)
    lc.backward()
    e_flow, e_moved = rel(flow.detach().cpu(), fc.detach()), rel(y.detach().cpu(), yc.detach())
    e_loss = abs(float(loss) - float(lc)) / abs(float(lc))
    gerr = sorted(rel(p.grad.cpu(), sdc[k].grad) for k, p in model.named_parameters())
    print("\n[64x96x112 doubled, %s] flow %.2e moved %.2e loss %.2e | gradient rel err: median %.2e max %.2e"
          % (engine, e_flow, e_moved, e_loss, gerr[len(gerr) // 2], gerr[-1]))
    tol = dict(bf16=(2e-2, 1e-3, 1e-4), bf16x3=(1e-4, 1e-4, 1e-5))[engine]
    assert e_flow <= tol[0] and e_moved <= tol[1] and e_loss <= tol[2]
    assert gerr[len(gerr) // 2] <= 2e-2 and gerr[-1] <= 5e-2


@pytest.mark.parametrize("feats", [
    [[4, 8, 8, 8], [8, 8, 8, 8, 8, 4, 4]],
    [[16, 24, 24, 24], [24, 24, 24, 24, 24, 16, 16]],
    [[32, 128, 64, 64], [64, 64, 64, 64, 64, 32, 32]],
    [[16, 32, 32, 32], [32, 16, 32, 32, 32, 16, 16]],          # a 16 + 32 concatenation: no kernel takes it
])
def test_wide_refusals_name_the_fp32_engine(vxm_env, cuda, feats):
    vxm = vxm_env("bf16")
    m = vxm.networks.VxmDense((16, 16, 16), nb_unet_features=feats).to(cuda)
    with pytest.raises(vxm._lib.VxmError, match="VXM_B200_CONV_ENGINE=f32"):
        m(torch.rand(1, 1, 16, 16, 16, device=cuda), torch.rand(1, 1, 16, 16, 16, device=cuda))
