"""GPU tests of the tensor-core (bf16) U-Net engine: Unet + flow head forward and the hand-written backward against the
CPU oracle with bf16 storage emulated at the same points (oracle/ref_torch.emulate_bf16), and the measured deviation from
the pure-fp32 oracle (reported; bf16 operands cannot meet the 1e-4 parity the fp32 engine meets)."""
import numpy as np
import pytest
import torch

from oracle import cases, ref_torch

from test_oracle import full_cfg

pytestmark = pytest.mark.gpu

F16 = [[16, 16, 16, 16], [16, 16, 16, 16, 16, 16, 16]]
BF16_VARIANTS = {
    "default3d": dict(inshape=(32, 32, 48)),
    "feat16_3d": dict(inshape=(16, 32, 32), nb_unet_features=F16),
    "halfres3d": dict(inshape=(16, 16, 32), unet_half_res=True),
    "ncpl2_3d": dict(inshape=(16, 16, 16), nb_unet_features=16, nb_unet_levels=3, unet_feat_mult=1, nb_unet_conv_per_level=2),
    "config1_2d": dict(inshape=(64, 64), int_steps=0),
    "bidir2d": dict(inshape=(32, 48), bidir=True, int_steps=5),
}


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.fixture()
def vxm_bf16(cuda, monkeypatch):
    import voxelmorph_b200 as v
    v._lib.load()
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "bf16")
    yield v
    ref_torch.emulate_bf16(False)


@pytest.mark.parametrize("name", sorted(BF16_VARIANTS))
def test_bf16_engine_forward_backward(vxm_bf16, cuda, name):
    vxm = vxm_bf16
    kw = BF16_VARIANTS[name]
    cfg = full_cfg(kw)
    model = vxm.networks.VxmDense(**kw)
    sd = ref_torch.init_state_dict(cfg, seed=77, flow_std=2e-2)
    model.load_state_dict(sd, strict=False)
    model.to(cuda).train()
    shape = kw["inshape"]
    s, tr = cases.volume_pair(93, shape, sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    out = model(S, T)
    flow = out[-1]
    gen = torch.Generator().manual_seed(1)
    gflow = torch.randn(flow.shape, generator=gen)
    gy = torch.randn(out[0].shape, generator=gen)
    loss = (flow * gflow.to(cuda)).sum() + (out[0] * gy.to(cuda)).sum()
    loss.backward()
    # oracle with bf16 storage emulation
    ref_torch.emulate_bf16(True)
    sdc = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    outc = ref_torch.vxm_forward(sdc, cfg, t(s), t(tr))
    ((outc[-1] * gflow).sum() + (outc[0] * gy).sum()).backward()
    ref_torch.emulate_bf16(False)
    with torch.no_grad():
        out32 = ref_torch.vxm_forward(sd, cfg, t(s), t(tr))
    e_flow, e_moved = rel(flow.detach().cpu(), outc[-1].detach()), rel(out[0].detach().cpu(), outc[0].detach())
    d_flow, d_moved = rel(flow.detach().cpu(), out32[-1]), rel(out[0].detach().cpu(), out32[0])
    print("\n[%s] vs bf16-emulating oracle: flow %.2e moved %.2e | vs fp32 oracle: flow %.2e moved %.2e"
          % (name, e_flow, e_moved, d_flow, d_moved))
    assert e_flow <= 1e-2 and e_moved <= 1e-2      # measured <= 5e-3 (DESIGN 4.3)
    assert d_flow <= 2e-2 and d_moved <= 2e-2      # measured <= 1e-2 vs the pure fp32 oracle
    errs = sorted(((rel(p.grad.cpu(), sdc[k].grad), k) for k, p in model.named_parameters()), reverse=True)
    print("[%s] worst parameter-gradient rel errs vs emulating oracle: %s" % (name, ", ".join("%s %.2e" % (k, e) for e, k in errs[:3])))
    # bf16 gradient storage costs ~0.4% per layer; the tiny deepest levels (a handful of voxels) are the noisiest
    assert errs[0][0] <= 1.5e-1, (name, errs[:3])
    assert np.median([e for e, _ in errs]) <= 5e-2


def test_bf16_engine_train_step_tracks_fp32(vxm_bf16, cuda, golden):
    """One full training step (NCC + Grad, Adam) in bf16 mode lands within 1e-2 of the fp32 reference loss."""
    vxm = vxm_bf16
    g = golden("vxmdense")
    kw = dict(inshape=(32, 32, 48))
    cfg = full_cfg(kw)
    model = vxm.networks.VxmDense(**kw)
    model.load_state_dict(ref_torch.init_state_dict(cfg, seed=1234, flow_std=2e-2), strict=False)
    model.to(cuda).train()
    s, tr = cases.volume_pair(91, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4)
    opt.zero_grad()
    y, flow = model(S, T)
    loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
    loss.backward()
    opt.step()
    ref = float(g["default3d/loss"])
    assert abs(float(loss.item()) - ref) <= 1e-2 * abs(ref)
    # second step exercises the refreshed packed weights
    opt.zero_grad()
    y, flow = model(S, T)
    loss2 = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
    loss2.backward()
    opt.step()
    assert np.isfinite(float(loss2.item()))


def test_bf16_engine_rejects_unsupported_shapes(vxm_bf16, cuda):
    vxm = vxm_bf16
    m = vxm.networks.VxmDense((16, 16, 16), nb_unet_features=[[4, 8, 8, 8], [8, 8, 8, 8, 8, 4, 4]]).to(cuda)
    with pytest.raises(vxm._lib.VxmError, match="VXM_B200_CONV_ENGINE=f32"):
        m(torch.rand(1, 1, 16, 16, 16, device=cuda), torch.rand(1, 1, 16, 16, 16, device=cuda))


def test_graphed_train_step_matches_eager(vxm_bf16, cuda):
    """The CUDA-graph replay of the whole step produces the same loss sequence / parameters as eager launches."""
    vxm = vxm_bf16
    from voxelmorph_b200.trainer import GraphedTrainStep
    kw = dict(inshape=(32, 32, 32))
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
    for _ in range(6):
        o1.zero_grad()
        y, flow = m1(S, T)
        loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
        loss.backward()
        o1.step()
        eager.append(float(loss))
    m2, o2 = make()
    tr2 = GraphedTrainStep(m2, o2, warmup=3).capture(S, T)      # the 3 warm-up steps are rolled back; capture executes nothing
    graphed = [float(tr2(S, T)) for _ in range(3)]
    # replays are steps 1, 2, 3 of the eager trajectory (atomics in the VecInt / warp backward make the two runs agree
    # only to rounding)
    for i in range(3):
        assert abs(graphed[i] - eager[i]) <= 2e-3 * abs(eager[i]), (i, graphed, eager)
    assert int(o2.step_dev.item()) == 3
    m3, o3 = make()
    tr3 = GraphedTrainStep(m3, o3, warmup=3, keep_warmup=True).capture(S, T)
    kept = [float(tr3(S, T)) for _ in range(3)]
    for i in range(3):
        assert abs(kept[i] - eager[3 + i]) <= 2e-3 * abs(eager[3 + i]), (i, kept, eager)
    assert int(o3.step_dev.item()) == 6


def test_eager_forward_after_graph_replays_sees_current_weights(vxm_bf16, cuda):
    """Replays update the fp32 parameters inside the graph; an eager (validation) forward afterwards must repack them
    every time, not only the first time (round-1 advisor finding)."""
    vxm = vxm_bf16
    from voxelmorph_b200.trainer import GraphedTrainStep
    kw = dict(inshape=(32, 32, 32))
    cfg = full_cfg(kw)
    s, tr = cases.volume_pair(96, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    m = vxm.networks.VxmDense(**kw)
    m.load_state_dict(ref_torch.init_state_dict(cfg, seed=6, flow_std=2e-2), strict=False)
    m.to(cuda).train()
    o = vxm.optim.FusedAdam(m.parameters(), lr=1e-2)       # large steps: stale weights would be visible
    step = GraphedTrainStep(m, o).capture(S, T)
    for _ in range(2):
        for _ in range(4):
            step(S, T)
        with torch.no_grad():
            flow_eager = m(S, T)[1]
        # oracle on the CURRENT fp32 weights, bf16 storage emulated
        sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
        ref_torch.emulate_bf16(True)
        with torch.no_grad():
            flow_ref = ref_torch.vxm_forward(sd, cfg, t(s), t(tr))[1]
        ref_torch.emulate_bf16(False)
        assert rel(flow_eager.cpu(), flow_ref) <= 2e-2


# ---------------------------------------------------------------------------------------------------------------------
# split precision ("bf16x3"): the in-tolerance tensor-core mode.  Same wgmma kernels, every operand a bf16 (hi, lo)
# pair, three MMAs passes per layer -> flow and moved image within north_star's 1e-4 of the fp32 reference.
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def vxm_x3(cuda, monkeypatch):
    import voxelmorph_b200 as v
    v._lib.load()
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "bf16x3")
    return v


@pytest.mark.parametrize("name", sorted(BF16_VARIANTS))
def test_bf16x3_engine_within_reference_tolerance(vxm_x3, cuda, golden, name):
    vxm = vxm_x3
    kw = BF16_VARIANTS[name]
    cfg = full_cfg(kw)
    model = vxm.networks.VxmDense(**kw)
    sd = ref_torch.init_state_dict(cfg, seed=1234, flow_std=2e-2)
    model.load_state_dict(sd, strict=False)
    model.to(cuda).eval()
    shape = kw["inshape"]
    s, tr = cases.volume_pair(91, shape, sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    with torch.no_grad():
        out = model(S, T)
        reg = model(S, T, registration=True)
        ref = ref_torch.vxm_forward(sd, cfg, t(s), t(tr))
        ref_reg = ref_torch.vxm_forward(sd, cfg, t(s), t(tr), registration=True)
    errs = [rel(y.cpu(), r) for y, r in zip(out, ref)] + [rel(reg[1].cpu(), ref_reg[1])]
    print("\n[%s] bf16x3 vs fp32 oracle: %s" % (name, " ".join("%.2e" % e for e in errs)))
    assert max(errs) <= 1e-4, (name, errs)
    g = golden("vxmdense")
    from test_oracle import VARIANTS
    if VARIANTS.get(name) == kw:   # same constructor arguments as the frozen outputs of the unmodified reference
        for i, y in enumerate(out):
            assert rel(y.cpu(), t(g["%s/train%d" % (name, i)])) <= 1e-4, (name, i)
        assert rel(reg[1].cpu(), t(g["%s/reg_flow" % name])) <= 1e-4


def test_bf16x3_training_step(vxm_x3, cuda, golden):
    """Training step with the split-precision forward (backward on bf16 operands): loss within 1e-4 of the reference's,
    gradients at bf16 grade."""
    vxm = vxm_x3
    g = golden("vxmdense")
    kw = dict(inshape=(32, 32, 48))
    cfg = full_cfg(kw)
    model = vxm.networks.VxmDense(**kw)
    model.load_state_dict(ref_torch.init_state_dict(cfg, seed=1234, flow_std=2e-2), strict=False)
    model.to(cuda).train()
    s, tr = cases.volume_pair(91, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    y, flow = model(S, T)
    loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
    opt.zero_grad()
    loss.backward()
    ref = float(g["default3d/loss"])
    assert abs(float(loss.item()) - ref) <= 1e-4 * abs(ref)
    params = dict(model.named_parameters())
    worst = 0.0
    for k in ("flow.weight", "unet_model.encoder.0.0.main.weight", "unet_model.decoder.0.0.main.weight"):
        e = rel(params[k].grad.cpu(), t(g["default3d/grad/%s" % k]))
        worst = max(worst, e)
    print("\nbf16x3 training step: worst sampled gradient error vs reference %.2e" % worst)
    assert worst <= 5e-2
    opt.step()


# ---------------------------------------------------------------------------------------------------------------------
# the timed configuration itself: 160x192x224, default features, bf16 engine (what bench.py times) and bf16x3
# ---------------------------------------------------------------------------------------------------------------------
FULL = (160, 192, 224)
# tolerances: about twice the errors the tensor-core engines show at this size (bf16 operands cost the flow field most;
# see DESIGN.md section 4.4)
FULL_TOL = {"bf16": dict(flow=1.5e-2, moved=1e-4, loss=1e-5, grad_med=2e-2, grad_max=4e-2),
            "bf16x3": dict(flow=1e-4, moved=1e-4, loss=1e-5, grad_med=1e-2, grad_max=2e-2)}


@pytest.mark.parametrize("engine", ["bf16", "bf16x3"])
def test_full_size_step_vs_oracle(cuda, monkeypatch, engine):
    """BASELINE config 2 at its own size: forward, NCC + Grad loss and the flat gradient of the tensor-core engines
    against oracle/ref_torch (fp32 CPU restatement of the reference) on the same weights and the same pair."""
    import voxelmorph_b200 as vxm
    vxm._lib.load()
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", engine)
    kw = dict(inshape=FULL)
    cfg = full_cfg(kw)
    sd = ref_torch.init_state_dict(cfg, seed=1234, flow_std=1e-2)
    model = vxm.networks.VxmDense(**kw)
    model.load_state_dict(sd, strict=False)
    model.to(cuda).train()
    gsrc = torch.Generator().manual_seed(7)
    coarse = torch.rand((1, 1, 20, 24, 28), generator=gsrc)
    S_c = torch.nn.functional.interpolate(coarse, size=FULL, mode="trilinear", align_corners=True)
    S_c = (S_c + 0.05 * torch.rand(S_c.shape, generator=gsrc)).clamp_(0, 1).contiguous()
    fl = torch.nn.functional.interpolate(torch.randn((1, 3, 10, 12, 14), generator=gsrc) * 3.0, size=FULL, mode="trilinear",
                                         align_corners=True).contiguous()
    T_c = ref_torch.spatial_transform(S_c, fl).contiguous()
    S, T = S_c.to(cuda), T_c.to(cuda)
    y, flow = model(S, T)
    loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
    loss.backward()
    torch.cuda.synchronize()
    # oracle (fp32, CPU): same step
    torch.set_num_threads(max(1, min(64, (torch.get_num_threads() or 1))))
    sdc = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    yc, fc = ref_torch.vxm_forward(sdc, cfg, S_c, T_c)
    lc = ref_torch.ncc_loss(T_c, yc) + 0.01 * ref_torch.grad_loss(fc, "l2", 2)
    lc.backward()
    tol = FULL_TOL[engine]
    e_flow, e_moved = rel(flow.detach().cpu(), fc.detach()), rel(y.detach().cpu(), yc.detach())
    e_loss = abs(float(loss) - float(lc)) / abs(float(lc))
    gerr = sorted(rel(p.grad.cpu(), sdc[k].grad) for k, p in model.named_parameters())
    print("\n[full size, %s] flow %.2e moved %.2e loss %.2e (%.6f vs %.6f) | gradient rel err: median %.2e max %.2e"
          % (engine, e_flow, e_moved, e_loss, float(loss), float(lc), gerr[len(gerr) // 2], gerr[-1]))
    assert e_flow <= tol["flow"] and e_moved <= tol["moved"] and e_loss <= tol["loss"]
    assert gerr[len(gerr) // 2] <= tol["grad_med"] and gerr[-1] <= tol["grad_max"]


def test_kd_folded_layers_match_unfolded_step(vxm_bf16, cuda, monkeypatch):
    """The kd-folded first convolution / flow-head backward compute the same sums as the 3-D kernels (other MMA grouping only)."""
    import voxelmorph_b200 as vxm
    from oracle import cases
    shape = (16, 32, 32)
    s, t = cases.volume_pair(5, shape, sigma=1.5)
    S, T = torch.from_numpy(s).to(cuda), torch.from_numpy(t).to(cuda)
    res = {}
    for fold in ("1", "0"):
        monkeypatch.setenv("VXM_B200_KDFOLD", fold)
        torch.manual_seed(3)
        model = vxm.networks.VxmDense(inshape=shape).to(cuda).train()
        with torch.no_grad():
            model.flow.weight.normal_(0, 2e-2)
        y, flow = model(S, T)
        loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
        loss.backward()
        torch.cuda.synchronize()
        res[fold] = (flow.detach().cpu(), {n: p.grad.detach().cpu().clone() for n, p in model.named_parameters() if p.grad is not None})
    f1, g1 = res["1"]
    f0, g0 = res["0"]
    assert float((f1 - f0).abs().max()) <= 2e-3 * float(f0.abs().max())
    assert set(g1) == set(g0)
    for n in g0:
        den = float(g0[n].abs().max()) + 1e-12
        assert float((g1[n] - g0[n]).abs().max()) <= 2e-2 * den, n
