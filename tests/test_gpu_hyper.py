"""HyperVxmDense on the GPU: the hypernetwork and weight-generation kernels against fp64 (tests/hyper_ref.py), their
determinism, flat-gradient path and refusals, exactness against VxmDense when the generated weights are a VxmDense's,
the whole step on every engine against fp64 autograd, and the graphed step (eager parity, a new lambda between replays,
full size).  Run with -s to see every measured error next to its bound."""
import numpy as np
import pytest
import torch

from oracle import cases, ref_torch

import hyper_ref
from test_gpu_fp32_step_kernels import report
from test_gpu_image_grads import relmax, t
from test_gpu_probabilistic import STEP_TOL
from test_oracle import full_cfg

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
DEFAULT_FEATS = [[16, 32, 32, 32], [32, 32, 32, 32, 32, 16, 16]]
WIDE_FEATS = [[64] * 4, [64] * 7]


@pytest.fixture(scope="module")
def vxm(cuda):
    import voxelmorph_b200 as v
    v._lib.load()
    return v


@pytest.fixture()
def engine(monkeypatch):
    def set_engine(name):
        monkeypatch.setenv("VXM_B200_CONV_ENGINE", name)
    yield set_engine
    ref_torch.emulate_bf16(False)


def _shapes(vxm, feats, inshape=(8, 8, 8)):
    return vxm.networks.HyperVxmDense(inshape, nb_unet_features=feats, nb_hyp_units=8).hyper.shapes


# ---- 1. the kernels ---------------------------------------------------------------------------------------------------

# (generated shapes, P, U, layers): the default U-Net's N = 326 032 and the 64-channel U-Net's, then ragged N (410: 8-byte
# loads, 165: 4-byte loads) and P in {1, 3}, U in {32, 128, 256}
KERNEL_CASES = {
    "default": ("default", 1, 128, 6),
    "default-p3-u256": ("default", 3, 256, 6),
    "default-u32-l8": ("default", 1, 32, 8),
    "wide64": ("wide", 1, 128, 6),
    "ragged410-p3-u256": ([(5, 3, 3, 3, 3)], 3, 256, 2),
    "ragged165-p1-u32": ([(3, 2, 3, 3, 3)], 1, 32, 3),
}


def _hyper_module(vxm, cuda, name, seed=0, cases=KERNEL_CASES):
    shapes, P, U, L = cases[name]
    if isinstance(shapes, str):
        shapes = _shapes(vxm, DEFAULT_FEATS if shapes == "default" else WIDE_FEATS)
    torch.manual_seed(seed)
    mod = vxm.layers.HyperWeights(shapes, P, L, U).to(cuda)
    g = torch.Generator(device=cuda).manual_seed(seed)
    with torch.no_grad():
        mod.hyper_bias.copy_(0.1 * torch.randn(mod.hyper_bias.shape, generator=g, device=cuda))
        for lin in mod.hypernet:          # non-zero biases, both ReLU branches in use
            lin.bias.copy_(0.1 * torch.randn(lin.bias.shape, generator=g, device=cuda))
    hyp = torch.rand(1, P, generator=g, device=cuda)
    dW = torch.randn(mod.hyper_bias.shape, generator=g, device=cuda)
    return mod, hyp, dW


def _run(mod, hyp, dW):
    for p in mod.parameters():
        p.grad = None
    w = mod(hyp)
    w.backward(dW)
    return [w.detach().clone()] + [p.grad.clone() for p in mod.parameters()]


@pytest.mark.parametrize("name", sorted(KERNEL_CASES))
def test_kernels_vs_fp64(vxm, cuda, name):
    mod, hyp, dW = _hyper_module(vxm, cuda, name)
    check_vs_fp64(mod, hyp, dW, _run(mod, hyp, dW), name)


def check_vs_fp64(mod, hyp, dW, got, name):
    """got = [Wflat, then every parameter's gradient] against fp64 autograd, each within its counted bound"""
    L = len(mod.hypernet)
    P, U = mod.hypernet[0].in_features, mod.hypernet[0].out_features
    prm = [p.detach().double().requires_grad_(True) for p in mod.parameters()]
    mlp = [(prm[2 + 2 * i], prm[3 + 2 * i]) for i in range(L)]
    A, a = prm[0], prm[1]
    hd, dWd = hyp.double(), dW.double()
    w = a + hyper_ref.hypernet(hd, mlp) @ A
    w.backward(dWd)
    with torch.no_grad():
        # magnitudes the fp32 roundings scale with: every term taken by its absolute value
        ax = [hd.abs().reshape(-1)]
        for wl, bl in mlp:
            ax.append(wl.abs() @ ax[-1] + bl.abs())
        ah = ax[-1]
        s_w = a.abs() + ah @ A.abs()
        s_gA = torch.outer(ah, dWd.abs())
        s_dh = A.abs() @ dWd.abs()
        ag, s_mlp = s_dh, []
        for i in reversed(range(L)):
            wl = mlp[i][0]
            s_mlp = [torch.outer(ag, ax[i]), ag] + s_mlp
            ag = wl.abs().t() @ ag
        c_h = L * (max(U, P) + 2)                      # the hypernetwork's fma chains
        c_dh = 32 + 5 + 2 + c_h                        # a lane's 32-term chain, the warp tree, the fp64 tile sum's rounding

        def ratio(x, ref, scale):
            return float(((x.double() - ref).abs() / scale.clamp_min(1e-300)).max())
        tag = "hyper %s P=%d U=%d L=%d N=%d" % (name, P, U, L, a.numel())
        report(tag + " Wflat", ratio(got[0], w, s_w), (c_h + U + 2) * U32)
        report(tag + " grad A", ratio(got[1], A.grad, s_gA), (c_h + 2) * U32)
        assert torch.equal(got[2], dW), "grad a = dW exactly"
        for i in range(L):
            report(tag + " grad hypernet.%d.weight" % i, ratio(got[3 + 2 * i], mlp[i][0].grad, s_mlp[2 * i]),
                   (c_dh + 2 * L * (U + 2)) * U32)
            report(tag + " grad hypernet.%d.bias" % i, ratio(got[4 + 2 * i], mlp[i][1].grad, s_mlp[2 * i + 1]),
                   (c_dh + 2 * L * (U + 2)) * U32)


@pytest.mark.parametrize("name", ["default", "ragged410-p3-u256", "ragged165-p1-u32"])
def test_kernels_are_deterministic_and_flat_grads_equal_autograd(vxm, cuda, name):
    mod, hyp, dW = _hyper_module(vxm, cuda, name, seed=3)
    a, b = _run(mod, hyp, dW), _run(mod, hyp, dW)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    opt = vxm.optim.FusedAdam(mod.parameters(), lr=1e-3)
    opt.zero_grad()
    flat = [p.grad for p in mod.parameters()]
    w = mod(hyp)
    w.backward(dW)
    assert all(p.grad is g for p, g in zip(mod.parameters(), flat))         # written in place, autograd got None
    assert torch.equal(w, a[0]) and all(torch.equal(g, x) for g, x in zip(flat, a[1:]))
    mod(hyp).backward(dW)                                                  # accumulates: a rounded sum, as autograd's
    assert all(torch.equal(g, x + x) for g, x in zip(flat, a[1:]))


def test_bad_sizes_are_refused(vxm, cuda):
    L = vxm._lib
    with pytest.raises(ValueError, match="nb_hyp_units"):
        vxm.layers.HyperWeights([(8, 2, 3, 3, 3)], 1, 6, 257)
    mod = vxm.layers.HyperWeights([(8, 2, 3, 3, 3)], 2, 2, 16).to(cuda)
    with pytest.raises(L.VxmError, match=r"\(1, 2\)"):
        mod(torch.zeros(2, 2, device=cuda))
    with pytest.raises(L.VxmError, match="CUDA tensors"):
        mod(torch.zeros(1, 2))
    m = vxm.networks.HyperVxmDense((16, 16, 16), nb_unet_features=[[16, 16], [16, 16, 16]]).to(cuda)
    x = torch.zeros(2, 1, 16, 16, 16, device=cuda)
    with pytest.raises(L.VxmError, match=r"\(2, 1\)"):
        m(x, x, torch.zeros(2, 1, device=cuda))


# ---- 2. exactness against VxmDense ------------------------------------------------------------------------------------

EXACT = dict(inshape=(32, 32, 48), nb_unet_features=DEFAULT_FEATS)


@pytest.mark.parametrize("eng_name", ["f32", "bf16", "bf16x3"])
def test_zero_kernel_is_vxmdense_bit_for_bit(vxm, cuda, engine, eng_name):
    """hyper_kernel = 0 and hyper_bias = a VxmDense's U-Net parameters (flattened in execution order): flow, moved image and
    loss equal the VxmDense's bit for bit, and so do hyper_bias.grad and the flow head's gradients against the VxmDense's
    parameter gradients for one fixed gradient of the U-Net's field (the step's VecInt and warp backward scatter with
    atomics, so a whole step's gradients are not bit-reproducible for either model)."""
    engine(eng_name)
    cfg = full_cfg(EXACT)
    sd = ref_torch.init_state_dict(cfg, seed=5, flow_std=2e-2)
    plain = vxm.networks.VxmDense(**EXACT)
    plain.load_state_dict(sd, strict=False)
    hyper = vxm.networks.HyperVxmDense(**EXACT)
    with torch.no_grad():
        hyper.hyper.hyper_kernel.zero_()
        hyper.hyper.hyper_bias.copy_(torch.cat([p.reshape(-1) for p in plain.unet_model.parameters()]))
        hyper.flow.weight.copy_(plain.flow.weight)
        hyper.flow.bias.copy_(plain.flow.bias)
    plain, hyper = plain.to(cuda).train(), hyper.to(cuda).train()
    s, tr = cases.volume_pair(31, EXACT["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    hyp = torch.tensor([[0.37]], device=cuda)
    outs = []
    with torch.no_grad():
        for m, extra in ((plain, ()), (hyper, (hyp,))):
            y, flow = m(S, T, *extra)
            loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
            outs.append((y, flow, loss))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    g = torch.Generator(device=cuda).manual_seed(2)
    G = 1e-3 * torch.randn((1, 3) + EXACT["inshape"], generator=g, device=cuda)
    plain._head(S, T).backward(G)
    hyper._assign(hyper.hyper(hyp))
    hyper._head(S, T).backward(G)
    want = torch.cat([p.grad.reshape(-1) for p in plain.unet_model.parameters()])
    assert torch.equal(hyper.hyper.hyper_bias.grad, want)
    assert torch.equal(hyper.flow.weight.grad, plain.flow.weight.grad) and torch.equal(hyper.flow.bias.grad, plain.flow.bias.grad)
    print("\n[hyper exact %s] flow, moved, loss %.6f and the U-Net weight gradients bit-identical to VxmDense"
          % (eng_name, float(outs[0][2])))


# ---- 3. the step end to end --------------------------------------------------------------------------------------------

STEP = {
    "3d": dict(inshape=(32, 32, 32), nb_unet_features=[[16, 16, 16, 16], [16, 16, 16, 16, 16, 16, 16]]),
    "bidir3d": dict(inshape=(32, 32, 48), bidir=True),
    "2d": dict(inshape=(64, 64)),
}


def _hyper_model(vxm, kw, seed=21, kernel_scale=1.0):
    """A HyperVxmDense whose hyper_bias is an ordinary U-Net initialisation and whose flow head is the oracle's."""
    cfg = full_cfg(kw)
    sd0 = ref_torch.init_state_dict(cfg, seed=seed, flow_std=2e-2)
    torch.manual_seed(seed)
    model = vxm.networks.HyperVxmDense(**kw)
    with torch.no_grad():
        model.hyper.hyper_bias.copy_(torch.cat([sd0[k].reshape(-1) for k in sd0 if k.startswith("unet_model.")]))
        model.hyper.hyper_kernel.mul_(kernel_scale)
        model.flow.weight.copy_(sd0["flow.weight"])
        model.flow.bias.copy_(sd0["flow.bias"])
    return model, cfg


def _loss(vxm, hyp, outs, T):
    return vxm.losses.hyper_loss(hyp, vxm.losses.NCC().loss(T, outs[0]), vxm.losses.Grad("l2", loss_mult=2).loss(None, outs[-1]))


@pytest.mark.parametrize("name", sorted(STEP))
@pytest.mark.parametrize("eng_name", ["f32", "bf16x3", "bf16"])
def test_hyper_step_vs_oracle(vxm, cuda, engine, eng_name, name):
    check_step_vs_oracle(vxm, cuda, engine, eng_name, name)


def check_step_vs_oracle(vxm, cuda, engine, eng_name, name, flat=False):
    """One step's flow, moved image, loss and every parameter gradient against fp64 autograd (STEP_TOL), then the
    registration form.  flat: the parameters are FusedAdam's views, zeroed, as in training — the gradients are read from
    the flat buffer.  Returns the model and the optimizer (None unless flat)."""
    engine(eng_name)
    kw = STEP[name]
    model, cfg = _hyper_model(vxm, kw)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    model = model.to(cuda).train()
    opt = None
    if flat:
        opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-3)
        opt.zero_grad()
    s, tr = cases.volume_pair(41, kw["inshape"], sigma=1.5)
    S_c, T_c = t(s), t(tr)
    hyp = torch.tensor([[0.3]])
    outs = model(S_c.to(cuda), T_c.to(cuda), hyp.to(cuda))
    loss = _loss(vxm, hyp.to(cuda), outs, T_c.to(cuda))
    loss.backward()
    ref_torch.emulate_bf16(eng_name == "bf16")
    try:
        sdc = {k: v.double().requires_grad_(True) for k, v in sd.items()}
        ref = hyper_ref.hyper_forward(sdc, cfg, S_c.double(), T_c.double(), hyp.double())
        lc = hyper_ref.hyper_loss(ref, T_c.double(), hyp)
        lc.backward()
        reg = hyper_ref.hyper_forward({k: v.detach() for k, v in sdc.items()}, cfg, S_c.double(), T_c.double(), hyp.double(),
                                      registration=True)
    finally:
        ref_torch.emulate_bf16(False)
    tol = STEP_TOL[eng_name]
    e_fp, e_moved = relmax(outs[-1].detach().cpu(), ref[-1].detach()), relmax(outs[0].detach().cpu(), ref[0].detach())
    e_loss = abs(float(loss.detach()) - float(lc.detach())) / abs(float(lc.detach()))
    gerr = {k: relmax(p.grad.cpu(), sdc[k].grad) for k, p in model.named_parameters()}
    g = sorted(gerr.values())
    print("\n[hyper step %s %s] flow %.2e moved %.2e loss %.2e | gradient rel err median %.2e max %.2e (%s) | bounds %s"
          % (eng_name, name, e_fp, e_moved, e_loss, g[len(g) // 2], g[-1], max(gerr, key=gerr.get), tol))
    assert e_fp <= tol["fp"] and e_moved <= tol["moved"] and e_loss <= tol["loss"]
    assert g[len(g) // 2] <= tol["grad_med"] and g[-1] <= tol["grad_max"], gerr
    # registration form, eval mode
    model.eval()
    y_reg, pos = model(S_c.to(cuda), T_c.to(cuda), hyp.to(cuda), registration=True)
    assert not y_reg.requires_grad
    e_reg, e_pos = relmax(y_reg.cpu(), reg[0]), relmax(pos.cpu(), reg[1])
    print("[hyper registration %s %s] moved %.2e pos_flow %.2e" % (eng_name, name, e_reg, e_pos))
    assert e_reg <= tol["moved"] and e_pos <= tol["fp"]
    return model, opt


def test_two_lambdas_give_different_flows(vxm, cuda, engine):
    engine("bf16")
    kw = STEP["3d"]
    model, _ = _hyper_model(vxm, kw, kernel_scale=5.0)
    model = model.to(cuda).eval()
    s, tr = cases.volume_pair(42, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    flows = [model(S, T, torch.tensor([[lam]], device=cuda), registration=True)[1] for lam in (0.0, 1.0)]
    again = model(S, T, torch.tensor([[0.0]], device=cuda), registration=True)[1]
    d = relmax(flows[1], flows[0])
    print("\n[hyper lambdas] flow(1) vs flow(0): %.2e of its max-norm" % d)
    assert d > 1e-2 and torch.equal(again, flows[0])


# ---- 4. the graphed step -----------------------------------------------------------------------------------------------

LR = 1e-4
WEIGHT_TOL = 3 * LR


def _graph_run(vxm, cuda, mode, hyps, inputs, kw):
    from voxelmorph_b200.trainer import GraphedTrainStep
    model, _ = _hyper_model(vxm, kw, kernel_scale=5.0)
    model = model.to(cuda).train()
    opt = vxm.optim.FusedAdam(model.parameters(), lr=LR)
    S, T = inputs

    def loss_fn(model, src, trg, hyp):
        return _loss(vxm, hyp, model(src, trg, hyp), trg)
    losses, wflats = [], []
    if mode == "eager":
        for h in hyps:
            opt.zero_grad()
            loss = loss_fn(model, S, T, h)
            loss.backward()
            wflats.append(model.hyper.wflat.clone())
            opt.step()
            losses.append(float(loss))
    else:
        start = opt.fp.flat.clone()
        step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=3).capture(S, T, hyps[0])
        assert torch.equal(opt.fp.flat, start)
        for h in hyps:
            losses.append(float(step(None, None, h)))
            wflats.append(model.hyper.wflat.clone())
    torch.cuda.synchronize()
    return losses, wflats, opt.fp.flat.clone()


def test_graphed_step_matches_eager_and_takes_a_new_lambda(vxm, cuda, engine):
    """Three replays at one lambda, then two at others: the static hyp changes between replays without a re-capture, and
    each replay equals an eager step at that lambda — the weight generation and the pack launch are in the graph."""
    engine("bf16")
    kw = STEP["3d"]
    s, tr = cases.volume_pair(43, kw["inshape"], sigma=1.5)
    inputs = (t(s).to(cuda), t(tr).to(cuda))
    hyps = [torch.tensor([[v]], device=cuda) for v in (0.2, 0.2, 0.2, 0.9, 0.0)]
    le, we, pe = _graph_run(vxm, cuda, "eager", hyps, inputs, kw)
    lg, wg, pg = _graph_run(vxm, cuda, "graphed", hyps, inputs, kw)
    d_param = float((pg - pe).abs().max())
    d_w = [relmax(a, b) for a, b in zip(wg, we)]
    jump = relmax(we[3], we[2])
    print("\n[graphed hyper step] losses %s vs eager %s | generated weights %s (lambda change moves them %.2e) | params %.2e "
          "(bound %.0e)" % (lg, le, ["%.1e" % d for d in d_w], jump, d_param, WEIGHT_TOL))
    for i in range(len(hyps)):
        assert abs(lg[i] - le[i]) <= 2e-3 * abs(le[i]), (i, lg, le)
    assert max(d_w) <= 1e-2 * jump and jump > 1e-2
    assert d_param <= WEIGHT_TOL


def test_full_size_graphed_hyper_step(vxm, cuda, engine):
    engine("bf16")
    from voxelmorph_b200.trainer import GraphedTrainStep
    shape = (160, 192, 224)
    s, tr = cases.volume_pair(95, shape, sigma=3.0)
    torch.manual_seed(0)
    model = vxm.networks.HyperVxmDense(shape).to(cuda).train()
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4)

    def loss_fn(model, src, trg, hyp):
        return _loss(vxm, hyp, model(src, trg, hyp), trg)
    start = model.hyper.hyper_kernel.detach().clone()
    hyp = torch.tensor([[0.5]], device=cuda)
    step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=2).capture(t(s).to(cuda), t(tr).to(cuda), hyp)
    losses = [float(step(None, None, torch.tensor([[v]], device=cuda))) for v in (0.1, 0.5, 0.9)]
    moved = float((model.hyper.hyper_kernel.detach() - start).abs().max())
    print("\n[full-size graphed hyper step] losses %s, hyper_kernel moved by up to %.2e" % (losses, moved))
    assert all(np.isfinite(losses)) and moved > 0
