"""Probabilistic VoxelMorph on the GPU: the sampler against the numpy restatement of its noise stream (tests/probs_ref.py),
the KL and sigma-weighted MSE kernels against fp64, the model's step on every engine against the oracle with the noise the
kernel drew, its registration form against VxmDense, checkpoints, and graphed steps.  Run with -s to see every measured
error next to its bound."""
import numpy as np
import pytest
import torch

from oracle import cases, ref_torch

import probs_ref
from test_gpu_fp32_step_kernels import report
from test_gpu_image_grads import relmax, t
from test_gpu_template import FLOW_WGRAD_TOL
from test_oracle import full_cfg

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


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


def _state(cuda, seed, call):
    return torch.tensor([seed, call], dtype=torch.int64, device=cuda)


# ---- 1. the sampler ---------------------------------------------------------------------------------------------------

# eps in fp32: u1, u2 are exact; logf (1 ulp), the product by -2 (exact), sqrtf (0.5 ulp, halving the log's relative
# error), sincospif (1 ulp) and the product r * cos (0.5 ulp) give under 3 ulp of |eps|; 8 ulp is the bound.  An error
# in the index mapping, the seed or the counter is an O(1) mismatch
EPS_REL = 8 * U
SAMPLE_SHAPES = {"full": (1, 3, 160, 192, 224), "2d-b2": (2, 2, 192, 224), "ragged": (2, 3, 5, 7, 9)}


@pytest.mark.parametrize("name", sorted(SAMPLE_SHAPES))
def test_sampler_draws_the_restated_stream(vxm, cuda, name):
    shape = SAMPLE_SHAPES[name]
    nd = shape[1]
    seed, call = 0x1234_5678_9ABC_DEF0 + len(name), (1 << 32) + 5
    state = _state(cuda, seed, call)
    params = torch.zeros((shape[0], 2 * nd) + shape[2:], device=cuda)
    z = vxm.layers.sample_normal_logvar(params, state)
    torch.cuda.synchronize()
    assert state.tolist() == [seed, call + 1]
    want = probs_ref.normal_stream(z.numel(), seed, call)
    got = z.detach().cpu().double().numpy().reshape(-1)
    err = float((np.abs(got - want) / (np.abs(want) + 1e-30)).max())
    report("sampler eps %s %s: rel err vs numpy stream" % (name, shape), err, EPS_REL)
    mb, vb = probs_ref.standard_error_bounds(want)
    report("sampler eps %s: |mean| (5 s.e.)" % name, abs(float(got.mean())), mb)
    report("sampler eps %s: |var - 1| (5 s.e.)" % name, abs(float(got.var()) - 1), vb)


@pytest.mark.parametrize("name", ["2d-b2", "ragged"])
def test_sampler_general_mean_and_variance_and_backward(vxm, cuda, name):
    shape = SAMPLE_SHAPES[name]
    nd = shape[1]
    g = torch.Generator(device=cuda).manual_seed(4)
    params = torch.randn((shape[0], 2 * nd) + shape[2:], generator=g, device=cuda)
    params[:, nd:] -= 2.0
    params.requires_grad_(True)
    state = _state(cuda, 99, 7)
    z = vxm.layers.sample_normal_logvar(params, state)
    gz = torch.randn(z.shape, generator=g, device=cuda)
    z.backward(gz)
    p = params.detach().cpu().double().numpy()
    zw, eps = probs_ref.sample_normal_logvar(p[:, :nd], p[:, nd:], 99, 7)
    s = np.exp(p[:, nd:] / 2)
    # z = fma(expf(l / 2), eps, mu): the product l / 2 is exact, expf 2 ulp, eps 8 ulp (above), one rounding of the fma
    bound_z = (10 * np.abs(s * eps) + np.abs(zw)) * U + 1e-30
    report("sampler z %s: max err / bound" % name, float((np.abs(z.detach().cpu().double().numpy() - zw) / bound_z).max()), 1.0)
    gp = params.grad.cpu()
    assert torch.equal(gp[:, :nd], gz.cpu()), "d mu must be d z bit for bit"
    dl = gz.cpu().double().numpy() * eps * 0.5 * s
    # (dz * eps) * (0.5 * expf(l / 2)): eps 8 ulp, expf 2 ulp, two products
    report("sampler d logvar %s: max rel err" % name, float((np.abs(gp[:, nd:].double().numpy() - dl) / (np.abs(dl) + 1e-30)).max()),
           12 * U)


def test_sampler_state_advances_and_reproduces(vxm, cuda):
    params = torch.zeros((1, 6, 8, 12, 16), device=cuda)
    state = _state(cuda, 5, 0)
    a = vxm.layers.sample_normal_logvar(params, state)
    b = vxm.layers.sample_normal_logvar(params, state)
    assert state.tolist() == [5, 2]
    assert float((a - b).abs().max()) > 1.0            # two forwards draw different eps
    state.copy_(_state(cuda, 5, 0))
    assert torch.equal(vxm.layers.sample_normal_logvar(params, state), a)     # the same (seed, call) reproduces it
    other = vxm.layers.sample_normal_logvar(params, _state(cuda, 6, 0))
    assert float((other - a).abs().max()) > 1.0
    # the backward regenerates the forward's eps even after the state moved on: d logvar at l = 0 is dz eps / 2
    pr = params.clone().requires_grad_(True)
    st = _state(cuda, 5, 0)
    z = vxm.layers.sample_normal_logvar(pr, st)
    vxm.layers.sample_normal_logvar(params, st)
    z.backward(torch.ones_like(z))
    assert torch.equal(pr.grad[:, 3:], a * 0.5)


# ---- 2. KL and MSE(sigma) ---------------------------------------------------------------------------------------------

KL_SHAPES = {"full-b2": (2, 6, 160, 192, 224), "2d-b8": (8, 4, 192, 224), "odd": (2, 6, 13, 17, 19),
             "deg-3d": (1, 6, 1, 5, 7), "deg-2d": (2, 4, 1, 9), "size2": (3, 6, 2, 2, 3)}
LAM = 10.0


def _kl_magnitude(p, lam):
    """sum of the absolute values of the loss's terms (fp64), for the rounding bound of the fp32 terms"""
    nd = p.ndim - 2
    B, V = p.shape[0], int(np.prod(p.shape[2:]))
    lv = p[:, nd:]
    a = 0.5 / (B * V) * np.sum(lam * probs_ref.degree(p.shape[2:]) * np.exp(lv) + np.abs(lv))
    for ax in range(2, p.ndim):
        n = p.shape[ax]
        if n > 1:
            a += lam / (4.0 * B * nd * (n - 1) * (V / n)) * np.sum(np.diff(p[:, :nd], axis=ax) ** 2)
    return a


@pytest.mark.parametrize("name", sorted(KL_SHAPES))
def test_kl_vs_fp64(vxm, cuda, name):
    shape = KL_SHAPES[name]
    nd = shape[1] // 2
    g = torch.Generator(device=cuda).manual_seed(12)
    params = torch.randn(shape, generator=g, device=cuda)
    params[:, nd:] = params[:, nd:] * 0.5 - 3.0
    params.requires_grad_(True)
    loss = vxm.losses.KL(LAM, flow_vol_shape=shape[2:]).loss(None, params)
    loss.backward()
    p = params.detach().cpu().double().numpy()
    want = probs_ref.kl_loss(p, LAM)
    # per term: expf 2 ulp, three products / one difference in fp32 (4 roundings), the fp64 sum exact to 2^-50
    report("KL %s %s loss: |err| / (8 ulp of the terms' magnitude)" % (name, shape),
           abs(float(loss) - want) / (8 * U * _kl_magnitude(p, LAM) + U * abs(want)), 1.0)
    gw, mag = probs_ref.kl_grad(p, LAM)
    # per element: every stencil term and the pointwise term round a few times in fp32 (differences, coefficient products,
    # sums of up to 6 terms): 8 ulp of the magnitude
    e = np.abs(params.grad.cpu().double().numpy() - gw) / (8 * U * mag + 1e-38)
    report("KL %s gradient: max err / bound" % name, float(e.max()), 1.0)


@pytest.mark.parametrize("sigma", [0.02, 0.5])
def test_mse_sigma_vs_fp64(vxm, cuda, sigma):
    shape = (2, 1, 40, 48, 56)
    g = torch.Generator(device=cuda).manual_seed(3)
    a = torch.rand(shape, generator=g, device=cuda)
    b = torch.rand(shape, generator=g, device=cuda).requires_grad_(True)
    loss = vxm.losses.MSE(sigma).loss(a, b)
    loss.backward()
    ad, bd = a.cpu().double(), b.detach().cpu().double()
    want = float(probs_ref.mse_sigma(ad, bd, sigma))
    report("MSE(%g) loss rel err" % sigma, abs(float(loss) - want) / want, 4 * U)
    gw = 2.0 / a.numel() / sigma ** 2 * (bd - ad)
    report("MSE(%g) gradient rel err" % sigma, float(((b.grad.cpu().double() - gw).abs() / (gw.abs() + 1e-30)).max()), 3 * U)
    # MSE() runs the unscaled kernels as before; MSE(1.0) is the same loss
    b.grad = None
    plain = vxm.losses.MSE().loss(a, b)
    plain.backward()
    lib, L = vxm._lib.load(), vxm._lib
    direct = torch.empty((), device=cuda)
    L.check(lib.vxm_mse_fwd(L.ptr(a), L.ptr(b.detach()), L.ptr(direct), L.ptr(L.reduce_workspace(cuda)), a.numel(),
                            L.stream_ptr()), "mse")
    assert torch.equal(plain.detach(), direct) and torch.equal(vxm.losses.MSE(1.0).loss(a, b).detach(), direct)
    assert torch.equal(b.grad, (2.0 / a.numel()) * (b.detach() - a)) or \
        float((b.grad - (2.0 / a.numel()) * (b.detach() - a)).abs().max()) <= 2 * U * float(b.grad.abs().max())


# ---- 3. the model's step against the oracle ----------------------------------------------------------------------------

STEP = {
    "smoke3d": dict(inshape=(32, 32, 32), nb_unet_features=[[16, 16, 16, 16], [16, 16, 16, 16, 16, 16, 16]]),
    "default2d": dict(inshape=(64, 64)),
    "bidir3d": dict(inshape=(32, 32, 48), bidir=True),
}
# the deterministic step's bounds per engine (test_gpu_bf16_engine.FULL_TOL, smoke()): the bf16 engine against the oracle
# with bf16 operands emulated.  The f32 engine's weight gradients take the bound of test_gpu_template.FLOW_WGRAD_TOL: they
# are sums of the flow-field gradient, which the step's fp32 tail (resize, VecInt, resize, warp) puts up to 2.3e-3 of its
# max-norm from fp64 where samples land in other trilinear cells in fp32 and fp64 (DESIGN section 7).  Over 10 noise draws
# per case (H100) the median parameter error was 1e-6 to 4e-5 in most draws and reached 1.3e-3 (max 2.1e-3) in one
# bidirectional draw, with 90 % of the flow_params gradient error in 10 voxels; the same jump appears without noise
STEP_TOL = {"f32": dict(fp=1e-4, moved=1e-4, loss=1e-4, grad_med=FLOW_WGRAD_TOL, grad_max=FLOW_WGRAD_TOL),
            "bf16x3": dict(fp=1e-4, moved=1e-4, loss=1e-4, grad_med=1e-2, grad_max=5e-2),
            "bf16": dict(fp=2e-2, moved=2e-3, loss=2e-3, grad_med=5e-2, grad_max=1.5e-1)}


def _prob_model(vxm, cuda, kw, seed=1234, ls_bias=-6.0):
    cfg = full_cfg(kw)
    sd = probs_ref.init_log_sigma(ref_torch.init_state_dict(cfg, seed=seed, flow_std=2e-2), cfg, seed=seed, bias=ls_bias)
    model = vxm.networks.VxmDenseProbabilistic(**kw)
    model.load_state_dict(sd, strict=True)
    # the constructor draws the noise seed from torch's global generator, whose state depends on what ran before: pin it
    model.noise_state.copy_(torch.tensor([seed, 0], dtype=torch.int64))
    return model.to(cuda).train(), sd, cfg


def _recover_eps(vxm, state0, fp_shape, nd, cuda):
    """the eps a forward drew from noise_state = state0: the sampler on mu = 0, l = 0 at the same (seed, call)"""
    zeros = torch.zeros((fp_shape[0], 2 * nd) + tuple(fp_shape[2:]), device=cuda)
    return vxm.layers.sample_normal_logvar(zeros, state0.clone()).cpu()


def _gpu_loss(vxm, outs, S, T):
    mse, kl = vxm.losses.MSE(0.02).loss, vxm.losses.KL(10.0).loss
    loss = mse(T, outs[0]) + 0.01 * kl(None, outs[-1])
    if len(outs) == 3:
        loss = loss + mse(S, outs[1])
    return loss


def _step_check(vxm, cuda, engine, eng_name, kw, tag, vols=None, dtype=torch.float64):
    engine(eng_name)
    model, sd, cfg = _prob_model(vxm, cuda, kw)
    if vols is None:
        vols = cases.volume_pair(91, kw["inshape"], sigma=1.5)
    S_c, T_c = t(vols[0]), t(vols[1])
    S, T = S_c.to(cuda), T_c.to(cuda)
    state0 = model.noise_state.clone()
    outs = model(S, T)
    loss = _gpu_loss(vxm, outs, S, T)
    loss.backward()
    nd = len(kw["inshape"])
    assert model.noise_state.tolist() == [state0[0].item(), state0[1].item() + 1]
    eps = _recover_eps(vxm, state0, outs[-1].shape, nd, cuda).to(dtype)
    ref_torch.emulate_bf16(eng_name == "bf16")
    try:
        sdc = {k: v.to(dtype).requires_grad_(True) for k, v in sd.items()}
        ref = probs_ref.prob_forward(sdc, cfg, S_c.to(dtype), T_c.to(dtype), eps)
        lc = probs_ref.prob_loss(ref, T_c.to(dtype), S_c.to(dtype))
        lc.backward()
    finally:
        ref_torch.emulate_bf16(False)
    tol = STEP_TOL[eng_name]
    e_fp, e_moved = relmax(outs[-1].detach().cpu(), ref[-1].detach()), relmax(outs[0].detach().cpu(), ref[0].detach())
    e_loss = abs(float(loss) - float(lc)) / abs(float(lc))
    gerr = sorted(relmax(p.grad.cpu(), sdc[k].grad) for k, p in model.named_parameters())
    print("\n[probabilistic step %s %s] flow_params %.2e moved %.2e loss %.2e (%.6f vs %.6f) | gradient rel err median "
          "%.2e max %.2e | bounds %s" % (eng_name, tag, e_fp, e_moved, e_loss, float(loss), float(lc), gerr[len(gerr) // 2],
                                        gerr[-1], tol))
    assert e_fp <= tol["fp"] and e_moved <= tol["moved"] and e_loss <= tol["loss"]
    assert gerr[len(gerr) // 2] <= tol["grad_med"] and gerr[-1] <= tol["grad_max"]
    return model


@pytest.mark.parametrize("name", sorted(STEP))
@pytest.mark.parametrize("eng_name", ["f32", "bf16x3", "bf16"])
def test_probabilistic_step_vs_oracle(vxm, cuda, engine, eng_name, name):
    _step_check(vxm, cuda, engine, eng_name, STEP[name], name)


def test_full_size_probabilistic_step_bf16(vxm, cuda, engine):
    shape = (160, 192, 224)
    gsrc = torch.Generator().manual_seed(7)
    coarse = torch.rand((1, 1, 20, 24, 28), generator=gsrc)
    S = torch.nn.functional.interpolate(coarse, size=shape, mode="trilinear", align_corners=True).contiguous()
    fl = torch.nn.functional.interpolate(torch.randn((1, 3, 10, 12, 14), generator=gsrc) * 3.0, size=shape, mode="trilinear",
                                         align_corners=True).contiguous()
    T = ref_torch.spatial_transform(S, fl).contiguous()
    torch.set_num_threads(max(1, min(64, (torch.get_num_threads() or 1))))
    _step_check(vxm, cuda, engine, "bf16", dict(inshape=shape), "160x192x224", vols=(S.numpy(), T.numpy()), dtype=torch.float32)


@pytest.mark.parametrize("eng_name", ["f32", "bf16x3", "bf16"])
@pytest.mark.parametrize("name", ["smoke3d", "default2d"])
def test_registration_form_is_vxmdense_on_the_mean(vxm, cuda, engine, eng_name, name):
    """registration=True integrates mu: the flow of a VxmDense with the same U-Net and flow weights.  On the tensor-core
    engines the head's 2 nd outputs pad to the same MMA width (16) as nd outputs, so each output column sums its K terms in
    the same order and the result is bit-identical as well."""
    engine(eng_name)
    kw = STEP[name]
    model, sd, _ = _prob_model(vxm, cuda, kw)
    plain = vxm.networks.VxmDense(**kw)
    plain.load_state_dict({k: v for k, v in sd.items() if not k.startswith("log_sigma")}, strict=True)
    plain.to(cuda).eval()
    model.eval()
    S, T = (t(v).to(cuda) for v in cases.volume_pair(92, kw["inshape"], sigma=1.5))
    state0 = model.noise_state.clone()
    ys, flow = model(S, T, registration=True)
    yp, fp = plain(S, T, registration=True)
    assert torch.equal(model.noise_state, state0)            # nothing sampled
    print("\n[registration %s %s] flow max |diff| %.3e" % (eng_name, name, float((flow - fp).abs().max())))
    assert torch.equal(flow, fp) and torch.equal(ys, yp)


def test_checkpoint_round_trip(vxm, cuda, tmp_path, engine):
    engine("bf16")
    model, _, _ = _prob_model(vxm, cuda, STEP["smoke3d"])
    p = tmp_path / "prob.pt"
    model.save(p)
    m2 = vxm.networks.VxmDenseProbabilistic.load(p, "cuda").to(cuda)
    for k, v in model.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k
    model.eval()
    m2.eval()
    S, T = (t(v).to(cuda) for v in cases.volume_pair(93, STEP["smoke3d"]["inshape"], sigma=1.5))
    assert all(torch.equal(a, b) for a, b in zip(model(S, T, registration=True), m2(S, T, registration=True)))
    # the training form with the same noise state draws the same field
    m2.noise_state.copy_(model.noise_state)
    assert all(torch.equal(a, b) for a, b in zip(model(S, T), m2(S, T)))


# ---- 4. graphs ---------------------------------------------------------------------------------------------------------

LR = 1e-4
# the step is not bit-reproducible run to run: the VecInt backward scatters with atomics (DESIGN section 5).  Within one
# replay the noise is the eager step's bit for bit (same (seed, call)); the runs then differ by rounding, which Adam turns
# into steps of up to lr on weights whose gradient is at rounding level: 3 steps bound the weights by 3 lr
WEIGHT_TOL = 3 * LR


def test_graphed_probabilistic_step_matches_eager(vxm, cuda, engine):
    eng_name = "bf16"
    engine(eng_name)
    from voxelmorph_b200.trainer import GraphedTrainStep
    kw = STEP["smoke3d"]
    S, T = (t(v).to(cuda) for v in cases.volume_pair(94, kw["inshape"], sigma=1.5))
    runs = {}
    for mode in ("eager", "graphed"):
        model, _, _ = _prob_model(vxm, cuda, kw, seed=5)
        model.noise_state.copy_(_state(cuda, 77, 0))
        opt = vxm.optim.FusedAdam(model.parameters(), lr=LR)

        def loss_fn(model, s, tr):
            return _gpu_loss(vxm, model(s, tr), s, tr)
        if mode == "eager":
            losses = []
            for _ in range(3):
                opt.zero_grad()
                loss = loss_fn(model, S, T)
                loss.backward()
                opt.step()
                losses.append(float(loss))
        else:
            step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=3).capture(S, T)
            assert model.noise_state.tolist() == [77, 0]          # the warm-up's draws are rolled back
            losses, calls = [], []
            for _ in range(3):
                losses.append(float(step(S, T)))
                calls.append(model.noise_state.tolist()[1])
            assert calls == [1, 2, 3]                              # every replay draws the next call: fresh noise
        torch.cuda.synchronize()
        runs[mode] = (losses, opt.fp.flat.clone(), model.noise_state.clone())
    (le, pe, ne), (lg, pg, ng) = runs["eager"], runs["graphed"]
    d = float((pg - pe).abs().max())
    print("\n[graphed probabilistic step %s] losses %s vs eager %s | weights %.2e (bound %.0e)" % (eng_name, lg, le, d, WEIGHT_TOL))
    assert torch.equal(ne, ng)
    assert abs(lg[0] - le[0]) <= 1e-5 * abs(le[0])
    for i in range(3):
        assert abs(lg[i] - le[i]) <= 2e-3 * abs(le[i]), (i, lg, le)
    assert d <= WEIGHT_TOL
