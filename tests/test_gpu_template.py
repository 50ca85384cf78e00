"""TemplateCreation on the GPU: the MeanStream kernels against the fp64 restatement (tests/template_ref.py), the template
step end to end on every engine against fp64 autograd of the oracle, a graphed template step against an eager one, and the
full-size graphed step.  Run with -s to see every measured error next to its bound."""
import numpy as np
import pytest
import torch

from oracle import cases, ref_torch

import template_ref
from test_gpu_fp32_step_kernels import report
from test_gpu_image_grads import DOUBLED, E2E_TOL, relmax, t
from test_oracle import full_cfg

pytestmark = pytest.mark.gpu


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


# ---- 1. the MeanStream kernels ---------------------------------------------------------------------------------------

MS_SHAPES = {"full": (3, 160, 192, 224), "2d": (2, 192, 224), "ragged": (3, 13, 17, 19)}
MS_STEPS, MS_CAP = 8, 5.0
# fp32 against fp64: the state update rounds a handful of times per step (sum over b, alpha, 1 - alpha, two products, one
# add) and carries the previous error scaled by 1 - alpha < 1, so 8 roundings per step over 8 steps bound it; the output
# adds one product, the gradient's scalar and sum a few more roundings
MS_STATE_TOL = MS_STEPS * 8 * 2.0 ** -24
MS_GRAD_TOL = 8 * 2.0 ** -24


def _ms_run(vxm, cuda, shape, B, seed):
    """8 training steps of layers.MeanStream; returns the per-step (x, gout, out, grad, mean, count), on the device."""
    ms = vxm.layers.MeanStream(shape, cap=MS_CAP).to(cuda).train()
    g = torch.Generator(device=cuda).manual_seed(seed)
    res = []
    for _ in range(MS_STEPS):
        x = torch.randn((B,) + shape, generator=g, device=cuda).requires_grad_(True)
        gout = torch.randn((B,) + shape, generator=g, device=cuda)
        out = ms(x)
        assert out.shape == x.shape and (B == 1 or out.stride(0) == 0)
        out.backward(gout)
        res.append((x.detach(), gout, out[0].detach(), x.grad, ms.mean.clone(), float(ms.count)))
    return res


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("name", sorted(MS_SHAPES))
def test_mean_stream_kernels_vs_fp64(vxm, cuda, name, B):
    shape = MS_SHAPES[name]
    res = _ms_run(vxm, cuda, shape, B, 3 + B)
    mean, count = torch.zeros(shape, dtype=torch.float64), 0.0
    e_state = e_out = e_grad = 0.0
    for step, (x, gout, out, gx, m_gpu, c_gpu) in enumerate(res):
        xd = x.cpu().double().requires_grad_(True)
        want, m1, n1 = template_ref.mean_stream(xd, mean, count, MS_CAP)
        (want * gout.cpu().double()).sum().backward()
        assert c_gpu == n1 == (step + 1) * B                      # count is exact
        e_state = max(e_state, relmax(m_gpu.cpu(), m1.detach()))
        e_out = max(e_out, relmax(out.cpu(), want[0].detach()))
        e_grad = max(e_grad, relmax(gx.cpu(), xd.grad))
        mean, count = m1.detach(), n1
    tag = "mean stream %s %s B=%d, %d steps, cap %g" % (name, shape, B, MS_STEPS, MS_CAP)
    report(tag + " state", e_state, MS_STATE_TOL)
    report(tag + " output", e_out, MS_STATE_TOL)
    report(tag + " d/dx", e_grad, MS_GRAD_TOL)


@pytest.mark.parametrize("name", sorted(MS_SHAPES))
def test_mean_stream_is_deterministic_and_eval_commits_nothing(vxm, cuda, name):
    shape = MS_SHAPES[name]
    a, b = _ms_run(vxm, cuda, shape, 2, 9), _ms_run(vxm, cuda, shape, 2, 9)
    for ra, rb in zip(a, b):
        for u, v in zip(ra, rb):
            assert torch.equal(u, v) if torch.is_tensor(u) else u == v
    ms = vxm.layers.MeanStream(shape, cap=MS_CAP).to(cuda)
    x0 = torch.randn((2,) + shape, device=cuda)
    ms(x0)
    m0, c0 = ms.mean.clone(), ms.count.clone()
    ms.eval()
    x = torch.randn((2,) + shape, device=cuda).requires_grad_(True)
    out = ms(x)
    assert torch.equal(ms.mean, m0) and torch.equal(ms.count, c0)
    want, _, _ = template_ref.mean_stream(x.detach().cpu().double(), m0.cpu().double(), float(c0), MS_CAP)
    report("mean stream %s eval output" % name, relmax(out[0].detach().cpu(), want[0]), MS_GRAD_TOL)
    # a gradient broadcast over the batch (stride 0) is summed in the kernel like a materialised one
    g1 = torch.randn((1,) + shape, device=cuda)
    out.backward(g1.expand_as(out))
    want_g = x.grad.clone()
    x.grad = None
    ms(x).backward(g1.expand_as(out).contiguous())
    assert torch.equal(x.grad, want_g)


def test_mean_stream_reports_bad_arguments(vxm, cuda):
    lib, L = vxm._lib.load(), vxm._lib
    x = torch.zeros(8, device=cuda)
    ws = L.reduce_workspace(cuda)
    rc = lib.vxm_mean_stream_fwd(L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(ws), 1, 8, 0.0, 1, L.stream_ptr())
    assert rc != 0 and "cap" in L.last_error()
    rc = lib.vxm_mean_stream_fwd(L.ptr(x), None, L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(ws), 1, 8, 3.0, 1, L.stream_ptr())
    assert rc != 0 and "null pointer" in L.last_error()
    rc = lib.vxm_mean_stream_bwd(L.ptr(x), L.ptr(x), L.ptr(x), 2, 4, 3, L.stream_ptr())
    assert rc != 0 and "stride" in L.last_error()
    with pytest.raises(L.VxmError, match="does not match"):
        vxm.layers.MeanStream((2, 4, 4), cap=3).to(cuda)(torch.zeros(1, 3, 4, 4, device=cuda))


# ---- 2. the template step end to end ----------------------------------------------------------------------------------

# the image sizes of test_gpu_image_grads.E2E, plus B = 2 in 3-D and 2-D
TEMPLATE_E2E = {
    "default3d": (dict(inshape=(32, 32, 48)), 1),
    "doubled3d": (dict(inshape=(16, 32, 32), nb_unet_features=DOUBLED), 1),
    "default2d": (dict(inshape=(64, 64)), 1),
    "b2-3d": (dict(inshape=(32, 32, 48)), 2),
    "b2-2d": (dict(inshape=(32, 48), int_steps=5), 2),
}
W_IMG = 0.75        # every term of the step active: the inverse image term differentiates NCC w.r.t. the atlas (y_true)
CAP = 5.0
# the flow head's weight gradient is a sum over voxels of the flow-field gradient, which the step's fp32 tail (resize,
# VecInt, resize, warp) puts 2.3e-3 of its max-norm from fp64 on every engine (DESIGN section 7: samples that land in
# other trilinear cells in fp32 and fp64 coordinates); measured <= 1.2e-3 here on all three engines, f32 included
FLOW_WGRAD_TOL = 3e-3


def _template(vxm, cuda, kw, B, seed=77):
    """GPU model and fp64 oracle state on the same parameters: the atlas and the images are smooth volumes, the mean
    stream starts part-way (count 3, a random mean) so that both of its terms count."""
    cfg = full_cfg(dict(kw, bidir=True))
    sd = {"vxm_model." + k: v for k, v in ref_torch.init_state_dict(cfg, seed=seed, flow_std=2e-2).items()}
    shape = kw["inshape"]
    s, _ = cases.volume_pair(93, shape, sigma=1.5)
    sd["atlas"] = t(s)
    imgs = np.concatenate([cases.volume_pair(94 + b, shape, sigma=1.5)[1] for b in range(B)], axis=0)
    g = torch.Generator().manual_seed(seed)
    mean0 = 0.1 * torch.randn((len(shape),) + tuple(shape), generator=g)
    model = vxm.networks.TemplateCreation(mean_cap=CAP, **kw)
    model.load_state_dict(sd, strict=False)
    with torch.no_grad():
        model.mean_stream.mean.copy_(mean0)
        model.mean_stream.count.fill_(3)
    tcfg = dict(cfg, mean_cap=CAP)
    return model.to(cuda).train(), sd, tcfg, t(imgs), mean0


def _gpu_step_loss(vxm, model, image, zeros, w_img=1.0):
    """train_template.py's loss: w_img NCC(image, y_source) [+ (1 - w_img) NCC(atlas, y_target)] + MSE(0, mean_stream) +
    Grad('l2', 2)(pos_flow); `zeros` is a device-resident constant"""
    ncc = vxm.losses.NCC().loss
    y_source, y_target, ms, pos = model(image)
    loss = w_img * ncc(image, y_source) + vxm.losses.MSE().loss(zeros, ms) + vxm.losses.Grad("l2", loss_mult=2).loss(None, pos)
    if w_img != 1.0:
        atlas_b = model.atlas.expand((image.shape[0],) + tuple(model.atlas.shape[1:]))
        loss = loss + (1 - w_img) * ncc(atlas_b, y_target)
    return loss


@pytest.mark.parametrize("name", sorted(TEMPLATE_E2E))
@pytest.mark.parametrize("eng_name", ["bf16", "bf16x3", "f32"])
def test_template_step_end_to_end(vxm, cuda, engine, eng_name, name):
    engine(eng_name)
    kw, B = TEMPLATE_E2E[name]
    model, sd, tcfg, img, mean0 = _template(vxm, cuda, kw, B)
    image = img.to(cuda)
    zeros = torch.zeros((B, len(kw["inshape"])) + tuple(kw["inshape"]), device=cuda)
    loss = _gpu_step_loss(vxm, model, image, zeros, W_IMG)
    loss.backward()
    ref_torch.emulate_bf16(eng_name == "bf16")
    try:
        sdc = {k: v.double().requires_grad_(True) for k, v in sd.items()}
        outs, (m1, n1) = template_ref.template_forward(sdc, tcfg, img.double(), mean0.double(), 3.0)
        atlas_b = sdc["atlas"].expand((B,) + tuple(sdc["atlas"].shape[1:]))
        lc = template_ref.template_loss(outs, atlas_b, img.double(), w_img=W_IMG)
        lc.backward()
    finally:
        ref_torch.emulate_bf16(False)
    vm = model.vxm_model
    errs = {"loss": abs(float(loss) - float(lc)) / abs(float(lc)),
            "atlas.grad": relmax(model.atlas.grad.cpu(), sdc["atlas"].grad),
            "flow.weight.grad": relmax(vm.flow.weight.grad.cpu(), sdc["vxm_model.flow.weight"].grad),
            "mean stream": relmax(model.mean_stream.mean.cpu(), m1.detach())}
    print("\n[template step %s %s B=%d] " % (eng_name, name, B) + ", ".join("%s %.2e" % kv for kv in errs.items())
          + " | bound %.0e, flow.weight.grad %.0e" % (E2E_TOL[eng_name], FLOW_WGRAD_TOL))
    assert float(model.mean_stream.count) == n1 == 3 + B
    assert errs.pop("flow.weight.grad") <= FLOW_WGRAD_TOL
    assert max(errs.values()) <= E2E_TOL[eng_name], errs


# ---- 3. graphed against eager ------------------------------------------------------------------------------------------

LR = 1e-4


def _template_opt_and_loss(vxm, model, zeros):
    opt = vxm.optim.FusedAdam(model.parameters(), lr=LR)         # the weights and the atlas

    def loss_fn(model, image):
        return _gpu_step_loss(vxm, model, image, zeros)
    return opt, loss_fn


# two runs of one build differ by rounding (atomics in the VecInt and warp backward; 3.6e-6 of the parameters at full
# size, DESIGN section 5).  The atlas, whose gradient is large everywhere, stays within a few times that (measured
# 3.1e-6).  Adam scales every element's step to about lr, so a weight whose gradient is at rounding level can step by up
# to lr in either direction in either run: 3 steps bound the weights by 3 lr (measured 1.1e-4).  The mean stream is a
# flow computed from those weights (measured 1.7e-3 of its max-norm)
ATLAS_TOL, WEIGHT_TOL, MEAN_TOL = 1e-5, 3 * LR, 1e-2


def test_graphed_template_step_matches_eager(vxm, cuda, engine):
    engine("bf16")
    from voxelmorph_b200.trainer import GraphedTrainStep
    kw = dict(inshape=(32, 32, 32))
    zeros = torch.zeros((1, 3) + kw["inshape"], device=cuda)
    runs = {}
    for mode in ("eager", "graphed"):
        model, _, _, img, _ = _template(vxm, cuda, kw, 1, seed=5)
        with torch.no_grad():
            model.mean_stream.mean.zero_()
            model.mean_stream.count.zero_()
        image = img.to(cuda)
        opt, loss_fn = _template_opt_and_loss(vxm, model, zeros)
        start = model.atlas.detach().clone()
        if mode == "eager":
            losses = []
            for _ in range(3):
                opt.zero_grad()
                loss = loss_fn(model, image)
                loss.backward()
                opt.step()
                losses.append(float(loss))
        else:
            step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=3).capture(image)
            # the warm-up is rolled back, the mean stream included
            assert torch.equal(model.atlas.detach(), start)
            assert float(model.mean_stream.count) == 0 and float(model.mean_stream.mean.abs().max()) == 0
            losses = [float(step(image)) for _ in range(3)]
        torch.cuda.synchronize()
        assert float(model.mean_stream.count) == 3 and int(opt.step_dev.item()) == 3
        runs[mode] = (losses, model.atlas.detach().clone(), opt.fp.flat.clone(), model.mean_stream.mean.clone())
    (le, ae, pe, me), (lg, ag, pg, mg) = runs["eager"], runs["graphed"]
    d_atlas, d_param, e_mean = float((ag - ae).abs().max()), float((pg - pe).abs().max()), relmax(mg.cpu(), me.cpu())
    print("\n[graphed template step] losses %s vs eager %s | atlas %.2e (bound %.0e), weights and atlas %.2e (bound %.0e), "
          "mean stream %.2e (bound %.0e)" % (lg, le, d_atlas, ATLAS_TOL, d_param, WEIGHT_TOL, e_mean, MEAN_TOL))
    for i in range(3):
        assert abs(lg[i] - le[i]) <= 2e-3 * abs(le[i]), (i, lg, le)
    assert d_atlas <= ATLAS_TOL and d_param <= WEIGHT_TOL and e_mean <= MEAN_TOL


# ---- 4. the full-size graphed step ------------------------------------------------------------------------------------

# library launches the template step adds to the bidirectional learnable-source step with the same losses bar the mean
# term: MeanStream forward and backward, MSE forward and backward, and the backward of the inverse flow's VecInt and x2
# resize (in the plain bidirectional step nothing differentiates neg_flow)
TEMPLATE_EXTRA_LAUNCHES = 6


def _captured_launches(vxm, step, *inputs):
    n0 = vxm._lib.launch_count()
    step.capture(*inputs)
    n1 = vxm._lib.launch_count()
    return n1 - n0, step


def test_full_size_graphed_template_step(vxm, cuda, engine):
    engine("bf16")
    from voxelmorph_b200.trainer import GraphedTrainStep
    shape = (160, 192, 224)
    s, tr = cases.volume_pair(95, shape, sigma=3.0)
    image = t(tr).to(cuda)
    zeros = torch.zeros((1, 3) + shape, device=cuda)
    ncc, grad = vxm.losses.NCC().loss, vxm.losses.Grad("l2", loss_mult=2).loss

    # the bidirectional VxmDense step whose moving image is a learnable Parameter
    torch.manual_seed(0)
    vm = vxm.networks.VxmDense(shape, bidir=True).to(cuda).train()
    src = torch.nn.Parameter(t(s).to(cuda))
    opt_b = vxm.optim.FusedAdam(list(vm.parameters()) + [src], lr=1e-4)

    def bidir_loss(model, image):
        pos, neg, _ = model.flows(src, image)
        y_source = model.transformer(src, pos)
        model.transformer(image, neg)
        return ncc(image, y_source) + grad(None, pos)
    n_bidir, step_b = _captured_launches(vxm, GraphedTrainStep(vm, opt_b, loss_fn=bidir_loss, warmup=2), image)
    del step_b, vm, opt_b, src
    torch.cuda.empty_cache()

    torch.manual_seed(0)
    model = vxm.networks.TemplateCreation(shape).to(cuda).train()
    model.set_atlas(s)
    start = model.atlas.detach().clone()
    opt, loss_fn = _template_opt_and_loss(vxm, model, zeros)
    n_tmpl, step = _captured_launches(vxm, GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=2), image)
    # launches counted over the capture: the warm-up's plus the captured step's, each the same step
    per_bidir, per_tmpl = n_bidir / 3, n_tmpl / 3
    losses = [float(step(image)) for _ in range(3)]
    moved = float((model.atlas.detach() - start).abs().max())
    print("\n[full-size graphed template step] losses %s, atlas moved by up to %.2e, launches per step %g (bidirectional "
          "learnable-source step %g)" % (losses, moved, per_tmpl, per_bidir))
    assert all(np.isfinite(losses)), losses
    assert moved > 0 and float(model.mean_stream.count) == 3
    assert n_tmpl == n_bidir + 3 * TEMPLATE_EXTRA_LAUNCHES, (n_tmpl, n_bidir)
