"""ConditionalTemplateCreation on the GPU: the phenotype decoder kernels against the fp64 restatement
(tests/cond_template_ref.py), their determinism, flat-gradient path and refusals, the conditional template step end to end
on every engine against fp64 autograd, a graphed step against an eager one, and the full-size graphed step.  Run with -s
to see every measured error next to its bound."""
import math

import numpy as np
import pytest
import torch

from oracle import cases, ref_torch

import cond_template_ref
from test_gpu_fp32_step_kernels import report
from test_gpu_image_grads import E2E_TOL, relmax, t
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


# ---- 1. the decoder kernels -------------------------------------------------------------------------------------------

# (vol, P, F, B): the script's configuration at full size, then 2-D and a ragged volume over F in {1, 3, 8, 32} and
# P in {1, 3, 16}; B = 5 runs the batch in two chunks
DEC_CASES = {
    "full-b1": ((160, 192, 224), 2, 4, 1),
    "full-b2": ((160, 192, 224), 2, 4, 2),
    "2d-p1-f1": ((192, 224), 1, 1, 2),
    "2d-p3-f8": ((192, 224), 3, 8, 3),
    "2d-p16-f32": ((192, 224), 16, 32, 2),
    "ragged-p16-f3": ((13, 17, 19), 16, 3, 5),
    "ragged-p3-f32": ((13, 17, 19), 3, 32, 3),
    "ragged-p1-f8": ((13, 17, 19), 1, 8, 1),
}


def _dec_inputs(vxm, cuda, vol, P, F, B, seed=0):
    """A decoder with both ELU branches in use, its pheno and an output gradient."""
    g = torch.Generator(device=cuda).manual_seed(seed)
    dec = vxm.layers.PhenoDecoder(P, F, vol).to(cuda)
    with torch.no_grad():
        dec.weight.copy_(torch.randn(dec.weight.shape, generator=g, device=cuda) / math.sqrt(P))
        dec.bias.copy_(0.5 * torch.randn(dec.bias.shape, generator=g, device=cuda))
        dec.like_weight.copy_(torch.randn(dec.like_weight.shape, generator=g, device=cuda) / math.sqrt(F))
        dec.like_bias.copy_(torch.randn(dec.like_bias.shape, generator=g, device=cuda))
    pheno = torch.randn(B, P, generator=g, device=cuda)
    gout = torch.randn((B, F) + tuple(vol), generator=g, device=cuda)
    return dec, pheno, gout


def _dec_run(dec, pheno, gout):
    for p in dec.parameters():
        p.grad = None
    out = dec(pheno)
    out.backward(gout)
    return [out.detach()] + [p.grad.clone() for p in dec.parameters()]


def _bwd_chain(vxm, V, B, F):
    """Longest per-thread fp32 chain of the backward's voxel sums: at least 32 threads in each of min(V / 32, 4 SMs) CTAs"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return math.ceil(V / min(V, 4 * sms * 32)) * B


@pytest.mark.parametrize("name", sorted(DEC_CASES))
def test_decoder_kernels_vs_fp64(vxm, cuda, name):
    vol, P, F, B = DEC_CASES[name]
    dec, pheno, gout = _dec_inputs(vxm, cuda, vol, P, F, B)
    out, gW, gb, glw, glb = _dec_run(dec, pheno, gout)
    # the restatement in fp64 (on the device), and the magnitudes the fp32 roundings scale with
    W, bias, lw, lb = [p.detach().double().requires_grad_(True) for p in dec.parameters()]
    ph, go = pheno.double(), gout.double()
    want = cond_template_ref.decoder(ph, W, bias, lw, lb)
    want.backward(go)
    with torch.no_grad():
        lw2, aph = lw.reshape(F, F).abs(), ph.abs()
        h_abs = bias.abs().unsqueeze(0) + torch.einsum("bp,pf...->bf...", aph, W.abs())        # >= |pre| >= |h|
        a_out = lb.abs().reshape((1, F) + (1,) * len(vol)) + torch.einsum("gf,bf...->bg...", lw2, h_abs)
        g_abs = torch.einsum("gf,bg...->bf...", lw2, go.abs()) * (1 + h_abs)                   # >= |g_pre|, error scale
        a_gw, a_gb = torch.einsum("bp,bf...->pf...", aph, g_abs), g_abs.sum(0)
        a_glw = torch.einsum("bg...,bf...->gf", go.abs(), h_abs).reshape(lw.shape)
        a_glb = go.abs().sum(dim=tuple(i for i in range(go.dim()) if i != 1))
        n = _bwd_chain(vxm, int(np.prod(vol)), B, F)

        def ratio(got, ref, scale):
            return float(((got.double() - ref).abs() / scale.clamp_min(1e-300)).max())
        tag = "decoder %s %s P=%d F=%d B=%d" % (name, vol, P, F, B)
        # forward: P-term fma chain, expm1f (2 ulp), F-term fma chain; backward: the forward's pre and h, an F-term chain
        # for g_h, the ELU derivative, then B terms for gW / gbias, or an n-term fp32 chain, a 5-level warp tree and one
        # rounding to fp32 for the voxel sums
        report(tag + " out", ratio(out, want, a_out), (P + F + 4) * U)
        report(tag + " dW", ratio(gW, W.grad, a_gw), (P + F + B + 8) * U)
        report(tag + " dbias", ratio(gb, bias.grad, a_gb), (P + F + B + 8) * U)
        report(tag + " dlike_w", ratio(glw, lw.grad, a_glw), (n + P + 12) * U)
        report(tag + " dlike_b", ratio(glb, lb.grad, a_glb), (n + 8) * U)


@pytest.mark.parametrize("name", ["full-b2", "2d-p16-f32", "ragged-p16-f3"])
def test_decoder_is_deterministic(vxm, cuda, name):
    vol, P, F, B = DEC_CASES[name]
    dec, pheno, gout = _dec_inputs(vxm, cuda, vol, P, F, B, seed=3)
    a, b = _dec_run(dec, pheno, gout), _dec_run(dec, pheno, gout)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("name", ["full-b1", "ragged-p3-f32", "ragged-p16-f3"])
def test_decoder_flat_grads_equal_autograd(vxm, cuda, name):
    """FusedAdam's flat views receive the autograd path's gradients bit for bit, and a second backward accumulates."""
    vol, P, F, B = DEC_CASES[name]
    dec, pheno, gout = _dec_inputs(vxm, cuda, vol, P, F, B, seed=4)
    want = _dec_run(dec, pheno, gout)[1:]
    opt = vxm.optim.FusedAdam(dec.parameters(), lr=1e-3)
    opt.zero_grad()
    flat = [p.grad for p in dec.parameters()]
    dec(pheno).backward(gout)
    assert all(p.grad is g for p, g in zip(dec.parameters(), flat))          # written in place, autograd got None
    assert all(torch.equal(g, w) for g, w in zip(flat, want))
    dec(pheno).backward(gout)
    # the voxel-summed gradients add their total once; gW and gbias add the batch sum at once when the batch fits the
    # kernel's register chunk (64 / F entries, rounded down to 1, 2 or 4) and chunk by chunk otherwise
    chunk = min(4, 64 // next(m for m in (4, 8, 16, 32) if F <= m))
    for i, (g, w) in enumerate(zip(flat, want)):
        if i >= 2 or B <= chunk:
            assert torch.equal(g, w + w), i
        else:
            assert relmax(g, w + w) <= 4 * U, i


def test_decoder_reports_bad_arguments(vxm, cuda):
    lib, L = vxm._lib.load(), vxm._lib
    x = torch.zeros(64, device=cuda)
    ws = torch.zeros(int(lib.vxm_pheno_decoder_workspace_bytes(4)), dtype=torch.uint8, device=cuda)
    args = [L.ptr(x)] * 6
    assert lib.vxm_pheno_decoder_fwd(*args, 1, 17, 4, 8, L.stream_ptr()) != 0 and "P = 17" in L.last_error()
    assert lib.vxm_pheno_decoder_fwd(*args, 1, 2, 33, 8, L.stream_ptr()) != 0 and "F = 33" in L.last_error()
    assert lib.vxm_pheno_decoder_fwd(*args, 0, 2, 4, 8, L.stream_ptr()) != 0 and "non-positive" in L.last_error()
    bargs = [L.ptr(x)] * 9 + [L.ptr(ws)]
    assert lib.vxm_pheno_decoder_bwd(*bargs, 1, 2, 40, 8, 0, L.stream_ptr()) != 0 and "1 to 32" in L.last_error()
    assert lib.vxm_pheno_decoder_bwd(*bargs, 1, 2, 4, 8, 2, L.stream_ptr()) != 0 and "accumulate" in L.last_error()
    bargs[0] = None
    assert lib.vxm_pheno_decoder_bwd(*bargs, 1, 2, 4, 8, 0, L.stream_ptr()) != 0 and "null pointer" in L.last_error()
    assert lib.vxm_pheno_decoder_workspace_bytes(33) == 0
    dec = vxm.layers.PhenoDecoder(2, 4, (4, 5, 6)).to(cuda)
    with pytest.raises(L.VxmError, match="does not match"):
        dec(torch.zeros(1, 3, device=cuda))
    with pytest.raises(L.VxmError, match="CUDA tensors"):
        dec(torch.zeros(1, 2))


# ---- 2. the conditional template step end to end ---------------------------------------------------------------------

COND_E2E = {
    "3d": (dict(inshape=(32, 32, 48)), 1),
    "b2-3d": (dict(inshape=(32, 32, 48)), 2),
    "b2-2d": (dict(inshape=(32, 48), int_steps=5), 2),
}
CAP, P_ATTR, F_GEN = 5.0, 2, 4
# the flow field's bound per engine, as smoke() and test_gpu_probabilistic.STEP_TOL hold it: bf16 operands move the flow
# by up to 2e-2 of its max-norm (the moved image far less)
FLOW_TOL = {"f32": 1e-4, "bf16x3": 1e-4, "bf16": 2e-2}


def _cond(vxm, cuda, kw, B, seed=77):
    """GPU model and fp64 oracle state on the same parameters.  The generator is scaled up from its N(0, 1e-7) output
    layer so that the template depends on the attributes; the mean stream starts part-way (count 3, a random mean)."""
    cfg = full_cfg(dict(kw, bidir=True))
    shape = kw["inshape"]
    torch.manual_seed(seed)
    model = vxm.networks.ConditionalTemplateCreation(pheno_input_shape=(P_ATTR,), conv_nb_features=F_GEN, mean_cap=CAP, **kw)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        model.pheno_decoder.bias.copy_(0.3 * torch.randn(model.pheno_decoder.bias.shape, generator=g))
        model.pheno_decoder.weight.mul_(30.0)
        model.atlas_gen.weight.copy_(0.05 * torch.randn(model.atlas_gen.weight.shape, generator=g))
        model.mean_stream.mean.copy_(0.1 * torch.randn(model.mean_stream.mean.shape, generator=g))
        model.mean_stream.count.fill_(3)
    sd = {k: v.clone() for k, v in model.state_dict().items() if not k.startswith("mean_stream")}
    sd.update({"vxm_model." + k: v for k, v in ref_torch.init_state_dict(cfg, seed=seed, flow_std=2e-2).items()})
    model.load_state_dict(sd, strict=False)
    s, _ = cases.volume_pair(93, shape, sigma=1.5)
    imgs = np.concatenate([cases.volume_pair(94 + b, shape, sigma=1.5)[1] for b in range(B)], axis=0)
    pheno = torch.randn(B, P_ATTR, generator=g)
    return model.to(cuda).train(), sd, cfg, pheno, t(s), t(imgs), model.mean_stream.mean.detach().cpu().clone()


def _gpu_loss(vxm, outs, image, zeros):
    """train_cond_template.py's loss: NCC(image, y_source) + MSE(0, mean_stream) + Grad('l2', 2)(pos) + 0.01 MSE(0, pos)"""
    y_source, ms, pos, _ = outs
    mse = vxm.losses.MSE().loss
    return vxm.losses.NCC().loss(image, y_source) + mse(zeros, ms) + vxm.losses.Grad("l2", loss_mult=2).loss(None, pos) \
        + 0.01 * mse(zeros, pos)


@pytest.mark.parametrize("name", sorted(COND_E2E))
@pytest.mark.parametrize("eng_name", ["bf16", "bf16x3", "f32"])
def test_cond_template_step_end_to_end(vxm, cuda, engine, eng_name, name):
    engine(eng_name)
    kw, B = COND_E2E[name]
    model, sd, cfg, pheno, atlas, img, mean0 = _cond(vxm, cuda, kw, B)
    zeros = torch.zeros((B, len(kw["inshape"])) + tuple(kw["inshape"]), device=cuda)
    outs = model(pheno.to(cuda), atlas.to(cuda), img.to(cuda))
    assert len(outs) == 4 and outs[2] is outs[3]
    loss = _gpu_loss(vxm, outs, img.to(cuda), zeros)
    loss.backward()
    ref_torch.emulate_bf16(eng_name == "bf16")
    try:
        sdc = {k: v.double().requires_grad_(True) for k, v in sd.items()}
        ref, (m1, n1), atlas_t = cond_template_ref.cond_template_forward(sdc, cfg, pheno.double(), atlas.double(),
                                                                          img.double(), mean0.double(), 3.0, CAP)
        lc = cond_template_ref.cond_template_loss(ref, img.double())
        lc.backward()
    finally:
        ref_torch.emulate_bf16(False)
    params = dict(model.named_parameters())
    errs = {"loss": abs(float(loss.detach()) - float(lc)) / abs(float(lc)),
            "y_source": relmax(outs[0].detach().cpu(), ref[0].detach()),
            "mean stream": relmax(model.mean_stream.mean.cpu(), m1.detach())}
    for k in ("pheno_decoder.weight", "pheno_decoder.bias", "pheno_decoder.like_weight", "pheno_decoder.like_bias"):
        errs[k] = relmax(params[k].grad.cpu(), sdc[k].grad)
    wgrad = {k: relmax(params[k].grad.cpu(), sdc[k].grad) for k in params
             if k.startswith(("extra_convs.", "atlas_gen.")) or k == "vxm_model.flow.weight"}
    print("\n[cond template step %s %s B=%d] " % (eng_name, name, B) + ", ".join("%s %.2e" % kv for kv in errs.items())
          + " | bound %.0e; weight gradients %s, bound %.0e" % (E2E_TOL[eng_name], ", ".join("%s %.2e" % kv for kv in wgrad.items()),
                                                               FLOW_WGRAD_TOL))
    assert float(model.mean_stream.count) == n1 == 3 + B
    assert max(errs.values()) <= E2E_TOL[eng_name], errs
    assert max(wgrad.values()) <= FLOW_WGRAD_TOL, wgrad
    # registration form and the template alone
    model.eval()
    y_reg, pos_reg = model(pheno.to(cuda), atlas.to(cuda), img.to(cuda), registration=True)
    tmpl = model.template(pheno.to(cuda), atlas.to(cuda))
    assert not tmpl.requires_grad and float(model.mean_stream.count) == 3 + B
    e_reg, e_flow = relmax(y_reg.detach().cpu(), ref[0].detach()), relmax(pos_reg.detach().cpu(), ref[2].detach())
    e_tmpl = relmax(tmpl.cpu(), atlas_t.detach())
    print("[cond template %s %s] registration y_source %.2e, pos_flow %.2e (bound %.0e), template %.2e"
          % (eng_name, name, e_reg, e_flow, FLOW_TOL[eng_name], e_tmpl))
    assert e_reg <= E2E_TOL[eng_name] and e_flow <= FLOW_TOL[eng_name] and e_tmpl <= 1e-5


# ---- 3. graphed against eager ------------------------------------------------------------------------------------------

LR = 1e-4
# as test_gpu_template: Adam moves a weight whose gradient is at rounding level by up to lr per step in either run (3 lr
# over 3 steps); the mean stream is a flow computed from those weights
WEIGHT_TOL, MEAN_TOL = 3 * LR, 1e-2


def _opt_and_loss(vxm, model, zeros):
    opt = vxm.optim.FusedAdam(model.parameters(), lr=LR)

    def loss_fn(model, pheno, atlas, image):
        return _gpu_loss(vxm, model(pheno, atlas, image), image, zeros)
    return opt, loss_fn


def test_graphed_cond_template_step_matches_eager(vxm, cuda, engine):
    engine("bf16")
    from voxelmorph_b200.trainer import GraphedTrainStep
    kw = dict(inshape=(32, 32, 32))
    zeros = torch.zeros((1, 3) + kw["inshape"], device=cuda)
    runs = {}
    for mode in ("eager", "graphed"):
        model, _, _, pheno, atlas, img, _ = _cond(vxm, cuda, kw, 1, seed=5)
        with torch.no_grad():
            model.mean_stream.mean.zero_()
            model.mean_stream.count.zero_()
        inputs = (pheno.to(cuda), atlas.to(cuda), img.to(cuda))
        opt, loss_fn = _opt_and_loss(vxm, model, zeros)
        start = opt.fp.flat.clone()
        if mode == "eager":
            losses = []
            for _ in range(3):
                opt.zero_grad()
                loss = loss_fn(model, *inputs)
                loss.backward()
                opt.step()
                losses.append(float(loss))
        else:
            step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=3).capture(*inputs)
            # the warm-up is rolled back, the mean stream included
            assert torch.equal(opt.fp.flat, start)
            assert float(model.mean_stream.count) == 0 and float(model.mean_stream.mean.abs().max()) == 0
            losses = [float(step(*inputs)) for _ in range(3)]
        torch.cuda.synchronize()
        assert float(model.mean_stream.count) == 3 and int(opt.step_dev.item()) == 3
        runs[mode] = (losses, opt.fp.flat.clone(), model.mean_stream.mean.clone(), model.pheno_decoder.weight.detach().clone())
    (le, pe, me, de), (lg, pg, mg, dg) = runs["eager"], runs["graphed"]
    d_param, d_dec, e_mean = float((pg - pe).abs().max()), float((dg - de).abs().max()), relmax(mg.cpu(), me.cpu())
    print("\n[graphed cond template step] losses %s vs eager %s | weights %.2e, decoder weight %.2e (bound %.0e), mean "
          "stream %.2e (bound %.0e)" % (lg, le, d_param, d_dec, WEIGHT_TOL, e_mean, MEAN_TOL))
    for i in range(3):
        assert abs(lg[i] - le[i]) <= 2e-3 * abs(le[i]), (i, lg, le)
    assert d_param <= WEIGHT_TOL and e_mean <= MEAN_TOL


# ---- 4. the full-size graphed step ------------------------------------------------------------------------------------

def test_full_size_graphed_cond_template_step(vxm, cuda, engine):
    engine("bf16")
    from voxelmorph_b200.trainer import GraphedTrainStep
    shape = (160, 192, 224)
    s, tr = cases.volume_pair(95, shape, sigma=3.0)
    zeros = torch.zeros((1, 3) + shape, device=cuda)
    torch.manual_seed(0)
    model = vxm.networks.ConditionalTemplateCreation(shape, (2,), conv_nb_features=4).to(cuda).train()
    opt, loss_fn = _opt_and_loss(vxm, model, zeros)
    pheno = torch.tensor([[0.3, -1.0]], device=cuda)
    start = model.pheno_decoder.weight.detach().clone()
    step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=2).capture(pheno, t(s).to(cuda), t(tr).to(cuda))
    losses = [float(step(pheno, t(s).to(cuda), t(tr).to(cuda))) for _ in range(3)]
    moved = float((model.pheno_decoder.weight.detach() - start).abs().max())
    print("\n[full-size graphed cond template step] losses %s, decoder weight moved by up to %.2e" % (losses, moved))
    assert all(np.isfinite(losses)), losses
    assert moved > 0 and float(model.mean_stream.count) == 3
