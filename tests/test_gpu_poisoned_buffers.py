"""Every buffer the library allocates without initialising it must be written before it is read.

The outputs, packed operands, channel-block accumulators and workspaces of the convolution engines and the fp32 kernels
come from torch.empty, including the persistent weight-gradient workspace (tc.WgradBatch.work, 512 MB).  Channels are
padded in many places (2, 3 or 6 planes of an 8-channel tensor, coutp = 16 for 2 to 6 outputs, 9 of 16 channels of the
kd-folded flow gradient, the K padding of transposed head operands, the fp32 accumulator of channel blocks).  In a fresh
process that memory is usually zero or finite, so a kernel that read padding it never wrote, or added into an output it
should overwrite, would pass every other test; in a long run or a CUDA-graph pool it holds other data.

Here torch.empty, torch.empty_like and Tensor.new_empty return tensors with every byte 0xFF (NaN in fp32 and bf16, -1 in
integers), the weight-gradient workspaces are filled with 0xFF, and fresh models are built so that their pack plans are
allocated under the patch; NaN * 0 = NaN, so any such read shows.  torch.zeros is left alone: the reduction and decoder
workspaces are zeroed once by contract and the kernels leave them zeroed.  Each case runs once without and once with the
poison and compares: the U-Net forward and backward on every engine, the fp32 kernels one by one, and one eager training
step of each model family."""
import pytest
import torch

from oracle import cases

LR = 1e-4


def _fill(t):
    """every byte of t's storage 0xFF (bool tensors, whose only valid bytes are 0 and 1, are left as they are)"""
    if t.dtype != torch.bool and t.numel():
        t.untyped_storage().fill_(0xFF)
    return t


def _poison(monkeypatch, device=None):
    empty, empty_like, new_empty = torch.empty, torch.empty_like, torch.Tensor.new_empty
    monkeypatch.setattr(torch, "empty", lambda *a, **k: _fill(empty(*a, **k)))
    monkeypatch.setattr(torch, "empty_like", lambda *a, **k: _fill(empty_like(*a, **k)))
    monkeypatch.setattr(torch.Tensor, "new_empty", lambda self, *a, **k: _fill(new_empty(self, *a, **k)))
    if device is not None:
        from voxelmorph_b200 import tc
        tc.WgradBatch.get(device).work.fill_(0xFF)
        monkeypatch.setattr(tc, "_wgrad_ws", {})          # the wgrad workspaces are allocated again, under the patch


@pytest.fixture()
def poisoned(monkeypatch):
    """call it (with the device, on the GPU) to poison every allocation of the rest of the test"""
    return lambda device=None: _poison(monkeypatch, device)


def test_poison_fills_nan_and_minus_one(poisoned):
    poisoned()
    f32, bf16 = torch.empty(7), torch.empty((2, 3), dtype=torch.bfloat16)
    i32 = torch.empty_like(torch.zeros(5, dtype=torch.int32))
    i64, u8 = torch.zeros(2, dtype=torch.int64).new_empty(4), torch.empty(9, dtype=torch.uint8)
    assert bool(f32.isnan().all()) and bool((f32.view(torch.int32) == -1).all())
    assert bool(bf16.isnan().all()) and bool((bf16.view(torch.int16) == -1).all())
    assert bool((i32 == -1).all()) and bool((i64 == -1).all()) and bool((u8 == 255).all())
    assert bool((torch.zeros(3) == 0).all())


@pytest.fixture(scope="module")
def vxm(cuda):
    import voxelmorph_b200 as v
    v._lib.load()
    return v


def relmax(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


# ---- 1. the U-Net and its head, every engine --------------------------------------------------------------------------

DOUBLED = [[32, 64, 64, 64], [64, 64, 64, 64, 64, 32, 32]]
# name: (constructor, arguments, B)
UNETS = {
    "default": ("VxmDense", dict(inshape=(160, 192, 224)), 1),
    "2d": ("VxmDense", dict(inshape=(192, 224)), 8),
    "halfres": ("VxmDense", dict(inshape=(160, 192, 224), unet_half_res=True), 1),
    "doubled": ("VxmDense", dict(inshape=(64, 96, 112), nb_unet_features=DOUBLED), 1),
    "probs": ("VxmDenseProbabilistic", dict(inshape=(96, 128, 160)), 1),
    "probs_2d": ("VxmDenseProbabilistic", dict(inshape=(192, 224)), 8),
    "template": ("TemplateCreation", dict(inshape=(96, 128, 160)), 1),
    "hyper": ("HyperVxmDense", dict(inshape=(96, 128, 160)), 1),
    "hyper_2d": ("HyperVxmDense", dict(inshape=(192, 224)), 8),
}


def _unet_run(vxm, cuda, name):
    """a fresh model (fixed weights, a head of ordinary size), its U-Net and head on images that ask for their gradient,
    backward with a fixed flow gradient: [flow, every parameter's gradient, the source image's gradient].  A
    HyperVxmDense's parameters include the hypernetwork's, reached through the generated weights' flat gradient."""
    cls, kw, B = UNETS[name]
    torch.manual_seed(3)
    model = getattr(vxm.networks, cls)(**kw)
    net = model.vxm_model if cls == "TemplateCreation" else model
    net = net.to(cuda).train()
    g = torch.Generator(device=cuda).manual_seed(4)
    with torch.no_grad():
        for m in (net.flow, getattr(net, "log_sigma", None)):
            if m is not None:
                m.weight.copy_(torch.randn(m.weight.shape, generator=g, device=cuda) * 0.05)
    planes = net.unet_model.encoder[0][0].main.in_channels
    S = torch.rand((B, 1) + kw["inshape"], generator=g, device=cuda).requires_grad_(True)
    T = torch.rand((B, planes - 1) + kw["inshape"], generator=g, device=cuda)
    if cls == "HyperVxmDense":            # the generated weights (hypernetwork and weight generation) for one lambda
        net._assign(net.hyper(torch.tensor([[0.4]], device=cuda)))
    out = net._head(S, T)
    out.backward(torch.randn(out.shape, generator=g, device=cuda))
    torch.cuda.synchronize()
    return [out.detach()] + [p.grad for p in net.parameters()] + [S.grad]


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["bf16", "bf16x3", "f32"])
@pytest.mark.parametrize("name", sorted(UNETS))
def test_unet_on_poisoned_buffers(vxm, cuda, monkeypatch, poisoned, name, engine):
    """flow, every parameter gradient and the image gradient bit-identical with and without the poison"""
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", engine)
    clean = _unet_run(vxm, cuda, name)
    poisoned(cuda)
    dirty = _unet_run(vxm, cuda, name)
    assert all(t is not None for t in clean) and len(clean) == len(dirty)
    bad = [(i, int((a != b).sum()), int(b.isnan().sum())) for i, (a, b) in enumerate(zip(clean, dirty)) if not torch.equal(a, b)]
    assert not bad, "(output 0 = flow, then the parameters, last the image gradient; mismatches, NaNs): %s" % bad


# ---- 2. the fp32 kernels one by one -------------------------------------------------------------------------------------

def _randn(g, shape, scale=1.0, grad=False):
    return (torch.randn(shape, generator=g, device=g.device) * scale).requires_grad_(grad)


def _rand(g, shape, grad=False):
    return torch.rand(shape, generator=g, device=g.device).requires_grad_(grad)


def k_resize(vxm, g):
    out = []
    for shape, vel_resize in (((1, 3, 80, 96, 112), 2), ((1, 3, 40, 48, 56), 0.5), ((8, 2, 96, 112), 2), ((3, 2, 48, 56), 0.5)):
        x = _randn(g, shape, grad=True)
        y = vxm.layers.ResizeTransform(vel_resize, len(shape) - 2)(x)
        y.backward(_randn(g, y.shape))
        out += [y.detach(), x.grad]
    return out, []


def k_vecint(vxm, g):
    exact, atomic = [], []
    for shape in ((1, 3, 80, 96, 112), (8, 2, 96, 112)):
        v = _randn(g, shape, 2.0, grad=True)
        y = vxm.layers.VecInt(shape[2:], 7)(v)
        y.backward(_randn(g, y.shape))
        exact.append(y.detach())
        atomic.append(v.grad)
    return exact, atomic


def k_warp(vxm, g):
    exact, atomic = [], []
    for shape in ((1, 1, 80, 96, 112), (8, 1, 96, 112)):
        nd = len(shape) - 2
        src, flow = _rand(g, shape, grad=True), _randn(g, (shape[0], nd) + shape[2:], 3.0, grad=True)
        y = vxm.layers.SpatialTransformer(shape[2:])(src, flow)
        y.backward(_randn(g, y.shape))
        exact.append(y.detach())
        atomic += [src.grad, flow.grad]
    return exact, atomic


def k_ncc(vxm, g, wins):
    out = []
    for shape, win in wins:
        I, J = _rand(g, shape, grad=True), _rand(g, shape, grad=True)
        loss = vxm.losses.NCC(win).loss(I, J)
        loss.backward()
        J1 = J.detach().clone().requires_grad_(True)             # the training step's call: d/dJ alone
        loss1 = vxm.losses.NCC(win).loss(I.detach(), J1)
        loss1.backward()
        out += [loss.detach(), I.grad, J.grad, loss1.detach(), J1.grad]
    return out, []


def k_grad(vxm, g):
    out = []
    for shape in ((2, 3, 37, 45, 51), (8, 2, 96, 112)):
        for penalty, mult in (("l1", None), ("l2", 2)):
            y = _randn(g, shape, grad=True)
            loss = vxm.losses.Grad(penalty, loss_mult=mult).loss(None, y)
            loss.backward()
            out += [loss.detach(), y.grad]
    return out, []


def k_mse(vxm, g):
    out = []
    for shape in ((2, 1, 80, 96, 112), (8, 1, 96, 112)):
        a, b = _rand(g, shape, grad=True), _rand(g, shape, grad=True)
        loss = vxm.losses.MSE().loss(a, b)
        loss.backward()
        out += [loss.detach(), a.grad, b.grad]
    return out, []


def k_dice(vxm, g):
    labels = torch.randint(0, 5, (2, 40, 48, 56), generator=g, device=g.device)
    y_true = torch.nn.functional.one_hot(labels, 6).permute(0, 4, 1, 2, 3).float().requires_grad_(True)   # label 5 absent
    y_pred = torch.softmax(_randn(g, (2, 6, 40, 48, 56)), 1).requires_grad_(True)
    loss = vxm.losses.Dice().loss(y_true, y_pred)
    loss.backward()
    return [loss.detach(), y_true.grad, y_pred.grad], []


def k_kl(vxm, g):
    out = []
    for shape in ((2, 6, 40, 48, 56), (8, 4, 96, 112)):
        p = _randn(g, shape, grad=True)
        loss = vxm.losses.KL(10.0).loss(None, p)
        loss.backward()
        out += [loss.detach(), p.grad]
    return out, []


def k_sampler(vxm, g):
    out = []
    for shape in ((2, 6, 40, 48, 56), (8, 4, 96, 112)):
        p = _randn(g, shape, grad=True)
        state = torch.tensor([7, 2], dtype=torch.int64, device=g.device)
        z = vxm.layers.sample_normal_logvar(p, state)
        z.backward(_randn(g, z.shape))
        out += [z.detach(), p.grad, state]
    return out, []


def k_mean_stream(vxm, g):
    out = []
    for shape, B in (((3, 40, 48, 56), 2), ((2, 96, 112), 8)):
        ms = vxm.layers.MeanStream(shape, cap=5).to(g.device).train()
        with torch.no_grad():
            ms.mean.copy_(_randn(g, shape))
            ms.count.fill_(3)
        x = _randn(g, (B,) + shape, grad=True)
        y = ms(x)
        y.backward(_randn(g, y.shape))
        out += [y.detach(), ms.mean, ms.count, x.grad]
    return out, []


def k_decoder(vxm, g):
    """the phenotype decoder forward, its backward into fresh tensors (autograd) and into FusedAdam's flat views"""
    dec = vxm.layers.PhenoDecoder(3, 8, (40, 48, 56)).to(g.device)
    with torch.no_grad():
        for p in dec.parameters():
            p.copy_(_randn(g, p.shape, 0.3))
    pheno, gout = _randn(g, (2, 3)), _randn(g, (2, 8, 40, 48, 56))
    y = dec(pheno)
    y.backward(gout)
    out = [y.detach()] + [p.grad for p in dec.parameters()]
    fp = vxm.optim.FlatParams(list(dec.parameters()))
    fp.zero_grad()
    dec(pheno).backward(gout)
    return out + [fp.grad.clone()], []


def k_hyper(vxm, g):
    """the hypernetwork and weight generation forward (pre, h and the generated buffer), the backward into fresh tensors
    (autograd; dh and its partial workspace) and into FusedAdam's flat views behind a 1-float pad (unaligned, 4-byte
    loads; 16-byte loads for the fresh tensors, N = 14 736), U = 37 (the unrolled rows' tail)"""
    mod = vxm.layers.HyperWeights([(16, 2, 3, 3, 3), (32, 16, 3, 3, 3)], 3, 4, 37).to(g.device)
    with torch.no_grad():
        for p in mod.parameters():
            p.copy_(_randn(g, p.shape, 0.3))
    hyp, gout = _rand(g, (1, 3)), _randn(g, mod.hyper_bias.shape)
    w = mod(hyp)
    out = [w.detach().clone()]
    w.backward(gout)
    out += [p.grad for p in mod.parameters()]
    fp = vxm.optim.FlatParams([torch.nn.Parameter(torch.zeros(1, device=g.device))] + list(mod.parameters()))
    fp.zero_grad()
    mod(hyp).backward(gout)
    return out + [fp.grad.clone()], []


def k_jacdet(vxm, g):
    out = []
    for shape in ((2, 3, 40, 48, 56), (8, 2, 96, 112)):
        det, folds = vxm.utils.jacobian_determinant_device(_randn(g, shape, 0.5), return_folds=True)
        out += [det, torch.tensor(folds)]
    return out, []


KERNELS = {
    "resize": k_resize, "vecint": k_vecint, "warp": k_warp,
    "ncc9": lambda vxm, g: k_ncc(vxm, g, [((1, 1, 80, 96, 112), None), ((8, 1, 96, 112), None)]),
    "ncc_generic": lambda vxm, g: k_ncc(vxm, g, [((2, 1, 45, 70, 121), (5, 9, 7)), ((3, 1, 64, 80), (5, 5))]),
    "grad": k_grad, "mse": k_mse, "dice": k_dice, "kl": k_kl, "sampler": k_sampler, "mean_stream": k_mean_stream,
    "decoder": k_decoder, "jacdet": k_jacdet, "hyper": k_hyper,
}
# the VecInt and warp backwards scatter with atomics, so two runs differ in the last bits: each is within 1e-5 of the fp64
# adjoint in its own test (test_gpu_fp32_step_kernels.py, test_gpu_fp32_other_paths.py), so two runs within twice that
ATOMIC_TOL = 2e-5


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_fp32_kernel_on_poisoned_buffers(vxm, cuda, poisoned, kernel):
    """deterministic outputs and gradients bit-identical with and without the poison; the gradients summed with atomics
    NaN-free and within ATOMIC_TOL"""
    clean = KERNELS[kernel](vxm, torch.Generator(device=cuda).manual_seed(5))
    poisoned(cuda)
    dirty = KERNELS[kernel](vxm, torch.Generator(device=cuda).manual_seed(5))
    torch.cuda.synchronize()
    bad = [(i, int((a != b).sum()), int(b.isnan().sum())) for i, (a, b) in enumerate(zip(clean[0], dirty[0])) if not torch.equal(a, b)]
    assert len(clean[0]) == len(dirty[0]) and not bad, "(output, mismatches, NaNs): %s" % bad
    errs = [relmax(b, a) if bool(b.isfinite().all()) else float("inf") for a, b in zip(clean[1], dirty[1])]
    print("\n[poisoned %s] %d outputs bit-identical; atomic gradients rel err %s (bound %.0e)" % (kernel, len(clean[0]), errs, ATOMIC_TOL))
    assert all(e <= ATOMIC_TOL for e in errs), errs


# ---- 3. one eager training step of each model family ------------------------------------------------------------------

STEP_SHAPE = (32, 32, 48)
# the graphed-vs-eager step tests' tolerances (test_gpu_template.py): losses within 2e-3, and the weights within 3 lr, since
# Adam scales each element's step to about lr whatever the size of its gradient, and the VecInt and warp atomics make the
# gradients of two runs differ at rounding level
LOSS_TOL, WEIGHT_TOL = 2e-3, 3 * LR


def _step(vxm, cuda, family):
    torch.manual_seed(21)
    s, t = cases.volume_pair(23, STEP_SHAPE, sigma=1.5)
    S, T = torch.from_numpy(s).to(cuda), torch.from_numpy(t).to(cuda)
    mse, ncc, grad = vxm.losses.MSE().loss, vxm.losses.NCC().loss, vxm.losses.Grad("l2", loss_mult=2).loss
    zeros = torch.zeros((1, 3) + STEP_SHAPE, device=cuda)
    if family == "vxm":
        model = vxm.networks.VxmDense(STEP_SHAPE)
    elif family == "probs":
        model = vxm.networks.VxmDenseProbabilistic(STEP_SHAPE)
        model.noise_state.copy_(torch.tensor([5, 0]))
    elif family == "template":
        model = vxm.networks.TemplateCreation(STEP_SHAPE)
        model.set_atlas(torch.from_numpy(s))
    elif family == "hyper":
        model = vxm.networks.HyperVxmDense(STEP_SHAPE)
    else:
        model = vxm.networks.ConditionalTemplateCreation(STEP_SHAPE, (2,), conv_nb_features=4)
    model = model.to(cuda).train()
    opt = vxm.optim.FusedAdam(model.parameters(), lr=LR)
    opt.zero_grad()
    if family == "vxm":
        y, flow = model(S, T)
        loss = ncc(T, y) + 0.01 * grad(None, flow)
    elif family == "probs":
        y, params = model(S, T)
        loss = vxm.losses.MSE(0.02).loss(T, y) + 0.01 * vxm.losses.KL(10.0).loss(None, params)
    elif family == "template":
        y_source, y_target, ms, pos = model(T)
        loss = 0.5 * ncc(T, y_source) + 0.5 * ncc(model.atlas, y_target) + mse(zeros, ms) + 0.01 * grad(None, pos)
    elif family == "hyper":
        hyp = torch.tensor([[0.3]], device=cuda)
        y, flow = model(S, T, hyp)
        loss = vxm.losses.hyper_loss(hyp, ncc(T, y), grad(None, flow))
    else:
        y_source, ms, pos, _ = model(torch.tensor([[0.3, -1.0]], device=cuda), S, T)
        loss = ncc(T, y_source) + mse(zeros, ms) + grad(None, pos) + 0.01 * mse(zeros, pos)
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    return float(loss), opt.fp.flat.clone()


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["vxm", "probs", "template", "cond_template", "hyper"])
def test_training_step_on_poisoned_buffers(vxm, cuda, monkeypatch, poisoned, family):
    """one bf16 step with FusedAdam and the family's own losses: loss and updated flat parameters finite and within the step
    tests' tolerances of the unpoisoned step"""
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "bf16")
    l0, p0 = _step(vxm, cuda, family)
    poisoned(cuda)
    l1, p1 = _step(vxm, cuda, family)
    d = float((p1 - p0).abs().max())
    print("\n[poisoned step %s] loss %.6f vs %.6f | parameters max |diff| %.2e (bound %.0e)" % (family, l1, l0, d, WEIGHT_TOL))
    assert bool(p1.isfinite().all()) and abs(l1 - l0) <= LOSS_TOL * abs(l0) and d <= WEIGHT_TOL
