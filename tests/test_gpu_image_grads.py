"""The gradients the registration step owes its IMAGES: the first convolution's dgrad on the tensor-core engine (exact
tier), source.grad / target.grad end to end on every engine against fp64 autograd of oracle/ref_torch, NCC and Dice
differentiated w.r.t. y_true, and the checks that a step whose images need no gradient runs as before.  Run with -s to see
every measured error next to its bound."""
import numpy as np
import pytest
import torch

from oracle import cases, ref_torch, spec_np

import conv_exact_ref as ref
import image_grads_ref
from test_gpu_fp32_step_kernels import _ncc_fp32, _pair, rel, report
from test_oracle import full_cfg

pytestmark = pytest.mark.gpu

DOUBLED = [[32, 64, 64, 64], [64, 64, 64, 64, 64, 32, 32]]
WIDE64 = [[64, 64, 64, 64], [64, 64, 64, 64, 64, 64, 64]]


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def relmax(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


@pytest.fixture(scope="module")
def vx(cuda):
    import voxelmorph_b200 as vxm
    from voxelmorph_b200 import engine_bf16, tc
    vxm._lib.load()
    return vxm, engine_bf16, tc


@pytest.fixture()
def engine(monkeypatch):
    def set_engine(name):
        monkeypatch.setenv("VXM_B200_CONV_ENGINE", name)
    yield set_engine
    ref_torch.emulate_bf16(False)


# ---- 1. the first convolution's dgrad into the image planes, exactly ---------------------------------------------------

def ternary(shape, g):
    nz = torch.randint(0, 2, shape, generator=g, device=g.device)
    return (nz * (2 * torch.randint(0, 2, shape, generator=g, device=g.device) - 1)).to(torch.bfloat16)


def _first_dgrad_mismatches(vx, cuda, kw, B, seed):
    """The plan's own image dgrad (form, lazily built operand, launch) of VxmDense(**kw) on a gradient in {-1, 0, 1} and
    weights 2^-6 k, |k| <= 8: every fp32 sum is exact whatever its order, so the fp32 planes must EQUAL the fp64 tap sums."""
    vxm, eng, tc = vx
    g = torch.Generator(device=cuda).manual_seed(seed)
    model = vxm.networks.VxmDense(**kw).to(cuda)
    first = model.unet_model.encoder[0][0].main
    with torch.no_grad():
        first.weight.copy_(torch.randint(-8, 9, first.weight.shape, generator=g, device=cuda).float() * 2.0 ** -6)
    plan = eng._plan_of(model, False)
    L = plan.layers[0]
    assert L.role == "first" and L.dgrad is None and L.dgrad_img is not None
    shape = tuple(kw["inshape"])
    kd = 3 if len(shape) == 3 else 1
    vol = shape if kd == 3 else (1,) + shape
    gz = ternary((B,) + vol + (L.cout,), g)
    out = eng._run(L.dgrad_img, plan.image_dgrad_packs(), gz, None, L.cin, kd, out_fp32_planar=True)
    torch.cuda.synchronize()
    assert out.shape == (B, L.cin) + vol and out.dtype == torch.float32
    # |partial sums| <= 27 taps x cout channels x 8 units of 2^-6: far below the 2^22 units the exact tier allows
    assert 27 * L.cout * 8 < 2 ** 22
    w5 = first.weight.detach() if kd == 3 else first.weight.detach().unsqueeze(2)
    got = out.permute(0, 2, 3, 4, 1)
    n = sum(ref.conv([(gz, False)], ref.dgrad_weight(w5), vol[0],
                     finish=lambda y, d0, d1: int((got[:, d0:d1] != y.float()).sum())))
    return n, L


FIRST_CASES = {
    "16to2-full": (dict(inshape=(160, 192, 224)), 1),
    "32to2": (dict(inshape=(64, 96, 112), nb_unet_features=DOUBLED), 1),
    "64to2": (dict(inshape=(64, 96, 112), nb_unet_features=WIDE64), 1),
    "16to3": (dict(inshape=(32, 48, 64), src_feats=2, trg_feats=1), 1),
    "16to8": (dict(inshape=(32, 48, 64), src_feats=4, trg_feats=4), 2),
    "64to8": (dict(inshape=(16, 32, 48), nb_unet_features=WIDE64, src_feats=4, trg_feats=4), 1),
    "2d-16to2": (dict(inshape=(192, 224)), 2),
    "2d-64to3": (dict(inshape=(96, 112), nb_unet_features=WIDE64, src_feats=1, trg_feats=2), 2),
}


@pytest.mark.parametrize("name", sorted(FIRST_CASES))
def test_first_layer_image_dgrad_exact(vx, cuda, name):
    kw, B = FIRST_CASES[name]
    n, L = _first_dgrad_mismatches(vx, cuda, kw, B, 11 + len(name))
    print("\n[image dgrad %s] %d -> %d planes, form %s: %d mismatches" % (name, L.cout, L.cin, L.dgrad_img, n))
    assert n == 0


@pytest.mark.parametrize("ctas", ["1", "5", None])
def test_first_layer_image_dgrad_exact_ragged_under_cta_caps(vx, cuda, monkeypatch, ctas):
    """A ragged shape (partial tiles along h and w, odd depth is not poolable so the model is 2 levels deep) with B = 2, the
    persistent grid capped at 1 and 5 CTAs (many items per CTA, other depth chunkings) and uncapped."""
    if ctas is None:
        monkeypatch.delenv("VXM_B200_CONV_CTAS", raising=False)
    else:
        monkeypatch.setenv("VXM_B200_CONV_CTAS", ctas)
    kw = dict(inshape=(22, 42, 134), nb_unet_features=[[16], [16, 16]], src_feats=1, trg_feats=2)
    n, _ = _first_dgrad_mismatches(vx, cuda, kw, 2, 5)
    assert n == 0


# ---- 2. / 3. source.grad and target.grad end to end ------------------------------------------------------------------

E2E = {
    "default3d": dict(inshape=(32, 32, 48)),
    "doubled3d": dict(inshape=(16, 32, 32), nb_unet_features=DOUBLED),
    "default2d": dict(inshape=(64, 64)),
    "bidir2d": dict(inshape=(32, 48), bidir=True, int_steps=5),
}
# max-norm bounds on the image gradients of the step's loss.  The tensor-core engines (bf16-operand backward, gradients
# stored in bf16 between layers) measure <= 1.8e-4 on the models below, the bound is ten times that; most of this gradient
# reaches the images through the warp and the NCC directly, the part through the U-Net alone is held to UNET_PATH_L2 below.
# The f32 engine meets 1e-4 (measured <= 1.7e-5)
E2E_TOL = {"bf16": 2e-3, "bf16x3": 2e-3, "f32": 1e-4}


def _step_loss(lib, out, S, T, bidir):
    """NCC(target, y_source) + 0.01 Grad(preint_flow) (+ NCC(source, y_target) when both images are warped); `lib` is the
    package's losses or the oracle's functions"""
    ncc, grad = lib
    loss = ncc(T, out[0]) + 0.01 * grad(out[-1])
    if bidir:
        loss = loss + ncc(S, out[1])
    return loss


def _gpu_losses(vxm):
    return vxm.losses.NCC().loss, lambda f: vxm.losses.Grad("l2", loss_mult=2).loss(None, f)


_ORACLE = (ref_torch.ncc_loss, lambda f: ref_torch.grad_loss(f, "l2", 2))


def _oracle_image_grads(sd, cfg, s, tr, emulate):
    """fp64 autograd of the reference restatement; `emulate`: bf16 storage emulated where the bf16 engine stores bf16"""
    ref_torch.emulate_bf16(emulate)
    try:
        sdc = {k: v.double() for k, v in sd.items()}
        Sc, Tc = t(s).double().requires_grad_(True), t(tr).double().requires_grad_(True)
        out = ref_torch.vxm_forward(sdc, cfg, Sc, Tc)
        _step_loss(_ORACLE, out, Sc, Tc, cfg.get("bidir", False)).backward()
    finally:
        ref_torch.emulate_bf16(False)
    return Sc.grad, Tc.grad


def _model(vxm, cuda, kw, seed=77):
    cfg = full_cfg(kw)
    sd = ref_torch.init_state_dict(cfg, seed=seed, flow_std=2e-2)
    model = vxm.networks.VxmDense(**kw)
    model.load_state_dict(sd, strict=False)
    return model.to(cuda).train(), sd, cfg


@pytest.mark.parametrize("name", sorted(E2E))
@pytest.mark.parametrize("eng_name", ["bf16", "bf16x3", "f32"])
def test_image_gradients_end_to_end(vx, cuda, engine, eng_name, name):
    vxm = vx[0]
    engine(eng_name)
    kw = E2E[name]
    model, sd, cfg = _model(vxm, cuda, kw)
    s, tr = cases.volume_pair(93, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda).requires_grad_(True), t(tr).to(cuda).requires_grad_(True)
    _step_loss(_gpu_losses(vxm), model(S, T), S, T, kw.get("bidir", False)).backward()
    gS, gT = _oracle_image_grads(sd, cfg, s, tr, emulate=eng_name == "bf16")
    eS, eT = relmax(S.grad.cpu(), gS), relmax(T.grad.cpu(), gT)
    print("\n[image grads %s %s] max-norm rel err source %.2e target %.2e | rel L2 source %.2e target %.2e"
          % (eng_name, name, eS, eT, rel_l2(S.grad.cpu(), gS), rel_l2(T.grad.cpu(), gT)))
    assert eS <= E2E_TOL[eng_name] and eT <= E2E_TOL[eng_name]


@pytest.mark.parametrize("which", ["source", "target"])
@pytest.mark.parametrize("eng_name", ["bf16", "bf16x3"])
def test_one_image_alone_requires_a_gradient(vx, cuda, engine, eng_name, which):
    vxm = vx[0]
    engine(eng_name)
    kw = E2E["default3d"]
    model, sd, cfg = _model(vxm, cuda, kw)
    s, tr = cases.volume_pair(93, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda).requires_grad_(which == "source"), t(tr).to(cuda).requires_grad_(which == "target")
    _step_loss(_gpu_losses(vxm), model(S, T), S, T, False).backward()
    gS, gT = _oracle_image_grads(sd, cfg, s, tr, emulate=eng_name == "bf16")
    got, want, other = (S.grad, gS, T) if which == "source" else (T.grad, gT, S)
    assert other.grad is None
    assert relmax(got.cpu(), want) <= E2E_TOL[eng_name]
    assert all(p.grad is not None for p in model.parameters())


@pytest.mark.parametrize("eng_name", ["bf16", "bf16x3", "f32"])
def test_semi_supervised_image_gradients(vx, cuda, engine, eng_name):
    """VxmDenseSemiSupervisedSeg: NCC + Grad + Dice on the linearly warped one-hot segmentation; gradients of both images
    and of the (probabilistic) source segmentation."""
    vxm = vx[0]
    engine(eng_name)
    shape, nlab = (32, 32, 32), 5
    model = vxm.networks.VxmDenseSemiSupervisedSeg(shape, nlab)
    cfg = model.vxm_model.config
    sd = ref_torch.init_state_dict(cfg, seed=21, flow_std=2e-2)
    model.vxm_model.load_state_dict(sd, strict=False)
    model.to(cuda).train()
    s, tr = cases.volume_pair(401, shape, sigma=1.5)
    oh = lambda lab: (lab[:, 0, ::2, ::2, ::2][:, None] == np.arange(nlab, dtype=np.float32)[None, :, None, None, None]).astype(np.float32)  # noqa: E731
    seg_m, seg_f = oh(cases.label_volume(402, shape, nlab)), oh(cases.label_volume(403, shape, nlab))
    S, T = t(s).to(cuda).requires_grad_(True), t(tr).to(cuda).requires_grad_(True)
    M = t(seg_m).to(cuda).requires_grad_(True)
    y, pre, yseg = model(S, T, M)
    ncc, grad = _gpu_losses(vxm)
    (ncc(T, y) + 0.01 * grad(pre) + 0.1 * vxm.losses.Dice().loss(t(seg_f).to(cuda), yseg)).backward()
    ref_torch.emulate_bf16(eng_name == "bf16")
    sdc = {k: v.double() for k, v in sd.items()}
    Sc, Tc = t(s).double().requires_grad_(True), t(tr).double().requires_grad_(True)
    Mc = t(seg_m).double().requires_grad_(True)
    yc, prec = ref_torch.vxm_forward(sdc, cfg, Sc, Tc)
    _, posc = ref_torch.vxm_forward(sdc, cfg, Sc, Tc, registration=True)
    ysegc = ref_torch.spatial_transform(Mc, ref_torch.resize_transform(posc, 2))
    (ref_torch.ncc_loss(Tc, yc) + 0.01 * ref_torch.grad_loss(prec, "l2", 2) + 0.1 * ref_torch.dice_loss(t(seg_f).double(), ysegc)).backward()
    ref_torch.emulate_bf16(False)
    errs = relmax(S.grad.cpu(), Sc.grad), relmax(T.grad.cpu(), Tc.grad), relmax(M.grad.cpu(), Mc.grad)
    print("\n[semi-supervised %s] max-norm rel err source %.2e target %.2e source segmentation %.2e" % ((eng_name,) + errs))
    assert max(errs) <= E2E_TOL[eng_name]


# rel L2 between the image gradients of bf16x3 (bf16-operand backward) and f32 through the U-Net alone: measured 5.5e-2
# (source) and 5.9e-2 (target) on the default model, the sum of a bf16 rounding of the gradient at every one of its 12
# layers; the weight gradients of the same backward are allowed a median of 5e-2 and a maximum of 1.5e-1
# (test_gpu_bf16_engine.py)
UNET_PATH_L2 = 1e-1


def test_engines_agree_on_the_image_gradient(vx, cuda, engine):
    """source.grad and target.grad of bf16x3 against f32 on the same weights, (a) for the step's loss, (b) for a loss on
    the flow field alone, whose whole image gradient flows through the U-Net: an engine that drops that part returns None
    (or the warp's share only) and fails here."""
    vxm = vx[0]
    kw = E2E["default3d"]
    s, tr = cases.volume_pair(93, kw["inshape"], sigma=1.5)
    gen = torch.Generator().manual_seed(1)
    res = {}
    for eng_name in ("f32", "bf16x3"):
        engine(eng_name)
        model, _, _ = _model(vxm, cuda, kw)
        S, T = t(s).to(cuda).requires_grad_(True), t(tr).to(cuda).requires_grad_(True)
        _step_loss(_gpu_losses(vxm), model(S, T), S, T, False).backward()
        step = (S.grad.clone(), T.grad.clone())
        S.grad = T.grad = None
        flow = model(S, T)[-1]
        if "gflow" not in res:
            res["gflow"] = torch.randn(flow.shape, generator=gen).to(cuda)
        (flow * res["gflow"]).sum().backward()
        assert S.grad is not None and T.grad is not None, eng_name
        res[eng_name] = step + (S.grad.clone(), T.grad.clone())
    names = ("step source", "step target", "flow-only source", "flow-only target")
    errs = [rel_l2(a, b) for a, b in zip(res["bf16x3"], res["f32"])]
    print("\n[bf16x3 vs f32] rel L2: " + ", ".join("%s %.2e" % p for p in zip(names, errs)))
    assert float(res["f32"][2].abs().max()) > 0
    assert max(errs) <= UNET_PATH_L2, dict(zip(names, errs))


# ---- 4. NCC differentiated w.r.t. either image -----------------------------------------------------------------------

_ncc_ref_cache = {}


def _ncc_refs(kind, B, shape, win):
    key = (kind, B, shape, win)
    if key not in _ncc_ref_cache:
        I, J = _pair(kind, B, shape)
        l64 = spec_np.ncc_loss(I, J, list(win))
        gI64, gJ64 = image_grads_ref.ncc_grad_true(I, J, list(win)), spec_np.ncc_grad_pred(I, J, list(win))
        It, Jt = t(I).requires_grad_(True), t(J).requires_grad_(True)
        l32 = _ncc_fp32(It, Jt, win)
        l32.backward()
        _ncc_ref_cache[key] = (I, J, l64, gI64, gJ64, abs(float(l32.detach()) - l64) / abs(l64), rel(It.grad, gI64), rel(Jt.grad, gJ64))
    return _ncc_ref_cache[key]


def _ncc_both_ways(vxm, cuda, kind, B, shape, win, tag):
    """d/dI alone, d/dJ alone and both in one call, each within twice the fp64 distance of the reference's own fp32
    arithmetic (+1e-6); d/dJ of the two-sided call EQUALS the one-sided kernel's; d/dI of NCC(I, J) against d/dJ of NCC(J, I)."""
    I, J, l64, gI64, gJ64, e_loss, e_gI, e_gJ = _ncc_refs(kind, B, shape, win)
    ncc = vxm.losses.NCC(win=list(win)).loss
    tag = "ncc %s %s B=%d %s win=%s" % (tag, kind, B, shape, win)

    def run(a, b, need_a, need_b):
        A, Bt = t(a).to(cuda).requires_grad_(need_a), t(b).to(cuda).requires_grad_(need_b)
        loss = ncc(A, Bt)
        loss.backward()
        return float(loss.detach()), A.grad, Bt.grad

    l1, gI1, none = run(I, J, True, False)
    assert none is None
    l2, none, gJ2 = run(I, J, False, True)
    assert none is None
    l3, gI3, gJ3 = run(I, J, True, True)
    for name, l in (("y_true", l1), ("y_pred", l2), ("both", l3)):
        report(tag + " loss, %s (fp32 ref %.1e)" % (name, e_loss), abs(l - l64) / abs(l64), 2 * e_loss + 1e-6)
    report(tag + " d/dI alone (fp32 ref %.1e)" % e_gI, rel(gI1.cpu(), gI64), 2 * e_gI + 1e-6)
    report(tag + " d/dI both (fp32 ref %.1e)" % e_gI, rel(gI3.cpu(), gI64), 2 * e_gI + 1e-6)
    report(tag + " d/dJ both (fp32 ref %.1e)" % e_gJ, rel(gJ3.cpu(), gJ64), 2 * e_gJ + 1e-6)
    assert torch.equal(gJ3, gJ2), tag + ": d/dJ of the two-sided call differs from the one-sided kernel's"
    _, _, gJ_swapped = run(J, I, False, True)
    report(tag + " d/dI NCC(I,J) vs d/dJ NCC(J,I)", rel(gI3.cpu(), gJ_swapped.cpu()), 2 * e_gI + 1e-6)


KINDS = ["smooth", "stripped", "offset"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B,shape,win", [(1, (160, 192, 224), (9, 9, 9)), (2, (192, 224), (9, 9))], ids=["3d-full", "2d"])
def test_ncc9_both_ways_vs_fp64(vx, cuda, B, shape, win, kind):
    _ncc_both_ways(vx[0], cuda, kind, B, shape, win, "fast")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("zchunk", ["1", "5", "45"])
def test_ncc9_both_ways_depth_chunks(vx, cuda, monkeypatch, zchunk, kind):
    monkeypatch.setenv("VXM_B200_NCC_ZCHUNK", zchunk)
    _ncc_both_ways(vx[0], cuda, kind, 2, (45, 70, 121), (9, 9, 9), "fast zchunk=" + zchunk)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("win", [(3, 3, 3), (5, 9, 9), (5, 5)], ids=["3", "5-9-9", "2d-5"])
def test_ncc_generic_both_ways_vs_fp64(vx, cuda, win, kind):
    shape = (45, 70, 121) if len(win) == 3 else (70, 121)
    _ncc_both_ways(vx[0], cuda, kind, 2, shape, win, "generic")


def test_ncc_entry_points_report_bad_arguments(vx, cuda):
    vxm = vx[0]
    lib, L = vxm._lib.load(), vxm._lib
    x = torch.zeros(8, device=cuda)
    rc = lib.vxm_ncc_fwd2(L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(L.reduce_workspace(cuda)), 4, 1, 1, 2, 4, 1, 1, 1, L.stream_ptr())
    assert rc != 0 and "which" in L.last_error()
    rc = lib.vxm_ncc_bwd2(L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(x), None, L.ptr(x), 3, 1, 1, 2, 4, 1, 1, 1, L.stream_ptr())
    assert rc != 0 and "null pointer" in L.last_error()
    rc = lib.vxm_ncc_bwd2(L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(x), L.ptr(x), 3, 1, 1, 2, 4, 1, 1, 4, L.stream_ptr())
    assert rc != 0 and "window" in L.last_error()


# ---- 5. Dice w.r.t. y_true ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B,L,shape", [(1, 30, (80, 96, 112)), (2, 7, (13, 17, 19))], ids=["30-labels", "ragged"])
def test_dice_gradient_of_y_true_vs_fp64(vx, cuda, B, L, shape):
    """Probability maps with one label absent from BOTH (bottom at the clamp floor: zero gradient, as torch.clamp gives)."""
    vxm = vx[0]
    g = torch.Generator().manual_seed(L)
    a = torch.softmax(3 * torch.randn((B, L) + shape, generator=g), 1)
    b = torch.softmax(3 * torch.randn((B, L) + shape, generator=g), 1)
    a[:, 3] = 0
    b[:, 3] = 0
    A, Bt = a.to(cuda).requires_grad_(True), b.to(cuda).requires_grad_(True)
    loss = vxm.losses.Dice().loss(A, Bt)
    loss.backward()
    a64, b64 = a.double().requires_grad_(True), b.double().requires_grad_(True)
    l64 = ref_torch.dice_loss(a64, b64)
    l64.backward()
    assert abs(float(loss) - float(l64)) <= 1e-6 * abs(float(l64))
    report("dice d/dy_true %s L=%d" % (shape, L), rel(A.grad.cpu(), a64.grad), 1e-5)
    report("dice d/dy_pred %s L=%d" % (shape, L), rel(Bt.grad.cpu(), b64.grad), 1e-5)
    assert float(A.grad[:, 3].abs().max()) == 0.0
    A2 = a.to(cuda).requires_grad_(True)
    vxm.losses.Dice().loss(A2, b.to(cuda)).backward()
    assert torch.equal(A2.grad, A.grad)


# ---- 6. a step whose images need no gradient runs as before; a learnable image trains under graph capture ---------------

# kernel launches of the second eager step (forward, NCC + Grad, backward, fused Adam) of the default model at 32 x 32 x 48,
# images without requires_grad: the figures of the build before the image gradients existed
STEP_LAUNCHES = {"bf16": 69, "bf16x3": 94}


def _count_step(vxm, model, opt, S, T):
    n0 = vxm._lib.launch_count()
    opt.zero_grad()
    y, flow = model(S, T)
    loss = vxm.losses.NCC().loss(T, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    return vxm._lib.launch_count() - n0


@pytest.mark.parametrize("eng_name", ["bf16", "bf16x3"])
def test_step_without_image_gradients_launches_what_it_did(vx, cuda, engine, eng_name):
    vxm = vx[0]
    engine(eng_name)
    kw = E2E["default3d"]
    model, _, _ = _model(vxm, cuda, kw)
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4)
    s, tr = cases.volume_pair(93, kw["inshape"], sigma=1.5)
    S, T = t(s).to(cuda), t(tr).to(cuda)
    _count_step(vxm, model, opt, S, T)
    plain = _count_step(vxm, model, opt, S, T)
    assert model._vxm_pack_plan.img_table is None          # the image operand is not even built
    Sg = S.clone().requires_grad_(True)
    _count_step(vxm, model, opt, Sg, T)
    with_image = _count_step(vxm, model, opt, Sg, T)
    again = _count_step(vxm, model, opt, S, T)
    print("\n[launches %s] step %d, with source.grad %d, step again %d" % (eng_name, plain, with_image, again))
    assert plain == again == STEP_LAUNCHES[eng_name]
    assert with_image > plain


def test_graphed_step_trains_a_learnable_image(vx, cuda, engine):
    """The consumer's shape: the moving image is an nn.Parameter (an atlas) held by the optimizer next to the weights; the
    whole step is captured, replayed three times, and the image moves."""
    vxm = vx[0]
    engine("bf16")
    from voxelmorph_b200.trainer import GraphedTrainStep
    kw = dict(inshape=(32, 32, 32))
    model, _, _ = _model(vxm, cuda, kw, seed=5)
    s, tr = cases.volume_pair(95, kw["inshape"], sigma=1.5)
    atlas = torch.nn.Parameter(t(s).to(cuda))
    start = atlas.detach().clone()
    opt = vxm.optim.FusedAdam(list(model.parameters()) + [atlas], lr=1e-3)
    ncc, grad = _gpu_losses(vxm)

    def loss_fn(model, target):
        y, flow = model(atlas, target)
        return ncc(target, y) + 0.01 * grad(flow)

    step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=3).capture(t(tr).to(cuda))
    assert torch.equal(atlas.detach(), start)               # the warm-up steps are rolled back
    losses = [float(step(t(tr).to(cuda))) for _ in range(3)]
    assert all(np.isfinite(losses)), losses
    moved = float((atlas.detach() - start).abs().max())
    print("\n[graphed atlas step] losses %s, image moved by up to %.2e" % (losses, moved))
    assert moved > 0 and int(opt.step_dev.item()) == 3
