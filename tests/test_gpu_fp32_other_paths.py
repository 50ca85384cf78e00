"""The fp32 kernels real models run outside the 3-D fast tail of tests/test_gpu_fp32_step_kernels.py, voxel by voxel
against float64 (or bit for bit where the kernel replays fp32 arithmetic), at the sizes they serve: the exact-replay
VecInt and warp (every 2-D model's VecInt, `VXM_B200_LINEAR_ARITH=exact` training, both divisions), the 2-D resize and
Grad, MSE, Dice, the fused Adam over a real model's flat buffer, the Jacobian determinant, and the 2-D step's fp32
tail.  Run with -s to see every measured error next to its bound.

Each bound rests on an explicit mechanism:
* bit-exact replay: the exact-arithmetic kernels and oracle/spec_np round every operation of torch's fp32 sequence once,
  so forward outputs and VecInt's saved states must be identical;
* the trajectory method: VecInt's adjoint is evaluated in fp64 along the kernel's own states at the replayed fp32
  coordinates (oracle/at_coords.py); each Adam step is taken in fp64 from the kernel's previous fp32 state;
* operation counts: a bound of k roundings (u = 2^-24) of the magnitudes the fp32 sequence forms (MSE, Adam, Jacobian);
* the reference's own fp32 error (resize), as in the fast tier.
"""
import numpy as np
import pytest
import torch

from oracle import at_coords, cases, ref_torch, spec_np

pytestmark = pytest.mark.gpu

FULL = (160, 192, 224)
HALF = (80, 96, 112)
U = 2.0 ** -24


@pytest.fixture(scope="module")
def vxm(cuda):
    import voxelmorph_b200 as v
    v._lib.load()
    return v


def rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def report(what, err, bound):
    print("%-66s err %.3e  bound %.3e" % (what, err, bound))
    assert err <= bound, (what, err, bound)


def batch(fn, seeds):
    return np.concatenate([fn(s) for s in seeds], axis=0)


def exact_arith(monkeypatch, div):
    """The exact-arithmetic linear resampler with torch CPU's division ('true') or torch CUDA's reciprocal ('recip')."""
    monkeypatch.setenv("VXM_B200_LINEAR_ARITH", "exact")
    if div == "recip":
        monkeypatch.setenv("VXM_B200_NEAREST_ARITH", "cuda")
    else:
        monkeypatch.delenv("VXM_B200_NEAREST_ARITH", raising=False)


def border_samples(coords):
    """Number of samples whose cell is not entirely inside the volume (the kernels' border corners)."""
    c = np.floor(coords)
    S = np.array(coords.shape[2:]).reshape((1, -1) + (1,) * (coords.ndim - 2))
    return int(((c < 0) | (c >= S - 1)).any(axis=1).sum())


def field(seed, nd, shape, B, scale):
    return batch(lambda b: cases.smooth_field(seed + b, nd, shape, scale=scale), range(B))


DIVS = ["true", "recip"]


# ---------------------------------------------------------------- VecInt, exact replay -----------------------------

VECINT_CASES = [((96, 112), 8), ((192, 224), 8), ((45, 71), 3), (HALF, 1), ((37, 45, 51), 2)]


@pytest.mark.parametrize("nsteps", [0, 1, 2, 3, 4, 7])
@pytest.mark.parametrize("div", DIVS)
@pytest.mark.parametrize("shape,B", VECINT_CASES, ids=["2d-half-B8", "2d-full-B8", "2d-ragged-B3", "3d-half", "3d-B2"])
def test_vecint_exact_replay(vxm, cuda, monkeypatch, shape, B, div, nsteps):
    """Output and every saved state bit-identical to spec_np's fp32 replay (training path; the no-grad ping-pong path
    gives the same output); the backward against the fp64 chain adjoint along the kernel's states at the replayed
    coordinates.  nsteps covers both parities of the forward ping-pong and of the backward's two-buffer rotation."""
    exact_arith(monkeypatch, div)
    nd = len(shape)
    vel = field(60, nd, shape, B, 10.0)
    gout = field(70, nd, shape, B, 1.0)
    nvox = B * int(np.prod(shape))
    threads = torch.cuda.get_device_properties(cuda).multi_processor_count * 2048
    tag = "vecint exact %s %s B=%d n=%d" % (div, shape, B, nsteps)
    print("%s: %d voxels, SMs x 2048 = %d" % (tag, nvox, threads))
    states = []
    out_ref = spec_np.vecint(vel, nsteps, div=div, states=states)
    v = torch.from_numpy(vel).to(cuda).requires_grad_(True)
    out = vxm.layers.VecInt(shape, nsteps)(v)
    assert np.array_equal(out.detach().cpu().numpy(), out_ref)
    if nsteps:
        st = out.grad_fn.states
        assert tuple(st.shape) == (nsteps,) + vel.shape
        for k in range(nsteps):
            assert np.array_equal(st[k].cpu().numpy(), states[k]), k
    with torch.no_grad():
        assert torch.equal(vxm.layers.VecInt(shape, nsteps)(v.detach()), out.detach())
    out.backward(torch.from_numpy(gout).to(cuda))
    grad = v.grad.cpu().numpy()
    if nsteps == 0:
        assert np.array_equal(grad, gout)
        return
    replayed = lambda s: at_coords.coords_replayed(s, div)    # noqa: E731
    assert sum(border_samples(replayed(s)) for s in states) > 0
    ref = at_coords.vecint_adjoint(states, gout, 1.0 / 2 ** nsteps, coords=replayed)
    report(tag + " bwd", rel(grad, ref), 1e-5)


# ---------------------------------------------------------------- warp, exact replay -------------------------------

@pytest.mark.parametrize("div", DIVS)
@pytest.mark.parametrize("shape,B,C", [(FULL, 1, 1), ((37, 45, 51), 2, 3), ((192, 224), 8, 1)],
                         ids=["full", "3d-B2-C3", "2d-B8"])
def test_warp_exact_vs_fp64(vxm, cuda, monkeypatch, shape, B, C, div):
    """Linear: the moved image bit-identical to spec_np.warp; d/dsrc and d/dflow against the fp64 adjoints of sampling
    at the replayed coordinates (d coord / d flow = 1: source and flow have the same size).  Nearest: the moved labels
    bit-identical, d/dsrc the scatter of gout to the rounded index (fp64 bincount), d/dflow zero."""
    exact_arith(monkeypatch, div)
    nd = len(shape)
    src = batch(lambda b: np.concatenate([cases.smooth_volume(100 * b + c, shape) for c in range(C)], axis=1), range(B))
    flow = field(17, nd, shape, B, 8.0)
    gout = field(40, C, shape, B, 1.0) if C == 1 else batch(
        lambda b: np.concatenate([cases.smooth_field(40 + 10 * b + c, 1, shape, scale=1.0) for c in range(C)], axis=1), range(B))
    coords = at_coords.coords_replayed(flow, div)
    assert border_samples(coords) > 0
    tag = "warp exact %s %s B=%d C=%d" % (div, shape, B, C)
    s_g = torch.from_numpy(src).to(cuda).requires_grad_(True)
    f_g = torch.from_numpy(flow).to(cuda).requires_grad_(True)
    out = vxm.layers.SpatialTransformer(shape)(s_g, f_g)
    assert np.array_equal(out.detach().cpu().numpy(), spec_np.warp(src, flow, div=div))
    out.backward(torch.from_numpy(gout).to(cuda))
    gs, gc = at_coords.sample_adjoint(src, coords, gout)
    report(tag + " d/dsrc", rel(s_g.grad.cpu(), gs), 1e-5)
    report(tag + " d/dflow", rel(f_g.grad.cpu(), gc), 1e-5)
    # nearest
    lab = batch(lambda b: np.concatenate([cases.label_volume(50 * b + c, shape) for c in range(C)], axis=1), range(B))
    s_g = torch.from_numpy(lab).to(cuda).requires_grad_(True)
    f_g = torch.from_numpy(flow).to(cuda).requires_grad_(True)
    out = vxm.layers.SpatialTransformer(shape, mode="nearest")(s_g, f_g)
    assert np.array_equal(out.detach().cpu().numpy(), spec_np.warp(lab, flow, "nearest", div=div))
    out.backward(torch.from_numpy(gout).to(cuda))
    idx = np.rint(coords).astype(np.int64)
    Sa = np.array(shape).reshape((1, nd) + (1,) * nd)
    ok = ((idx >= 0) & (idx < Sa)).all(axis=1).reshape(B, -1)
    flat = np.ravel_multi_index(tuple(np.clip(idx[:, a], 0, shape[a] - 1) for a in range(nd)), shape).reshape(B, -1)
    ref = np.zeros((B, C, int(np.prod(shape))))
    go = gout.reshape(B, C, -1).astype(np.float64)
    for b in range(B):
        for c in range(C):
            ref[b, c] = np.bincount(flat[b][ok[b]], weights=go[b, c][ok[b]], minlength=ref.shape[2])
    report(tag + " nearest d/dsrc", rel(s_g.grad.cpu().reshape(B, C, -1), ref), 1e-6)
    assert not f_g.grad.any()


# ---------------------------------------------------------------- resize, 2-D --------------------------------------

@pytest.mark.parametrize("B,shape,vel_resize", [
    (8, (192, 224), 2), (8, (96, 112), 0.5),      # the 2-D default model (B.C = 16: two channels per marching thread)
    (3, (192, 224), 2), (3, (96, 112), 0.5),      # B.C = 6: three channels per thread, spanning two batch entries
    (8, (192, 224), 4), (8, (48, 56), 0.25),      # int_downsize 4
], ids=["down2-B8", "up2-B8", "down2-B3", "up2-B3", "down4-B8", "up4-B8"])
def test_resize_2d_vs_fp64(vxm, cuda, B, shape, vel_resize):
    """Forward and adjoint against fp64 autograd of F.interpolate(bilinear, align_corners=True).  Bound 1e-5, or twice
    the reference's own fp32 error where that is larger (both place output q at fl32(ratio) * q in the input)."""
    x = field(90, 2, shape, B, 4.0)
    x_c = torch.from_numpy(x).double().requires_grad_(True)
    o_c = ref_torch.resize_transform(x_c, vel_resize)
    w = torch.from_numpy(np.random.default_rng(9).standard_normal(tuple(o_c.shape)).astype(np.float32))
    (o_c * w.double()).sum().backward()
    x_32 = torch.from_numpy(x).requires_grad_(True)
    o_32 = ref_torch.resize_transform(x_32, vel_resize)
    (o_32 * w).sum().backward()
    x_g = torch.from_numpy(x).to(cuda).requires_grad_(True)
    o_g = vxm.layers.ResizeTransform(vel_resize, 2)(x_g)
    assert tuple(o_g.shape) == tuple(o_c.shape)
    (o_g * w.to(cuda)).sum().backward()
    tag = "resize 2d B=%d %s x%g" % (B, shape, 1 / vel_resize)
    e_fwd, e_bwd = rel(o_32.detach(), o_c.detach()), rel(x_32.grad, x_c.grad)
    report(tag + " fwd (fp32 ref %.1e)" % e_fwd, rel(o_g.detach().cpu(), o_c.detach()), max(1e-5, 2 * e_fwd))
    report(tag + " bwd (fp32 ref %.1e)" % e_bwd, rel(x_g.grad.cpu(), x_c.grad), max(1e-5, 2 * e_bwd))


# ---------------------------------------------------------------- Grad, 2-D ----------------------------------------

@pytest.mark.parametrize("kind", ["smooth", "ties"])
@pytest.mark.parametrize("penalty", ["l1", "l2"])
@pytest.mark.parametrize("B,shape", [(8, (192, 224)), (3, (45, 71))])
def test_grad_2d_vs_fp64(vxm, cuda, B, shape, penalty, kind):
    """Loss <= 1e-6 and gradient <= 1e-5 against fp64 autograd of ref_torch.grad_loss.  'ties': a piecewise-constant
    field (integers), so most differences are exactly 0 and |d|'s derivative there must be torch's, 0."""
    y = field(500, 2, shape, B, 4.0)
    if kind == "ties":
        y = np.round(y).astype(np.float32)
        assert (np.diff(y, axis=-1) == 0).mean() > 0.5
    y_c = torch.from_numpy(y).double().requires_grad_(True)
    l_c = ref_torch.grad_loss(y_c, penalty, loss_mult=2)
    l_c.backward()
    y_g = torch.from_numpy(y).to(cuda).requires_grad_(True)
    l_g = vxm.losses.Grad(penalty, loss_mult=2).loss(None, y_g)
    l_g.backward()
    tag = "grad 2d %s %s B=%d %s" % (penalty, kind, B, shape)
    report(tag + " loss", abs(l_g.item() - l_c.item()) / abs(l_c.item()), 1e-6)
    report(tag + " d/dy", rel(y_g.grad.cpu(), y_c.grad), 1e-5)


# ---------------------------------------------------------------- MSE ----------------------------------------------

# d/dy_pred = fl(fl(gl * fl32(2 / n)) * fl(b - a)): three fp32 roundings of the exact 2 (b - a) / n (gl = 1 exactly)
MSE_GRAD_TOL = 3.01 * U


@pytest.mark.parametrize("case", ["template", "full-B2", "2d-B8"])
def test_mse_vs_fp64(vxm, cuda, case):
    """Loss relative <= 1e-6 (each term rounded twice in fp32, summed in double); d/dy_pred and d/dy_true elementwise
    within three fp32 roundings of +-2 (b - a) / n."""
    if case == "template":      # TemplateCreation's MSE(0, mean stream) over 3 x 160 x 192 x 224
        b = field(700, 3, FULL, 1, 2.0)
        a = np.zeros_like(b)
    else:
        B, shape = (2, FULL) if case == "full-B2" else (8, (192, 224))
        pairs = [cases.volume_pair(710 + i, shape, sigma=2.0) for i in range(B)]
        a = np.concatenate([p[1] for p in pairs])
        b = np.concatenate([p[0] for p in pairs])
    a_g = torch.from_numpy(a).to(cuda).requires_grad_(True)
    b_g = torch.from_numpy(b).to(cuda).requires_grad_(True)
    loss = vxm.losses.MSE().loss(a_g, b_g)
    loss.backward()
    d = b.astype(np.float64) - a.astype(np.float64)
    l64 = float(np.mean(d * d))
    tag = "mse %s %s" % (case, a.shape)
    report(tag + " loss", abs(float(loss) - l64) / l64, 1e-6)
    ref = 2.0 * d / d.size
    scale = np.maximum(np.abs(ref), 1e-300)
    report(tag + " d/dy_pred (per element, of |ref|)", float((np.abs(b_g.grad.cpu().numpy() - ref) / scale).max()), MSE_GRAD_TOL)
    report(tag + " d/dy_true (per element, of |ref|)", float((np.abs(a_g.grad.cpu().numpy() + ref) / scale).max()), MSE_GRAD_TOL)


# ---------------------------------------------------------------- Dice ---------------------------------------------

def test_dice_config5_scale_vs_fp64(vxm, cuda):
    """The one-hot of a 30-label map at 160 x 192 x 224, B = 2, against its linear warp (config 5's Dice on the warped
    segmentation), with one label absent from both maps: loss <= 1e-6 absolute, d/dy_pred and d/dy_true <= 1e-5 of
    max |ref| against the fp64 oracle (spec_np.dice_coefs, floor fl32(1e-5))."""
    L = 30
    lab = np.concatenate([cases.label_volume(800 + b, FULL, L) for b in range(2)])
    lab[lab == L - 1] = L - 2                                   # label 29 absent from y_true, hence from its warp
    lab_g = torch.from_numpy(lab).to(cuda)
    onehot = torch.cat([(lab_g == k).float() for k in range(L)], dim=1)
    flow = torch.from_numpy(field(810, 3, FULL, 2, 3.0)).to(cuda)
    with torch.no_grad():
        warped = vxm.layers.SpatialTransformer(FULL)(onehot, flow)
    yt = onehot.requires_grad_(True)
    yp = warped.clone().requires_grad_(True)
    loss = vxm.losses.Dice().loss(yt, yp)
    loss.backward()
    yt_c, yp_c = onehot.detach().cpu().numpy(), warped.cpu().numpy()
    assert not yt_c[:, L - 1].any() and not yp_c[:, L - 1].any()
    l64, k1, k2 = spec_np.dice_coefs(yt_c, yp_c)
    report("dice 2 x 30 x %s loss (absolute)" % (FULL,), abs(float(loss) - l64), 1e-6)
    for name, g, other in (("d/dy_pred", yp.grad, yt_c), ("d/dy_true", yt.grad, yp_c)):
        err = big = 0.0
        for b in range(2):
            for k in range(L):
                r = k1[b, k] * other[b, k].astype(np.float64) - k2[b, k]
                err = max(err, float(np.abs(g[b, k].cpu().numpy() - r).max()))
                big = max(big, float(np.abs(r).max()))
        report("dice 2 x 30 x %s %s" % (FULL, name), err / big, 1e-5)


def test_dice_floor_vs_torch_fp32(vxm, cuda):
    """Sums exactly at the fp32 floor, a step below and a step above it, an ordinary label and an empty one, in one
    call: both gradients equal torch's fp32 CPU autograd of the reference's formula (at the floor torch's clamp passes
    the gradient: [-0.5, 0.5] / L at the sample, not [-1, 0] / L)."""
    yt, yp = cases.dice_floor_pair()
    a, b = torch.from_numpy(yt).requires_grad_(True), torch.from_numpy(yp).requires_grad_(True)
    ref_torch.dice_loss(a, b).backward()
    a_g = torch.from_numpy(yt).to(cuda).requires_grad_(True)
    b_g = torch.from_numpy(yp).to(cuda).requires_grad_(True)
    vxm.losses.Dice().loss(a_g, b_g).backward()
    for name, mine, ref in (("d/dy_pred", b_g.grad, b.grad), ("d/dy_true", a_g.grad, a.grad)):
        mine = mine.cpu().numpy()
        print("dice floor %s at the floor: kernel %s, torch %s" % (name, mine[0, 0, 0, :2], ref.numpy()[0, 0, 0, :2]))
        np.testing.assert_allclose(mine, ref.numpy(), rtol=1e-6, atol=1e-6 * float(ref.abs().max()), err_msg=name)


# ---------------------------------------------------------------- Adam ---------------------------------------------

DOUBLED = [[32, 64, 64, 64], [64, 64, 64, 64, 64, 32, 32]]


def _model(vxm, cuda, features=None, seed=0):
    torch.manual_seed(seed)
    return vxm.networks.VxmDense(FULL, nb_unet_features=features).to(cuda)


def _grads(rng, n):
    """Seeded gradients of mixed magnitude (1e-6 .. 10) with 10 % exact zeros."""
    g = rng.standard_normal(n) * 10.0 ** rng.uniform(-6, 1, n)
    g[rng.random(n) < 0.1] = 0
    return g.astype(np.float32)


def _adam64(p, g, m, v, step, opt):
    """One Adam step in fp64 from the kernel's fp32 state, with the fp32 constants the kernel receives, and the
    elementwise error bounds of the kernel's fp32 op sequence (u = 2^-24):
    g' = fma(wd, p, g * gscale): 1 rounding of |g'| (g * 0.5 is exact);
    m' = b1 m + (1 - b1) g': 2 roundings of M = b1 |m| + (1 - b1) |g'|, plus g''s: 3u M;
    v' = b2 v + (1 - b2) g' g': 4 roundings of v' (all terms >= 0), plus 2u v' through g': 6u v';
    d = sqrtf(v') * fl32(1 / sqrt(bc2)) + eps: 3u (half v''s) + 4 roundings: 7u of d;
    p' = p - fl32(lr / bc1) * (m' / d): the quotient carries 3u M / d + (7 + 1)u |m'| / d, the two products 2u |m'| / d
    times lr_c, the subtraction u |p'|.  Bounds used: 3u M, 6u v', and u (2 |p'| + 12 lr_c (M + |m'|) / d)."""
    f = lambda x: float(np.float32(x))    # noqa: E731
    lr, b1, b2, eps, wd = f(opt.param_groups[0]["lr"]), f(opt.betas[0]), f(opt.betas[1]), f(opt.eps), f(opt.weight_decay)
    p, g, m, v = (np.asarray(x, np.float64) for x in (p, g, m, v))
    gg = g * f(opt.grad_scale) + wd * p
    m1 = b1 * m + (1 - b1) * gg
    v1 = b2 * v + (1 - b2) * gg * gg
    lr_c = lr / (1 - b1 ** step)
    d = np.sqrt(v1) / np.sqrt(1 - b2 ** step) + eps
    p1 = p - lr_c * m1 / d
    M = b1 * np.abs(m) + (1 - b1) * np.abs(gg)
    return (p1, m1, v1), (U * (2 * np.abs(p1) + 12 * lr_c * (M + np.abs(m1)) / d), 3 * U * M, 6 * U * v1)


def _state(opt):
    return [t.detach().cpu().numpy().copy() for t in (opt.fp.flat, opt.m, opt.v)]


def _adam_trajectory(opt, steps, seed, tag, none_param=None, lr_at=None):
    """`steps` steps with seeded gradients, each checked against one fp64 step from the kernel's previous state.
    none_param: index of a parameter whose .grad is None at every step (it must see a zero gradient).
    lr_at: (step, lr) an eager learning-rate change through param_groups before that step."""
    rng = np.random.default_rng(seed)
    n = opt.fp.numel
    worst = [0.0, 0.0, 0.0]
    prev = _state(opt)
    for i in range(steps):
        if lr_at and i == lr_at[0]:
            opt.param_groups[0]["lr"] = lr_at[1]
        g = _grads(rng, n)
        opt.zero_grad()
        opt.fp.grad.copy_(torch.from_numpy(g))
        if none_param is not None:
            p = opt.fp.params[none_param]
            off = sum(q.numel() for q in opt.fp.params[:none_param])
            p.grad = None
            g[off:off + p.numel()] = 0
        opt.step()
        step = int(opt.step_dev.item())
        cur = _state(opt)
        ref, bounds = _adam64(prev[0], g, prev[1], prev[2], step, opt)
        for j in range(3):
            err = np.abs(cur[j] - ref[j])
            ratio = np.where(err > 0, err / np.maximum(bounds[j], 1e-300), 0.0)
            worst[j] = max(worst[j], float(ratio.max()))
        prev = cur
    for j, name in enumerate(("p", "m", "v")):
        report("adam %s %s (max err / bound over %d steps)" % (tag, name, steps), worst[j], 1.0)
    return prev


@pytest.mark.parametrize("run", ["default", "wd", "world2", "lr-change", "none-grad", "doubled"])
def test_adam_trajectory_vs_fp64(vxm, cuda, run):
    """25 steps over the real flat buffer of VxmDense (default features, or the doubled model), per step against fp64."""
    model = _model(vxm, cuda, DOUBLED if run == "doubled" else None)
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4, weight_decay=1e-2 if run == "wd" else 0.0,
                              world_size=2 if run == "world2" else 1)
    print("adam %s: %d parameters" % (run, opt.fp.numel))
    _adam_trajectory(opt, 25, 1, run, none_param=3 if run == "none-grad" else None,
                     lr_at=(12, 3e-5) if run == "lr-change" else None)
    if run == "none-grad":
        assert opt.fp.params[3].grad is not None and not opt.fp.params[3].grad.any()


def test_adam_resume_late_step_and_graph_replay(vxm, cuda):
    """load_state_dict at step 1000 (bias corrections near 1) continues on the fp64 trajectory; state_dict -> a fresh
    optimizer -> continue is bit-identical to the uninterrupted run; k replays of a captured opt.step() are
    bit-identical to k eager steps from the same state (the device step counter advances the bias corrections)."""
    torch.manual_seed(0)
    init = {k: v.clone() for k, v in _model(vxm, cuda).state_dict().items()}

    def fresh():
        m = _model(vxm, cuda)
        m.load_state_dict(init)
        return vxm.optim.FusedAdam(m.parameters(), lr=1e-4, weight_decay=1e-2), m

    # late step
    opt, _ = fresh()
    gen = torch.Generator().manual_seed(5)
    m0 = torch.randn(opt.fp.numel, generator=gen) * 1e-3
    sd = dict(step=1000, m=m0, v=m0 * m0 * 4 + 1e-12, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)
    opt.load_state_dict(sd)
    _adam_trajectory(opt, 10, 2, "step 1000")
    assert int(opt.step_dev.item()) == 1010
    # resume
    opt_a, _ = fresh()
    _adam_trajectory(opt_a, 20, 3, "uninterrupted")
    opt_b, model_b = fresh()
    rng = np.random.default_rng(3)
    for _ in range(10):
        opt_b.zero_grad()
        opt_b.fp.grad.copy_(torch.from_numpy(_grads(rng, opt_b.fp.numel)))
        opt_b.step()
    sd = opt_b.state_dict()
    opt_c = vxm.optim.FusedAdam(model_b.parameters(), lr=1.0)
    opt_c.load_state_dict(sd)
    for _ in range(10):
        opt_c.zero_grad()
        opt_c.fp.grad.copy_(torch.from_numpy(_grads(rng, opt_c.fp.numel)))
        opt_c.step()
    for x, y in zip(_state(opt_a), _state(opt_c)):
        assert np.array_equal(x, y)
    # graph replay
    k = 6
    opt_a.fp.grad.copy_(torch.from_numpy(_grads(rng, opt_a.fp.numel)))
    snap = opt_a.snapshot()
    for _ in range(k):
        opt_a.step()
    torch.cuda.synchronize()
    eager = _state(opt_a)
    opt_a.restore(snap)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt_a.step()
    opt_a.restore(snap)
    for _ in range(k):
        graph.replay()
    torch.cuda.synchronize()
    assert int(opt_a.step_dev.item()) == int(snap["step_dev"].item()) + k
    for x, y in zip(eager, _state(opt_a)):
        assert np.array_equal(x, y)


# ---------------------------------------------------------------- Jacobian determinant -----------------------------

def _jac_bound(disp):
    """Per-voxel bound on the fp32 determinant's error, for a (*vol, nd) displacement: each J entry is rounded at most
    twice (the difference, relative to the displacement gradient G, and the + 1, relative to J): u (|G| + |J|) = u M;
    the expansion's 2 (2-D) or 5 (3-D) products and sums are rounded once each.  So |err| <= 10 u * sum over the
    expansion's terms of the products of M (M >= |J| covers the expansion's own roundings)."""
    d = np.asarray(disp, np.float64)
    nd = d.ndim - 1
    G = [spec_np._central_diff(d, a) for a in range(nd)]
    M = [np.abs(G[a]) + np.abs(G[a] + np.eye(nd)[a]) for a in range(nd)]
    if nd == 2:
        P = M[0][..., 0] * M[1][..., 1] + M[1][..., 0] * M[0][..., 1]
    else:
        x, y, z = M
        P = (x[..., 0] * (y[..., 1] * z[..., 2] + y[..., 2] * z[..., 1]) + x[..., 1] * (y[..., 0] * z[..., 2] + y[..., 2] * z[..., 0])
             + x[..., 2] * (y[..., 0] * z[..., 1] + y[..., 1] * z[..., 0]))
    return 10 * U * P


def _jacdet(vxm, cuda, flow):
    f = torch.from_numpy(flow).to(cuda)
    det, folds = vxm.utils.jacobian_determinant_device(f, return_folds=True)
    det2, folds2 = vxm.utils.jacobian_determinant_device(f, return_folds=True)
    assert folds2 == folds and torch.equal(det2, det)
    return det.cpu().numpy(), folds


@pytest.mark.parametrize("shape,B", [(FULL, 2), ((192, 224), 8)], ids=["full-B2", "2d-B8"])
def test_jacdet_vs_fp64(vxm, cuda, shape, B):
    nd = len(shape)
    flow = field(900, nd, shape, B, 12.0)
    det, folds = _jacdet(vxm, cuda, flow)
    assert folds == int((det <= 0).sum())
    worst, sure, amb = 0.0, 0, 0
    for b in range(B):
        disp = np.moveaxis(flow[b], 0, -1)
        d64 = spec_np.jacobian_determinant(disp)
        bound = _jac_bound(disp)
        worst = max(worst, float((np.abs(det[b] - d64) / bound).max()))
        clear = np.abs(d64) > bound
        assert np.array_equal((det[b] <= 0)[clear], (d64 <= 0)[clear])
        sure += int((d64 <= 0)[clear].sum())
        amb += int((~clear).sum())
    tag = "jacdet %s B=%d" % (shape, B)
    print("%s: %d folds (fp64: %d outside the bound, %d voxels within it)" % (tag, folds, sure, amb))
    assert sure > 0 and sure <= folds <= sure + amb
    report(tag + " det (max err / per-voxel bound)", worst, 1.0)


@pytest.mark.parametrize("shape,B", [((40, 48, 56), 2), ((96, 112), 3)], ids=["3d-B2", "2d-B3"])
def test_jacdet_exact(vxm, cuda, shape, B):
    """Displacements in 2^-3 units with |v| <= 4: every J entry is a multiple of 2^-4 with |J| <= 5, every product of
    three a multiple of 2^-12 below 6 * 80^3 units < 2^24, so the fp32 determinant is exact in any order.  Boxes of
    7 voxels per axis map onto their centre (phi constant, J = 0): det == 0 there, and those ties count as folds."""
    nd = len(shape)
    flow = np.round(field(950, nd, shape, B, 3.5) * 8) / 8
    grid = np.stack(np.meshgrid(*[np.arange(s) for s in shape], indexing="ij"))
    rng = np.random.default_rng(7)
    for b in range(B):
        for _ in range(6):
            lo = [int(rng.integers(0, s - 7)) for s in shape]
            box = tuple(slice(l, l + 7) for l in lo)
            for a in range(nd):
                flow[(b, a) + box] = (lo[a] + 3) - grid[(a,) + box]
    flow = flow.astype(np.float32)
    assert np.abs(flow).max() <= 4 and np.array_equal(flow * 8, np.round(flow * 8))
    det, folds = _jacdet(vxm, cuda, flow)
    d64 = np.stack([spec_np.jacobian_determinant(np.moveaxis(flow[b], 0, -1)) for b in range(B)])
    assert (d64 == 0).sum() >= 5 ** nd
    assert torch.equal(torch.from_numpy(det).double(), torch.from_numpy(d64))
    assert folds == int((d64 <= 0).sum())
    print("jacdet exact %s B=%d: %d folds, %d of them det == 0" % (shape, B, folds, int((d64 == 0).sum())))


# ---------------------------------------------------------------- the 2-D step's fp32 tail ---------------------------

# Samples that fall into different cells in the kernels' fp32 coordinates and in fp64, where the flow gradient jumps,
# make the difference; the 3-D tail measures 1.6e-4 against the same bound
TAIL_REL_L2 = 5e-4


def test_step_tail_2d_flow_gradient_vs_fp64(vxm, cuda):
    """2-D field at 192 x 224, B = 8 -> resize x1/2 -> VecInt(7) (the exact kernels every 2-D model runs) -> resize x2
    -> warp -> NCC(9^2) + 0.01 Grad(preint): d/d(field) against ref_torch in fp64, as a relative L2."""
    shape, B = (192, 224), 8
    pairs = [cases.volume_pair(600 + b, shape, sigma=3.0) for b in range(B)]
    src = np.concatenate([p[0] for p in pairs])
    trg = np.concatenate([p[1] for p in pairs])
    fld = field(601, 2, shape, B, 3.0)

    f_c = torch.from_numpy(fld).double().requires_grad_(True)
    pre = ref_torch.resize_transform(f_c, 2)
    pos = ref_torch.resize_transform(ref_torch.vec_int(pre, 7), 0.5)
    moved = ref_torch.spatial_transform(torch.from_numpy(src).double(), pos)
    l_c = ref_torch.ncc_loss(torch.from_numpy(trg).double(), moved) + 0.01 * ref_torch.grad_loss(pre, "l2", 2)
    l_c.backward()

    f_g = torch.from_numpy(fld).to(cuda).requires_grad_(True)
    pre = vxm.layers.ResizeTransform(2, 2)(f_g)
    pos = vxm.layers.ResizeTransform(0.5, 2)(vxm.layers.VecInt((96, 112), 7)(pre))
    moved = vxm.layers.SpatialTransformer(shape)(torch.from_numpy(src).to(cuda), pos)
    l_g = vxm.losses.NCC().loss(torch.from_numpy(trg).to(cuda), moved) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, pre)
    l_g.backward()
    g, r = f_g.grad.cpu().double(), f_c.grad
    l2 = float((g - r).norm() / r.norm())
    print("2-D step tail: loss %.8f (fp64 %.8f), d/dfield rel-L2 %.3e, rel-max %.3e" % (float(l_g), float(l_c), l2, rel(g, r)))
    assert abs(float(l_g) - float(l_c)) <= 1e-5 * abs(float(l_c))
    report("2-D step tail d/d(flow field) rel-L2", l2, TAIL_REL_L2)
