"""The fp32 kernels of the training step after the flow head (ResizeTransform, VecInt, SpatialTransformer, NCC,
Grad), voxel by voxel against float64, at the step's full size and on every kernel path the step or a common
model variant takes.  Run with -s to see every measured error next to its bound.

Each bound rests on an explicit mechanism:
* exact-cell fp64: quantised fields (every displacement an odd multiple of 2^-11, |v| < 2^7) make p + v exact in
  fp32 and never integral, so the kernel and fp64 autograd of oracle/ref_torch sample the same trilinear cells;
* the trajectory method (multi-step VecInt): every squaring and the adjoint of the whole chain are evaluated in
  fp64 along the kernel's own saved states and fp32 coordinates (oracle/at_coords.py);
* the reference's own fp32 error (NCC): ref_torch.ncc_loss in fp32 against the same fp64 result; the kernel may
  be at most twice as far from fp64, plus 1e-6.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import at_coords, cases, ref_torch, spec_np

pytestmark = pytest.mark.gpu

FULL = (160, 192, 224)
HALF = (80, 96, 112)


@pytest.fixture(scope="module")
def vxm(cuda):
    import voxelmorph_b200 as v
    v._lib.load()
    return v


@pytest.fixture(autouse=True)
def fast_arith(monkeypatch):
    monkeypatch.setenv("VXM_B200_LINEAR_ARITH", "fast")     # the step's linear resampler (the default)


def rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def report(what, err, bound):
    print("%-58s err %.3e  bound %.3e" % (what, err, bound))
    assert err <= bound, (what, err, bound)


def batch(fn, seeds):
    return np.concatenate([fn(s) for s in seeds], axis=0)


def border_samples(flow):
    """Number of samples whose trilinear cell is not entirely inside the volume (the kernels' border branch)."""
    c = np.floor(at_coords.coords_fp32(flow))
    S = np.array(flow.shape[2:]).reshape((1, -1) + (1,) * (flow.ndim - 2))
    return int(((c < 0) | (c >= S - 1)).any(axis=1).sum())


# ---------------------------------------------------------------- SpatialTransformer (fast path) ------------------

WARP_CASES = [(FULL, 1, 1), ((37, 45, 51), 2, 1), ((37, 45, 51), 2, 3), ((45, 71), 2, 3)]


@pytest.mark.parametrize("src_grad", [False, True], ids=["nosrc", "srcgrad"])
@pytest.mark.parametrize("shape,B,C", WARP_CASES)
def test_warp_quantised_vs_fp64(vxm, cuda, shape, B, C, src_grad):
    """Moved image and d/dflow per voxel (and d/dsrc when the source needs a gradient) against fp64 autograd.
    src_grad=False is the step's call (the moving image has no gradient: the NOSRC kernel)."""
    nd = len(shape)
    src = batch(lambda b: np.concatenate([cases.smooth_volume(100 * b + c, shape) for c in range(C)], axis=1), range(B))
    flow = batch(lambda b: at_coords.quantised(7 + b, nd, shape, 8.0), range(B))
    gout = batch(lambda b: cases.smooth_field(30 + b, C, shape, scale=1.0), range(B))
    assert border_samples(flow) > 0
    s_c = torch.from_numpy(src).double().requires_grad_(src_grad)
    f_c = torch.from_numpy(flow).double().requires_grad_(True)
    out_c = ref_torch.spatial_transform(s_c, f_c)
    out_c.backward(torch.from_numpy(gout).double())
    s_g = torch.from_numpy(src).to(cuda).requires_grad_(src_grad)
    f_g = torch.from_numpy(flow).to(cuda).requires_grad_(True)
    out_g = vxm.layers.SpatialTransformer(shape)(s_g, f_g)
    out_g.backward(torch.from_numpy(gout).to(cuda))
    tag = "warp %s B=%d C=%d %s" % (shape, B, C, "src-grad" if src_grad else "nosrc")
    report(tag + " moved", rel(out_g.detach().cpu(), out_c.detach()), 1e-5)
    report(tag + " d/dflow", rel(f_g.grad.cpu(), f_c.grad), 1e-5)
    if src_grad:
        report(tag + " d/dsrc", rel(s_g.grad.cpu(), s_c.grad), 1e-5)


@pytest.mark.parametrize("shape,B,C", WARP_CASES)
def test_warp_src_grad_unquantised_vs_fp64(vxm, cuda, shape, B, C):
    """d/dsrc is continuous in the sample coordinates, so it needs no quantisation."""
    nd = len(shape)
    src = batch(lambda b: np.concatenate([cases.smooth_volume(200 * b + c, shape) for c in range(C)], axis=1), range(B))
    flow = batch(lambda b: cases.smooth_field(17 + b, nd, shape, scale=8.0), range(B))
    gout = batch(lambda b: cases.smooth_field(40 + b, C, shape, scale=1.0), range(B))
    s_c = torch.from_numpy(src).double().requires_grad_(True)
    ref_torch.spatial_transform(s_c, torch.from_numpy(flow).double()).backward(torch.from_numpy(gout).double())
    s_g = torch.from_numpy(src).to(cuda).requires_grad_(True)
    vxm.layers.SpatialTransformer(shape)(s_g, torch.from_numpy(flow).to(cuda)).backward(torch.from_numpy(gout).to(cuda))
    report("warp %s B=%d C=%d d/dsrc (unquantised)" % (shape, B, C), rel(s_g.grad.cpu(), s_c.grad), 1e-5)


# ---------------------------------------------------------------- VecInt (fast path, training) --------------------

# per-step forward: the kernel's lerp tree rounds each of its ~7 levels once, the final add once: 2^-20 of max|v|
STEP_TOL = 2.0 ** -20
_traj_cache = {}


def _vecint_run(vxm, cuda, vel, nsteps, gout):
    v = torch.from_numpy(vel).to(cuda).requires_grad_(True)
    out = vxm.layers.VecInt(vel.shape[2:], nsteps)(v)
    B, _, D, H, W = vel.shape
    st = out.grad_fn.states.view(torch.float32).view(nsteps, B, D, H, W, 4)
    assert not st[..., 3].any()
    states = [st[k, ..., :3].permute(0, 4, 1, 2, 3).contiguous().cpu().numpy() for k in range(nsteps)]
    out.backward(torch.from_numpy(gout).to(cuda))
    return out.detach().cpu().numpy(), states, v.grad.cpu().numpy()


@pytest.mark.parametrize("nsteps", [1, 2, 3, 4, 7])
@pytest.mark.parametrize("shape,B", [(HALF, 1), ((37, 45, 51), 2), ((2, 37, 64), 1)])
def test_vecint_trajectory_vs_fp64(vxm, cuda, shape, B, nsteps):
    """Every squaring and the backward of the whole chain (grid-stride walk with next-voxel prefetch) against fp64
    along the kernel's own states; a second run gives the same output and states."""
    vel = batch(lambda b: cases.smooth_field(60 + b, 3, shape, scale=10.0), range(B))
    gout = batch(lambda b: cases.smooth_field(70 + b, 3, shape, scale=1.0), range(B))
    out, states, grad = _vecint_run(vxm, cuda, vel, nsteps, gout)
    scale = 1.0 / 2 ** nsteps
    assert np.array_equal(states[0], (vel * np.float32(scale)).astype(np.float32))
    tag = "vecint %s B=%d n=%d" % (shape, B, nsteps)
    nxt = states[1:] + [out]
    err = max(np.abs(nxt[k] - at_coords.vecint_step(states[k])).max() / np.abs(nxt[k]).max() for k in range(nsteps))
    report(tag + " per-step fwd (max over steps)", err, STEP_TOL)
    assert sum(border_samples(s) for s in states) > 0
    ref = at_coords.vecint_adjoint(states, gout, scale)
    report(tag + " bwd", rel(grad, ref), 1e-5)
    out2, states2, _ = _vecint_run(vxm, cuda, vel, nsteps, gout)
    assert np.array_equal(out2, out) and all(np.array_equal(a, b) for a, b in zip(states, states2))


def test_vecint_one_step_quantised_full_size_vs_autograd(vxm, cuda):
    """nsteps = 1 at the step's size with a quantised field: plain fp64 autograd of ref_torch is the yardstick."""
    v0 = at_coords.quantised(80, 3, HALF, 10.0)
    vel = 2 * v0                                   # VecInt(., 1) scales by 1/2 exactly
    gout = cases.smooth_field(81, 3, HALF, scale=1.0)
    v_c = torch.from_numpy(vel).double().requires_grad_(True)
    out_c = ref_torch.vec_int(v_c, 1)
    out_c.backward(torch.from_numpy(gout).double())
    v_g = torch.from_numpy(vel).to(cuda).requires_grad_(True)
    out_g = vxm.layers.VecInt(HALF, 1)(v_g)
    out_g.backward(torch.from_numpy(gout).to(cuda))
    assert border_samples(v0) > 0
    report("vecint %s n=1 quantised fwd" % (HALF,), rel(out_g.detach().cpu(), out_c.detach()), STEP_TOL)
    report("vecint %s n=1 quantised bwd" % (HALF,), rel(v_g.grad.cpu(), v_c.grad), 1e-5)


# ---------------------------------------------------------------- ResizeTransform ----------------------------------

@pytest.mark.parametrize("B,shape,vel_resize,env", [
    (1, FULL, 2, None),             # the step's down path (pre 1, post 0.5)
    (1, HALF, 0.5, None),           # the step's up path (pre 2): column-marching shared-memory adjoint
    (1, HALF, 0.5, "march"),        # ... and the plain marching adjoint
    (1, FULL, 4, None),             # int_downsize 4: marching adjoint
    (1, (40, 48, 56), 0.25, None),  # int_downsize 4 up: generic adjoint
    (2, (37, 45, 51), 4, None),
    (2, (10, 12, 13), 0.25, None),
], ids=["down2", "up2", "up2-march", "down4", "up4", "down4-B2", "up4-B2"])
def test_resize_vs_fp64(vxm, cuda, monkeypatch, B, shape, vel_resize, env):
    """Forward and adjoint against fp64 autograd of F.interpolate.  Bound 1e-5, or twice the error of the reference
    in fp32 where that is larger: the kernels and torch's fp32 path both place output q at fl32(ratio) * q in the
    input, and against a non-smooth cotangent the resulting weight error (~1e-7 * position) shows in the adjoint."""
    if env:
        monkeypatch.setenv("VXM_B200_RESIZE_BWD", env)
    x = batch(lambda b: cases.smooth_field(90 + b, 3, shape, scale=4.0), range(B))
    x_c = torch.from_numpy(x).double().requires_grad_(True)
    o_c = ref_torch.resize_transform(x_c, vel_resize)
    w = torch.from_numpy(np.random.default_rng(9).standard_normal(tuple(o_c.shape)).astype(np.float32))
    (o_c * w.double()).sum().backward()
    x_32 = torch.from_numpy(x).requires_grad_(True)
    o_32 = ref_torch.resize_transform(x_32, vel_resize)
    (o_32 * w).sum().backward()
    x_g = torch.from_numpy(x).to(cuda).requires_grad_(True)
    o_g = vxm.layers.ResizeTransform(vel_resize, 3)(x_g)
    assert tuple(o_g.shape) == tuple(o_c.shape)
    (o_g * w.to(cuda)).sum().backward()
    tag = "resize B=%d %s x%g%s" % (B, shape, 1 / vel_resize, " (%s)" % env if env else "")
    e_fwd, e_bwd = rel(o_32.detach(), o_c.detach()), rel(x_32.grad, x_c.grad)
    report(tag + " fwd (fp32 ref %.1e)" % e_fwd, rel(o_g.detach().cpu(), o_c.detach()), max(1e-5, 2 * e_fwd))
    report(tag + " bwd (fp32 ref %.1e)" % e_bwd, rel(x_g.grad.cpu(), x_c.grad), max(1e-5, 2 * e_bwd))


# ---------------------------------------------------------------- NCC ----------------------------------------------

def _pair(kind, B, shape):
    """(I, J) float32 (B, 1, *shape): 'smooth' as the other tests use; 'stripped' an object with exact zeros outside
    it (at least 5 voxels of pure background on every side) and its warp, so the rims disagree; 'offset'
    100 + 50 * the smooth pair."""
    Is, Js = [], []
    for b in range(B):
        I, J = cases.volume_pair(300 + b, shape, sigma=3.0)
        if kind == "stripped":
            ax = [np.abs(np.arange(n) - (n - 1) / 2.0) / (0.36 * n) for n in shape]
            r2 = sum(np.square(a).reshape([-1 if i == k else 1 for i in range(len(shape))]) for k, a in enumerate(ax))
            I = np.where(r2 <= 1.0, np.float32(0.2) + np.float32(0.8) * I, np.float32(0)).astype(np.float32)
            J = spec_np.warp(I, cases.smooth_field(400 + b, len(shape), shape, scale=3.0))
            for a in range(2, I.ndim):
                assert not np.take(I, np.r_[0:5, -5:0], axis=a).any()
        elif kind == "offset":
            I, J = (np.float32(100) + np.float32(50) * I).astype(np.float32), (np.float32(100) + np.float32(50) * J).astype(np.float32)
        Is.append(I)
        Js.append(J)
    return np.concatenate(Is), np.concatenate(Js)


def _ncc_fp32(I, J, win):
    """The reference's NCC (ref_torch.ncc_loss) in fp32 on CPU; a window that is not a cube is padded per axis, as
    the CUDA kernels and spec_np do (the reference pads every axis by win[0] // 2)."""
    if len(set(win)) == 1:
        return ref_torch.ncc_loss(I, J, win)
    nd = I.dim() - 2
    filt = torch.ones([1, 1, *win], dtype=I.dtype)
    conv = (F.conv1d, F.conv2d, F.conv3d)[nd - 1]

    def S(t):
        return conv(t, filt, padding=[w // 2 for w in win])

    I_sum, J_sum, I2_sum, J2_sum, IJ_sum = S(I), S(J), S(I * I), S(J * J), S(I * J)
    n = float(np.prod(win))
    u_I, u_J = I_sum / n, J_sum / n
    cross = IJ_sum - u_J * I_sum - u_I * J_sum + u_I * u_J * n
    I_var = I2_sum - 2 * u_I * I_sum + u_I * u_I * n
    J_var = J2_sum - 2 * u_J * J_sum + u_J * u_J * n
    return -(cross * cross / (I_var * J_var + 1e-5)).mean()


_ncc_ref_cache = {}


def _ncc_refs(kind, B, shape, win):
    key = (kind, B, shape, win)
    if key not in _ncc_ref_cache:
        I, J = _pair(kind, B, shape)
        l64 = spec_np.ncc_loss(I, J, list(win))
        g64 = spec_np.ncc_grad_pred(I, J, list(win))
        Jt = torch.from_numpy(J).requires_grad_(True)
        l32 = _ncc_fp32(torch.from_numpy(I), Jt, win)
        l32.backward()
        e_loss = abs(float(l32.detach()) - l64) / abs(l64)
        e_grad = rel(Jt.grad, g64)
        _ncc_ref_cache[key] = (I, J, l64, g64, e_loss, e_grad)
    return _ncc_ref_cache[key]


def _ncc_check(vxm, cuda, kind, B, shape, win, tag):
    I, J, l64, g64, e_loss, e_grad = _ncc_refs(kind, B, shape, win)
    Jg = torch.from_numpy(J).to(cuda).requires_grad_(True)
    loss = vxm.losses.NCC(win=list(win)).loss(torch.from_numpy(I).to(cuda), Jg)
    loss.backward()
    tag = "ncc %s %s B=%d %s win=%s" % (tag, kind, B, shape, win)
    report(tag + " loss (fp32 ref %.1e)" % e_loss, abs(float(loss) - l64) / abs(l64), 2 * e_loss + 1e-6)
    report(tag + " d/dJ (fp32 ref %.1e)" % e_grad, rel(Jg.grad.cpu(), g64), 2 * e_grad + 1e-6)


KINDS = ["smooth", "stripped", "offset"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B,shape,win", [(1, FULL, (9, 9, 9)), (2, (192, 224), (9, 9))], ids=["3d-full", "2d"])
def test_ncc9_full_size_vs_fp64(vxm, cuda, B, shape, win, kind):
    _ncc_check(vxm, cuda, kind, B, shape, win, "fast")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("zchunk", ["1", "5", "45"])
def test_ncc9_depth_chunks_vs_fp64(vxm, cuda, monkeypatch, zchunk, kind):
    """A ragged shape with partial 32 x 56 tiles on both axes, B = 2, and fixed depth chunks, so the H / W tile seams
    and the chunk seams checked here do not depend on the GPU's SM count."""
    monkeypatch.setenv("VXM_B200_NCC_ZCHUNK", zchunk)
    _ncc_check(vxm, cuda, kind, 2, (45, 70, 121), (9, 9, 9), "fast zchunk=" + zchunk)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("win,env", [((3, 3, 3), None), ((7, 7, 7), None), ((5, 9, 9), None), ((9, 5, 7), None),
                                     ((5, 5), None), ((9, 9, 9), "generic"), ((9, 9, 9), "generic-zchunk4")],
                         ids=["3", "7", "5-9-9", "9-5-7", "2d-5", "9-generic", "9-generic-zchunk4"])
def test_ncc_generic_vs_fp64(vxm, cuda, monkeypatch, win, env, kind):
    if env:
        monkeypatch.setenv("VXM_B200_NCC_KERNEL", "generic")
    if env == "generic-zchunk4":
        monkeypatch.setenv("VXM_B200_NCC_ZCHUNK", "4")
    shape = (45, 70, 121) if len(win) == 3 else (70, 121)
    _ncc_check(vxm, cuda, kind, 2, shape, win, "generic" if env is None else env)


# ---------------------------------------------------------------- Grad ---------------------------------------------

@pytest.mark.parametrize("penalty", ["l1", "l2"])
@pytest.mark.parametrize("B,shape", [(1, HALF), (2, (37, 45, 51))])
def test_grad_vs_fp64(vxm, cuda, B, shape, penalty):
    y = batch(lambda b: cases.smooth_field(500 + b, 3, shape, scale=4.0), range(B))
    y_c = torch.from_numpy(y).double().requires_grad_(True)
    l_c = ref_torch.grad_loss(y_c, penalty, loss_mult=2)
    l_c.backward()
    y_g = torch.from_numpy(y).to(cuda).requires_grad_(True)
    l_g = vxm.losses.Grad(penalty, loss_mult=2).loss(None, y_g)
    l_g.backward()
    tag = "grad %s B=%d %s" % (penalty, B, shape)
    report(tag + " loss", abs(float(l_g) - float(l_c)) / abs(float(l_c)), 1e-6)
    report(tag + " d/dy", rel(y_g.grad.cpu(), y_c.grad), 1e-5)


# ---------------------------------------------------------------- the step's fp32 tail -----------------------------

def _ncc64_separable(I, J, win=9):
    """ref_torch.ncc_loss in float64 with the box sum done one axis at a time (the same sum; a 9^3 fp64 convolution at
    160x192x224 is out of reach on a CPU)."""
    def S(t):
        for ax in range(3):
            k = [1, 1, 1]
            k[ax] = win
            p = [0, 0, 0]
            p[ax] = win // 2
            t = F.avg_pool3d(t, k, stride=1, padding=p, count_include_pad=True) * win
        return t

    I_sum, J_sum, I2_sum, J2_sum, IJ_sum = S(I), S(J), S(I * I), S(J * J), S(I * J)
    n = float(win ** 3)
    u_I, u_J = I_sum / n, J_sum / n
    cross = IJ_sum - u_J * I_sum - u_I * J_sum + u_I * u_J * n
    I_var = I2_sum - 2 * u_I * I_sum + u_I * u_I * n
    J_var = J2_sum - 2 * u_J * J_sum + u_J * u_J * n
    return -(cross * cross / (I_var * J_var + 1e-5)).mean()


# Samples that fall into different trilinear cells in the kernels' fp32 coordinates and in fp64, where the flow
# gradient jumps, make the difference: 1.6e-4 measured on an H100 80GB HBM3 (max-norm 2.3e-3 of max|ref|)
TAIL_REL_L2 = 5e-4


def test_step_tail_flow_gradient_vs_fp64(vxm, cuda):
    """flow field -> resize -> VecInt(7) -> resize -> warp -> NCC + 0.01 Grad(preint): d/d(flow field), the gradient
    the U-Net's flow head receives, against ref_torch in fp64."""
    src, trg = cases.volume_pair(600, FULL, sigma=3.0)
    field = cases.smooth_field(601, 3, FULL, scale=3.0)

    def tail64(f):
        pre = ref_torch.resize_transform(f, 2)
        pos = ref_torch.resize_transform(ref_torch.vec_int(pre, 7), 0.5)
        moved = ref_torch.spatial_transform(torch.from_numpy(src).double(), pos)
        return _ncc64_separable(torch.from_numpy(trg).double(), moved) + 0.01 * ref_torch.grad_loss(pre, "l2", 2)

    f_c = torch.from_numpy(field).double().requires_grad_(True)
    l_c = tail64(f_c)
    l_c.backward()
    f_g = torch.from_numpy(field).to(cuda).requires_grad_(True)
    pre = vxm.layers.ResizeTransform(2, 3)(f_g)
    pos = vxm.layers.ResizeTransform(0.5, 3)(vxm.layers.VecInt(HALF, 7)(pre))
    moved = vxm.layers.SpatialTransformer(FULL)(torch.from_numpy(src).to(cuda), pos)
    l_g = vxm.losses.NCC().loss(torch.from_numpy(trg).to(cuda), moved) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, pre)
    l_g.backward()
    g, r = f_g.grad.cpu().double(), f_c.grad
    l2 = float((g - r).norm() / r.norm())
    print("step tail: loss %.8f (fp64 %.8f), d/dfield rel-L2 %.3e, rel-max %.3e"
          % (float(l_g), float(l_c), l2, rel(g, r)))
    assert abs(float(l_g) - float(l_c)) <= 1e-5 * abs(float(l_c))
    report("step tail d/d(flow field) rel-L2", l2, TAIL_REL_L2)
