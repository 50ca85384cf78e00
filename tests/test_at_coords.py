"""oracle/at_coords.py (fp64 sampling at given coordinates, its adjoints, the VecInt chain adjoint) pinned against
fp64 autograd of oracle/ref_torch on CPU.

Quantised fields (every displacement an odd multiple of 2^-11, |v| < 2^7) make p + v exact in fp32 and never
integral, so ref_torch's coordinate round trip and the helpers' fp32 coordinates pick the same cells and the two
agree to rounding (~1e-12).  The multi-step VecInt case makes torch use the helpers' coordinates and states by
rounding both to fp32 with a straight-through gradient."""
import numpy as np
import pytest
import torch

from oracle import at_coords, cases, ref_torch, spec_np

TOL = 1e-12


def rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(b).max(), 1e-300)


def grid(shape, B):
    return at_coords.coords_fp32(np.zeros((B, len(shape)) + tuple(shape), np.float32))


@pytest.mark.parametrize("shape,B,C,scale", [((9, 11, 13), 2, 2, 6.0), ((7, 5, 12), 1, 3, 1.5), ((13, 17), 2, 3, 5.0)])
def test_sample_and_adjoints_vs_autograd(shape, B, C, scale):
    nd = len(shape)
    src = np.concatenate([np.concatenate([cases.smooth_volume(10 * b + c, shape) for c in range(C)], axis=1)
                          for b in range(B)], axis=0)
    flow = np.concatenate([at_coords.quantised(50 + b, nd, shape, scale) for b in range(B)], axis=0)
    coords = at_coords.coords_fp32(flow)
    assert np.array_equal(coords.astype(np.float64), grid(shape, B).astype(np.float64) + flow)   # p + flow is exact
    s = torch.from_numpy(src).double().requires_grad_(True)
    f = torch.from_numpy(flow).double().requires_grad_(True)
    out = ref_torch.spatial_transform(s, f)
    gout = np.random.default_rng(1).standard_normal(out.shape)
    out.backward(torch.from_numpy(gout))
    mine = at_coords.sample(src, coords)
    gs, gc = at_coords.sample_adjoint(src, coords, gout)
    lo = np.floor(coords)
    assert ((lo < 0) | (lo >= np.array(shape).reshape((1, nd) + (1,) * nd) - 1)).any()   # some samples use padding
    assert rel(mine, out.detach().numpy()) <= TOL
    assert rel(gs, s.grad.numpy()) <= TOL
    assert rel(gc, f.grad.numpy()) <= TOL


@pytest.mark.parametrize("shape", [(8, 10, 12), (12, 14)])
def test_vecint_one_step_quantised_vs_autograd(shape):
    nd = len(shape)
    v0 = at_coords.quantised(7, nd, shape, 3.0)
    vel = torch.from_numpy(2 * v0).double().requires_grad_(True)     # vec_int(., 1) halves it back to v0 exactly
    out = ref_torch.vec_int(vel, 1)
    gout = np.random.default_rng(2).standard_normal(out.shape)
    out.backward(torch.from_numpy(gout))
    assert rel(at_coords.vecint_step(v0), out.detach().numpy()) <= TOL
    assert rel(at_coords.vecint_adjoint([v0], gout, 0.5), vel.grad.numpy()) <= TOL


def _st_round(x):
    """Round to fp32 in the forward pass, identity in the backward pass."""
    return x + (x.float().double() - x).detach()


def _warp_fp32_coords(src, flow):
    """ref_torch.spatial_transform with the sample location rounded to fp32 (straight through)."""
    shape = flow.shape[2:]
    loc = _st_round(ref_torch.identity_grid(shape, dtype=flow.dtype) + flow)
    comps = [2 * (loc[:, i] / (shape[i] - 1) - 0.5) for i in range(len(shape))]
    return torch.nn.functional.grid_sample(src, torch.stack(comps[::-1], dim=-1), align_corners=True)


def test_vecint_chain_adjoint_vs_straight_through_autograd():
    shape, n = (9, 10, 11), 4
    vel_np = cases.smooth_field(8, 3, shape, scale=12.0)
    vel = torch.from_numpy(vel_np).double().requires_grad_(True)
    v = vel * (1.0 / 2 ** n)
    states, fwd = [], []
    for _ in range(n):
        v = _st_round(v)
        states.append(v.detach().float().numpy())
        v = v + _warp_fp32_coords(v, v)
        fwd.append(v.detach().numpy())
    gout = np.random.default_rng(3).standard_normal(v.shape)
    v.backward(torch.from_numpy(gout))
    for k in range(n):
        assert rel(at_coords.vecint_step(states[k]), fwd[k]) <= TOL, k
    c = np.concatenate([at_coords.coords_fp32(s) for s in states])
    assert not (c == np.floor(c)).any()     # an integral coordinate could fall on either side of a face
    assert rel(at_coords.vecint_adjoint(states, gout, 1.0 / 2 ** n), vel.grad.numpy()) <= TOL


# ---------------------------------------------------------------- the replayed coordinates of the exact kernels ----

DIVS = ["true", "recip"]


@pytest.mark.parametrize("div", DIVS)
@pytest.mark.parametrize("shape,B,C", [((9, 11, 13), 2, 2), ((13, 17), 2, 3)])
def test_coords_replayed_vs_spec_warp(shape, B, C, div):
    """Sampling at coords_replayed reproduces spec_np.warp (linear: to fp32 rounding of the weights; nearest: the same
    selection), in both divisions."""
    nd = len(shape)
    src = np.concatenate([np.concatenate([cases.smooth_volume(20 * b + c, shape) for c in range(C)], axis=1)
                          for b in range(B)], axis=0)
    lab = np.concatenate([cases.label_volume(30 + b, shape) for b in range(B)], axis=0)
    flow = np.concatenate([cases.smooth_field(40 + b, nd, shape, scale=4.0) for b in range(B)], axis=0)
    c = at_coords.coords_replayed(flow, div)
    assert c.dtype == np.float32 and c.shape == flow.shape
    assert rel(at_coords.sample(src, c), spec_np.warp(src, flow, div=div)) <= 1e-6
    idx = np.rint(c).astype(np.int64)
    S = np.array(shape).reshape((1, nd) + (1,) * nd)
    ok = ((idx >= 0) & (idx < S)).all(axis=1)
    near = lab[(np.arange(B).reshape((B,) + (1,) * nd), 0) + tuple(np.clip(idx[:, a], 0, shape[a] - 1) for a in range(nd))]
    assert np.array_equal(np.where(ok, near, 0)[:, None], spec_np.warp(lab, flow, "nearest", div=div))


def _warp_replayed_coords(src, flow, div):
    """ref_torch.spatial_transform with the sample location replaced by the reference's fp32 round trip
    (coords_replayed) in the forward pass, straight through (d coord / d flow = 1) in the backward pass."""
    shape = flow.shape[2:]
    loc = ref_torch.identity_grid(shape, dtype=flow.dtype) + flow
    loc = loc + (torch.from_numpy(at_coords.coords_replayed(flow.detach().float().numpy(), div)).double() - loc).detach()
    comps = [2 * (loc[:, i] / (shape[i] - 1) - 0.5) for i in range(len(shape))]
    return torch.nn.functional.grid_sample(src, torch.stack(comps[::-1], dim=-1), align_corners=True)


@pytest.mark.parametrize("div", DIVS)
@pytest.mark.parametrize("shape", [(9, 10, 11), (14, 17)])
def test_vecint_replayed_adjoint_vs_straight_through_autograd(shape, div):
    """vecint_adjoint(coords=coords_replayed) against fp64 autograd of the chain whose states and sample coordinates
    are rounded to the fp32 values of the reference's arithmetic (straight through)."""
    n = 4
    vel = torch.from_numpy(cases.smooth_field(9, len(shape), shape, scale=12.0)).double().requires_grad_(True)
    v = vel * (1.0 / 2 ** n)
    states = []
    for _ in range(n):
        v = _st_round(v)
        states.append(v.detach().float().numpy())
        v = v + _warp_replayed_coords(v, v, div)
    gout = np.random.default_rng(4).standard_normal(v.shape)
    v.backward(torch.from_numpy(gout))
    c = np.concatenate([at_coords.coords_replayed(s, div) for s in states])
    assert not (c == np.floor(c)).any()
    lo = np.floor(c)
    assert ((lo < 0) | (lo >= np.array(shape).reshape((1, len(shape)) + (1,) * len(shape)) - 1)).any()
    replayed = lambda s: at_coords.coords_replayed(s, div)
    assert rel(at_coords.vecint_adjoint(states, gout, 1.0 / 2 ** n, coords=replayed), vel.grad.numpy()) <= TOL


@pytest.mark.parametrize("shape", [(8, 10, 12), (15, 13)])
def test_spec_vecint_recip_is_composed_warps(shape):
    """spec_np.vecint(div='recip') is the scaling and squaring of spec_np.warp(div='recip'), states included, and
    differs from the true-division replay somewhere."""
    vel = cases.smooth_field(11, len(shape), shape, scale=6.0)
    for n in (0, 1, 4):
        states = []
        out = spec_np.vecint(vel, n, div="recip", states=states)
        v = (vel * np.float32(1.0 / 2 ** n)).astype(np.float32)
        for k in range(n):
            assert np.array_equal(states[k], v)
            v = (v + spec_np.warp(v, v, div="recip")).astype(np.float32)
        assert np.array_equal(out, v) and len(states) == n
    assert not np.array_equal(spec_np.vecint(vel, 4, div="recip"), spec_np.vecint(vel, 4))
