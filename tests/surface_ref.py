"""fp64 restatements of the surface-point operators of VxmDenseSemiSupervisedPointCloud: the point warp
(point_spatial_transformer, reference voxelmorph/tf/utils/utils.py:465-499), the distance lookup (value_at_location,
utils.py:71-88) and their adjoints, twice:

* a closed form (`point_warp`, `point_warp_flow_grad`, `value_at`, `value_at_grad`), the oracle the GPU tests use;
* `*_tf`: a literal torch transcription of the TF graph (floor, clip, gather, product of weights), differentiated by
  autograd.

Both sample with neurite's ne.utils.interpn(vol, loc, 'linear', fill_value=None), which the reference tree does not
contain; its semantics, per axis of size n at coordinate x:
    c = clip(x, 0, n-1),  i0 = clip(floor(x), 0, n-1),  i1 = clip(i0 + 1, 0, n-1),
    weight i1 - c on i0 and 1 - (i1 - c) on i1; the weights of the axes multiply;
so a point outside the volume reads the border value, and the derivative in x is 0 there (the clip passes its
gradient for 0 <= x <= n-1, ends included; floor and the integer cast pass none).

Layouts are the package's: points (B, N, nd+1) with the label index last, flow (B, nd, *S), sdt (B, L, *S).
"""
import itertools

import torch

F64 = torch.float64


def _taps(x, n):
    c = x.clamp(0, n - 1)
    i0 = torch.floor(x).clamp(0, n - 1)
    i1 = (i0 + 1).clamp(0, n - 1)
    w0 = i1 - c
    return i0.long(), i1.long(), w0, 1 - w0, ((x >= 0) & (x <= n - 1)).to(F64)


def _interp(vol, loc):
    """Closed form.  vol (*S, C) channel-last, loc (N, len(S)).  Returns the values (N, C) and the derivatives
    (len(S), N, C) with respect to each coordinate."""
    S = vol.shape[:-1]
    nd = len(S)
    taps = [_taps(loc[:, d], S[d]) for d in range(nd)]
    flat = vol.reshape(-1, vol.shape[-1])
    strides = [1] * nd
    for d in range(nd - 2, -1, -1):
        strides[d] = strides[d + 1] * S[d + 1]
    val = 0
    der = [0] * nd
    for corner in itertools.product((0, 1), repeat=nd):
        idx = sum(taps[d][corner[d]] * strides[d] for d in range(nd))
        v = flat[idx]
        w = [taps[d][2 + corner[d]] for d in range(nd)]
        val = val + torch.prod(torch.stack(w), 0)[:, None] * v
        for d in range(nd):
            others = [w[e] for e in range(nd) if e != d]
            wo = torch.prod(torch.stack(others), 0) if others else torch.ones_like(w[d])
            sgn = 1.0 if corner[d] else -1.0
            der[d] = der[d] + (sgn * wo * taps[d][4])[:, None] * v
    return val, torch.stack(der)


def _scatter(shape, loc, g):
    """Adjoint of _interp in vol: vol-shaped (*shape, C) sum of weight * g (N, C)."""
    nd = len(shape)
    taps = [_taps(loc[:, d], shape[d]) for d in range(nd)]
    strides = [1] * nd
    for d in range(nd - 2, -1, -1):
        strides[d] = strides[d + 1] * shape[d + 1]
    out = torch.zeros(int(torch.tensor(shape).prod()), g.shape[1], dtype=F64)
    for corner in itertools.product((0, 1), repeat=nd):
        idx = sum(taps[d][corner[d]] * strides[d] for d in range(nd))
        w = torch.prod(torch.stack([taps[d][2 + corner[d]] for d in range(nd)]), 0)
        out.index_add_(0, idx, w[:, None] * g)
    return out.reshape(*shape, g.shape[1])


def _last(t):
    """(B, C, *S) -> (B, *S, C)"""
    return t.permute(0, *range(2, t.dim()), 1)


def point_warp(points, flow, r=1.0):
    nd = flow.shape[1]
    out = points.clone().to(F64)
    for b in range(points.shape[0]):
        v, _ = _interp(_last(flow.to(F64))[b], points[b, :, :nd].to(F64))
        out[b, :, :nd] = points[b, :, :nd].to(F64) + r * v
    return out


def point_warp_flow_grad(points, gout, flow_shape, r=1.0):
    nd = flow_shape[1]
    g = torch.zeros(flow_shape[0], *flow_shape[2:], nd, dtype=F64)
    for b in range(points.shape[0]):
        g[b] = _scatter(tuple(flow_shape[2:]), points[b, :, :nd].to(F64), r * gout[b, :, :nd].to(F64))
    return g.permute(0, nd + 1, *range(1, nd + 1)).contiguous()


def value_at(sdt, q):
    out = torch.empty(q.shape[0], q.shape[1], 1, dtype=F64)
    for b in range(q.shape[0]):
        v, _ = _interp(_last(sdt.to(F64))[b][..., None], q[b].to(F64))
        out[b] = v.abs()
    return out


def value_at_grad(sdt, q, gout):
    nd = sdt.dim() - 2
    g = torch.zeros(q.shape, dtype=F64)
    for b in range(q.shape[0]):
        v, dv = _interp(_last(sdt.to(F64))[b][..., None], q[b].to(F64))
        s = torch.sign(v[:, 0]) * gout[b, :, 0].to(F64)
        for d in range(nd):
            g[b, :, d] = s * dv[d, :, 0]
    return g


# ---- literal transcription of the TF graph, differentiated by autograd ----

def interpn_tf(vol, loc):
    """ne.utils.interpn(vol, loc, 'linear', fill_value=None) step by step (vol channel-last)."""
    nb_dims = loc.shape[-1]
    if vol.dim() == nb_dims:
        vol = vol[..., None]
    volshape = list(vol.shape)
    max_loc = [d - 1 for d in volshape[:-1]]
    loc0 = torch.floor(loc)
    clipped_loc = [loc[..., d].clamp(0, max_loc[d]) for d in range(nb_dims)]
    loc0lst = [loc0[..., d].clamp(0, max_loc[d]) for d in range(nb_dims)]
    loc1 = [(loc0lst[d] + 1).clamp(0, max_loc[d]) for d in range(nb_dims)]
    locs = [[f.detach().long() for f in loc0lst], [f.detach().long() for f in loc1]]
    diff_loc1 = [loc1[d] - clipped_loc[d] for d in range(nb_dims)]
    diff_loc0 = [1 - d for d in diff_loc1]
    weights_loc = [diff_loc1, diff_loc0]
    interp_vol = 0
    for c in itertools.product([0, 1], repeat=nb_dims):
        subs = [locs[c[d]][d] for d in range(nb_dims)]
        idx = 0
        for d in range(nb_dims):      # sub2ind2d: row-major
            idx = idx * volshape[d] + subs[d]
        vol_val = vol.reshape(-1, volshape[-1])[idx]
        wt = weights_loc[c[0]][0]
        for d in range(1, nb_dims):   # prod_n
            wt = wt * weights_loc[c[d]][d]
        interp_vol = interp_vol + wt[..., None] * vol_val
    return interp_vol


def point_warp_tf(points, flow, r=1.0):
    trf = _last(flow) * r
    li = points[..., -1:]
    sp = points[..., :-1]
    diff = torch.stack([interpn_tf(trf[b], sp[b]) for b in range(points.shape[0])])
    return torch.cat([sp + diff, li], -1)


def value_at_tf(sdt, q):
    vol = _last(sdt)
    return torch.stack([interpn_tf(vol[b], q[b]) for b in range(q.shape[0])]).abs()
