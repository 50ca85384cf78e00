"""Linear sampling at given coordinates, and its adjoints, evaluated in float64 (numpy).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  `ref_torch.spatial_transform` samples at coordinates it
derives itself (p + flow, then grid_sample's normalise / un-normalise round trip); the fast CUDA paths sample at
fl32(p + flow).  The two can pick different trilinear cells for the same input, and the derivative with respect to
the coordinates jumps across a cell face, so a per-voxel check of a large field needs a reference that samples
at the kernel's own fp32 coordinates.  These helpers take the coordinates as given (any float array, read
exactly) and do everything else in float64:

* `sample` / `sample_adjoint`: trilinear (3-D) or bilinear (2-D) interpolation with zero padding, as
  F.grid_sample(align_corners=True, padding_mode="zeros") defines it, and its adjoints with respect to the
  source and to the coordinates;
* `coords_fp32`: fl32(p + v), the coordinates the fast warp and VecInt kernels form;
* `coords_replayed`: the fp32 coordinates of torch's normalise / un-normalise round trip (`spec_np._sample_coords`),
  which the exact-arithmetic warp and VecInt kernels form;
* `quantised`: a smooth field whose values are odd multiples of 2^-11 with |v| < 2^7, so that p + v is exact in fp32
  and never integral: every sampler, whatever its coordinate arithmetic, then picks the same trilinear cell;
* `vecint_step` / `vecint_adjoint`: one scaling-and-squaring step v + v(p + v), and the adjoint of the whole
  chain over a given list of states v_0 .. v_{n-1} (e.g. the ones the CUDA kernel saved).
"""
import numpy as np


def _cell(S, c):
    """Per spatial axis a of the (nd, N) coordinate array c: the lower corner index, the fraction t, and for the
    two taps (bit 0 / 1) the clamped index, the weight (0 outside the volume) and the validity (1 / 0)."""
    axes = []
    for a, n in enumerate(S):
        f = np.floor(c[a])
        t = c[a] - f
        i0 = f.astype(np.int64)
        taps = []
        for bit in (0, 1):
            i = i0 + bit
            ok = ((i >= 0) & (i < n)).astype(np.float64)
            w = (t if bit else 1.0 - t) * ok
            taps.append((np.clip(i, 0, n - 1), w, ok))
        axes.append(taps)
    return axes


def _corners(S, c):
    """Yield, for each of the 2^nd corners: flat source index (clamped), weight, and per axis the derivative of the
    weight with respect to that axis' coordinate."""
    nd = len(S)
    axes = _cell(S, c)
    for k in range(1 << nd):
        bits = [(k >> (nd - 1 - a)) & 1 for a in range(nd)]
        idx = np.ravel_multi_index(tuple(axes[a][bits[a]][0] for a in range(nd)), S)
        w = np.ones(c.shape[1])
        for a in range(nd):
            w = w * axes[a][bits[a]][1]
        dw = []
        for a in range(nd):
            d = axes[a][bits[a]][2] * (1.0 if bits[a] else -1.0)
            for o in range(nd):
                if o != a:
                    d = d * axes[o][bits[o]][1]
            dw.append(d)
        yield idx, w, dw


def _flat(src, coords):
    src = np.asarray(src, np.float64)
    coords = np.asarray(coords)
    B, C = src.shape[:2]
    S = src.shape[2:]
    nd = len(S)
    assert coords.shape[:2] == (B, nd), (src.shape, coords.shape)
    O = coords.shape[2:]
    return src.reshape(B, C, -1), coords.reshape(B, nd, -1).astype(np.float64), S, O


def sample(src, coords):
    """src (B, C, *S) sampled at coords (B, nd, *O) (voxel units, spatial axis order): (B, C, *O) float64."""
    s, c, S, O = _flat(src, coords)
    out = np.zeros(s.shape[:2] + (c.shape[2],))
    for b in range(s.shape[0]):
        for idx, w, _ in _corners(S, c[b]):
            out[b] += s[b][:, idx] * w
    return out.reshape(s.shape[:2] + tuple(O))


def sample_adjoint(src, coords, gout):
    """Adjoints of `sample` applied to gout (B, C, *O): (d/d src, d/d coords), shaped like src and coords."""
    s, c, S, O = _flat(src, coords)
    B, C, N = s.shape
    go = np.asarray(gout, np.float64).reshape(B, C, -1)
    gsrc = np.zeros_like(s)
    gc = np.zeros_like(c)
    for b in range(B):
        for idx, w, dw in _corners(S, c[b]):
            for ch in range(C):
                gsrc[b, ch] += np.bincount(idx, weights=w * go[b, ch], minlength=N)
            vg = (s[b][:, idx] * go[b]).sum(axis=0)
            for a in range(len(S)):
                gc[b, a] += vg * dw[a]
    return gsrc.reshape(np.shape(src)), gc.reshape(np.shape(coords))


def coords_fp32(v):
    """fl32(p + v) for a (B, nd, *S) field: the sample coordinates of the fast warp / VecInt kernels."""
    v = np.asarray(v, np.float32)
    S = v.shape[2:]
    grid = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float32) for n in S], indexing="ij"))
    return (grid[None] + v).astype(np.float32)


def coords_replayed(v, div="true"):
    """The fp32 sample coordinates of the reference's round trip p + v -> [-1, 1] -> voxel units for a (B, nd, *S) field
    (spec_np._sample_coords, stacked on axis 1): those of the exact-arithmetic warp / VecInt kernels.  `div` as in
    spec_np.warp ('true': torch CPU's division, 'recip': torch CUDA's multiply by the reciprocal)."""
    from . import spec_np
    return np.stack(spec_np._sample_coords(v, div), axis=1)


def quantised(seed, channels, shape, scale):
    """cases.smooth_field(seed, channels, shape, scale) rounded to odd multiples of 2^-11 (|v| < 2^7 asserted): p + v is
    exact in fp32 for any voxel index p < 2^12 and never an integer, so fp64 round-off cannot move a sample across a
    cell face either."""
    from . import cases
    f = cases.smooth_field(seed, channels, shape, scale=scale).astype(np.float64)
    q = (2.0 * np.floor(f * 2.0 ** 10) + 1.0) * 2.0 ** -11
    assert np.abs(q).max() < 2.0 ** 7
    return q.astype(np.float32)


def vecint_step(v):
    """One squaring of a float32 state v (B, nd, *S): v + v(fl32(p + v)), in float64."""
    return np.asarray(v, np.float64) + sample(v, coords_fp32(v))


def vecint_adjoint(states, gout, scale, coords=coords_fp32):
    """d(v_n)/d(vel)^T gout for the chain v_0 = scale * vel, v_{k+1} = v_k + v_k(c(v_k)), evaluated along the given
    states v_0 .. v_{n-1} (each (B, nd, *S)) at the coordinates `coords(v_k)`: fl32(p + v_k) by default, or e.g.
    `coords_replayed`.  Both have d c / d v = 1 in exact arithmetic, which is what the adjoint uses."""
    g = np.asarray(gout, np.float64)
    for v in reversed(states):
        gs, gc = sample_adjoint(v, coords(v), g)
        g = g + gs + gc
    return g * scale
