"""fp64 / numpy restatement of probabilistic diffeomorphic VoxelMorph for the tests, composed from the oracle's primitives
(oracle/ref_torch.py, which stays untouched).

* The sampler's noise stream (include/vxm_b200.h, vxm_sample_normal_logvar_fwd): Philox4x32-10 keyed by the 64-bit
  seed, element i = (b nd + c) V + v taking word i mod 4 of the block with counter (lo32(i / 4), hi32(i / 4), lo32(call),
  hi32(call)), Box-Muller on the word pairs (0, 1) and (2, 3) with u1 = ((w0 >> 8) + 1) 2^-24 in (0, 1] and
  u2 = (w1 >> 8) 2^-24: eps0 = sqrt(-2 log u1) cos(2 pi u2), eps1 = sqrt(-2 log u1) sin(2 pi u2).
* SampleNormalLogVar (neurite; not in the reference tree): z = mu + exp(logvar / 2) eps.
* KL(prior_lambda) (reference voxelmorph/tf/losses.py:247-349) in closed form, and a literal transcription of it.
* The probabilistic step: flow_params = cat(flow(x), log_sigma(x)) (voxelmorph/tf/networks.py:155-165), the sampled
  field through resize / VecInt / resize / warp as ref_torch.vxm_forward does with its field, eps given as an input.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ref_torch

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: four uint32 arrays (counter words), key: two uint32 values -> four uint32 arrays."""
    c = [np.asarray(w, dtype=np.uint64) for w in ctr]
    k0, k1 = int(key[0]), int(key[1])
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
    return [w.astype(np.uint32) for w in c]


def _sinpi(x):
    """sin(pi x) for x in [0, 2), with the exact zeros and ones of the kernel's sincospif (x is a multiple of 2^-23)."""
    neg = x >= 1
    r = np.where(neg, x - 1, x)
    v = np.sin(np.pi * np.minimum(r, 1 - r))
    return np.where(neg, -v, v)


def normal_stream(n, seed, call):
    """eps[0:n] (float64) of the stream (seed, call)."""
    seed, call = int(seed) & ((1 << 64) - 1), int(call) & ((1 << 64) - 1)
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    ctr = [q & _MASK, q >> np.uint64(32), np.full_like(q, call & 0xFFFFFFFF), np.full_like(q, call >> 32)]
    w = philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))
    out = np.empty((q.size, 4), dtype=np.float64)
    for j, (a, b) in enumerate(((w[0], w[1]), (w[2], w[3]))):
        u1 = ((a >> 8).astype(np.float64) + 1.0) * 2.0 ** -24
        u2 = (b >> 8).astype(np.float64) * 2.0 ** -24
        r = np.sqrt(-2.0 * np.log(u1))
        x = 2 * u2                                   # sincospif(2 u2): cos(2 pi u2) = sin(pi ((x + 0.5) mod 2))
        out[:, 2 * j] = r * _sinpi(np.mod(x + 0.5, 2.0))
        out[:, 2 * j + 1] = r * _sinpi(x)
    return out.reshape(-1)[:n]


def sample_normal_logvar(mu, logvar, seed, call):
    """(z, eps) in float64 for mu, logvar of shape (B, nd, *vol)."""
    mu, logvar = np.asarray(mu, dtype=np.float64), np.asarray(logvar, dtype=np.float64)
    eps = normal_stream(mu.size, seed, call).reshape(mu.shape)
    return mu + np.exp(logvar / 2) * eps, eps


# ---- KL (reference voxelmorph/tf/losses.py:247-349) -------------------------------------------------------------------

def degree(shape):
    """Number of in-volume axial neighbours of every voxel of a volume of `shape`."""
    deg = np.zeros(shape, dtype=np.float64)
    for ax, n in enumerate(shape):
        idx = np.arange(n).reshape([-1 if a == ax else 1 for a in range(len(shape))])
        deg = deg + (idx > 0) + (idx < n - 1)
    return deg


def kl_loss(params, prior_lambda):
    """Closed form on flow_params (B, 2 nd, *vol), float64: 0.5 nd (sigma_term + prec_term); an axis of size 1 has no
    differences and contributes 0 to prec_term."""
    p = np.asarray(params, dtype=np.float64)
    nd = p.ndim - 2
    mu, lv = p[:, :nd], p[:, nd:]
    sigma = np.mean(prior_lambda * degree(p.shape[2:]) * np.exp(lv) - lv)
    prec = 0.0
    for ax in range(2, p.ndim):
        if p.shape[ax] > 1:
            prec += np.mean(np.diff(mu, axis=ax) ** 2)
    return 0.5 * nd * (sigma + prior_lambda * 0.5 / nd * prec)


def kl_grad(params, prior_lambda):
    """d kl_loss / d params in closed form: pointwise in l, the axis-scaled 2 nd-point Laplacian of mu; and the magnitude
    (sum of the absolute values of the terms, for rounding bounds)."""
    p = np.asarray(params, dtype=np.float64)
    nd = p.ndim - 2
    B, V = p.shape[0], int(np.prod(p.shape[2:]))
    mu, lv = p[:, :nd], p[:, nd:]
    g, mag = np.zeros_like(p), np.zeros_like(p)
    a = prior_lambda * degree(p.shape[2:]) * np.exp(lv)
    g[:, nd:] = 0.5 / (B * V) * (a - 1)
    mag[:, nd:] = 0.5 / (B * V) * (a + 1)
    for ax in range(2, p.ndim):
        n = p.shape[ax]
        if n < 2:
            continue
        c = prior_lambda / (4.0 * B * nd * (n - 1) * (V / n))
        d = np.diff(mu, axis=ax) * 2 * c              # d/d(mu_{x+1}) of c (mu_{x+1} - mu_x)^2
        lo = [slice(None)] * p.ndim
        hi = [slice(None)] * p.ndim
        lo[ax], hi[ax] = slice(0, n - 1), slice(1, n)
        gm, mm = g[:, :nd], mag[:, :nd]
        gm[tuple(hi)] += d
        gm[tuple(lo)] -= d
        mm[tuple(hi)] += np.abs(d)
        mm[tuple(lo)] += np.abs(d)
    return g, mag


def kl_literal(params, prior_lambda):
    """A literal torch transcription of tf/losses.py:257-349 on the NCDHW layout (channels moved last as in TF): the
    degree matrix as the SAME-padded conv of ones with _adj_filt, prec_loss by permute / diff / mean.  A size-1 axis gives
    an empty difference tensor whose mean is NaN; such terms are dropped here (the closed form counts them as 0)."""
    y = params.permute(0, *range(2, params.dim()), 1)              # NDHWC, as TF holds it
    nd = y.dim() - 2
    vol = list(y.shape[1:-1])
    # _adj_filt(nd): [3]*nd + [nd, nd], 1 at the axial neighbours of the centre, feature i -> feature i
    inner = np.zeros([3] * nd)
    for j in range(nd):
        o = [[1]] * nd
        o[j] = [0, 2]
        inner[np.ix_(*o)] = 1
    filt = np.zeros([3] * nd + [nd, nd])
    for i in range(nd):
        filt[..., i, i] = inner
    conv = (F.conv1d, F.conv2d, F.conv3d)[nd - 1]
    w = torch.from_numpy(filt).to(y.dtype).permute(nd + 1, nd, *range(nd))          # (out, in, k...)
    ones = torch.ones([1, nd] + vol, dtype=y.dtype)
    D = conv(ones, w, padding=1).permute(0, *range(2, nd + 2), 1)                   # (1, *vol, nd)
    mean, log_sigma = y[..., 0:nd], y[..., nd:]
    sigma_term = (prior_lambda * D * torch.exp(log_sigma) - log_sigma).mean()
    sm = 0
    for i in range(nd):
        d = i + 1
        r = [d, *range(d), *range(d + 1, nd + 2)]
        yy = mean.permute(*r)
        df = yy[1:, ...] - yy[:-1, ...]
        if df.numel():
            sm = sm + (df * df).mean()
    prec_term = prior_lambda * (0.5 * sm / nd)
    return 0.5 * nd * (sigma_term + prec_term)


def mse_sigma(y_true, y_pred, image_sigma):
    """tf/losses.py:112-134."""
    return 1.0 / image_sigma ** 2 * ((y_true - y_pred) ** 2).mean()


# ---- the probabilistic step -----------------------------------------------------------------------------------------

def flow_params(sd, cfg, source, target):
    """cat(flow(x), log_sigma(x)) of the U-Net output x (state-dict keys of VxmDenseProbabilistic)."""
    x = ref_torch.unet_forward(torch.cat([source, target], dim=1), sd, cfg)
    return torch.cat([ref_torch._conv(x, sd, "flow", False), ref_torch._conv(x, sd, "log_sigma", False)], dim=1)


def prob_forward(sd, cfg, source, target, eps, registration=False):
    """VxmDenseProbabilistic.forward with the noise `eps` (B, nd, *) given: training form (y_source[, y_target],
    flow_params), registration form (y_source, pos_flow) from the mean."""
    int_steps = cfg.get("int_steps", 7)
    int_downsize = cfg.get("int_downsize", 2)
    bidir = cfg.get("bidir", False)
    fp = flow_params(sd, cfg, source, target)
    nd = fp.shape[1] // 2
    mu, lv = fp[:, :nd], fp[:, nd:]
    pos = mu if registration else mu + torch.exp(lv / 2) * eps
    if (not cfg.get("unet_half_res", False)) and int_steps > 0 and int_downsize > 1:
        pos = ref_torch.resize_transform(pos, int_downsize)
    neg = -pos if bidir else None
    if int_steps > 0:
        pos = ref_torch.vec_int(pos, int_steps)
        neg = ref_torch.vec_int(neg, int_steps) if bidir else None
        if int_downsize > 1:
            pos = ref_torch.resize_transform(pos, 1 / int_downsize)
            neg = ref_torch.resize_transform(neg, 1 / int_downsize) if bidir else None
    y_source = ref_torch.spatial_transform(source, pos)
    if registration:
        return y_source, pos
    y_target = ref_torch.spatial_transform(target, neg) if bidir else None
    return (y_source, y_target, fp) if bidir else (y_source, fp)


def kl_torch(fp, prior_lambda):
    """kl_loss in torch (autograd reference for the step's gradient)."""
    nd = fp.dim() - 2
    mu, lv = fp[:, :nd], fp[:, nd:]
    deg = torch.from_numpy(degree(tuple(fp.shape[2:]))).to(fp.dtype)
    sigma = (prior_lambda * deg * torch.exp(lv) - lv).mean()
    prec = 0
    for ax in range(2, fp.dim()):
        if fp.shape[ax] > 1:
            prec = prec + (torch.diff(mu, dim=ax) ** 2).mean()
    return 0.5 * nd * (sigma + prior_lambda * 0.5 / nd * prec)


def prob_loss(outs, target, source=None, image_sigma=0.02, kl_lambda=10.0, kl_weight=0.01):
    """train.py --use-probs: MSE(image_sigma)(target, y_source) [+ the same on (source, y_target) when bidir]
    + kl_weight KL(kl_lambda)(flow_params)."""
    y_source, fp = outs[0], outs[-1]
    loss = mse_sigma(target, y_source, image_sigma)
    if len(outs) == 3:
        loss = loss + mse_sigma(source, outs[1], image_sigma)
    return loss + kl_weight * kl_torch(fp, kl_lambda)


def init_log_sigma(sd, cfg, seed=0, std=1e-2, bias=-3.0):
    """Adds log_sigma.* to an oracle state dict: spread-out values (the model's own init, N(0, 1e-10) and -10, makes the
    noise vanish), so that the sampled term counts in a test."""
    g = torch.Generator().manual_seed(seed + 1)
    nd = len(cfg["inshape"])
    w = sd["flow.weight"]
    out = dict(sd)
    out["log_sigma.weight"] = torch.randn((nd,) + tuple(w.shape[1:]), generator=g, dtype=w.dtype) * std
    out["log_sigma.bias"] = torch.full((nd,), float(bias), dtype=w.dtype)
    return out


def standard_error_bounds(eps, k=5.0):
    """|mean| and |var - 1| bounds of k standard errors for n N(0, 1) samples."""
    n = eps.size
    return k / math.sqrt(n), k * math.sqrt(2.0 / n)
