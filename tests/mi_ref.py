"""fp64 restatements of the MutualInformation loss (neurite's soft-binned MI behind reference
voxelmorph/tf/losses.py:352-367), used to pin the spec on the CPU and to check the CUDA kernels.

- `mi_closed_form`: numpy, the loss and the closed-form gradient of both inputs (the chain rule the backward kernel runs),
  computed over voxel chunks so a full 160x192x224 volume fits in memory.
- `mi_torch_graph`: a literal torch transcription of the TF graph (soft quantize with linspace centres, then `maps`),
  differentiated by autograd.
"""
import numpy as np
import torch

EPS = 1e-7   # Keras' epsilon


def default_alpha(nb_bins=None, bin_centers=None):
    if bin_centers is not None:
        sigma = 0.5 * float(np.mean(np.diff(np.asarray(bin_centers, np.float64))))
    else:
        sigma = 0.5 / (nb_bins - 1)
    return 1.0 / (2.0 * sigma ** 2)


def _centres(t, nb_bins, bin_centers):
    if bin_centers is not None:
        return np.asarray(bin_centers, np.float64)
    lo, hi = float(t.min()), float(t.max())
    return lo + (hi - lo) * np.arange(nb_bins, dtype=np.float64) / (nb_bins - 1)


def _weights(tc, c, alpha):
    s = -alpha * (tc[:, None] - c[None, :]) ** 2
    s -= s.max(axis=1, keepdims=True)
    e = np.exp(s)
    return e / e.sum(axis=1, keepdims=True)


def _tables(P, sx, sy):
    """MI of one item and dMI/dP, dMI/dsx, dMI/dsy (fp64)."""
    S1, SX1, SY1 = P.sum() + EPS, sx.sum() + EPS, sy.sum() + EPS
    pxy, px, py = P / S1, sx / SX1, sy / SY1
    den = px[:, None] * py[None, :] + EPS
    r = pxy / den
    lg = np.log(r + EPS)
    mi = float((pxy * lg).sum())
    A = lg + pxy / ((r + EPS) * den)                      # dMI/dpxy
    Q = -pxy * pxy / ((r + EPS) * den * den)              # dMI/d(px py)
    gpx, gpy = Q @ py, Q.T @ px
    gP = A / S1 - (A * P).sum() / S1 ** 2
    gsx = gpx / SX1 - (gpx * sx).sum() / SX1 ** 2
    gsy = gpy / SY1 - (gpy * sy).sum() / SY1 ** 2
    return mi, gP, gsx, gsy


def mi_closed_form(x, y, nb_bins=None, bin_centers=None, alpha=None, min_clip=-np.inf, max_clip=np.inf,
                   chunk=1 << 18, grads=True):
    """loss, d loss / d x, d loss / d y for x = y_true, y = y_pred of shape (N, 1, *vol) (any float dtype; computed in
    fp64).  Returns (loss, gx, gy) with gx, gy float64 arrays of x's shape (None when grads=False)."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    N = x.shape[0]
    xf, yf = x.reshape(N, -1), y.reshape(N, -1)
    V = xf.shape[1]
    B = len(bin_centers) if bin_centers is not None else (16 if nb_bins is None else int(nb_bins))
    if alpha is None:
        alpha = default_alpha(B, bin_centers)
    cx, cy = _centres(xf, B, bin_centers), _centres(yf, B, bin_centers)
    clip = lambda t: np.clip(t, min_clip, max_clip)
    tabs, mis = [], []
    for n in range(N):
        P, sx, sy = np.zeros((B, B)), np.zeros(B), np.zeros(B)
        for v0 in range(0, V, chunk):
            wx = _weights(clip(xf[n, v0:v0 + chunk]), cx, alpha)
            wy = _weights(clip(yf[n, v0:v0 + chunk]), cy, alpha)
            P += wx.T @ wy
            sx += wx.sum(0)
            sy += wy.sum(0)
        mi, gP, gsx, gsy = _tables(P, sx, sy)
        mis.append(mi)
        tabs.append((gP, gsx, gsy))
    loss = -float(np.mean(mis))
    if not grads:
        return loss, None, None
    s = -1.0 / N
    gx, gy = np.zeros_like(xf), np.zeros_like(yf)
    dcx, dcy = np.zeros(B), np.zeros(B)
    for n in range(N):
        gP, gsx, gsy = tabs[n]
        for v0 in range(0, V, chunk):
            tx, ty = xf[n, v0:v0 + chunk], yf[n, v0:v0 + chunk]
            txc, tyc = clip(tx), clip(ty)
            wx, wy = _weights(txc, cx, alpha), _weights(tyc, cy, alpha)
            for w, wo, G, gs, tc, t, c, g, dc in ((wx, wy, gP, gsx, txc, tx, cx, gx, dcx),
                                                  (wy, wx, gP.T, gsy, tyc, ty, cy, gy, dcy)):
                a = wo @ G.T + gs[None, :]                            # a_vb = sum_c G_bc wo_vc + gs_b
                d = w * (a - (w * a).sum(1, keepdims=True))           # softmax backward
                e = s * d * 2.0 * alpha * (tc[:, None] - c[None, :])  # dL/dc_b per voxel
                mask = (t >= min_clip) & (t <= max_clip)
                g[n, v0:v0 + chunk] = np.where(mask, -e.sum(1), 0.0)
                dc += e.sum(0)
    if bin_centers is None:   # the linspace centres' path to the min and max, split among ties
        f = np.arange(B) / (B - 1)
        for tf, g, dc in ((xf, gx, dcx), (yf, gy, dcy)):
            lo, hi = tf.min(), tf.max()
            at_lo, at_hi = tf == lo, tf == hi
            g += at_lo * ((dc * (1 - f)).sum() / at_lo.sum()) + at_hi * ((dc * f).sum() / at_hi.sum())
    return loss, gx.reshape(x.shape), gy.reshape(y.shape)


def mi_torch_graph(x, y, nb_bins=None, bin_centers=None, alpha=None, min_clip=-np.inf, max_clip=np.inf):
    """The TF graph op for op in torch fp64, differentiated by autograd: (loss, gx, gy)."""
    B = len(bin_centers) if bin_centers is not None else (16 if nb_bins is None else int(nb_bins))
    if alpha is None:
        alpha = default_alpha(B, bin_centers)
    xt = torch.tensor(np.asarray(x, np.float64), requires_grad=True)
    yt = torch.tensor(np.asarray(y, np.float64), requires_grad=True)

    def soft_quantize(t):   # neurite.utils.soft_quantize(..., return_log=False)
        if bin_centers is None:
            lo, hi = torch.amin(t), torch.amax(t)
            c = lo + (hi - lo) * torch.arange(B, dtype=torch.float64) / (B - 1)   # tf.linspace(lo, hi, B)
        else:
            c = torch.tensor(np.asarray(bin_centers, np.float64))
        t = torch.clamp(t, min_clip, max_clip)
        return torch.softmax(-alpha * (t[..., None] - c) ** 2, dim=-1)

    N = xt.shape[0]
    qx = soft_quantize(xt).reshape(N, -1, B)
    qy = soft_quantize(yt).reshape(N, -1, B)
    # neurite MutualInformation.maps
    pxy = torch.bmm(qx.transpose(1, 2), qy)
    pxy = pxy / (pxy.sum(dim=(1, 2), keepdim=True) + EPS)
    px = qx.sum(1, keepdim=True)
    px = px / (px.sum(2, keepdim=True) + EPS)
    py = qy.sum(1, keepdim=True)
    py = py / (py.sum(2, keepdim=True) + EPS)
    pxpy = torch.bmm(px.transpose(1, 2), py) + EPS
    mi = (pxy * torch.log(pxy / pxpy + EPS)).sum(dim=(1, 2))
    loss = -mi.mean()   # Keras' batch mean of -volumes(...)
    loss.backward()
    return float(loss.detach()), xt.grad.numpy(), yt.grad.numpy()


def make_case(seed, shape, n=1, ties=False, constant=False):
    """A correlated, non-monotonic pair of intensity volumes in [0, 1] of shape (n, 1, *shape), float32."""
    rng = np.random.default_rng(seed)
    x = rng.random((n, 1) + tuple(shape)).astype(np.float32)
    y = np.cos(3.0 * x) ** 2 * 0.8 + 0.2 * rng.random(x.shape)
    y = y.astype(np.float32)
    if ties:   # a skull-stripped look: about half the voxels at the minimum 0
        x[rng.random(x.shape) < 0.5] = 0.0
        y[rng.random(y.shape) < 0.4] = 0.0
    if constant:
        x[...] = 0.25
    return x, y
