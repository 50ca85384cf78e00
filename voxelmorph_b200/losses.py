"""NCC / MSE / Dice / Grad losses with the reference's surface
(reference voxelmorph/torch/losses.py), and the KL loss and sigma-weighted MSE of the probabilistic
model and the soft-binned MutualInformation (reference voxelmorph/tf/losses.py): plain classes whose bound `.loss(y_true, y_pred)`
returns a 0-d tensor supporting `.item()`, `*`, `+`, `.backward()`.
Each loss is one fused sm_90a kernel (plus a fused backward) from libvxm_b200.so.
"""
import numpy as np
import torch

from . import _lib
from .layers import _dims


def _scalar(device):
    return torch.empty((), dtype=torch.float32, device=device)


class _NccFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y_true, y_pred, win):
        _lib.require_cuda(y_true, y_pred, what="NCC")
        I, J = _lib.contig(y_true), _lib.contig(y_pred)
        B, C, D, H, W, nd = _dims(I)
        if C != 1 or tuple(J.shape) != tuple(I.shape):
            # the reference's ones(1,1,*win) filter only accepts single-channel volumes (losses.py:29,51)
            raise _lib.VxmError("NCC: expected two single-channel volumes of equal shape, got %s and %s"
                                % (tuple(I.shape), tuple(J.shape)))
        wd, wh, ww = (1, win[0], win[1]) if nd == 2 else tuple(win)
        lib = _lib.load()
        loss = _scalar(I.device)
        # which gradients the backward owes: bit 0 = y_true, bit 1 = y_pred.  y_pred alone (the training loop) runs the
        # three-field kernels as ever; y_true adds Bp, Tp to the saved fields (5 per voxel for both, 3 for y_true alone)
        which = (1 if ctx.needs_input_grad[0] else 0) | (2 if ctx.needs_input_grad[1] else 0)
        saved = torch.empty((B, 5 if which == 3 else 3, D, H, W), dtype=torch.float32, device=I.device) if which else None
        ws = _lib.reduce_workspace(I.device)
        if which in (0, 2):
            _lib.check(lib.vxm_ncc_fwd(_lib.ptr(I), _lib.ptr(J), _lib.ptr(loss), _lib.ptr(saved), _lib.ptr(ws),
                                       B, D, H, W, wd, wh, ww, _lib.stream_ptr()), "vxm_ncc_fwd")
        else:
            _lib.check(lib.vxm_ncc_fwd2(_lib.ptr(I), _lib.ptr(J), _lib.ptr(loss), _lib.ptr(saved), _lib.ptr(ws), which,
                                        B, D, H, W, wd, wh, ww, _lib.stream_ptr()), "vxm_ncc_fwd2")
        ctx.save_for_backward(I, J)
        ctx.saved_fields = saved
        ctx.cfg = (B, D, H, W, wd, wh, ww, which)
        return loss

    @staticmethod
    def backward(ctx, gl):
        I, J = ctx.saved_tensors
        B, D, H, W, wd, wh, ww, which = ctx.cfg
        gl = gl.contiguous().float()
        gI = torch.empty_like(I) if which & 1 else None
        gJ = torch.empty_like(J) if which & 2 else None
        lib = _lib.load()
        if which == 2:
            _lib.check(lib.vxm_ncc_bwd(_lib.ptr(I), _lib.ptr(J), _lib.ptr(ctx.saved_fields), _lib.ptr(gl), _lib.ptr(gJ),
                                       B, D, H, W, wd, wh, ww, _lib.stream_ptr()), "vxm_ncc_bwd")
        else:
            _lib.check(lib.vxm_ncc_bwd2(_lib.ptr(I), _lib.ptr(J), _lib.ptr(ctx.saved_fields), _lib.ptr(gl), _lib.ptr(gI), _lib.ptr(gJ),
                                        which, B, D, H, W, wd, wh, ww, _lib.stream_ptr()), "vxm_ncc_bwd2")
        return gI, gJ, None


class NCC:
    """Local (over window) normalized cross correlation loss (reference losses.py:7-67)."""

    def __init__(self, win=None):
        self.win = win

    def loss(self, y_true, y_pred):
        ndims = len(list(y_true.size())) - 2
        assert ndims in [1, 2, 3], "volumes should be 1 to 3 dimensions. found: %d" % ndims
        if ndims == 1:
            raise _lib.VxmError("NCC: 1-D volumes are not supported by the GPU path")
        win = [9] * ndims if self.win is None else list(self.win)
        return _NccFn.apply(y_true, y_pred, tuple(int(w) for w in win))


class _MseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y_true, y_pred, scale):
        _lib.require_cuda(y_true, y_pred, what="MSE")
        if tuple(y_true.shape) != tuple(y_pred.shape):
            y_true, y_pred = torch.broadcast_tensors(y_true, y_pred)
        a, b = _lib.contig(y_true), _lib.contig(y_pred)
        lib = _lib.load()
        loss = _scalar(a.device)
        ws = _lib.reduce_workspace(a.device)
        if scale == 1.0:
            _lib.check(lib.vxm_mse_fwd(_lib.ptr(a), _lib.ptr(b), _lib.ptr(loss), _lib.ptr(ws), a.numel(), _lib.stream_ptr()),
                       "vxm_mse_fwd")
        else:
            _lib.check(lib.vxm_mse_scaled_fwd(_lib.ptr(a), _lib.ptr(b), _lib.ptr(loss), _lib.ptr(ws), a.numel(), scale,
                                              _lib.stream_ptr()), "vxm_mse_scaled_fwd")
        ctx.save_for_backward(a, b)
        ctx.scale = scale
        return loss

    @staticmethod
    def backward(ctx, gl):
        a, b = ctx.saved_tensors
        gl = gl.contiguous().float()
        gp = torch.empty_like(b)
        lib = _lib.load()
        if ctx.scale == 1.0:
            _lib.check(lib.vxm_mse_bwd(_lib.ptr(a), _lib.ptr(b), _lib.ptr(gl), _lib.ptr(gp), a.numel(), _lib.stream_ptr()),
                       "vxm_mse_bwd")
        else:
            _lib.check(lib.vxm_mse_scaled_bwd(_lib.ptr(a), _lib.ptr(b), _lib.ptr(gl), _lib.ptr(gp), a.numel(), ctx.scale,
                                              _lib.stream_ptr()), "vxm_mse_scaled_bwd")
        gt = -gp if ctx.needs_input_grad[0] else None
        return gt, gp, None


class MSE:
    """Mean squared error loss (reference losses.py:70-76); with `image_sigma`, the sigma-weighted form of the reference's
    TensorFlow side, 1 / image_sigma^2 * mean((y_true - y_pred)^2) (voxelmorph/tf/losses.py:112-134), which
    train.py --use-probs sets through --legacy-image-sigma."""

    def __init__(self, image_sigma=1.0):
        self.image_sigma = image_sigma

    def loss(self, y_true, y_pred):
        return _MseFn.apply(y_true, y_pred, 1.0 / float(self.image_sigma) ** 2)


class _DiceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y_true, y_pred):
        _lib.require_cuda(y_true, y_pred, what="Dice")
        a, b = _lib.contig(y_true), _lib.contig(y_pred)
        if tuple(a.shape) != tuple(b.shape) or a.dim() < 3:
            raise _lib.VxmError("Dice: expected equal (B,L,*vol) shapes, got %s and %s" % (tuple(a.shape), tuple(b.shape)))
        BL = a.shape[0] * a.shape[1]
        V = a.numel() // BL
        lib = _lib.load()
        loss = _scalar(a.device)
        sums = torch.empty((BL, 2), dtype=torch.float32, device=a.device)
        work = torch.empty(int(lib.vxm_dice_workspace_bytes(BL)), dtype=torch.uint8, device=a.device)
        _lib.check(lib.vxm_dice_fwd(_lib.ptr(a), _lib.ptr(b), _lib.ptr(loss), _lib.ptr(sums), _lib.ptr(work), BL, V,
                                    _lib.stream_ptr()), "vxm_dice_fwd")
        # the backward of either argument reads the OTHER tensor (and the two sums)
        ctx.save_for_backward(a if ctx.needs_input_grad[1] else None, b if ctx.needs_input_grad[0] else None, sums)
        ctx.cfg = (BL, V)
        return loss

    @staticmethod
    def backward(ctx, gl):
        a, b, sums = ctx.saved_tensors
        BL, V = ctx.cfg
        gl = gl.contiguous().float()
        lib = _lib.load()
        grads = []
        # top = 2 sum(ab) and bottom = clamp(sum(a + b)) are symmetric in (a, b): d/dy_pred = k1 y_true - k2 and
        # d/dy_true = k1 y_pred - k2 with the same k1, k2 (clamp branch included), so one kernel serves both
        for other in (b, a):
            g = None
            if other is not None:
                g = torch.empty_like(other)
                _lib.check(lib.vxm_dice_bwd(_lib.ptr(other), _lib.ptr(sums), _lib.ptr(gl), _lib.ptr(g), BL, V, _lib.stream_ptr()),
                           "vxm_dice_bwd")
            grads.append(g)
        return tuple(grads)


class Dice:
    """N-D dice for segmentation (reference losses.py:79-90)."""

    def loss(self, y_true, y_pred):
        return _DiceFn.apply(y_true, y_pred)


class _GradFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, penalty, mult):
        _lib.require_cuda(y, what="Grad")
        y = _lib.contig(y)
        B, C, D, H, W, nd = _dims(y)
        lib = _lib.load()
        loss = _scalar(y.device)
        _lib.check(lib.vxm_gradloss_fwd(_lib.ptr(y), _lib.ptr(loss), _lib.ptr(_lib.reduce_workspace(y.device)), B, C, D,
                                        H, W, nd, penalty, mult, _lib.stream_ptr()), "vxm_gradloss_fwd")
        ctx.save_for_backward(y)
        ctx.cfg = (B, C, D, H, W, nd, penalty, mult)
        return loss

    @staticmethod
    def backward(ctx, gl):
        (y,) = ctx.saved_tensors
        B, C, D, H, W, nd, penalty, mult = ctx.cfg
        gl = gl.contiguous().float()
        gy = torch.empty_like(y)
        lib = _lib.load()
        _lib.check(lib.vxm_gradloss_bwd(_lib.ptr(y), _lib.ptr(gl), _lib.ptr(gy), B, C, D, H, W, nd, penalty, mult,
                                        _lib.stream_ptr()), "vxm_gradloss_bwd")
        return gy, None, None


class Grad:
    """N-D gradient loss (reference losses.py:93-135)."""

    def __init__(self, penalty='l1', loss_mult=None):
        self.penalty = penalty
        self.loss_mult = loss_mult

    def loss(self, _, y_pred):
        if self.penalty == 'l1':
            p = 1
        else:
            assert self.penalty == 'l2', 'penalty can only be l1 or l2. Got: %s' % self.penalty
            p = 2
        mult = 1.0 if self.loss_mult is None else float(self.loss_mult)
        return _GradFn.apply(y_pred, p, mult)


class _KlFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, params, prior_lambda):
        _lib.require_cuda(params, what="KL")
        params = _lib.contig(params)
        B, C, D, H, W, nd = _dims(params)
        if C != 2 * nd:
            raise _lib.VxmError("KL: expected flow_params with 2 * %d channels (mean, log sigma), got %d" % (nd, C))
        loss = _scalar(params.device)
        _lib.check(_lib.load().vxm_kl_fwd(_lib.ptr(params), _lib.ptr(loss), _lib.ptr(_lib.reduce_workspace(params.device)),
                                          B, D, H, W, nd, prior_lambda, _lib.stream_ptr()), "vxm_kl_fwd")
        ctx.save_for_backward(params)
        ctx.cfg = (B, D, H, W, nd, prior_lambda)
        return loss

    @staticmethod
    def backward(ctx, gl):
        (params,) = ctx.saved_tensors
        B, D, H, W, nd, prior_lambda = ctx.cfg
        gl = gl.contiguous().float()
        gp = torch.empty_like(params)
        _lib.check(_lib.load().vxm_kl_bwd(_lib.ptr(params), _lib.ptr(gl), _lib.ptr(gp), B, D, H, W, nd, prior_lambda,
                                          _lib.stream_ptr()), "vxm_kl_bwd")
        return gp, None


class KL:
    """Kullback-Leibler divergence of probabilistic flows (reference voxelmorph/tf/losses.py:247-349), on the NCDHW
    `flow_params` of networks.VxmDenseProbabilistic: channels [0, nd) the mean mu, [nd, 2 nd) l = log sigma^2.

        loss = 0.5 nd (mean_{B,V,nd}(prior_lambda D e^l - l) + prior_lambda 0.5 / nd sum_i mean((mu_{x+e_i} - mu_x)^2))

    with D the number of in-volume axial neighbours of each voxel (the reference's degree matrix) and each mean over axis
    i's own difference tensor; an axis of size 1 has no differences and contributes nothing (the reference's mean of an
    empty tensor would be NaN).  `y_true` is ignored; `flow_vol_shape`, if given, must be y_pred's spatial shape."""

    def __init__(self, prior_lambda, flow_vol_shape=None):
        self.prior_lambda = prior_lambda
        self.flow_vol_shape = flow_vol_shape

    def loss(self, y_true, y_pred):
        if self.flow_vol_shape is not None and tuple(int(s) for s in self.flow_vol_shape) != tuple(y_pred.shape[2:]):
            raise _lib.VxmError("KL: flow_vol_shape %s does not match flow_params of spatial shape %s"
                                % (tuple(self.flow_vol_shape), tuple(y_pred.shape[2:])))
        return _KlFn.apply(y_pred, float(self.prior_lambda))


class _MiFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y_true, y_pred, centers, nb_bins, alpha, min_clip, max_clip):
        _lib.require_cuda(y_true, y_pred, what="MutualInformation")
        x, y = _lib.contig(y_true), _lib.contig(y_pred)
        if x.dim() not in (4, 5) or x.shape[1] != 1 or tuple(x.shape) != tuple(y.shape):
            # neurite's `volumes` asserts one channel and equal shapes; 2-D and 3-D volumes only here
            raise _lib.VxmError("MutualInformation: expected two single-channel 2-D or 3-D volumes (N, 1, *vol) of equal "
                                "shape, got %s and %s" % (tuple(x.shape), tuple(y.shape)))
        N = x.shape[0]
        V = x.numel() // N
        lib = _lib.load()
        loss = _scalar(x.device)
        work = torch.empty(int(lib.vxm_mi_workspace_bytes(N, V, nb_bins)), dtype=torch.uint8, device=x.device)
        rw = _lib.reduce_workspace(x.device) if centers is None else None
        _lib.check(lib.vxm_mi_fwd(_lib.ptr(x), _lib.ptr(y), _lib.ptr(centers), _lib.ptr(loss), _lib.ptr(work), _lib.ptr(rw),
                                  N, V, nb_bins, alpha, min_clip, max_clip, _lib.stream_ptr()), "vxm_mi_fwd")
        # the backward re-reads both volumes and the forward's tables in `work`
        ctx.save_for_backward(x, y)
        ctx.work, ctx.centers = work, centers
        ctx.cfg = (N, V, nb_bins, alpha, min_clip, max_clip)
        return loss

    @staticmethod
    def backward(ctx, gl):
        x, y = ctx.saved_tensors
        N, V, nb_bins, alpha, min_clip, max_clip = ctx.cfg
        gl = gl.contiguous().float()
        # like _NccFn: only the sides autograd asks for are computed
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gy = torch.empty_like(y) if ctx.needs_input_grad[1] else None
        if gx is not None or gy is not None:
            _lib.check(_lib.load().vxm_mi_bwd(_lib.ptr(x), _lib.ptr(y), _lib.ptr(ctx.centers), _lib.ptr(gl), _lib.ptr(gx),
                                              _lib.ptr(gy), _lib.ptr(ctx.work), N, V, nb_bins, alpha, min_clip, max_clip,
                                              _lib.stream_ptr()), "vxm_mi_bwd")
        return gx, gy, None, None, None, None, None


class MutualInformation:
    """Soft-binned mutual information loss (reference voxelmorph/tf/losses.py:352-367 on neurite's MutualInformation;
    Guo 2019, Hoffmann et al. SynthMorph, TMI 2022), for registration across contrasts (T1 to T2, MR to CT).

    Each image's intensities are soft-assigned to B bins with weights softmax_b(-alpha (clip(t) - c_b)^2); the joint
    histogram of the two images gives MI per item, and `.loss(y_true, y_pred)` returns -mean_n MI_n as a 0-d tensor.
    Inputs are (N, 1, *vol) fp32 CUDA tensors of equal shape, 2-D or 3-D.

    - `bin_centers` and `nb_bins` are exclusive; with neither, nb_bins = 16.  Without centres, each image's centres are
      linspace(min, max, B) over its whole batch (the min/max gradient is split among tied voxels, as torch.amin/amax do).
    - `soft_bin_alpha` defaults to 1 / (2 sigma^2) with sigma = 0.5 / (B - 1) (centres not given: this assumes
      intensities in [0, 1], which vxm's loaders produce; rescale other data or pass alpha), or sigma = 0.5 mean(diff(
      bin_centers)).  So alpha = 450 at B = 16 and 1922 at B = 32.
    - `min_clip` / `max_clip` default to -inf / +inf; the gradient passes where min_clip <= t <= max_clip.
    - 2 <= B <= 64.  Loss and gradients are computed by fused kernels (csrc/mi.cu) that never store per-voxel bins."""

    def __init__(self, bin_centers=None, nb_bins=None, soft_bin_alpha=None, min_clip=None, max_clip=None):
        if bin_centers is not None and nb_bins is not None:
            raise _lib.VxmError("MutualInformation: give bin_centers or nb_bins, not both")
        if bin_centers is not None:
            c = np.asarray(bin_centers, dtype=np.float64).reshape(-1)
            if not np.all(np.isfinite(c)):
                raise _lib.VxmError("MutualInformation: bin_centers must be finite")
            nb_bins = c.size
        elif nb_bins is None:
            nb_bins = 16
        nb_bins = int(nb_bins)
        if nb_bins < 2 or nb_bins > 64:
            raise _lib.VxmError("MutualInformation: the number of bins must be in [2, 64], got %d" % nb_bins)
        if soft_bin_alpha is None:
            sigma = 0.5 * float(np.mean(np.diff(c))) if bin_centers is not None else 0.5 / (nb_bins - 1)
            soft_bin_alpha = 1.0 / (2.0 * sigma ** 2) if sigma != 0 else float("inf")
        soft_bin_alpha = float(soft_bin_alpha)
        if not (np.isfinite(soft_bin_alpha) and soft_bin_alpha > 0):
            raise _lib.VxmError("MutualInformation: soft_bin_alpha must be finite and positive, got %r" % soft_bin_alpha)
        self.nb_bins = nb_bins
        self.bin_centers = None if bin_centers is None else c.astype(np.float32)
        self.soft_bin_alpha = soft_bin_alpha
        self.min_clip = -np.inf if min_clip is None else float(min_clip)
        self.max_clip = np.inf if max_clip is None else float(max_clip)
        self._dev_centers = {}

    def _centers(self, device):
        if self.bin_centers is None:
            return None
        t = self._dev_centers.get(device)
        if t is None:
            t = torch.from_numpy(self.bin_centers).to(device)
            self._dev_centers[device] = t
        return t

    def loss(self, y_true, y_pred):
        return _MiFn.apply(y_true, y_pred, self._centers(y_true.device), self.nb_bins, self.soft_bin_alpha,
                           self.min_clip, self.max_clip)


def hyper_loss(hyp, image_loss, reg_loss):
    """HyperMorph's loss (reference scripts/tf/train_hypermorph.py:159-177): (1 - lam) image_loss + lam reg_loss with
    lam = hyp[0, 0], formed on the device from the (1, 1) hyp tensor (no host synchronisation, so a captured step takes
    the lambda of each replay's hyp).  lam receives no gradient.  The script's terms are image_loss = MSE(image_sigma=0.05)
    or NCC and reg_loss = Grad('l2', loss_mult=int_downsize) of the pre-integration flow."""
    lam = hyp.detach().reshape(-1)[0]
    return (1.0 - lam) * image_loss + lam * reg_loss
