"""Unet / VxmDense / ConvBlock with the reference's surface
(reference voxelmorph/torch/networks.py): same class names, constructor arguments, attributes
(`unet_model`, `flow`, `resize`, `fullsize`, `integrate`, `transformer`, `bidir`, `config`,
`Unet.final_nf`), forward signatures / return tuples and `state_dict` keys — so reference
checkpoints load unchanged — with every operator running in sm_90a kernels.
"""
import numpy as np
import torch
import torch.nn as nn
from torch.distributions.normal import Normal

from . import _lib, layers, ops
from .modelio import LoadableModel, store_config_args


def default_unet_features():
    """reference voxelmorph/py/utils.py:16-21"""
    return [[16, 32, 32, 32], [32, 32, 32, 32, 32, 16, 16]]


def _conv_cls(ndims):
    if ndims == 2:
        return _Conv2dK3
    if ndims == 3:
        return _Conv3dK3
    raise NotImplementedError("voxelmorph_b200: %d-D convolutions are not supported (2-D and 3-D only; the "
                              "reference's SpatialTransformer handles 2-D/3-D only as well, layers.py:41-46)" % ndims)


class _Conv3dK3(nn.Conv3d):
    """nn.Conv3d parameters (weight (Cout,Cin,3,3,3), bias, default init) + the vxm conv kernel."""

    def forward(self, x):
        _check_k3(self)
        return ops.conv_k3(x, self.weight, self.bias, None)


class _Conv2dK3(nn.Conv2d):
    def forward(self, x):
        _check_k3(self)
        return ops.conv_k3(x, self.weight, self.bias, None)


def _check_k3(m):
    nd = len(m.kernel_size)
    if tuple(m.kernel_size) != (3,) * nd or tuple(m.stride) != (1,) * nd or tuple(m.padding) != (1,) * nd \
            or tuple(m.dilation) != (1,) * nd or m.groups != 1:
        raise NotImplementedError("voxelmorph_b200 conv kernels implement kernel 3, stride 1, padding 1 only")


class ConvBlock(nn.Module):
    """Convolution followed by LeakyReLU(0.2) (reference networks.py:290-305), fused in one kernel."""

    def __init__(self, ndims, in_channels, out_channels, stride=1):
        super().__init__()
        self.main = _conv_cls(ndims)(in_channels, out_channels, 3, stride, 1)
        self.activation = nn.LeakyReLU(0.2)

    def forward(self, x):
        _check_k3(self.main)
        return ops.conv_k3(x, self.main.weight, self.main.bias, self.activation.negative_slope)


class _Pool2(nn.Module):
    def forward(self, x):
        return ops.maxpool2(x)


class Unet(nn.Module):
    """
    A unet architecture (reference networks.py:12-144). Layer features can be specified directly as a
    list of encoder and decoder features or as a single integer along with a number of unet levels.
    Default features: encoder [16, 32, 32, 32], decoder [32, 32, 32, 32, 32, 16, 16].
    """

    def __init__(self, inshape=None, infeats=None, nb_features=None, nb_levels=None, max_pool=2,
                 feat_mult=1, nb_conv_per_level=1, half_res=False):
        super().__init__()
        ndims = len(inshape)
        assert ndims in [1, 2, 3], 'ndims should be one of 1, 2, or 3. found: %d' % ndims
        self.half_res = half_res

        if nb_features is None:
            nb_features = default_unet_features()
        if isinstance(nb_features, int):
            if nb_levels is None:
                raise ValueError('must provide unet nb_levels if nb_features is an integer')
            feats = np.round(nb_features * feat_mult ** np.arange(nb_levels)).astype(int)
            nb_features = [np.repeat(feats[:-1], nb_conv_per_level), np.repeat(np.flip(feats), nb_conv_per_level)]
        elif nb_levels is not None:
            raise ValueError('cannot use nb_levels if nb_features is not an integer')

        enc_nf, dec_nf = nb_features
        nb_dec_convs = len(enc_nf)
        final_convs = dec_nf[nb_dec_convs:]
        dec_nf = dec_nf[:nb_dec_convs]
        self.nb_levels = int(nb_dec_convs / nb_conv_per_level) + 1

        if isinstance(max_pool, int):
            max_pool = [max_pool] * self.nb_levels
        if any(int(s) != 2 for s in max_pool):
            raise NotImplementedError("voxelmorph_b200: only max_pool=2 is implemented")
        self.pooling = [_Pool2() for _ in max_pool]
        self.upsampling = [nn.Upsample(scale_factor=s, mode='nearest') for s in max_pool]  # attribute parity only

        prev_nf = infeats
        encoder_nfs = [prev_nf]
        self.encoder = nn.ModuleList()
        for level in range(self.nb_levels - 1):
            convs = nn.ModuleList()
            for conv in range(nb_conv_per_level):
                nf = int(enc_nf[level * nb_conv_per_level + conv])
                convs.append(ConvBlock(ndims, prev_nf, nf))
                prev_nf = nf
            self.encoder.append(convs)
            encoder_nfs.append(prev_nf)

        encoder_nfs = np.flip(encoder_nfs)
        self.decoder = nn.ModuleList()
        for level in range(self.nb_levels - 1):
            convs = nn.ModuleList()
            for conv in range(nb_conv_per_level):
                nf = int(dec_nf[level * nb_conv_per_level + conv])
                convs.append(ConvBlock(ndims, prev_nf, nf))
                prev_nf = nf
            self.decoder.append(convs)
            if not half_res or level < (self.nb_levels - 2):
                prev_nf += int(encoder_nfs[level])

        self.remaining = nn.ModuleList()
        for nf in final_convs:
            self.remaining.append(ConvBlock(ndims, prev_nf, int(nf)))
            prev_nf = int(nf)
        self.final_nf = prev_nf

    def forward(self, x):
        skips = [x]
        for level, convs in enumerate(self.encoder):
            for conv in convs:
                x = conv(x)
            skips.append(x)
            x = self.pooling[level](x)
        for level, convs in enumerate(self.decoder):
            for conv in convs:
                x = conv(x)
            if not self.half_res or level < (self.nb_levels - 2):
                x = ops.upsample2_cat(x, skips.pop())   # nearest x2 + concat fused (networks.py:137-138)
        for conv in self.remaining:
            x = conv(x)
        return x


class VxmDense(LoadableModel):
    """VoxelMorph network for (unsupervised) nonlinear registration between two images
    (reference networks.py:147-287)."""

    @store_config_args
    def __init__(self, inshape, nb_unet_features=None, nb_unet_levels=None, unet_feat_mult=1,
                 nb_unet_conv_per_level=1, int_steps=7, int_downsize=2, bidir=False, use_probs=False,
                 src_feats=1, trg_feats=1, unet_half_res=False):
        super().__init__()
        self.training = True
        object.__setattr__(self, "_dp", None)            # dist.TransparentDP once attached (not a submodule / buffer)
        object.__setattr__(self, "_dp_checked", False)
        self.registration_no_grad = True     # eval-mode registration calls run without autograd bookkeeping (see forward)
        ndims = len(inshape)
        assert ndims in [1, 2, 3], 'ndims should be one of 1, 2, or 3. found: %d' % ndims

        self.unet_model = Unet(inshape, infeats=(src_feats + trg_feats), nb_features=nb_unet_features,
                               nb_levels=nb_unet_levels, feat_mult=unet_feat_mult,
                               nb_conv_per_level=nb_unet_conv_per_level, half_res=unet_half_res)

        self.flow = _conv_cls(ndims)(self.unet_model.final_nf, ndims, kernel_size=3, padding=1)
        self.flow.weight = nn.Parameter(Normal(0, 1e-5).sample(self.flow.weight.shape))
        self.flow.bias = nn.Parameter(torch.zeros(self.flow.bias.shape))

        if use_probs:
            raise NotImplementedError('Flow variance has not been implemented in pytorch - set use_probs to False')

        if not unet_half_res and int_steps > 0 and int_downsize > 1:
            self.resize = layers.ResizeTransform(int_downsize, ndims)
        else:
            self.resize = None
        if int_steps > 0 and int_downsize > 1:
            self.fullsize = layers.ResizeTransform(1 / int_downsize, ndims)
        else:
            self.fullsize = None

        self.bidir = bidir
        down_shape = [int(dim / int_downsize) for dim in inshape]
        self.integrate = layers.VecInt(down_shape, int_steps) if int_steps > 0 else None
        self.transformer = layers.SpatialTransformer(inshape)

    def _maybe_attach_dp(self):
        """Under torchrun the model becomes data parallel by itself on its first forward (dist.TransparentDP): the
        unmodified training loop then needs no DataParallel / DistributedDataParallel wrapper."""
        if not self._dp_checked:
            object.__setattr__(self, "_dp_checked", True)
            if self.training:
                from . import dist as vdist
                object.__setattr__(self, "_dp", vdist.attach_if_distributed(self))
        return self._dp

    def save(self, path):
        if self._dp is not None and not self._dp.is_writer():
            return                       # one checkpoint per job: rank 0 writes (SURVEY 8(e))
        super().save(path)

    def flows(self, source, target):
        """(pos_flow, neg_flow, preint_flow): the U-Net's field brought to the integration resolution (`preint_flow`,
        what train.py regularises), integrated and brought back to full resolution (`pos_flow`, what warps the moving
        image; `neg_flow` its inverse when bidir).  reference networks.py:253-276."""
        return self._integrate(self._head(source, target))

    def _head(self, source, target):
        """The U-Net and its head: the field `flow` predicts (a VxmDenseProbabilistic: cat(flow, log_sigma))."""
        engine = ops.resolve_engine(self)
        if engine in ('bf16', 'bf16x3'):
            # tensor-core engine: Unet + flow head as one hand-written forward/backward (engine_bf16.py)
            from . import engine_bf16
            return engine_bf16.unet_flow(self, source, target, split=(engine == 'bf16x3'))
        x = ops.upsample_free_cat(source, target)
        x = self.unet_model(x)
        if hasattr(self, 'log_sigma'):
            return torch.cat([self.flow(x), self.log_sigma(x)], dim=1)
        return self.flow(x)

    def _integrate(self, flow_field):
        """(pos_flow, neg_flow, preint_flow) of a field at the U-Net's resolution (see flows)."""
        pos_flow = flow_field
        if self.resize:
            pos_flow = self.resize(pos_flow)
        preint_flow = pos_flow
        neg_flow = -pos_flow if self.bidir else None

        if self.integrate:
            pos_flow = self.integrate(pos_flow)
            neg_flow = self.integrate(neg_flow) if self.bidir else None
            if self.fullsize:
                pos_flow = self.fullsize(pos_flow)
                neg_flow = self.fullsize(neg_flow) if self.bidir else None
        return pos_flow, neg_flow, preint_flow

    def forward(self, source, target, registration=False):
        self._maybe_attach_dp()
        if registration and not self.training and self.registration_no_grad and torch.is_grad_enabled():
            # inference (register.py:80-87 calls model.eval() but never torch.no_grad()): nothing downstream of a
            # registration call differentiates, so no activation / VecInt state is kept ("next" row N3)
            with torch.no_grad():
                return self.forward(source, target, registration=True)
        pos_flow, neg_flow, preint_flow = self.flows(source, target)
        y_source = self.transformer(source, pos_flow)
        y_target = self.transformer(target, neg_flow) if self.bidir else None

        if not registration:
            return (y_source, y_target, preint_flow) if self.bidir else (y_source, preint_flow)
        return y_source, pos_flow


def rank_seed(seed, rank):
    """The noise seed of data-parallel rank `rank` for a model constructed with `seed`: rank 0 keeps it, every other rank
    gets a splitmix64 mix of (seed, rank), so that replicas built from one torch seed draw independent noise."""
    if rank == 0:
        return int(seed)
    m = (1 << 64) - 1
    z = (int(seed) + (int(rank) * 0x9E3779B97F4A7C15)) & m
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return (z ^ (z >> 31)) & ((1 << 63) - 1)


class VxmDenseProbabilistic(VxmDense):
    """Probabilistic diffeomorphic VoxelMorph (Dalca et al., MICCAI 2018 / MedIA 2019): VxmDense with a second head,
    `log_sigma`, next to `flow`, as the reference's TensorFlow VxmDense builds it with use_probs=True
    (voxelmorph/tf/networks.py:155-165, 230-232).  The reference's torch VxmDense refuses use_probs, and so does this
    package's; this class takes VxmDense's constructor arguments bar use_probs.

    `log_sigma` = Conv(final_nf, nd, 3, padding=1), weight ~ N(0, 1e-10), bias -10.  flow_params = cat(mu, l) (B, 2 nd,
    *vol) with mu = flow(x) and l = log_sigma(x) = log sigma^2 (at half resolution with unet_half_res, as in TF).

    Training form (registration=False): z = mu + exp(l / 2) eps, eps ~ N(0, 1) — the formula of neurite's
    SampleNormalLogVar, which agrees with the KL loss reading exp(log_sigma) as the variance (voxelmorph/tf/losses.py:340)
    — goes through resize, VecInt, resize and the warp exactly as VxmDense's field does; returns (y_source, flow_params),
    or (y_source, y_target, flow_params) when bidir (neg_flow = -z, the same draw).  Attach losses.KL to flow_params.

    Registration form (registration=True): the mean mu is integrated and nothing is sampled, the papers' use of the model
    at test time.  This departs deliberately from the TF graph, whose sampling layer has no training switch.

    Noise: eps is drawn on the device (layers.sample_normal_logvar) from the non-persistent int64 buffer
    `noise_state` = (seed, call); `seed` is drawn from torch's default CPU generator at construction (torch.manual_seed
    makes runs reproducible; under data parallelism each rank mixes its rank in, see rank_seed), and every training
    forward advances `call` on the device, so CUDA-graph replays draw fresh noise.  The buffer stays out of checkpoints:
    the state-dict keys are VxmDense's plus log_sigma.weight and log_sigma.bias."""

    @store_config_args
    def __init__(self, inshape, nb_unet_features=None, nb_unet_levels=None, unet_feat_mult=1,
                 nb_unet_conv_per_level=1, int_steps=7, int_downsize=2, bidir=False,
                 src_feats=1, trg_feats=1, unet_half_res=False):
        config = self.config
        super().__init__(inshape, nb_unet_features, nb_unet_levels, unet_feat_mult, nb_unet_conv_per_level, int_steps,
                         int_downsize, bidir, False, src_feats, trg_feats, unet_half_res)
        self.config = config             # (VxmDense's decorator recorded its own arguments)
        ndims = len(inshape)
        self.log_sigma = _conv_cls(ndims)(self.unet_model.final_nf, ndims, kernel_size=3, padding=1)
        self.log_sigma.weight = nn.Parameter(Normal(0, 1e-10).sample(self.log_sigma.weight.shape))
        self.log_sigma.bias = nn.Parameter(torch.full(self.log_sigma.bias.shape, -10.0))
        seed = int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64))
        self.register_buffer("noise_state", torch.tensor([seed, 0], dtype=torch.int64), persistent=False)

    def _maybe_attach_dp(self):
        first = not self._dp_checked
        dp = super()._maybe_attach_dp()
        if first and dp is not None:
            with torch.no_grad():
                self.noise_state[0] = rank_seed(int(self.noise_state[0]), dp.rank)
        return dp

    def forward(self, source, target, registration=False):
        self._maybe_attach_dp()
        if registration and not self.training and self.registration_no_grad and torch.is_grad_enabled():
            with torch.no_grad():
                return self.forward(source, target, registration=True)
        flow_params = self._head(source, target)
        nd = flow_params.shape[1] // 2
        if registration:
            field = flow_params[:, :nd]
        else:
            field = layers.sample_normal_logvar(flow_params, self.noise_state)
        pos_flow, neg_flow, _ = self._integrate(field)
        y_source = self.transformer(source, pos_flow)
        y_target = self.transformer(target, neg_flow) if self.bidir else None
        if not registration:
            return (y_source, y_target, flow_params) if self.bidir else (y_source, flow_params)
        return y_source, pos_flow


class VxmDenseSemiSupervisedSeg(LoadableModel):
    """VoxelMorph network for semi-supervised registration with segmentations ("next" row N2; BASELINE config 5).

    The torch backend of the reference has no such class; the semantics are those of its TensorFlow model
    (voxelmorph/tf/networks.py:287-366) restated over the torch layers, as SURVEY.md section 8(a) A12 specifies: the
    full-resolution `pos_flow` of the inner VxmDense is rescaled to the segmentation resolution
    (`ResizeTransform(seg_resolution)`, i.e. RescaleTransform(1 / seg_resolution)), the probabilistic (one-hot) source
    segmentation is warped LINEARLY with it, and the result joins the outputs so that a Dice loss can be attached:

        y_source, preint_flow, y_seg = model(source, target, seg_source)
        loss = image_loss(target, y_source) + w_grad * Grad(preint_flow) + w_seg * Dice(seg_target, y_seg)

    `bidir_labels` additionally warps the target segmentation with `neg_flow` (and implies bidir).  The inner network is
    `self.vxm_model` (checkpoint keys `vxm_model.*`); `kwargs` are forwarded to it."""

    @store_config_args
    def __init__(self, inshape, nb_labels, nb_unet_features=None, seg_resolution=2, bidir=False, bidir_labels=False, **kwargs):
        super().__init__()
        if bidir_labels:
            bidir = True
        ndims = len(inshape)
        self.nb_labels = int(nb_labels)
        self.bidir_labels = bool(bidir_labels)
        self.vxm_model = VxmDense(inshape, nb_unet_features=nb_unet_features, bidir=bidir, **kwargs)
        self.seg_resize = layers.ResizeTransform(seg_resolution, ndims) if seg_resolution != 1 else None
        inshape_ds = [int(d / seg_resolution) for d in inshape]
        self.seg_transformer = layers.SpatialTransformer(inshape_ds)        # linear: the segmentation is a probability map

    def forward(self, source, target, seg_source, seg_target=None, registration=False):
        vm = self.vxm_model
        vm._maybe_attach_dp()
        pos_flow, neg_flow, preint_flow = vm.flows(source, target)
        y_source = vm.transformer(source, pos_flow)
        y_target = vm.transformer(target, neg_flow) if vm.bidir else None
        seg_flow = self.seg_resize(pos_flow) if self.seg_resize else pos_flow
        y_seg = self.seg_transformer(seg_source, seg_flow)
        outs = [y_source] + ([y_target] if vm.bidir else []) + [pos_flow if registration else preint_flow, y_seg]
        if self.bidir_labels:
            if seg_target is None:
                raise ValueError("bidir_labels=True needs the target segmentation")
            nseg_flow = self.seg_resize(neg_flow) if self.seg_resize else neg_flow
            outs.append(self.seg_transformer(seg_target, nseg_flow))
        return tuple(outs)

    def save(self, path):
        dp = self.vxm_model._dp
        if dp is not None and not dp.is_writer():
            return
        super().save(path)

    def register(self, source, target):
        """The transform from source to target (full resolution), like tf get_registration_model / register."""
        with torch.no_grad():
            return self.vxm_model.flows(source, target)[0]

    def apply_transform(self, source, target, img, interp_method='linear'):
        """Predict the transform from source to target and apply it to `img` ('linear' or 'nearest')."""
        mode = 'bilinear' if interp_method == 'linear' else interp_method
        flow = self.register(source, target)
        return layers.SpatialTransformer(tuple(img.shape[2:]), mode=mode)(img, flow)


class VxmDenseSemiSupervisedPointCloud(LoadableModel):
    """VoxelMorph network for registration aided by surface points (Dalca et al., "Unsupervised learning of
    probabilistic diffeomorphic registration for images and surfaces", MedIA 2019).

    The torch backend of the reference has no such class; the semantics are those of its TensorFlow model
    (voxelmorph/tf/networks.py:391-486).  A bidirectional VxmDense (`self.vxm_model`; a VxmDenseProbabilistic with
    `use_probs`) registers source to target.  `pos_flow` moves the atlas surface points into subject space and
    `neg_flow` the subject's into atlas space (layers.point_spatial_transformer); each side's signed distance
    transform (SDT) is read at the other side's moved points (layers.value_at_location), and a loss drives those
    distances to zero:

        y_source, y_target, flow, subj_dt_value, atl_dt_value = model(source, target, subj_dt, atl_dt,
                                                                       subj_surf, atl_surf)

    `flow` is preint_flow (or flow_params with use_probs).  SDTs are (B, nb_labels_sample, *sdt_shape) with
    sdt_shape = int(inshape * sdt_vol_resize); surfaces are (B, nb_surface_points, nd + 1), the last column the SDT
    channel.  Without `surf_bidir` the call is model(source, target, subj_dt, atl_surf) and atl_dt_value is dropped.

    As in the reference (voxelmorph/tf/utils/utils.py:480-493), with sdt_vol_resize != 1 the full-resolution flow,
    scaled by sdt_vol_resize, is sampled at the points' SDT-space coordinates, not at the matching full-resolution
    ones.  Checkpoint keys are `vxm_model.*`; `kwargs` are forwarded to the inner model."""

    @store_config_args
    def __init__(self, inshape, nb_surface_points, nb_labels_sample, nb_unet_features=None, sdt_vol_resize=1,
                 surf_bidir=True, use_probs=False, **kwargs):
        super().__init__()
        self.nb_surface_points = int(nb_surface_points)
        self.nb_labels_sample = int(nb_labels_sample)
        self.sdt_vol_resize = sdt_vol_resize
        self.surf_bidir = bool(surf_bidir)
        self.use_probs = bool(use_probs)
        self.sdt_shape = tuple(int(f * sdt_vol_resize) for f in inshape)
        cls = VxmDenseProbabilistic if use_probs else VxmDense
        self.vxm_model = cls(inshape, nb_unet_features=nb_unet_features, bidir=True, **kwargs)

    def _check_surface(self, sdt, surf, sdt_name, surf_name):
        B = sdt.shape[0]
        want_sdt = (B, self.nb_labels_sample) + self.sdt_shape
        want_surf = (B, self.nb_surface_points, len(self.sdt_shape) + 1)
        if tuple(sdt.shape) != want_sdt:
            raise _lib.VxmError("VxmDenseSemiSupervisedPointCloud: %s must be %s, got %s"
                                % (sdt_name, want_sdt, tuple(sdt.shape)))
        if tuple(surf.shape) != want_surf:
            raise _lib.VxmError("VxmDenseSemiSupervisedPointCloud: %s must be %s, got %s"
                                % (surf_name, want_surf, tuple(surf.shape)))

    def forward(self, source, target, *surface, registration=False):
        vm = self.vxm_model
        if registration:
            return vm(source, target, registration=True)
        if len(surface) != (4 if self.surf_bidir else 2):
            raise TypeError("VxmDenseSemiSupervisedPointCloud.forward takes (source, target, %s)"
                            % ("subj_dt, atl_dt, subj_surf, atl_surf" if self.surf_bidir else "subj_dt, atl_surf"))
        if self.surf_bidir:
            subj_dt, atl_dt, subj_surf, atl_surf = surface
            self._check_surface(atl_dt, subj_surf, "atl_dt", "subj_surf")
        else:
            subj_dt, atl_surf = surface
        self._check_surface(subj_dt, atl_surf, "subj_dt", "atl_surf")
        vm._maybe_attach_dp()
        if self.use_probs:
            flow_out = vm._head(source, target)
            pos_flow, neg_flow, _ = vm._integrate(layers.sample_normal_logvar(flow_out, vm.noise_state))
        else:
            pos_flow, neg_flow, flow_out = vm.flows(source, target)
        y_source = vm.transformer(source, pos_flow)
        y_target = vm.transformer(target, neg_flow)
        r = self.sdt_vol_resize
        subj_dt_value = layers.value_at_location(subj_dt, layers.point_spatial_transformer(atl_surf, pos_flow, r))
        outs = (y_source, y_target, flow_out, subj_dt_value)
        if self.surf_bidir:
            atl_dt_value = layers.value_at_location(atl_dt, layers.point_spatial_transformer(subj_surf, neg_flow, r))
            outs += (atl_dt_value,)
        return outs

    def save(self, path):
        dp = self.vxm_model._dp
        if dp is not None and not dp.is_writer():
            return
        super().save(path)

    def register(self, source, target):
        """The transform from source to target (full resolution; the mean's with use_probs), like tf register."""
        with torch.no_grad():
            return self.vxm_model(source, target, registration=True)[1]

    def apply_transform(self, source, target, img, interp_method='linear'):
        """Predict the transform from source to target and apply it to `img` ('linear' or 'nearest')."""
        mode = 'bilinear' if interp_method == 'linear' else interp_method
        flow = self.register(source, target)
        return layers.SpatialTransformer(tuple(img.shape[2:]), mode=mode)(img, flow)


class TemplateCreation(LoadableModel):
    """VoxelMorph network to learn an unconditional template (atlas) image.

    The torch backend of the reference has no such class; the semantics are those of its TensorFlow model
    (voxelmorph/tf/networks.py:761-853): the atlas is a learnable image, registered to every input by a bidirectional
    VxmDense (atlas = moving image, input = fixed image), and a MeanStream keeps the capped running mean of the
    full-resolution inverse flow so that a loss can pull the atlas towards the centre of the data:

        y_source, y_target, mean_stream, pos_flow = model(image)
        loss = w_img * L(image, y_source) + (1 - w_img) * L(atlas, y_target) + w_mean * MSE(0, mean_stream)
               + w_grad * Grad('l2', loss_mult=2)(pos_flow)

    `self.atlas` is an nn.Parameter of shape (1, atlas_feats, *inshape); the inner network is `self.vxm_model`
    (checkpoint keys `vxm_model.*`), the mean stream's state the buffers `mean_stream.mean` / `mean_stream.count`.
    `kwargs` are forwarded to the inner VxmDense."""

    @store_config_args
    def __init__(self, inshape, nb_unet_features=None, mean_cap=100, atlas_feats=1, src_feats=1, **kwargs):
        super().__init__()
        ndims = len(inshape)
        self.atlas = nn.Parameter(Normal(0, 1e-7).sample((1, atlas_feats) + tuple(inshape)))
        self.vxm_model = VxmDense(inshape, nb_unet_features, bidir=True, src_feats=atlas_feats, trg_feats=src_feats, **kwargs)
        self.mean_stream = layers.MeanStream((ndims,) + tuple(inshape), cap=mean_cap)

    def forward(self, image, registration=False):
        from . import dist as vdist
        if vdist.env_world()[0] > 1:
            raise _lib.VxmError("TemplateCreation does not run data parallel yet: each rank would keep its own mean "
                                "stream, and the atlas lies outside the inner model's gradient exchange; train it on "
                                "one GPU (WORLD_SIZE=1)")
        atlas_b = self.atlas.expand((image.shape[0],) + tuple(self.atlas.shape[1:]))
        pos_flow, neg_flow, _ = self.vxm_model.flows(atlas_b, image)
        y_source = self.vxm_model.transformer(atlas_b, pos_flow)
        if registration:
            return y_source, pos_flow
        y_target = self.vxm_model.transformer(image, neg_flow)
        return y_source, y_target, self.mean_stream(neg_flow), pos_flow

    def set_atlas(self, atlas):
        """Copy `atlas` into the atlas parameter in place (the Parameter object, and so an optimizer holding it, stays
        the same).  Accepts a tensor or an array of shape (1, C, *vol), (C, *vol), or *vol when C == 1."""
        a = torch.as_tensor(np.asarray(atlas) if not torch.is_tensor(atlas) else atlas, dtype=torch.float32)
        shape = tuple(self.atlas.shape)
        if a.dim() == len(shape) - 2 and shape[1] == 1:
            a = a.reshape(shape)
        elif a.dim() == len(shape) - 1:
            a = a.unsqueeze(0)
        if tuple(a.shape) != shape:
            raise ValueError("set_atlas: expected an atlas of shape %s, got %s" % (shape, tuple(np.shape(atlas))))
        with torch.no_grad():
            self.atlas.copy_(a)

    def get_atlas(self):
        """The atlas as a squeezed numpy array, like the reference's get_atlas."""
        return self.atlas.detach().cpu().numpy().squeeze()

    # the transform from source to target and its application to an image, through the inner VxmDense
    register = VxmDenseSemiSupervisedSeg.register
    apply_transform = VxmDenseSemiSupervisedSeg.apply_transform


def _glorot_conv_(conv):
    """Keras' default initialisation of a convolution: glorot-uniform kernel (fans = taps x channels), zero bias."""
    taps = int(np.prod(conv.weight.shape[2:]))
    lim = float(np.sqrt(6.0 / (taps * (conv.weight.shape[0] + conv.weight.shape[1]))))
    with torch.no_grad():
        conv.weight.uniform_(-lim, lim)
        conv.bias.zero_()
    return conv


class ConditionalTemplateCreation(LoadableModel):
    """VoxelMorph network to learn a conditional template: one atlas for every set of subject attributes (Dalca et al.,
    "Learning Conditional Deformable Templates with Convolutional Networks", NeurIPS 2019).

    The torch backend of the reference has no such class; the semantics are those of its TensorFlow model
    (voxelmorph/tf/networks.py:856-983).  For pheno (B, P), atlas (B or 1, atlas_feats, *inshape) and image
    (B, src_feats, *inshape):

        x0 = pheno_decoder(pheno)                 Dense(prod(inshape) F, 'elu') and neurite's conv_dec with no levels
                                                  (a 1x1 convolution F -> F, linear): layers.PhenoDecoder
        x_i = extra_convs[i](x_{i-1})             extra_conv_layers convolutions F -> F, 3^n, no activation
        atlas_t = atlas + atlas_gen(x)            F -> atlas_feats, 3^n, weight and bias ~ N(0, 1e-7)
        pos_flow, neg_flow = vxm_model.flows(atlas_t, image)     bidirectional VxmDense, atlas_t moving
        outputs = (y_source, mean_stream(neg_flow), pos_flow, pos_flow)   or (y_source, pos_flow, pos_flow) without
                                                  the mean stream; registration=True: (y_source, pos_flow)

    with F = conv_nb_features.  The warp of the image by neg_flow (TF's unused y_target) is not computed.  Keras'
    initialisation is kept: glorot-uniform kernels and zero biases in the decoder and the extra convolutions.  The extra
    convolutions and atlas_gen run on the fp32 CUDA-core kernels whatever the U-Net's engine.

    Checkpoint keys: `pheno_decoder.*`, `extra_convs.{i}.*`, `atlas_gen.*`, `vxm_model.*` and the mean stream's buffers
    `mean_stream.mean` / `mean_stream.count`.  `template(pheno, atlas)` returns the conditional atlas (TF's pheno_model).
    Not implemented (NotImplementedError): conv_nb_levels > 0, templcondsi, a conv_image_shape other than
    (*inshape, conv_nb_features) and conv_size other than 3.  `kwargs` are forwarded to the inner VxmDense."""

    @store_config_args
    def __init__(self, inshape, pheno_input_shape, nb_unet_features=None, src_feats=1, atlas_feats=None,
                 conv_image_shape=None, conv_size=3, conv_nb_levels=0, conv_nb_features=32, extra_conv_layers=3,
                 use_mean_stream=True, mean_cap=100, templcondsi=False, templcondsi_init=None, **kwargs):
        super().__init__()
        inshape = tuple(int(s) for s in inshape)
        ndims = len(inshape)
        F = int(conv_nb_features)
        if atlas_feats is None:
            atlas_feats = src_feats
        if templcondsi:
            raise NotImplementedError("ConditionalTemplateCreation: templcondsi is not implemented (the TF branch reads an "
                                      "undefined tensor and cannot run either)")
        if conv_nb_levels > 0:
            raise NotImplementedError("ConditionalTemplateCreation: conv_nb_levels > 0 (a conv_dec U-Net in the atlas "
                                      "generator) is not implemented; use conv_nb_levels=0")
        if conv_image_shape is not None and tuple(conv_image_shape) != inshape + (F,):
            raise NotImplementedError("ConditionalTemplateCreation: conv_image_shape must be (*inshape, conv_nb_features) "
                                      "= %s, got %s" % (inshape + (F,), tuple(conv_image_shape)))
        if conv_size != 3:
            raise NotImplementedError("ConditionalTemplateCreation: conv_size must be 3 (the convolution kernels are 3^n), "
                                      "got %r" % (conv_size,))
        P = int(np.prod(pheno_input_shape))
        self.pheno_decoder = layers.PhenoDecoder(P, F, inshape)
        Conv = _conv_cls(ndims)
        self.extra_convs = nn.ModuleList([_glorot_conv_(Conv(F, F, 3, padding=1)) for _ in range(extra_conv_layers)])
        self.atlas_gen = Conv(F, atlas_feats, 3, padding=1)
        self.atlas_gen.weight = nn.Parameter(Normal(0, 1e-7).sample(self.atlas_gen.weight.shape))
        self.atlas_gen.bias = nn.Parameter(Normal(0, 1e-7).sample(self.atlas_gen.bias.shape))
        self.vxm_model = VxmDense(inshape, nb_unet_features, bidir=True, src_feats=atlas_feats, trg_feats=src_feats, **kwargs)
        self.mean_stream = layers.MeanStream((ndims,) + inshape, cap=mean_cap) if use_mean_stream else None

    def _atlas(self, pheno, atlas):
        x = self.pheno_decoder(pheno)
        for conv in self.extra_convs:
            x = conv(x)
        return atlas + self.atlas_gen(x)

    def template(self, pheno, atlas):
        """The conditional atlas atlas + atlas_gen(...) for attributes `pheno` (B, P), without autograd."""
        with torch.no_grad():
            return self._atlas(pheno, atlas)

    def forward(self, pheno, atlas, image, registration=False):
        from . import dist as vdist
        if vdist.env_world()[0] > 1:
            raise _lib.VxmError("ConditionalTemplateCreation does not run data parallel yet: each rank would keep its own "
                                "mean stream, and the atlas generator lies outside the inner model's gradient exchange; "
                                "train it on one GPU (WORLD_SIZE=1)")
        atlas_t = self._atlas(pheno, atlas)
        pos_flow, neg_flow, _ = self.vxm_model.flows(atlas_t, image)
        y_source = self.vxm_model.transformer(atlas_t, pos_flow)
        if registration:
            return y_source, pos_flow
        if self.mean_stream is None:
            return y_source, pos_flow, pos_flow
        return y_source, self.mean_stream(neg_flow), pos_flow, pos_flow


class HyperVxmDense(VxmDense):
    """HyperMorph: VxmDense whose U-Net convolution weights are generated from the regularisation weight(s) by a
    hypernetwork, so that one model serves every lambda (Hoopes et al., "HyperMorph: Amortized Hyperparameter Learning
    for Image Registration", IPMI 2021 / MELBA 2022; reference voxelmorph/tf/networks.py:1192-1231, trained by
    scripts/tf/train_hypermorph.py).  The torch backend of the reference has no such class; this one restates the TF
    model over this package's VxmDense (zero-fill sampler, int_downsize, torch NCC):

        h = hypernet(hyp)                                 nb_hyp_layers Dense(nb_hyp_units, relu) layers, hyp (1, P)
        W_l, b_l = views of hyper_bias + h @ hyper_kernel every U-Net convolution (encoder, decoder, remaining), in
                                                          execution order, each [weight, bias]: layers.HyperWeights
        the U-Net with those weights (LeakyReLU(0.2) as before), then the flow head — a plain convolution with its own
        parameters `flow.*` — and VxmDense's integration, resize and warp.

    forward(source, target, hyp, registration=False) returns what VxmDense.forward returns.  One set of hyperparameters
    per step: hyp must have shape (1, P), and its weights are shared by every image of the batch (the engines' launches
    take one weight set; at batch size 1, the reference script's default, this is the script's behaviour).  Attach
    losses.hyper_loss to weigh the image and smoothness terms by lambda.  Parameters: `hyper.hypernet.{i}.weight/bias`,
    `hyper.hyper_kernel` (U, N), `hyper.hyper_bias` (N) and `flow.*`; the U-Net holds none of its own (N = 326 032 for
    the default features).  The generated weights live in one persistent buffer: run each forward's backward before the
    next forward.  use_probs is not implemented.  kwargs are VxmDense's."""

    @store_config_args
    def __init__(self, inshape, nb_hyp_params=1, nb_hyp_layers=6, nb_hyp_units=128, **kwargs):
        config = self.config
        if kwargs.get("use_probs", False):
            raise NotImplementedError("HyperVxmDense: use_probs (a flow-variance head) is not implemented")
        super().__init__(inshape, **kwargs)
        self.config = config             # (VxmDense's decorator recorded its own arguments)
        unet = self.unet_model
        self._convs = [blk.main for convs in list(unet.encoder) + list(unet.decoder) for blk in convs] + \
                      [blk.main for blk in unet.remaining]
        self.hyper = layers.HyperWeights([tuple(c.weight.shape) for c in self._convs], nb_hyp_params, nb_hyp_layers,
                                         nb_hyp_units)
        for c in self._convs:
            del c.weight, c.bias
        object.__setattr__(self, "_wflat", None)
        self._assign(self.hyper.wflat)

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self._assign(self.hyper.wflat)   # the generated buffer moved (.to, .cuda): re-point the U-Net at it
        return out

    def _assign(self, wflat):
        """Point every U-Net convolution at its (weight, bias) views of `wflat`."""
        object.__setattr__(self, "_wflat", wflat)
        for c, (w, b) in zip(self._convs, self.hyper.views(wflat)):
            c.weight, c.bias = w, b

    def _head(self, source, target):
        engine = ops.resolve_engine(self)
        if engine in ('bf16', 'bf16x3'):
            from . import engine_bf16
            return engine_bf16.unet_flow(self, source, target, split=(engine == 'bf16x3'), generated=self._wflat)
        return super()._head(source, target)

    def forward(self, source, target, hyp, registration=False):
        P = self.hyper.hypernet[0].in_features
        if hyp.dim() != 2 or tuple(hyp.shape) != (1, P):
            raise _lib.VxmError("HyperVxmDense: hyp must have shape (1, %d), one set of hyperparameters per step shared "
                                "by the whole batch (per-image values are not supported); got %s" % (P, tuple(hyp.shape)))
        self._maybe_attach_dp()
        if registration and not self.training and self.registration_no_grad and torch.is_grad_enabled():
            with torch.no_grad():
                return self.forward(source, target, hyp, registration=True)
        self._assign(self.hyper(hyp))
        try:
            pos_flow, neg_flow, preint_flow = self.flows(source, target)
        finally:
            # back to plain views of the buffer: the module keeps no autograd history from one step to the next (a kept
            # graph would also keep its AccumulateGrad nodes, bound to the stream they were made on, into a capture)
            self._assign(self.hyper.wflat)
        y_source = self.transformer(source, pos_flow)
        y_target = self.transformer(target, neg_flow) if self.bidir else None
        if not registration:
            return (y_source, y_target, preint_flow) if self.bidir else (y_source, preint_flow)
        return y_source, pos_flow
