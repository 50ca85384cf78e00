"""fp64 restatement of TemplateCreation (reference voxelmorph/tf/networks.py:761-853) and of its MeanStream, composed
from the oracle's primitives (oracle/ref_torch.py, which stays untouched) for the template tests.

MeanStream(cap) (neurite's layer; its semantics are restated here as the contract): for x (B, *shape), state mean
(*shape) and count, both zero at first,
    S = sum_b x_b,  n' = count + B,  alpha = B / min(n', cap),  m' = mean (1 - alpha) + (S / B) alpha,
    out = min(1, n' / cap) m'  for every b;  training commits mean <- m', count <- n' (eval commits nothing);
the gradient flows through S only: d out / d x_b = min(1, n' / cap) alpha / B.

The template step of scripts/tf/train_template.py:
    w_img L(image, y_source) + (1 - w_img) L(atlas, y_target) + w_mean MSE(0, mean_stream) + w_grad Grad('l2', 2)(pos_flow)
"""
import torch

from oracle import ref_torch


def mean_stream(x, mean, count, cap):
    """(out expanded over B, m', n'); autograd reaches x only (mean / count are plain values)."""
    B = x.shape[0]
    n1 = float(count) + B
    alpha = B / min(n1, float(cap))
    m1 = mean.detach() * (1 - alpha) + x.sum(0) / B * alpha
    out = min(1.0, n1 / float(cap)) * m1
    return out.unsqueeze(0).expand_as(x), m1, n1


def flows(sd, cfg, source, target):
    """(pos_flow, neg_flow, preint_flow) at full resolution: ref_torch.vxm_forward up to the warps, both directions."""
    int_steps = cfg.get("int_steps", 7)
    int_downsize = cfg.get("int_downsize", 2)
    x = ref_torch.unet_forward(torch.cat([source, target], dim=1), sd, cfg)
    pos = ref_torch._conv(x, sd, "flow", False)
    if (not cfg.get("unet_half_res", False)) and int_steps > 0 and int_downsize > 1:
        pos = ref_torch.resize_transform(pos, int_downsize)
    preint = pos
    neg = -pos
    if int_steps > 0:
        pos, neg = ref_torch.vec_int(pos, int_steps), ref_torch.vec_int(neg, int_steps)
        if int_downsize > 1:
            pos, neg = ref_torch.resize_transform(pos, 1 / int_downsize), ref_torch.resize_transform(neg, 1 / int_downsize)
    return pos, neg, preint


def vxm_cfg(tcfg):
    """The inner VxmDense's config of a TemplateCreation config (bidir, atlas_feats -> src_feats, src_feats -> trg_feats)."""
    c = {k: v for k, v in tcfg.items() if k not in ("mean_cap", "atlas_feats", "src_feats")}
    c.update(bidir=True, src_feats=tcfg.get("atlas_feats", 1), trg_feats=tcfg.get("src_feats", 1))
    return c


def template_forward(sd, tcfg, image, mean, count):
    """(y_source, y_target, mean_stream, pos_flow), (m', n') of TemplateCreation on `sd` (its state_dict keys: 'atlas',
    'vxm_model.*'); `tcfg` the full config, inner VxmDense defaults included."""
    inner = {k[len("vxm_model."):]: v for k, v in sd.items() if k.startswith("vxm_model.")}
    atlas_b = sd["atlas"].expand((image.shape[0],) + tuple(sd["atlas"].shape[1:]))
    pos, neg, _ = flows(inner, vxm_cfg(tcfg), atlas_b, image)
    y_source = ref_torch.spatial_transform(atlas_b, pos)
    y_target = ref_torch.spatial_transform(image, neg)
    ms, m1, n1 = mean_stream(neg, mean, count, tcfg.get("mean_cap", 100))
    return (y_source, y_target, ms, pos), (m1, n1)


def template_loss(outs, atlas_b, image, image_loss="ncc", w_img=1.0, w_mean=1.0, w_grad=1.0):
    """train_template.py's weighted sum (a zero weight drops its term)."""
    L = ref_torch.ncc_loss if image_loss == "ncc" else ref_torch.mse_loss
    y_source, y_target, ms, pos = outs
    loss = w_img * L(image, y_source) + w_mean * ref_torch.mse_loss(torch.zeros_like(ms), ms) \
        + w_grad * ref_torch.grad_loss(pos, "l2", 2)
    if w_img != 1.0:
        loss = loss + (1 - w_img) * L(atlas_b, y_target)
    return loss
