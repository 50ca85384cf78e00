"""fp64 restatement of ConditionalTemplateCreation (reference voxelmorph/tf/networks.py:856-983), composed from the
oracle's primitives (oracle/ref_torch.py) and the TemplateCreation restatement (tests/template_ref.py), both untouched.

neurite is not in the reference tree, so its part of the model is restated here as the contract.  The decoder is
neurite's conv_dec with nb_levels = 0: its level loop is empty and leaves one `{prefix}_likelihood` convolution with
kernel size 1, nb_labels = F outputs, a bias and a linear activation (final_pred_activation='linear').  For pheno (B, P),
atlas (B or 1, A, *vol) and image (B, S, *vol):

    pre[b,f,v] = bias[f,v] + sum_p pheno[b,p] W[p,f,v]     Dense(prod(vol) F, 'elu'), Keras Reshape to (*vol, F)
    h          = pre > 0 ? pre : expm1(pre)                ELU, alpha 1
    x0[b,g,v]  = like_b[g] + sum_f like_w[g,f] h[b,f,v]    conv_dec likelihood convolution, 1x1, F -> F
    x1..xn     = Conv(F, F, 3, pad 1, bias, no activation) extra_conv_layers = n
    atlas_t    = atlas + Conv(F, A, 3, pad 1)(xn)          atlas_gen, weight and bias ~ N(0, 1e-7)
    pos, neg   = VxmDense(bidir=True).flows(atlas_t, image)     atlas_t moving, image fixed
    outputs    = (warp(atlas_t, pos), MeanStream(cap)(neg), pos, pos)   TF get_output: [y_source, mean_stream, pos, pos]

W is laid out (P, F, *vol) and bias (F, *vol).  A Keras Dense kernel (P, V F) and bias (V F,) hold element (p, f, v) at
column v F + f (F fastest: Reshape to (*vol, F) reads the row in C order); `keras_dense` below is that literal form.
The ELU's gradient is TF's EluGrad, g (h < 0 ? h + 1 : 1), which autograd of expm1 reproduces: d expm1(x) = exp(x) = h + 1.

The step of scripts/tf/train_cond_template.py:
    L(image, y_source) + MSE(0, mean_stream) + Grad('l2', 2)(pos_flow) + 0.01 MSE(0, pos_flow)
"""
import torch
import torch.nn.functional as Fn

from oracle import ref_torch

import template_ref


def decoder(pheno, W, bias, like_w, like_b):
    """x0 (B, F, *vol) from pheno (B, P) and the (P, F, *vol) layout."""
    pre = bias.unsqueeze(0) + torch.einsum("bp,pf...->bf...", pheno, W)
    h = torch.where(pre > 0, pre, torch.expm1(pre))
    F = W.shape[1]
    return like_b.reshape((1, F) + (1,) * (W.dim() - 2)) + torch.einsum("gf,bf...->bg...", like_w.reshape(F, F), h)


def keras_dense(pheno, kernel, bias, vol, like_w, like_b):
    """The decoder written in Keras order: Dense over a (P, V F) kernel, ELU, Reshape to (*vol, F), the 1x1 convolution
    channels-last, and a final move of the channels to axis 1."""
    y = pheno @ kernel + bias
    y = torch.where(y > 0, y, torch.expm1(y)).reshape((pheno.shape[0],) + tuple(vol) + (-1,))
    F = y.shape[-1]
    y = y @ like_w.reshape(F, F).t() + like_b
    return y.movedim(-1, 1)


def conv(x, w, b):
    """3^n convolution, padding 1, bias, no activation (the fp32 generator convolutions: no bf16 emulation)."""
    fn = Fn.conv3d if x.dim() == 5 else Fn.conv2d
    return fn(x, w, b, padding=1)


def generator(sd, pheno, atlas, n_extra):
    """atlas_t from a state dict with the model's keys ('pheno_decoder.*', 'extra_convs.{i}.*', 'atlas_gen.*')."""
    x = decoder(pheno, sd["pheno_decoder.weight"], sd["pheno_decoder.bias"], sd["pheno_decoder.like_weight"],
                sd["pheno_decoder.like_bias"])
    for i in range(n_extra):
        x = conv(x, sd["extra_convs.%d.weight" % i], sd["extra_convs.%d.bias" % i])
    return atlas + conv(x, sd["atlas_gen.weight"], sd["atlas_gen.bias"])


def cond_template_forward(sd, vcfg, pheno, atlas, image, mean, count, cap, n_extra=3):
    """(y_source, mean_stream, pos_flow, pos_flow), (m', n'), atlas_t; `vcfg` the inner VxmDense's full config."""
    inner = {k[len("vxm_model."):]: v for k, v in sd.items() if k.startswith("vxm_model.")}
    atlas_t = generator(sd, pheno, atlas, n_extra)
    pos, neg, _ = template_ref.flows(inner, vcfg, atlas_t, image)
    y_source = ref_torch.spatial_transform(atlas_t, pos)
    ms, m1, n1 = template_ref.mean_stream(neg, mean, count, cap)
    return (y_source, ms, pos, pos), (m1, n1), atlas_t


def cond_template_loss(outs, image):
    """train_cond_template.py's loss with an NCC image term."""
    y_source, ms, pos, _ = outs
    return ref_torch.ncc_loss(image, y_source) + ref_torch.mse_loss(torch.zeros_like(ms), ms) \
        + ref_torch.grad_loss(pos, "l2", 2) + 0.01 * ref_torch.mse_loss(torch.zeros_like(pos), pos)
