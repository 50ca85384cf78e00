"""fp64 restatement of HyperMorph (reference voxelmorph/tf/networks.py:1192-1231 and scripts/tf/train_hypermorph.py),
composed from the oracle's VxmDense restatement (oracle/ref_torch.py), untouched.

neurite's HyperConvFromDense is not in the reference tree; its contract, restated here, is a Dense map from the
hypernetwork's last activation h (U,) to every convolution's kernel and bias.  In the package's flat layout (the U-Net's
convolutions in execution order, each [weight, bias]; N values in all):

    h     = relu(W_{L-1} relu(... relu(W_0 hyp + b_0)) + b_{L-1})       hyp (1, P), W_l torch.nn.Linear (out, in)
    Wflat = hyper_bias + h @ hyper_kernel                               hyper_kernel (U, N), hyper_bias (N)
    the U-Net's state-dict entries are views of Wflat; the flow head keeps its own parameters

and the step's loss is (1 - lam) image_loss + lam Grad('l2', loss_mult=int_downsize)(preint_flow), lam = hyp[0, 0].
"""
import torch

from oracle import ref_torch


def hypernet(hyp, mlp):
    """h (U,) for hyp (1, P) and mlp = [(weight, bias)] of nn.Linear layers."""
    x = hyp.reshape(-1)
    for w, b in mlp:
        x = torch.relu(w @ x + b)
    return x


def unet_keys(cfg):
    """The U-Net's state-dict prefixes in execution order (ref_torch.init_state_dict's insertion order)."""
    sd = ref_torch.init_state_dict(cfg)
    return [k[:-len(".weight")] for k in sd if k.endswith(".weight") and k.startswith("unet_model.")], sd


def layout(cfg):
    """[(prefix, weight shape, weight offset, bias offset)] and N."""
    keys, sd = unet_keys(cfg)
    out, n = [], 0
    for k in keys:
        s = tuple(sd[k + ".weight"].shape)
        out.append((k, s, n, n + sd[k + ".weight"].numel()))
        n += sd[k + ".weight"].numel() + s[0]
    return out, n


def generated_state_dict(wflat, cfg):
    """The U-Net's state-dict entries as views of the flat layout."""
    lay, _ = layout(cfg)
    sd = {}
    for k, s, ow, ob in lay:
        sd[k + ".weight"] = wflat[ow:ob].view(s)
        sd[k + ".bias"] = wflat[ob:ob + s[0]]
    return sd


def hyper_state(sd, cfg):
    """(hyp-independent) pieces of a HyperVxmDense state dict: mlp [(w, b)], hyper_kernel, hyper_bias, flow sd."""
    L = len([k for k in sd if k.startswith("hyper.hypernet.") and k.endswith(".weight")])
    mlp = [(sd["hyper.hypernet.%d.weight" % i], sd["hyper.hypernet.%d.bias" % i]) for i in range(L)]
    return mlp, sd["hyper.hyper_kernel"], sd["hyper.hyper_bias"], {k: sd[k] for k in ("flow.weight", "flow.bias")}


def hyper_forward(sd, cfg, source, target, hyp, registration=False):
    """HyperVxmDense.forward on a state dict with the package's keys."""
    mlp, A, a, flow = hyper_state(sd, cfg)
    h = hypernet(hyp, mlp)
    wflat = a + h @ A
    full = dict(generated_state_dict(wflat, cfg), **flow)
    return ref_torch.vxm_forward(full, cfg, source, target, registration=registration)


def hyper_loss(outs, target, hyp, image_loss="ncc", int_downsize=2, image_sigma=0.05):
    """train_hypermorph.py's loss on (y_source, preint_flow)."""
    lam = float(hyp.reshape(-1)[0])
    y, flow = outs[0], outs[-1]
    if image_loss == "ncc":
        img = ref_torch.ncc_loss(target, y)
    else:
        img = ref_torch.mse_loss(target, y) / image_sigma ** 2
    return (1 - lam) * img + lam * ref_torch.grad_loss(flow, "l2", int_downsize)
