"""What learning a conditional template costs: the CUDA-graphed ConditionalTemplateCreation step at 160x192x224, B = 1, on
the bf16 engine with train_cond_template.py's configuration (P = 2 attributes, conv_nb_features F = 4; NCC +
MSE(0, mean stream) + Grad('l2', 2)(pos) + 0.01 MSE(0, pos); FusedAdam over every parameter) against the graphed
TemplateCreation step (NCC + MSE(0, mean stream) + Grad).  Then the per-launch times of the phenotype decoder forward and
backward (accumulating into flat gradients, as in the step) with their bytes and share of the HBM bound, of the four
fp32 generator convolutions forward and backward, and of the FusedAdam step over each model's flat buffer.

The step legs alternate over `--rounds` rounds in one session, on a fresh model per leg; times are CUDA events around
`--steps` graph replays after `--warmup` replays.  Launch times are CUDA events around `--reps` calls.  The card's name
and power limit are printed with the numbers: they are part of them.

    python tools/cond_template_step.py [--steps 10] [--warmup 3] [--rounds 3] [--reps 20] [--size 160 192 224]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from image_grad_step import card, timed  # noqa: E402

HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet
P_ATTR, F_GEN = 2, 4


def _model(vxm, leg, shape, atlas0):
    import torch
    torch.manual_seed(1234)
    if leg == "template":
        model = vxm.networks.TemplateCreation(shape)
        model.set_atlas(atlas0.cpu())
    else:
        model = vxm.networks.ConditionalTemplateCreation(shape, (P_ATTR,), conv_nb_features=F_GEN)
    return model


def step_leg(vxm, dev, shape, image, atlas0, pheno, leg, steps, warmup):
    import torch
    from voxelmorph_b200.trainer import GraphedTrainStep
    ncc, grad, mse = vxm.losses.NCC().loss, vxm.losses.Grad("l2", loss_mult=2).loss, vxm.losses.MSE().loss
    zeros = torch.zeros((1, len(shape)) + tuple(shape), device=dev)
    model = _model(vxm, leg, shape, atlas0)
    if leg == "template":
        inputs = (image,)

        def loss_fn(model, image):
            y_source, _, mean_stream, pos = model(image)
            return ncc(image, y_source) + mse(zeros, mean_stream) + grad(None, pos)
    else:
        inputs = (pheno, atlas0, image)

        def loss_fn(model, pheno, atlas, image):
            y_source, mean_stream, pos, _ = model(pheno, atlas, image)
            return ncc(image, y_source) + mse(zeros, mean_stream) + grad(None, pos) + 0.01 * mse(zeros, pos)
    with torch.no_grad():
        model.to(dev).train()
        model.vxm_model.flow.weight.normal_(0, 1e-2)
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4)
    n0 = vxm._lib.launch_count()
    step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=3).capture(*inputs)
    launches = (vxm._lib.launch_count() - n0) // 4          # three warm-up steps and the captured one
    ms = timed(lambda: step(*inputs), steps, warmup)
    loss = float(step.loss)
    nparams = opt.fp.numel
    del step, opt, model
    torch.cuda.empty_cache()
    return dict(leg=leg, ms_per_step=round(ms, 3), loss=loss, launches_per_step=launches, parameters=nparams)


def _bound(ms, nbytes):
    return dict(us=round(ms * 1e3, 1), bytes=nbytes, hbm_bound_us=round(nbytes / HBM_BYTES_PER_S * 1e6, 1),
                share_of_hbm_bound=round(nbytes / HBM_BYTES_PER_S / (ms * 1e-3), 3))


def launch_legs(vxm, dev, shape, reps, atlas0, pheno):
    """us per launch of the decoder forward and backward (B = 1, accumulating), the generator convolutions, and FusedAdam
    over the conditional and the unconditional model's parameters"""
    import torch
    from voxelmorph_b200 import _lib, ops
    from voxelmorph_b200.layers import _pheno_decoder_workspace
    lib = _lib.load()
    out = {}
    V = 1
    for s in shape:
        V *= s
    P, F, B = P_ATTR, F_GEN, 1
    model = _model(vxm, "cond", shape, atlas0).to(dev)
    dec = model.pheno_decoder
    W, bias, lw, lb = dec.weight.detach(), dec.bias.detach(), dec.like_weight.detach(), dec.like_bias.detach()
    x0 = torch.empty((B, F) + tuple(shape), device=dev)
    gW, gb, glw, glb = (torch.zeros_like(p) for p in (W, bias, lw, lb))
    ws = _pheno_decoder_workspace(dev, F)
    fwd = timed(lambda: _lib.check(lib.vxm_pheno_decoder_fwd(_lib.ptr(pheno), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(lw), _lib.ptr(lb),
                                                             _lib.ptr(x0), B, P, F, V, _lib.stream_ptr()), "fwd"), reps)
    bwd = timed(lambda: _lib.check(lib.vxm_pheno_decoder_bwd(_lib.ptr(x0), _lib.ptr(pheno), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(lw),
                                                             _lib.ptr(gW), _lib.ptr(gb), _lib.ptr(glw), _lib.ptr(glb), _lib.ptr(ws),
                                                             B, P, F, V, 1, _lib.stream_ptr()), "bwd"), reps)
    # bytes from shapes: forward reads W and bias, writes the output; the accumulating backward reads W, bias and the
    # output gradient and reads and writes gW and gbias
    out["pheno_decoder_fwd"] = _bound(fwd, 4 * V * (P * F + F + B * F))
    out["pheno_decoder_bwd_accumulate"] = _bound(bwd, 4 * V * (P * F + F + B * F + 2 * (P * F + F)))
    del gW, gb
    # the four generator convolutions (3 x F -> F, F -> 1), forward and backward, fp32 CUDA-core kernels
    convs = list(model.extra_convs) + [model.atlas_gen]
    xin = x0.detach().requires_grad_(True)

    def gen_fwd():
        x = xin
        for c in convs:
            x = ops.conv_k3(x, c.weight, c.bias, None)
        return x
    fwd_ms = timed(lambda: gen_fwd(), reps)
    y = gen_fwd()
    gy = torch.randn_like(y)
    fb_ms = timed(lambda: torch.autograd.backward(gen_fwd(), gy), reps)
    out["generator_convs_fwd"] = dict(us=round(fwd_ms * 1e3, 1))
    out["generator_convs_bwd"] = dict(us=round((fb_ms - fwd_ms) * 1e3, 1))
    del y, gy, xin, x0, model, dec, W, bias
    torch.cuda.empty_cache()
    for leg in ("cond", "template"):
        m = _model(vxm, leg, shape, atlas0).to(dev)
        opt = vxm.optim.FusedAdam(m.parameters(), lr=1e-4)
        n = opt.fp.numel
        ms = timed(lambda: opt.step(), reps)
        out["fused_adam_%s" % leg] = dict(_bound(ms, 4 * 4 * n + 4 * 3 * n), parameters=n)   # p, m, v read + written, g read
        del m, opt
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--size", type=int, nargs=3, default=(160, 192, 224))
    args = ap.parse_args()
    import torch
    import voxelmorph_b200 as vxm
    from oracle import cases
    if not torch.cuda.is_available():
        raise SystemExit("cond_template_step.py measures on a CUDA device; none is available")
    os.environ["VXM_B200_CONV_ENGINE"] = "bf16"
    dev = torch.device("cuda:0")
    shape = tuple(args.size)
    s, tr = cases.volume_pair(3, shape, sigma=2.0)
    atlas0, image = torch.from_numpy(s).to(dev), torch.from_numpy(tr).to(dev)
    pheno = torch.tensor([[0.4, -1.0]], device=dev)
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=card(), size=shape, torch=torch.__version__)))
    results = {}
    for r in range(args.rounds):
        for leg in ("cond", "template"):
            res = step_leg(vxm, dev, shape, image, atlas0, pheno, leg, args.steps, args.warmup)
            res["round"] = r
            print(json.dumps(res), flush=True)
            results.setdefault(res["leg"], []).append(res["ms_per_step"])
    for leg, ms in results.items():
        print("%-10s ms/step per round: %s  (best %.3f)" % (leg, " ".join("%.3f" % m for m in ms), min(ms)))
    print(json.dumps(launch_legs(vxm, dev, shape, args.reps, atlas0, pheno)))


if __name__ == "__main__":
    main()
