"""What learning a template costs: the CUDA-graphed TemplateCreation step at 160x192x224 on the bf16 engine with
train_template.py's defaults (NCC; image-loss weight 1, so the inverse image term has weight 0 and is dropped; mean-stream
and Grad weights 1; FusedAdam over the weights and the atlas), against the graphed bidirectional VxmDense step whose
moving image is a learnable nn.Parameter (same losses bar the mean term), and one B = 2 template leg.  Then the
per-launch times of the MeanStream kernels with their bytes and share of the HBM bound, and of the first-layer image
dgrad (the largest launch the atlas adds) with its share of the template step.

The step legs alternate over `--rounds` rounds in one session, on a fresh model per leg; times are CUDA events around
`--steps` graph replays after `--warmup` replays.  Launch times are CUDA events around `--reps` launches.  The card's
name and power limit are printed with the numbers: they are part of them.

    python tools/template_step.py [--steps 10] [--warmup 3] [--rounds 3] [--reps 20] [--size 160 192 224]
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


def step_leg(vxm, dev, shape, images, atlas0, leg, steps, warmup):
    import torch
    from voxelmorph_b200.trainer import GraphedTrainStep
    ncc, grad, mse = vxm.losses.NCC().loss, vxm.losses.Grad("l2", loss_mult=2).loss, vxm.losses.MSE().loss
    B = images.shape[0]
    torch.manual_seed(1234)
    if leg == "bidir":
        model = vxm.networks.VxmDense(inshape=shape, bidir=True)
        src = torch.nn.Parameter(atlas0.clone())
        params = list(model.parameters()) + [src]

        def loss_fn(model, image):
            pos, neg, _ = model.flows(src, image)
            y_source = model.transformer(src, pos)
            model.transformer(image, neg)
            return ncc(image, y_source) + grad(None, pos)
    else:
        model = vxm.networks.TemplateCreation(shape)
        model.set_atlas(atlas0.cpu())
        params = list(model.parameters())
        zeros = torch.zeros((B, len(shape)) + tuple(shape), device=dev)     # device-resident target of the mean term

        def loss_fn(model, image):
            y_source, _, mean_stream, pos = model(image)
            return ncc(image, y_source) + mse(zeros, mean_stream) + grad(None, pos)
    with torch.no_grad():
        model.to(dev).train()
        (model.vxm_model if leg != "bidir" else model).flow.weight.normal_(0, 1e-2)
    opt = vxm.optim.FusedAdam(params, lr=1e-4)
    n0 = vxm._lib.launch_count()
    step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=3).capture(images)
    launches = (vxm._lib.launch_count() - n0) // 4          # three warm-up steps and the captured one
    ms = timed(lambda: step(images), steps, warmup)
    loss = float(step.loss)
    del step, opt, model
    torch.cuda.empty_cache()
    name = {"bidir": "bidir learnable source", "template": "template"}[leg] + " B=%d" % B
    return dict(leg=name, ms_per_step=round(ms, 3), loss=loss, launches_per_step=launches)


def launch_legs(vxm, dev, shape, reps, template_ms):
    """ms per launch of the MeanStream forward (training, commits the state) and backward at B = 1, and of the first-layer
    image dgrad of the template's U-Net"""
    import torch
    from voxelmorph_b200 import _lib
    from voxelmorph_b200 import engine_bf16 as eng
    lib = _lib.load()
    out = {}
    nd = len(shape)
    n = nd
    for s in shape:
        n *= s
    x = torch.randn((1, n), device=dev)
    mean, count = torch.zeros(n, device=dev), torch.zeros(1, device=dev)
    o, saved, gx = torch.empty(n, device=dev), torch.empty(1, device=dev), torch.empty(1, n, device=dev)
    ws = _lib.reduce_workspace(dev)
    fwd = timed(lambda: _lib.check(lib.vxm_mean_stream_fwd(_lib.ptr(x), _lib.ptr(mean), _lib.ptr(count), _lib.ptr(o), _lib.ptr(saved),
                                                           _lib.ptr(ws), 1, n, 100.0, 1, _lib.stream_ptr()), "mean_stream_fwd"), reps)
    bwd = timed(lambda: _lib.check(lib.vxm_mean_stream_bwd(_lib.ptr(x), _lib.ptr(saved), _lib.ptr(gx), 1, n, n, _lib.stream_ptr()),
                                   "mean_stream_bwd"), reps)
    for name, ms, nbytes in (("mean_stream_fwd", fwd, 4 * 4 * n), ("mean_stream_bwd", bwd, 2 * 4 * n)):
        out[name] = dict(us=round(ms * 1e3, 1), bytes=nbytes, hbm_bound_us=round(nbytes / HBM_BYTES_PER_S * 1e6, 1),
                         share_of_hbm_bound=round(nbytes / HBM_BYTES_PER_S / (ms * 1e-3), 3))
    del x, mean, o, gx
    model = vxm.networks.TemplateCreation(shape).to(dev)
    plan = eng._plan_of(model.vxm_model, False)
    L = plan.layers[0]
    gz = torch.randn((1,) + tuple(shape) + (L.cout,), device=dev).to(torch.bfloat16)
    packs = plan.image_dgrad_packs()
    ms = timed(lambda: eng._run(L.dgrad_img, packs, gz, None, L.cin, 3, out_fp32_planar=True), reps)
    out["first_layer_image_dgrad_%dto%d" % (L.cout, L.cin)] = dict(us=round(ms * 1e3, 1),
                                                                   share_of_template_step=round(ms / template_ms, 3))
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
        raise SystemExit("template_step.py measures on a CUDA device; none is available")
    os.environ["VXM_B200_CONV_ENGINE"] = "bf16"
    dev = torch.device("cuda:0")
    shape = tuple(args.size)
    vols = [cases.volume_pair(3 + i, shape, sigma=2.0) for i in range(2)]
    atlas0 = torch.from_numpy(vols[0][0]).to(dev)
    one = torch.from_numpy(vols[0][1]).to(dev)
    two = torch.cat([one, torch.from_numpy(vols[1][1]).to(dev)])
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=card(), size=shape, torch=torch.__version__)))
    results = {}
    for r in range(args.rounds):
        for leg, images in (("template", one), ("bidir", one), ("template", two)):
            res = step_leg(vxm, dev, shape, images, atlas0, leg, args.steps, args.warmup)
            res["round"] = r
            print(json.dumps(res), flush=True)
            results.setdefault(res["leg"], []).append(res["ms_per_step"])
    for leg, ms in results.items():
        print("%-28s ms/step per round: %s  (best %.3f)" % (leg, " ".join("%.3f" % m for m in ms), min(ms)))
    print(json.dumps(launch_legs(vxm, dev, shape, args.reps, min(results["template B=1"]))))


if __name__ == "__main__":
    main()
