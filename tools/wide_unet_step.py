"""Training-step throughput of the doubled VoxelMorph U-Net (`--enc 32 64 64 64 --dec 64 64 64 64 64 32 32`) on each
convolution engine, with the default U-Net on the bf16 engine for scale.

Every leg is the CUDA-graphed training step of bench.py (NCC + lam * Grad, FusedAdam, int_steps=7, int_downsize=2) at
160x192x224 on one GPU, on a fresh model per leg; the legs alternate over `--rounds` rounds so that drift of the shared
machine spreads over all of them.  Convolution FLOPs are computed from the layer shapes with the count of bench.py's
roofline (forward + weight gradient + data gradient, no data gradient for the first layer).

    python tools/wide_unet_step.py [--steps 5] [--warmup 2] [--rounds 2] [--size 160 192 224]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DOUBLED = [[32, 64, 64, 64], [64, 64, 64, 64, 64, 32, 32]]
DEFAULT = [[16, 32, 32, 32], [32, 32, 32, 32, 32, 16, 16]]


def conv_flops_per_step(model, shape):
    """Convolution FLOPs of one training step of a (full-resolution, 3-D) VxmDense, from its weight shapes: encoder level i
    runs at 1/8^i of the voxels, decoder level i at 1/8^(levels - i), the remaining convolutions and the flow head at full
    resolution."""
    import numpy as np
    V = float(np.prod(shape))
    unet = model.unet_model
    if unet.half_res:
        raise ValueError("half_res U-Nets are not counted here")
    n_enc = len(unet.encoder)
    layers = []    # (cin, cout, voxel fraction)
    for i, lvl in enumerate(unet.encoder):
        layers += [(b.main.weight.shape[1], b.main.weight.shape[0], 8.0 ** -i) for b in lvl]
    for i, lvl in enumerate(unet.decoder):
        layers += [(b.main.weight.shape[1], b.main.weight.shape[0], 8.0 ** -(n_enc - i)) for b in lvl]
    layers += [(b.main.weight.shape[1], b.main.weight.shape[0], 1.0) for b in unet.remaining]
    layers.append((model.flow.weight.shape[1], model.flow.weight.shape[0], 1.0))
    fwd = sum(2 * 27 * ci * co * V * f for ci, co, f in layers)
    bwd = sum(2 * 27 * ci * co * V * f * (1 if k == 0 else 2) for k, (ci, co, f) in enumerate(layers))
    return fwd + bwd


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - report, do not fail the measurement
        return "nvidia-smi unavailable (%s)" % e


def leg(vxm, dev, shape, pair, feats, engine, steps, warmup):
    import torch
    from voxelmorph_b200.trainer import GraphedTrainStep
    os.environ["VXM_B200_CONV_ENGINE"] = engine
    torch.manual_seed(1234)
    model = vxm.networks.VxmDense(inshape=shape, nb_unet_features=feats, int_steps=7, int_downsize=2)
    with torch.no_grad():
        model.flow.weight.normal_(0, 1e-2)
    flops = conv_flops_per_step(model, shape)
    model.to(dev).train()
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4)
    step = GraphedTrainStep(model, opt, image_loss="ncc", lam=0.01, int_downsize=2).capture(*pair)
    for _ in range(warmup):
        step(*pair)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step(*pair)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = dict(model="doubled" if feats is DOUBLED else "default", engine=engine, ms_per_step=round(ms, 2),
               vol_pairs_per_s=round(1e3 / ms, 3), conv_tflop_per_step=round(flops / 1e12, 3),
               conv_tflops=round(flops / (ms * 1e-3) / 1e12, 1), loss=float(loss), steps=steps, warmup=warmup)
    del step, opt, model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--size", type=int, nargs=3, default=(160, 192, 224))
    args = ap.parse_args()
    import torch
    import voxelmorph_b200 as vxm
    from oracle import cases
    if not torch.cuda.is_available():
        raise SystemExit("wide_unet_step.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    shape = tuple(args.size)
    s, t = cases.volume_pair(3, shape, sigma=2.0)
    pair = (torch.from_numpy(s).to(dev), torch.from_numpy(t).to(dev))
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=card(), size=shape, torch=torch.__version__)))
    legs = [(DOUBLED, "f32"), (DOUBLED, "bf16"), (DOUBLED, "bf16x3"), (DEFAULT, "bf16")]
    results = {}
    for r in range(args.rounds):
        for feats, engine in legs:
            res = leg(vxm, dev, shape, pair, feats, engine, args.steps, args.warmup)
            res["round"] = r
            print(json.dumps(res), flush=True)
            results.setdefault((res["model"], engine), []).append(res)
    print("\nmodel    engine   vol-pairs/s (per round)      conv TFLOP/step  conv TFLOP/s (best round)")
    for (m, e), rs in results.items():
        best = max(rs, key=lambda x: x["vol_pairs_per_s"])
        print("%-8s %-8s %-28s %-16s %s" % (m, e, " ".join("%.3f" % x["vol_pairs_per_s"] for x in rs), best["conv_tflop_per_step"],
                                           best["conv_tflops"]))
    f32 = max(x["vol_pairs_per_s"] for x in results[("doubled", "f32")])
    for e in ("bf16", "bf16x3"):
        print("doubled model, %s over f32: %.2fx" % (e, max(x["vol_pairs_per_s"] for x in results[("doubled", e)]) / f32))


if __name__ == "__main__":
    main()
