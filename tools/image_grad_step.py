"""What the image gradients cost: the CUDA-graphed default training step (bench.py's: NCC + lam * Grad, FusedAdam,
int_steps=7, int_downsize=2, bf16 engine) with the moving image a plain input, and with it a learnable nn.Parameter
held by the optimizer (the U-Net's first-layer dgrad, the warp's d/dsrc and the Adam update of the image run as well),
plus the per-launch times of the two launches the feature adds: the first convolution's dgrad into the image planes and
the two-sided NCC backward (next to today's one-sided one).

The two step legs alternate over `--rounds` rounds in one session, on a fresh model per leg; times are CUDA events
around `--steps` graph replays after `--warmup` replays.  Launch times are CUDA events around `--reps` launches.  The
card's name and power limit are printed with the numbers: they are part of them.

    python tools/image_grad_step.py [--steps 10] [--warmup 3] [--rounds 3] [--reps 20] [--size 160 192 224]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - report, do not fail the measurement
        return "nvidia-smi unavailable (%s)" % e


def timed(fn, reps, warm=3):
    """ms per call of fn(), CUDA events around `reps` calls after `warm` calls"""
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def step_leg(vxm, dev, shape, pair, learn_image, steps, warmup):
    import torch
    from voxelmorph_b200.trainer import GraphedTrainStep
    torch.manual_seed(1234)
    model = vxm.networks.VxmDense(inshape=shape, int_steps=7, int_downsize=2)
    with torch.no_grad():
        model.flow.weight.normal_(0, 1e-2)
    model.to(dev).train()
    params = list(model.parameters())
    loss_fn = None
    if learn_image:
        image = torch.nn.Parameter(pair[0].clone())
        params.append(image)
        ncc, grad = vxm.losses.NCC().loss, vxm.losses.Grad("l2", loss_mult=2).loss

        def loss_fn(model, source, target):       # the static `source` buffer is unused: the learnable image moves instead
            y, flow = model(image, target)
            return ncc(target, y) + 0.01 * grad(None, flow)
    opt = vxm.optim.FusedAdam(params, lr=1e-4)
    step = GraphedTrainStep(model, opt, image_loss="ncc", lam=0.01, int_downsize=2, loss_fn=loss_fn).capture(*pair)
    ms = timed(lambda: step(*pair), steps, warmup)
    loss = float(step.loss)
    del step, opt, model
    torch.cuda.empty_cache()
    return dict(leg="learnable image" if learn_image else "plain step", ms_per_step=round(ms, 3), loss=loss)


def launch_legs(vxm, dev, shape, pair, reps):
    """ms per launch: first-layer image dgrad (through the plan's own operand and form), NCC backward one- and two-sided"""
    import torch
    from voxelmorph_b200 import engine_bf16 as eng
    from voxelmorph_b200 import _lib
    lib = _lib.load()
    out = {}
    model = vxm.networks.VxmDense(inshape=shape).to(dev)
    plan = eng._plan_of(model, False)
    L = plan.layers[0]
    gz = torch.randn((1,) + tuple(shape) + (L.cout,), device=dev).to(torch.bfloat16)
    packs = plan.image_dgrad_packs()
    out["first_layer_image_dgrad_%dto%d_ms" % (L.cout, L.cin)] = timed(
        lambda: eng._run(L.dgrad_img, packs, gz, None, L.cin, 3, out_fp32_planar=True), reps)
    del gz
    I, J = pair
    B, D, H, W = I.shape[0], I.shape[2], I.shape[3], I.shape[4]
    gl = torch.ones((), device=dev)
    gI, gJ = torch.empty_like(I), torch.empty_like(J)
    ws = _lib.reduce_workspace(dev)
    loss = torch.empty((), device=dev)
    for which, nf in ((2, 3), (1, 3), (3, 5)):
        saved = torch.empty((B, nf, D, H, W), device=dev)
        name = {1: "y_true", 2: "y_pred", 3: "both"}[which]
        out["ncc_fwd_saving_for_%s_ms" % name] = timed(lambda: _lib.check(lib.vxm_ncc_fwd2(
            _lib.ptr(I), _lib.ptr(J), _lib.ptr(loss), _lib.ptr(saved), _lib.ptr(ws), which, B, D, H, W, 9, 9, 9, _lib.stream_ptr()), "ncc_fwd2"), reps)
        out["ncc_bwd_%s_ms" % name] = timed(lambda: _lib.check(lib.vxm_ncc_bwd2(
            _lib.ptr(I), _lib.ptr(J), _lib.ptr(saved), _lib.ptr(gl), _lib.ptr(gI), _lib.ptr(gJ), which, B, D, H, W, 9, 9, 9,
            _lib.stream_ptr()), "ncc_bwd2"), reps)
        del saved
    return {k: round(v, 4) for k, v in out.items()}


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
        raise SystemExit("image_grad_step.py measures on a CUDA device; none is available")
    os.environ["VXM_B200_CONV_ENGINE"] = "bf16"
    dev = torch.device("cuda:0")
    shape = tuple(args.size)
    s, t = cases.volume_pair(3, shape, sigma=2.0)
    pair = (torch.from_numpy(s).to(dev), torch.from_numpy(t).to(dev))
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=card(), size=shape, torch=torch.__version__)))
    results = {}
    for r in range(args.rounds):
        for learn in (False, True):
            res = step_leg(vxm, dev, shape, pair, learn, args.steps, args.warmup)
            res["round"] = r
            print(json.dumps(res), flush=True)
            results.setdefault(res["leg"], []).append(res["ms_per_step"])
    for leg, ms in results.items():
        print("%-16s ms/step per round: %s  (best %.3f)" % (leg, " ".join("%.3f" % m for m in ms), min(ms)))
    print(json.dumps(launch_legs(vxm, dev, shape, pair, args.reps)))


if __name__ == "__main__":
    main()
