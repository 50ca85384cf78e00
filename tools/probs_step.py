"""What the probabilistic model costs: the CUDA-graphed VxmDenseProbabilistic step at 160x192x224, B = 1, on the bf16
engine with train.py --use-probs's defaults (MSE(image_sigma = 0.02) + 0.01 KL(prior_lambda = 10)), against the graphed
deterministic VxmDense step with MSE + 0.01 Grad('l2', loss_mult=2).  Then the per-launch times of the sampler and KL
kernels with their bytes and share of the HBM bound, and of the 2 nd-output head's forward and dgrad next to the
nd-output ones of the deterministic model.

The step legs alternate over `--rounds` rounds in one session, on a fresh model per leg; times are CUDA events around
`--steps` graph replays after `--warmup` replays.  Launch times are CUDA events around `--reps` launches.  The card's
name and power limit are printed with the numbers: they are part of them.

    python tools/probs_step.py [--steps 10] [--warmup 3] [--rounds 3] [--reps 20] [--size 160 192 224]
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


def step_leg(vxm, dev, shape, S, T, leg, steps, warmup):
    import torch
    from voxelmorph_b200.trainer import GraphedTrainStep
    torch.manual_seed(1234)
    if leg == "probabilistic":
        model = vxm.networks.VxmDenseProbabilistic(shape)
        mse, kl = vxm.losses.MSE(0.02).loss, vxm.losses.KL(10.0).loss

        def loss_fn(model, s, t):
            y, flow_params = model(s, t)
            return mse(t, y) + 0.01 * kl(None, flow_params)
    else:
        model = vxm.networks.VxmDense(shape)
        mse, grad = vxm.losses.MSE().loss, vxm.losses.Grad("l2", loss_mult=2).loss

        def loss_fn(model, s, t):
            y, flow = model(s, t)
            return mse(t, y) + 0.01 * grad(None, flow)
    with torch.no_grad():
        model.to(dev).train()
        model.flow.weight.normal_(0, 1e-2)
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4)
    n0 = vxm._lib.launch_count()
    step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=3).capture(S, T)
    launches = (vxm._lib.launch_count() - n0) // 4          # three warm-up steps and the captured one
    ms = timed(lambda: step(S, T), steps, warmup)
    loss = float(step.loss)
    del step, opt, model
    torch.cuda.empty_cache()
    return dict(leg=leg, ms_per_step=round(ms, 3), loss=loss, launches_per_step=launches)


def _entry(ms, nbytes):
    return dict(us=round(ms * 1e3, 1), bytes=int(nbytes), hbm_bound_us=round(nbytes / HBM_BYTES_PER_S * 1e6, 1),
                share_of_hbm_bound=round(nbytes / HBM_BYTES_PER_S / (ms * 1e-3), 3))


def launch_legs(vxm, dev, shape, reps):
    import torch
    from voxelmorph_b200 import _lib, tc
    from voxelmorph_b200 import engine_bf16 as eng
    lib = _lib.load()
    out = {}
    nd = len(shape)
    V = 1
    for s in shape:
        V *= s
    n = nd * V                                               # elements of z at B = 1
    params = torch.randn((1, 2 * nd) + tuple(shape), device=dev) - 3.0
    z, gz, gp = torch.empty((1, nd) + tuple(shape), device=dev), torch.randn((1, nd) + tuple(shape), device=dev), torch.empty_like(params)
    state, ticket = torch.tensor([1, 0], dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev)
    ws = _lib.reduce_workspace(dev)
    loss, gl = torch.empty((), device=dev), torch.ones((), device=dev)
    legs = (
        ("sampler_fwd", 12 * n, lambda: lib.vxm_sample_normal_logvar_fwd(_lib.ptr(params), _lib.ptr(z), _lib.ptr(state), _lib.ptr(ticket),
                                                                          _lib.ptr(ws), 1, nd, V, _lib.stream_ptr())),
        ("sampler_bwd", 16 * n, lambda: lib.vxm_sample_normal_logvar_bwd(_lib.ptr(gz), _lib.ptr(params), _lib.ptr(state), _lib.ptr(ticket),
                                                                          _lib.ptr(gp), 1, nd, V, _lib.stream_ptr())),
        ("kl_fwd", 8 * n, lambda: lib.vxm_kl_fwd(_lib.ptr(params), _lib.ptr(loss), _lib.ptr(ws), 1, *shape, nd, 10.0, _lib.stream_ptr())),
        ("kl_bwd", 16 * n, lambda: lib.vxm_kl_bwd(_lib.ptr(params), _lib.ptr(gl), _lib.ptr(gp), 1, *shape, nd, 10.0, _lib.stream_ptr())),
    )
    for name, nbytes, fn in legs:
        out[name] = _entry(timed(lambda: _lib.check(fn(), name), reps), nbytes)
    del params, z, gz, gp
    # the heads: forward (bf16 input, fp32 planar output, bias) and dgrad (flow gradient in, masked LeakyReLU derivative)
    for cls in (vxm.networks.VxmDense, vxm.networks.VxmDenseProbabilistic):
        model = cls(shape).to(dev)
        plan = eng._plan_of(model, False)
        L = plan.layers[-1]
        x = torch.randn((1,) + tuple(shape) + (L.ca,), device=dev).to(torch.bfloat16)
        fwd = timed(lambda: eng._run(L.fwd, L.pk_fwd, x, None, L.cout, 3, L.bias.detach(), up=L.up, slope=None, out_fp32_planar=True), reps)
        planes = [torch.randn((1, 1) + tuple(shape), device=dev) for _ in range(L.cout)]
        g_in = tc.planar_fold_kd(planes, 16) if L.dgrad == "fold" else tc.planar_to_ndhwc8(planes)
        dg = timed(lambda: eng._run(L.dgrad, L.pk_dgrad, g_in, None, L.cin, 3, slope=0.2, mask=x), reps)
        form = "folded" if L.dgrad == "fold" else "non-folded"
        out["head_fwd_%d_outputs" % L.cout] = _entry(fwd, V * (2 * L.ca + 4 * L.cout))
        out["head_dgrad_%d_planes_%s" % (L.cout, form)] = _entry(dg, V * (2 * g_in.shape[-1] + 2 * L.cin + 2 * L.cin))
        del model, plan, x, planes, g_in
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
        raise SystemExit("probs_step.py measures on a CUDA device; none is available")
    os.environ["VXM_B200_CONV_ENGINE"] = "bf16"
    dev = torch.device("cuda:0")
    shape = tuple(args.size)
    s, t = cases.volume_pair(3, shape, sigma=2.0)
    S, T = torch.from_numpy(s).to(dev), torch.from_numpy(t).to(dev)
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=card(), size=shape, torch=torch.__version__)))
    results = {}
    for r in range(args.rounds):
        for leg in ("probabilistic", "deterministic"):
            res = step_leg(vxm, dev, shape, S, T, leg, args.steps, args.warmup)
            res["round"] = r
            print(json.dumps(res), flush=True)
            results.setdefault(leg, []).append(res["ms_per_step"])
    for leg, ms in results.items():
        print("%-16s ms/step per round: %s  (best %.3f)" % (leg, " ".join("%.3f" % m for m in ms), min(ms)))
    print(json.dumps(launch_legs(vxm, dev, shape, args.reps)))


if __name__ == "__main__":
    main()
