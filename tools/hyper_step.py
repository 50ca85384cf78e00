"""What HyperMorph costs: the CUDA-graphed HyperVxmDense step at 160x192x224, B = 1, default features, on the bf16 engine
(NCC, (1 - lambda) NCC + lambda Grad('l2', 2) through losses.hyper_loss; FusedAdam over every parameter) against the
graphed VxmDense step (NCC + 0.01 Grad).  Then the per-launch times of the four hypernetwork kernels — the hypernetwork
forward and backward, the weight generation and its backward (accumulating into flat gradients, as in the step) — with
their bytes and share of the HBM bound, the weight generation and its backward again on operands 1 and 2 floats past
16-byte alignment (the 4- and 8-byte loads the 3-D and 2-D steps take inside FusedAdam's buffer), and the FusedAdam step
over each model's flat buffer.

The step legs alternate over `--rounds` rounds in one session, on a fresh model per leg; times are CUDA events around
`--steps` graph replays after `--warmup` replays, with lambda changing between replays.  Launch times are CUDA events
around `--reps` calls.  The card's name and power limit are printed with the numbers: they are part of them.

    python tools/hyper_step.py [--steps 10] [--warmup 3] [--rounds 3] [--reps 50] [--size 160 192 224]
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
    ncc, grad = vxm.losses.NCC().loss, vxm.losses.Grad("l2", loss_mult=2).loss
    torch.manual_seed(1234)
    if leg == "hyper":
        model = vxm.networks.HyperVxmDense(shape)
        hyps = [torch.tensor([[v]], device=dev) for v in (0.1, 0.5, 0.9)]
        inputs = (S, T, hyps[0])

        def loss_fn(model, src, trg, hyp):
            y, flow = model(src, trg, hyp)
            return vxm.losses.hyper_loss(hyp, ncc(trg, y), grad(None, flow))
    else:
        model = vxm.networks.VxmDense(shape)
        hyps = [None]
        inputs = (S, T)

        def loss_fn(model, src, trg):
            y, flow = model(src, trg)
            return ncc(trg, y) + 0.01 * grad(None, flow)
    model.to(dev).train()
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4)
    n0 = vxm._lib.launch_count()
    step = GraphedTrainStep(model, opt, loss_fn=loss_fn, warmup=3).capture(*inputs)
    launches = (vxm._lib.launch_count() - n0) // 4          # three warm-up steps and the captured one
    i = [0]

    def replay():
        i[0] += 1
        step(None, None, hyps[i[0] % len(hyps)]) if leg == "hyper" else step()
    ms = timed(replay, steps, warmup)
    loss = float(step.loss)
    nparams = opt.fp.numel
    del step, opt, model
    torch.cuda.empty_cache()
    return dict(leg=leg, ms_per_step=round(ms, 3), loss=loss, launches_per_step=launches, parameters=nparams)


def _bound(ms, nbytes):
    return dict(us=round(ms * 1e3, 1), bytes=nbytes, hbm_bound_us=round(nbytes / HBM_BYTES_PER_S * 1e6, 1),
                share_of_hbm_bound=round(nbytes / HBM_BYTES_PER_S / (ms * 1e-3), 3))


def launch_legs(vxm, dev, shape, reps):
    """us per launch of the four hypernetwork kernels at the default sizes (P = 1, 6 layers of U = 128, N = 326 032), of
    the weight generation and its backward at each narrower load width, and of FusedAdam over the HyperVxmDense's and
    the VxmDense's parameters"""
    import torch
    from voxelmorph_b200 import _lib
    from voxelmorph_b200.layers import _ptr_array
    lib = _lib.load()
    torch.manual_seed(0)
    model = vxm.networks.HyperVxmDense(shape).to(dev)
    hw = model.hyper
    A, a, W = hw.hyper_kernel.detach(), hw.hyper_bias.detach(), hw.wflat
    U, N = A.shape
    mlp = [p.detach() for lin in hw.hypernet for p in (lin.weight, lin.bias)]
    L, P = len(mlp) // 2, mlp[0].shape[1]
    hyp = torch.tensor([[0.5]], device=dev)
    pre, h, dh = torch.empty(L, U, device=dev), torch.empty(U, device=dev), torch.empty(U, device=dev)
    gA, ga = torch.zeros_like(A), torch.zeros_like(a)
    gmlp = [torch.zeros_like(p) for p in mlp]
    dW = torch.randn(N, device=dev)
    work = torch.empty(int(lib.vxm_hyper_workspace_bytes(U, N)), dtype=torch.uint8, device=dev)
    _, wp = _ptr_array(mlp[0::2])
    _, bp = _ptr_array(mlp[1::2])
    _, gwp = _ptr_array(gmlp[0::2])
    _, gbp = _ptr_array(gmlp[1::2])
    s = _lib.stream_ptr
    out = {}
    nmlp = sum(p.numel() for p in mlp)
    ms = timed(lambda: _lib.check(lib.vxm_hyper_mlp_fwd(_lib.ptr(hyp), wp, bp, _lib.ptr(pre), _lib.ptr(h), P, U, L, s()), "mlp"), reps)
    out["hyper_mlp_fwd"] = _bound(ms, 4 * (nmlp + L * U + U))
    ms = timed(lambda: _lib.check(lib.vxm_hyper_mlp_bwd(_lib.ptr(dh), _lib.ptr(hyp), wp, _lib.ptr(pre), gwp, gbp, P, U, L, 1, s()),
                                  "mlp bwd"), reps)
    out["hyper_mlp_bwd_accumulate"] = _bound(ms, 4 * (nmlp + L * U + 2 * nmlp))
    # bytes from shapes: the forward reads A and a and writes W; the accumulating backward reads A and dW, reads and
    # writes gA and ga (its dh partials are U x N / 1024 floats)
    ms = timed(lambda: _lib.check(lib.vxm_hyper_weights_fwd(_lib.ptr(h), _lib.ptr(A), _lib.ptr(a), _lib.ptr(W), U, N, s()), "fwd"), reps)
    out["hyper_weights_fwd"] = _bound(ms, 4 * (U * N + 2 * N))
    ms = timed(lambda: _lib.check(lib.vxm_hyper_weights_bwd(_lib.ptr(h), _lib.ptr(A), _lib.ptr(dW), _lib.ptr(gA), _lib.ptr(ga),
                                                            _lib.ptr(dh), _lib.ptr(work), U, N, 1, s()), "bwd"), reps)
    out["hyper_weights_bwd_accumulate"] = _bound(ms, 4 * (3 * U * N + 3 * N))
    # the same two launches on A, a, W, gA, ga placed 1 and 2 floats into their buffers: the 4- and 8-byte loads of the
    # 3-D and 2-D steps, whose FusedAdam buffer puts hyper_kernel after the flow head's 1299 or 290 floats
    for off, width in ((1, 4), (2, 8)):
        bufs = [torch.zeros(n + off, device=dev) for n in (U * N, N, N, U * N, N)]
        Ao, ao, Wo, gAo, gao = [b[off:] for b in bufs]
        Ao.copy_(A.reshape(-1))
        ao.copy_(a)
        ms = timed(lambda: _lib.check(lib.vxm_hyper_weights_fwd(_lib.ptr(h), _lib.ptr(Ao), _lib.ptr(ao), _lib.ptr(Wo), U, N, s()),
                                      "fwd"), reps)
        out["hyper_weights_fwd_%dB_loads" % width] = _bound(ms, 4 * (U * N + 2 * N))
        ms = timed(lambda: _lib.check(lib.vxm_hyper_weights_bwd(_lib.ptr(h), _lib.ptr(Ao), _lib.ptr(dW), _lib.ptr(gAo),
                                                                _lib.ptr(gao), _lib.ptr(dh), _lib.ptr(work), U, N, 1, s()),
                                      "bwd"), reps)
        out["hyper_weights_bwd_accumulate_%dB_loads" % width] = _bound(ms, 4 * (3 * U * N + 3 * N))
        del bufs, Ao, ao, Wo, gAo, gao
    out["sizes"] = dict(P=P, U=U, layers=L, N=N)
    del gA, model, hw, A
    torch.cuda.empty_cache()
    for leg in ("hyper", "vxm"):
        torch.manual_seed(0)
        m = (vxm.networks.HyperVxmDense(shape) if leg == "hyper" else vxm.networks.VxmDense(shape)).to(dev)
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
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--size", type=int, nargs=3, default=(160, 192, 224))
    args = ap.parse_args()
    import torch
    import voxelmorph_b200 as vxm
    from oracle import cases
    if not torch.cuda.is_available():
        raise SystemExit("hyper_step.py measures on a CUDA device; none is available")
    os.environ["VXM_B200_CONV_ENGINE"] = "bf16"
    dev = torch.device("cuda:0")
    shape = tuple(args.size)
    s, tr = cases.volume_pair(3, shape, sigma=2.0)
    S, T = torch.from_numpy(s).to(dev), torch.from_numpy(tr).to(dev)
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=card(), size=shape, torch=torch.__version__)))
    results = {}
    for r in range(args.rounds):
        for leg in ("hyper", "vxm"):
            res = step_leg(vxm, dev, shape, S, T, leg, args.steps, args.warmup)
            res["round"] = r
            print(json.dumps(res), flush=True)
            results.setdefault(res["leg"], []).append(res["ms_per_step"])
    for leg, ms in results.items():
        print("%-6s ms/step per round: %s  (best %.3f)" % (leg, " ".join("%.3f" % m for m in ms), min(ms)))
    print(json.dumps(launch_legs(vxm, dev, shape, args.reps)))


if __name__ == "__main__":
    main()
