"""What the surface terms of VxmDenseSemiSupervisedPointCloud cost at 160x192x224, B = 1, on the bf16 engine:

* each surface launch through the C ABI at N = 5000 points (the TF training script's default) and L = 38 labels (the
  atlas's label count): the point warp forward and backward (pairs, CUB sort, run sums), the distance lookup forward
  and backward; CUDA events around `--reps` calls after three warm-up calls;
* the CUDA-graphed step with all five loss terms (0.5 MSE each way, 0.01 Grad, 0.25 / dt_sigma^2 MSE(0, value) per
  surface output) against the same model's graphed step without the surface terms, alternated over `--rounds`;
* the host-to-device copy of the two SDT inputs (2 x 38 x 160x192x224 fp32, 2.1 GB) from pinned memory;
* with `--feed L ...`, the host feed of one batch of generators.surf_semisupervised for each label count on a
  synthetic blob label map (the atlas preparation, once per generator, reported apart).

The card's name and power limit are printed with the numbers: they are part of them.

    python tools/surf_step.py [--steps 10] [--rounds 3] [--reps 20] [--points 5000] [--labels 38] [--feed 4 38]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from image_grad_step import card, timed  # noqa: E402

SHAPE = (160, 192, 224)


def points(rng, N, shape, L):
    import numpy as np
    cols = [rng.uniform(0, n - 1, N) for n in shape] + [rng.integers(0, L, N).astype(float)]
    return np.stack(cols, -1)[None].astype(np.float32)


def launch_legs(vxm, dev, N, L, reps):
    import numpy as np
    import torch
    from voxelmorph_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(0)
    pts = torch.from_numpy(points(rng, N, SHAPE, L)).to(dev)
    flow = torch.randn(1, 3, *SHAPE, device=dev) * 3
    sdt = torch.randn(1, L, *SHAPE, device=dev)
    q, v = torch.empty_like(pts), torch.empty(1, N, device=dev)
    gq, gv, gpts = torch.randn_like(pts), torch.randn(1, N, device=dev), torch.empty_like(pts)
    gflow = torch.zeros_like(flow)
    ws = int(lib.vxm_point_warp_workspace_bytes(1, N, *SHAPE, 3))
    work = torch.empty(ws, dtype=torch.uint8, device=dev)
    st = _lib.stream_ptr
    P = _lib.ptr
    legs = {
        "point_warp_fwd": lambda: lib.vxm_point_warp_fwd(P(pts), P(flow), P(q), 1, N, *SHAPE, 3, 1.0, st()),
        "point_warp_bwd": lambda: lib.vxm_point_warp_bwd(P(pts), P(gq), P(gflow), P(work), ws, 1, N, *SHAPE, 3, 1.0,
                                                         st()),
        "value_at_fwd": lambda: lib.vxm_value_at_fwd(P(sdt), P(q), P(v), 1, N, L, *SHAPE, 3, st()),
        "value_at_bwd": lambda: lib.vxm_value_at_bwd(P(sdt), P(q), P(gv), P(gpts), 1, N, L, *SHAPE, 3, st()),
    }
    out = dict(workspace_bytes=ws)
    for name, fn in legs.items():
        def call(fn=fn, name=name):
            _lib.check(fn(), name)
        out[name + "_us"] = round(timed(call, reps) * 1e3, 2)
    return out


def step_legs(vxm, dev, N, L, steps, rounds):
    import numpy as np
    import torch
    from oracle import cases
    from voxelmorph_b200.trainer import GraphedTrainStep
    rng = np.random.default_rng(1)
    s, t = cases.volume_pair(7, SHAPE, sigma=3.0)
    S, T = torch.from_numpy(s).to(dev), torch.from_numpy(t).to(dev)
    feed = (torch.randn(1, L, *SHAPE, device=dev), torch.randn(1, L, *SHAPE, device=dev),
            torch.from_numpy(points(rng, N, SHAPE, L)).to(dev), torch.from_numpy(points(rng, N, SHAPE, L)).to(dev))
    mse = vxm.losses.MSE().loss
    grad = vxm.losses.Grad("l2", loss_mult=2).loss

    def with_surface(model, src, trg, *f):
        y_s, y_t, flow, v1, v2 = model(src, trg, *f)
        z = torch.zeros_like(v1)
        return 0.5 * mse(trg, y_s) + 0.5 * mse(src, y_t) + 0.01 * grad(None, flow) + 0.25 / 4.0 * (mse(z, v1) + mse(z, v2))

    def without_surface(model, src, trg):
        y_s, y_t, flow = model.vxm_model(src, trg)
        return 0.5 * mse(trg, y_s) + 0.5 * mse(src, y_t) + 0.01 * grad(None, flow)

    torch.manual_seed(0)
    model = vxm.networks.VxmDenseSemiSupervisedPointCloud(SHAPE, N, L).to(dev).train()
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4)
    graphs = {"surface": GraphedTrainStep(model, opt, loss_fn=with_surface, warmup=3).capture(S, T, *feed),
              "no_surface": GraphedTrainStep(model, opt, loss_fn=without_surface, warmup=3).capture(S, T)}
    res = {k: [] for k in graphs}
    for _ in range(rounds):
        for name, g in graphs.items():
            g()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                g()
            torch.cuda.synchronize()
            res[name].append(round((time.perf_counter() - t0) / steps * 1e3, 3))
    return {"graphed_step_ms_" + k: v for k, v in res.items()}


def copy_leg(dev, L, reps):
    import torch
    host = [torch.empty(1, L, *SHAPE).pin_memory() for _ in range(2)]
    dst = [torch.empty(1, L, *SHAPE, device=dev) for _ in range(2)]

    def copy():
        for d, h in zip(dst, host):
            d.copy_(h, non_blocking=True)
    ms = timed(copy, reps)
    nbytes = sum(h.numel() * 4 for h in host)
    return dict(sdt_h2d_bytes=nbytes, sdt_h2d_ms=round(ms, 2), sdt_h2d_gb_per_s=round(nbytes / ms / 1e6, 2))


def feed_legs(labels_list, N, L):
    import tempfile

    import numpy as np
    from scipy import ndimage
    from voxelmorph_b200 import generators
    rng = np.random.default_rng(2)
    seg = np.argmax(ndimage.gaussian_filter(rng.random((L + 1,) + tuple(s // 8 for s in SHAPE)), (0, 1, 1, 1)), 0)
    seg = ndimage.zoom(seg, 8, order=0).astype(np.int32)
    img = (seg / L).astype(np.float32)
    out = {}
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "subj.npz")
        np.savez(f, vol=img, seg=seg)
        for nl in labels_list:
            np.random.seed(0)
            t0 = time.perf_counter()
            gen = generators.surf_semisupervised([f], img, seg, N, nb_labels_sample=nl)
            item = next(gen)          # the atlas preparation runs on the first draw
            t1 = time.perf_counter()
            next(gen)
            t2 = time.perf_counter()
            out["feed_labels%d" % nl] = dict(first_batch_s=round(t1 - t0, 2), batch_s=round(t2 - t1, 2),
                                             sdt_dtype=str(item[0][2].dtype))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--points", type=int, default=5000)
    ap.add_argument("--labels", type=int, default=38)
    ap.add_argument("--feed", type=int, nargs="*", default=[])
    args = ap.parse_args()
    os.environ["VXM_B200_CONV_ENGINE"] = "bf16"
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("surf_step.py measures on the GPU; no CUDA device found")
    import voxelmorph_b200 as vxm
    dev = torch.device("cuda")
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=card(), size=SHAPE, points=args.points,
                          labels=args.labels, torch=torch.__version__)), flush=True)
    print(json.dumps(launch_legs(vxm, dev, args.points, args.labels, args.reps)), flush=True)
    print(json.dumps(copy_leg(dev, args.labels, 5)), flush=True)
    print(json.dumps(step_legs(vxm, dev, args.points, args.labels, args.steps, args.rounds)), flush=True)
    if args.feed:
        print(json.dumps(feed_legs(args.feed, args.points, args.labels)), flush=True)


if __name__ == "__main__":
    main()
