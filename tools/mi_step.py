"""What MutualInformation costs at 160x192x224, B = 1: the isolated MI forward and backward (one-sided: y_pred only;
two-sided) at 16, 32 and 64 bins through the C ABI, next to the NCC forward and backward; the eager torch-op composition
of the same formula in fp32 on the same card (time and max_memory_allocated); and the CUDA-graphed VxmDense step with
MI + 0.01 Grad('l2') against NCC + 0.01 Grad, alternated over `--rounds` rounds.

Each launch leg reports its time with its bytes and FP32 FMAs, the HBM bound at 3.35 TB/s and the FMA bound at
33.5 T FMA/s (67 TFLOP/s), and its share of the larger bound.  Times are CUDA events around `--reps` calls after three
warm-up calls.  The card's name and power limit are printed with the numbers: they are part of them.

    python tools/mi_step.py [--steps 10] [--warmup 3] [--rounds 3] [--reps 20] [--size 160 192 224]
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
FMA_PER_S = 33.5e12              # 67 TFLOP/s FP32, data sheet


def _entry(ms, nbytes, fmas):
    hbm, fma = nbytes / HBM_BYTES_PER_S, fmas / FMA_PER_S
    bound = "hbm" if hbm >= fma else "fp32_fma"
    return dict(us=round(ms * 1e3, 1), bytes=int(nbytes), fmas=int(fmas), hbm_bound_us=round(hbm * 1e6, 1),
                fma_bound_us=round(fma * 1e6, 1), bound=bound, share_of_bound=round(max(hbm, fma) / (ms * 1e-3), 3))


def launch_legs(vxm, dev, S, T, reps):
    import torch
    from voxelmorph_b200 import _lib
    lib = _lib.load()
    shape = tuple(S.shape[2:])
    V = S.numel()
    out = {}
    loss, gl = torch.empty((), device=dev), torch.ones((), device=dev)
    gx, gy = torch.empty_like(S), torch.empty_like(T)
    rw = _lib.reduce_workspace(dev)
    st = _lib.stream_ptr
    for B in (16, 32, 64):
        BP = (B + 15) // 16 * 16
        alpha = 1.0 / (2.0 * (0.5 / (B - 1)) ** 2)
        work = torch.empty(int(lib.vxm_mi_workspace_bytes(1, V, B)), dtype=torch.uint8, device=dev)
        args = (1, V, B, alpha, float("-inf"), float("inf"))

        def fwd():
            _lib.check(lib.vxm_mi_fwd(_lib.ptr(T), _lib.ptr(S), None, _lib.ptr(loss), _lib.ptr(work), _lib.ptr(rw), *args,
                                      st()), "vxm_mi_fwd")

        def bwd(g_true, g_pred):
            _lib.check(lib.vxm_mi_bwd(_lib.ptr(T), _lib.ptr(S), None, _lib.ptr(gl), _lib.ptr(g_true), _lib.ptr(g_pred),
                                      _lib.ptr(work), *args, st()), "vxm_mi_bwd")
        fwd()
        # forward: min/max pass (8 B/voxel) + histogram pass (8 B/voxel), V BP^2 FMAs of P
        out["mi_fwd_B%d" % B] = _entry(timed(fwd, reps), 16 * V, V * BP * BP)
        # backward per side: 8 B/voxel read + 4 written, 4 re-read by the tie pass; V BP^2 FMAs of a = Gp w + gs
        out["mi_bwd_one_sided_B%d" % B] = _entry(timed(lambda: bwd(None, gy), reps), 16 * V, V * BP * BP)
        out["mi_bwd_two_sided_B%d" % B] = _entry(timed(lambda: bwd(gx, gy), reps), 24 * V, 2 * V * BP * BP)
        del work
    saved = torch.empty((1, 3) + shape, device=dev)
    ncc = lambda: _lib.check(lib.vxm_ncc_fwd(_lib.ptr(T), _lib.ptr(S), _lib.ptr(loss), _lib.ptr(saved), _lib.ptr(rw), 1,
                                             *shape, 9, 9, 9, st()), "vxm_ncc_fwd")
    ncc_b = lambda: _lib.check(lib.vxm_ncc_bwd(_lib.ptr(T), _lib.ptr(S), _lib.ptr(saved), _lib.ptr(gl), _lib.ptr(gy), 1,
                                           *shape, 9, 9, 9, st()), "vxm_ncc_bwd")
    ncc()
    out["ncc_fwd"] = _entry(timed(ncc, reps), 20 * V, 0)
    out["ncc_bwd_one_sided"] = _entry(timed(ncc_b, reps), 24 * V, 0)
    return out


def eager_legs(dev, S, T, reps):
    """The formula as torch ops in fp32, autograd for both inputs: time and peak memory of forward + backward."""
    import torch
    out = {}

    def mi_torch(x, y, B):
        alpha = 1.0 / (2.0 * (0.5 / (B - 1)) ** 2)

        def q(t):
            lo, hi = torch.amin(t), torch.amax(t)
            c = lo + (hi - lo) * torch.arange(B, dtype=t.dtype, device=t.device) / (B - 1)
            return torch.softmax(-alpha * (t[..., None] - c) ** 2, dim=-1).reshape(t.shape[0], -1, B)
        qx, qy = q(x), q(y)
        pxy = torch.bmm(qx.transpose(1, 2), qy)
        pxy = pxy / (pxy.sum(dim=(1, 2), keepdim=True) + 1e-7)
        px = qx.sum(1, keepdim=True)
        px = px / (px.sum(2, keepdim=True) + 1e-7)
        py = qy.sum(1, keepdim=True)
        py = py / (py.sum(2, keepdim=True) + 1e-7)
        pxpy = torch.bmm(px.transpose(1, 2), py) + 1e-7
        return -(pxy * torch.log(pxy / pxpy + 1e-7)).sum(dim=(1, 2)).mean()

    for B in (16, 32, 64):
        X, Y = T.clone().requires_grad_(True), S.clone().requires_grad_(True)

        def step():
            X.grad = Y.grad = None
            mi_torch(X, Y, B).backward()
        try:
            step()
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            ms = timed(step, max(3, reps // 4))
            peak = torch.cuda.max_memory_allocated(dev) - base
            out["eager_torch_fwd_bwd_B%d" % B] = dict(us=round(ms * 1e3, 1), extra_peak_mib=round(peak / 2 ** 20, 1))
        except torch.cuda.OutOfMemoryError:
            out["eager_torch_fwd_bwd_B%d" % B] = "out of memory"
        del X, Y
        torch.cuda.empty_cache()
    return out


def step_leg(vxm, dev, shape, S, T, leg, steps, warmup):
    import torch
    from voxelmorph_b200.trainer import GraphedTrainStep
    torch.manual_seed(1234)
    model = vxm.networks.VxmDense(shape)
    with torch.no_grad():
        model.to(dev).train()
        model.flow.weight.normal_(0, 1e-2)
    opt = vxm.optim.FusedAdam(model.parameters(), lr=1e-4)
    step = GraphedTrainStep(model, opt, image_loss=leg, warmup=3).capture(S, T)
    ms = timed(lambda: step(S, T), steps, warmup)
    loss = float(step.loss)
    del step, opt, model
    torch.cuda.empty_cache()
    return dict(leg=leg, ms_per_step=round(ms, 3), loss=loss)


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
        raise SystemExit("mi_step.py measures on a CUDA device; none is available")
    os.environ["VXM_B200_CONV_ENGINE"] = "bf16"
    dev = torch.device("cuda:0")
    shape = tuple(args.size)
    s, t = cases.volume_pair(3, shape, sigma=2.0)
    lo, hi = min(s.min(), t.min()), max(s.max(), t.max())
    S, T = (torch.from_numpy(((v - lo) / (hi - lo)).astype("float32")).to(dev) for v in (s, t))   # intensities in [0, 1]
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=card(), size=shape, torch=torch.__version__)))
    print(json.dumps(launch_legs(vxm, dev, S, T, args.reps)), flush=True)
    print(json.dumps(eager_legs(dev, S, T, args.reps)), flush=True)
    results = {}
    for r in range(args.rounds):
        for leg in ("mi", "ncc"):
            res = step_leg(vxm, dev, shape, S, T, leg, args.steps, args.warmup)
            res["round"] = r
            print(json.dumps(res), flush=True)
            results.setdefault(leg, []).append(res["ms_per_step"])
    for leg, ms in results.items():
        print("%-4s + Grad ms/step per round: %s  (best %.3f)" % (leg, " ".join("%.3f" % m for m in ms), min(ms)))


if __name__ == "__main__":
    main()
