"""Measurement aid for the memory-bound kernels: every kernel is called straight through the C ABI (no autograd
around it) at the benchmark shapes.

  python tools/r2_memprof.py time     -> CUDA-event timings (L2 flushed between launches), JSON on stdout
  python tools/r2_memprof.py launch   -> each kernel launched 3 times (wrap in `ncu --set full -k regex:...`)
"""
import ctypes
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import voxelmorph_b200 as vxm
from voxelmorph_b200 import _lib

HBM_GBS = 3350.0   # H100 SXM data-sheet HBM3 bandwidth (700 W); frac is relative to it
mode = sys.argv[1] if len(sys.argv) > 1 else "time"
dev = torch.device("cuda:0")
lib = _lib.load()
P, S = _lib.ptr, _lib.stream_ptr
shape = (160, 192, 224)
half = tuple(s // 2 for s in shape)
D, H, W = shape
Dh, Hh, Wh = half
V, Vh = D * H * W, Dh * Hh * Wh


def smooth(shp, sig):
    return torch.nn.functional.interpolate(torch.randn((1, 3) + tuple(max(2, s // 16) for s in shp), device=dev) * sig, size=shp,
                                           mode="trilinear", align_corners=True).contiguous()


src = torch.rand((1, 1) + shape, device=dev)
flow = smooth(shape, 3.0)
vel = smooth(half, 2.0)
out1 = torch.empty_like(src)
out3 = torch.empty_like(flow)
out3h = torch.empty_like(vel)
g1 = torch.rand_like(src)
g3 = torch.rand_like(flow)
g3h = torch.rand_like(vel)
I, J = torch.rand_like(src), torch.rand_like(src)
saved = torch.empty((1, 3) + shape, device=dev)
loss = torch.empty((), device=dev)
gl = torch.ones((), device=dev)
ws = _lib.reduce_workspace(dev)
states = torch.empty(int(lib.vxm_vecint_fast_states_bytes(1, Dh, Hh, Wh, 7)), dtype=torch.uint8, device=dev)
work_f = torch.empty(int(lib.vxm_vecint_fast_work_bytes(1, Dh, Hh, Wh, 0)), dtype=torch.uint8, device=dev)
work_b = torch.empty(int(lib.vxm_vecint_fast_work_bytes(1, Dh, Hh, Wh, 1)), dtype=torch.uint8, device=dev)
FAST = 2

K = {}
K["warp_fwd_fast"] = (lambda: lib.vxm_warp_fwd(P(src), P(flow), P(out1), 1, 1, D, H, W, D, H, W, 3, 0, FAST, S()), V * 20)
K["warp_fwd_nearest"] = (lambda: lib.vxm_warp_fwd(P(src), P(flow), P(out1), 1, 1, D, H, W, D, H, W, 3, 1, 0, S()), V * 20)
K["warp_bwd_fast(dflow)"] = (lambda: lib.vxm_warp_bwd(P(g1), P(src), P(flow), None, P(out3), 1, 1, D, H, W, D, H, W, 3, 0, FAST, S()), V * 36)
for n in (1, 3, 7):
    K["vecint_fwd_fast_n%d" % n] = (lambda n=n: lib.vxm_vecint_fwd(P(vel), P(out3h), None, P(work_f), 1, Dh, Hh, Wh, 3, n, FAST, S()), Vh * 24 * n)
K["vecint_fwd_fast_n7_states"] = (lambda: lib.vxm_vecint_fwd(P(vel), P(out3h), P(states), None, 1, Dh, Hh, Wh, 3, 7, FAST, S()), Vh * 24 * 7)
for n in (1, 7):
    K["vecint_bwd_fast_n%d" % n] = (lambda n=n: lib.vxm_vecint_bwd(P(g3h), P(states), P(out3h), P(work_b), 1, Dh, Hh, Wh, 3, n, FAST, S()), Vh * 36 * n)
K["resize_up"] = (lambda: lib.vxm_resize_fwd(P(vel), P(out3), 1, 3, Dh, Hh, Wh, D, H, W, 2.0, 1.0, S()), (V + Vh) * 12)
K["resize_down"] = (lambda: lib.vxm_resize_fwd(P(flow), P(out3h), 1, 3, D, H, W, Dh, Hh, Wh, 1.0, 0.5, S()), (V + Vh) * 12)
K["resize_up_bwd"] = (lambda: lib.vxm_resize_bwd(P(g3), P(out3h), 1, 3, Dh, Hh, Wh, D, H, W, 2.0, 1.0, S()), (V + Vh) * 12)
K["resize_down_bwd"] = (lambda: lib.vxm_resize_bwd(P(g3h), P(out3), 1, 3, D, H, W, Dh, Hh, Wh, 1.0, 0.5, S()), (V + Vh) * 12)
K["ncc_fwd"] = (lambda: lib.vxm_ncc_fwd(P(I), P(J), P(loss), None, P(ws), 1, D, H, W, 9, 9, 9, S()), V * 8)
K["ncc_fwd_saving"] = (lambda: lib.vxm_ncc_fwd(P(I), P(J), P(loss), P(saved), P(ws), 1, D, H, W, 9, 9, 9, S()), V * 20)
K["ncc_bwd"] = (lambda: lib.vxm_ncc_bwd(P(I), P(J), P(saved), P(gl), P(out1), 1, D, H, W, 9, 9, 9, S()), V * 24)
for n, c in ((1, 0), (8, 0), (8, 1), (16, 1)):
    K["gridsync_x%d_%s" % (n, "max" if c == 0 else "%dcta" % c)] = (lambda n=n, c=c: lib.vxm_debug_gridsync(n, c, S()), 0)

if mode == "launch":
    for name, (fn, _) in K.items():
        for _ in range(3):
            rc = fn()
            assert rc == 0, (name, _lib.last_error())
    torch.cuda.synchronize()
    sys.exit(0)

flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
res = {}
for name, (fn, nbytes) in K.items():
    for _ in range(3):
        assert fn() == 0, (name, _lib.last_error())
    ts = []
    for _ in range(10):
        flush.zero_()
        torch.cuda._sleep(300000)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    t = statistics.median(ts)
    res[name] = dict(us=round(t, 1), gbs=round(nbytes / t / 1e3, 1) if nbytes else None, frac=round(nbytes / t / 1e3 / HBM_GBS, 3) if nbytes else None)
    print("%-30s %8.1f us  %s" % (name, t, "" if not nbytes else "%7.1f GB/s  %.3f" % (nbytes / t / 1e3, nbytes / t / 1e3 / HBM_GBS)), file=sys.stderr)
print(json.dumps(res))
