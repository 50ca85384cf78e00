"""Per-layer timing of the tensor-core convolution kernels at the benchmark shapes (CUDA events, isolated launches)."""
import sys, os, statistics, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from voxelmorph_b200 import _lib, tc

lib = _lib.load()
dev = torch.device("cuda:0")
FULL = (160, 192, 224)


def timeit(fn, n=5):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(n):
        torch.cuda._sleep(200000)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def layer(name, shape, Ca, Cb, up, Cout):
    D, H, W = shape
    ash = (D // 2, H // 2, W // 2) if up else shape
    xa = torch.randn((1,) + ash + (Ca,), device=dev).to(torch.bfloat16)
    xb = torch.randn((1,) + shape + (Cb,), device=dev).to(torch.bfloat16) if Cb else None
    w = torch.randn((Cout, Ca + Cb, 3, 3, 3), device=dev) * 0.05
    b = torch.zeros(Cout, device=dev)
    wpk, NP = tc.pack_weights(w)
    V = D * H * W
    fl = 2.0 * 27 * (Ca + Cb) * Cout * V
    t = timeit(lambda: tc.conv_fwd(xa, xb, wpk, NP, b, Cout, 3, up=up, slope=0.2))
    gz = torch.randn((1,) + shape + (max(8, Cout),), device=dev).to(torch.bfloat16)
    tw = timeit(lambda: tc.conv_wgrad(xa, xb, gz, Ca + Cb, Cout, 3, up=up))
    tt = ts = None
    if lib.vxm_conv3d_tct_supported(Ca, Cb, Cout) and lib.vxm_conv3d_tcs_supported(Ca, Cb, Cout):
        wt, cp = tc.pack_weights_t(w, variant="t")
        tt = timeit(lambda: tc.conv_fwd_t(xa, xb, wt, cp, b, Cout, 3, up=up, slope=0.2))
        ws_, cps = tc.pack_weights_t(w, variant="s")
        ts = timeit(lambda: tc.conv_fwd_t(xa, xb, ws_, cps, b, Cout, 3, up=up, slope=0.2))
    print(json.dumps(dict(layer=name, fwd_ms=round(t, 3), fwd_tflops=round(fl / t / 1e9, 1),
                          fwd_t_ms=None if tt is None else round(tt, 3), fwd_t_tflops=None if tt is None else round(fl / tt / 1e9, 1),
                          fwd_s_ms=None if ts is None else round(ts, 3), fwd_s_tflops=None if ts is None else round(fl / ts / 1e9, 1),
                          wgrad_ms=round(tw, 3), wgrad_tflops=round(fl / tw / 1e9, 1))), flush=True)


half = tuple(s // 2 for s in FULL)
layer("rem0 48->32 @1", FULL, 32, 16, True, 32)
layer("rem1 32->16 @1", FULL, 32, 0, False, 16)
layer("rem2 16->16 @1", FULL, 16, 0, False, 16)
layer("dec3 64->32 @1/2", half, 32, 32, True, 32)
layer("enc1 16->32 @1/2", half, 16, 0, False, 32)
