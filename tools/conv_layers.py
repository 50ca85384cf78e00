"""Median CUDA-event time and rate of every full-resolution convolution launch of the benchmark step (forward, dgrad,
wgrad), under the environment switches given as KEY=VALUE,... sets on the command line (profiling aid; A/B of kernel
variants). The rate is the layer's useful work, 2*27*Cin*Cout*V FLOPs over its real (unpadded) channels, over the time."""
import sys, os, json, statistics
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from voxelmorph_b200 import tc

dev = torch.device("cuda:0")
FULL = (160, 192, 224)
HALF = tuple(s // 2 for s in FULL)
V = FULL[0] * FULL[1] * FULL[2]
FLOPS = {}          # layer name -> useful FLOPs of the launch (none for the layout kernels)


def flops(name, cin, cout, v=V):
    FLOPS[name] = 2 * 27 * cin * cout * v


def timeit(fn, n=7):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(n):
        torch.cuda._sleep(200000)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return round(statistics.median(ts) * 1e3, 1)


def rnd(shape, c):
    return torch.randn((1,) + shape + (c,), device=dev).to(torch.bfloat16)


def build():
    L = {}
    w = lambda co, ci: torch.randn((co, ci, 3, 3, 3), device=dev) * 0.05
    # forward layers
    for name, ca, cb, up, co in (("enc0_fwd 8->16", 8, 0, False, 16), ("rem0_fwd 32^+16->32", 32, 16, True, 32), ("rem1_fwd 32->16", 32, 0, False, 16),
                                 ("rem2_fwd 16->16", 16, 0, False, 16)):
        xa = rnd(HALF if up else FULL, ca)
        xb = rnd(FULL, cb) if cb else None
        W = w(co, max(ca + cb, 8) if ca + cb != 8 else 2)
        if ca + cb == 8:
            W = w(co, 2)
        pk, cp = tc.pack_weights_t(W, variant="s")
        b = torch.zeros(co, device=dev)
        L[name] = (lambda xa=xa, xb=xb, pk=pk, cp=cp, b=b, co=co, up=up: tc.conv_fwd_t(xa, xb, pk, cp, b, co, 3, up=up, slope=0.2))
        flops(name, 2 if ca + cb == 8 else ca + cb, co)
    # flow head: 16 -> 3, fp32 planar out
    x = rnd(FULL, 16); W = w(3, 16); pk, cp = tc.pack_weights_t(W, variant="s"); b3 = torch.zeros(3, device=dev)
    L["flow_fwd 16->3 planar"] = lambda: tc.conv_fwd_t(x, None, pk, cp, b3, 3, 3, out_fp32_planar=True)
    flops("flow_fwd 16->3 planar", 16, 3)
    # dgrads (transposed weights): g (Cout ch) -> Cin ch
    for name, cg, cin, mask, split in (("flow_dgrad 8->16 mask", 8, 16, True, None), ("rem2_dgrad 16->16 mask", 16, 16, True, None),
                                       ("rem1_dgrad 16->32 mask", 16, 32, True, None), ("rem0_dgrad 32->48 split", 32, 48, False, 32)):
        g = rnd(FULL, cg)
        W = w(cg if cg != 8 else 3, cin)
        pk, cp = tc.pack_weights_t(W, transposed=True, variant="s")
        m = rnd(FULL, cin) if mask else None
        L[name] = (lambda g=g, pk=pk, cp=cp, cin=cin, m=m, split=split: tc.conv_fwd_t(g, None, pk, cp, None, cin, 3, slope=0.2 if m is not None else None, mask=m, split=split))
        flops(name, cg if cg != 8 else 3, cin)
    # polyphase forms of rem0 (the engine's default; VXM_B200_POLYPHASE=0 runs the two launches above and the gradient
    # routing through the upsampler below, which the coarse dgrad does in its epilogue)
    from voxelmorph_b200 import engine_bf16
    xa, xb, g32, a32 = rnd(HALF, 32), rnd(FULL, 16), rnd(FULL, 32), rnd(HALF, 32)
    W = w(32, 48); b = torch.zeros(32, device=dev)
    pk_pf, pk_pd = tc.pack_weights_poly(W, 1, 32), tc.pack_weights_poly(W, 2, 32)
    pk_ps = tc.pack_weights_blocks(W, True, (((2, 0, 32),), ((32, 16, 0, 0),)))
    L["rem0_fwd poly 32^+16->32"] = lambda: tc.conv_fwd_poly(xa, xb, pk_pf, b, 32, 0.2)
    flops("rem0_fwd poly 32^+16->32", 48, 32)
    L["rem0_dgrad_up poly 32->32 coarse"] = lambda: tc.dgrad_poly(g32, pk_pd, a32, 0.2)
    flops("rem0_dgrad_up poly 32->32 coarse", 32, 32)
    L["rem0_dgrad_skip 32->16"] = lambda: tc.conv_fwd_t(g32, None, pk_ps[0, 0][0], (pk_ps[0, 0][1], "s"), None, 16, 3)
    flops("rem0_dgrad_skip 32->16", 32, 16)
    g_up = rnd(FULL, 32)
    L["rem0 sumpool_mask 2x2x2 (split dgrad)"] = lambda: engine_bf16._sumpool_mask(g_up, a32, 3, 0.2)
    # wgrads
    for name, cx, up, cg in (("flow_wgrad x16 g8", 16, False, 8), ("rem2_wgrad x16 g16", 16, False, 16), ("rem1_wgrad x32 g16", 32, False, 16),
                             ("rem0_wgrad_a x32^ g32", 32, True, 32), ("rem0_wgrad_b x16 g32", 16, False, 32), ("enc0_wgrad x8 g16", 8, False, 16)):
        xx = rnd(HALF if up else FULL, cx)
        g = rnd(FULL, cg)
        cout = 3 if cg == 8 else cg
        cin = 2 if cx == 8 else cx
        L[name] = (lambda xx=xx, g=g, cin=cin, cout=cout, up=up: tc.conv_wgrad(xx, None, g, cin, cout, 3, up=up))
        flops(name, cin, cout)
    # dec3's upsampled source at half resolution (the rates of the upsampled wgrads count the fine form's FLOPs; the
    # coarse form, VXM_B200_POLYPHASE=1, does a third of them)
    xx, g = rnd(tuple(s // 2 for s in HALF), 32), rnd(HALF, 32)
    L["dec3_wgrad_a x32^ g32 (half res)"] = lambda: tc.conv_wgrad(xx, None, g, 32, 32, 3, up=True)
    flops("dec3_wgrad_a x32^ g32 (half res)", 32, 32, V // 8)
    # kd-folded variants of the two layers with 2 / 3 real channels on one side
    planes2 = [torch.rand((1, 1) + FULL, device=dev) for _ in range(2)]
    planes3 = [torch.randn((1, 1) + FULL, device=dev) for _ in range(3)]
    L["fold: planar_fold_kd x (2 planes -> 8ch)"] = lambda: tc.planar_fold_kd(planes2, 8)
    L["fold: planar_fold_kd g (3 planes -> 16ch)"] = lambda: tc.planar_fold_kd(planes3, 16)
    L["plain: planar_to_ndhwc8 (3 planes)"] = lambda: tc.planar_to_ndhwc8(planes3)
    x3 = tc.planar_fold_kd(planes2, 8)
    W0 = w(16, 2); pk0, cp0 = tc.pack_weights_fold(W0); b16 = torch.zeros(16, device=dev)
    L["fold: enc0_fwd 2D (6 of 8)->16"] = lambda: tc.conv_fwd_t(x3, None, pk0, cp0, b16, 16, 1, slope=0.2)
    flops("fold: enc0_fwd 2D (6 of 8)->16", 2, 16)
    g3 = tc.planar_fold_kd(planes3, 16)
    Wf = w(3, 16); pkf, cpf = tc.pack_weights_fold(Wf, transposed=True); m16 = rnd(FULL, 16)
    L["fold: flow_dgrad 2D (9 of 16)->16 mask"] = lambda: tc.conv_fwd_t(g3, None, pkf, cpf, None, 16, 1, slope=0.2, mask=m16)
    flops("fold: flow_dgrad 2D (9 of 16)->16 mask", 3, 16)
    batch = tc.WgradBatch.get(dev)
    gw0 = torch.empty((16, 6, 1, 3, 3), device=dev); gb0 = torch.empty(16, device=dev); gz16 = rnd(FULL, 16)
    gwf = torch.empty((9, 16, 1, 3, 3), device=dev); gbf = torch.empty(9, device=dev); x16 = rnd(FULL, 16)

    def khm(x, g, gw, gb, ci, co):
        batch.add_khm(x, g, gw, gb, ci, co)
        batch.flush()
    L["fold: enc0_wgrad khm"] = lambda: khm(x3, gz16, gw0, gb0, 6, 16)
    L["fold: flow_wgrad khm"] = lambda: khm(x16, g3, gwf, gbf, 16, 9)
    flops("fold: enc0_wgrad khm", 2, 16)
    flops("fold: flow_wgrad khm", 16, 3)
    return L


if sys.argv[1:2] == ["--dump"]:
    # the output of every forward and dgrad launch on seeded operands, one file per launch under DIR, for a bit-for-bit
    # comparison of two builds: `tools/conv_layers.py --dump DIR` with each, then torch.equal on every pair of files
    out_dir = sys.argv[2]
    os.makedirs(out_dir, exist_ok=True)
    torch.manual_seed(0)
    for name, fn in build().items():
        if "wgrad" in name or "fold: planar" in name or "plain:" in name or "sumpool" in name:
            continue
        y = fn()
        ys = y if isinstance(y, tuple) else (y,)
        fname = "".join(c if c.isalnum() else "_" for c in name) + ".pt"
        torch.save([t.cpu() for t in ys], os.path.join(out_dir, fname))
    torch.cuda.synchronize()
    sys.exit(0)
if sys.argv[1:2] == ["--once"]:
    # every selected layer once (ncu replays the launch itself): `ncu --set full -k regex:"conv_tcs|wgrad2_kernel" ... tools/conv_layers.py --once`
    for name, fn in build().items():
        if sys.argv[2:] and not any(t in name for t in sys.argv[2:]):
            continue
        fn()
    torch.cuda.synchronize()
    sys.exit(0)
sets = sys.argv[1:] or [""]
L = build()
res = {}
for s in sets:
    kv = dict(x.split("=") for x in s.split(",") if x)
    for k, v in kv.items():
        os.environ[k] = v
    res[s or "default"] = {name: timeit(fn) for name, fn in L.items()}
    for k in kv:
        os.environ.pop(k, None)
names = list(L)


def rate(n, us):
    return "%8.1f TF/s" % (FLOPS[n] / (us * 1e-6) / 1e12) if n in FLOPS else " " * 13


print("%-40s" % "layer" + "".join("%26s" % (s or "default")[-26:] for s in sets))
for n in names:
    print("%-40s" % n + "".join("%10.1f us %s" % (res[s or "default"][n], rate(n, res[s or "default"][n])) for s in sets))
print("%-40s" % "sum" + "".join("%10.1f us %13s" % (sum(res[s or "default"].values()), "") for s in sets))
print(json.dumps(res))
