"""HyperMorph exactly, on the paths training runs.

A. The weight generation and its backward through the C ABI at every load width.  FusedAdam packs parameters back to
   back, so in a HyperVxmDense's flat buffer hyper_kernel starts after the flow head's 1296 + 3 floats (3-D) or 288 + 2
   (2-D): the step streams it with 4- or 8-byte loads, not the 16-byte loads of an aligned tensor.  Every operand is
   placed at float offsets 0, 1, 2 and 3, so each width the kernels pick (hyp_vec: N and the pointers' alignment) runs,
   fresh and accumulating, at the default and doubled U-Nets' N and at tile and block edges, for U with and without the
   8-row unroll's tail.  With operands on coarse power-of-two grids every fp32 partial sum is an integer below 2^24 of
   its unit (asserted from the operands), so the results must equal fp64 exactly; with randn operands the elementwise
   results are bit-identical across the widths and dh (a per-lane chain, whose terms depend on the width) stays within
   its counted bound.
B. The hypernetwork at its limits (P = 16, one and eight layers, U in {1, 7, 37, 200}) against fp64 with
   test_gpu_hyper's counted bounds: autograd's fresh outputs, FusedAdam's aligned flat views, flat views behind a 1-, 2-
   or 3-float pad parameter, and a flat layout with one .grad set to None (fresh outputs over an unaligned A).
C. The step against fp64 autograd with every parameter in FusedAdam's flat buffer, hyper_kernel unaligned as in training.
D. The generated weight gradients on every U-Net shape of test_gpu_conv_exact: a HyperVxmDense whose generated weights
   are a VxmDense's gives that VxmDense's flow, weight gradients and image gradient bit for bit, on both tensor-core
   engines under both polyphase / kd-fold settings, and on the fp32 engine where autograd sums the views' gradients.

Run with -s for the widths, the largest partial sums against 2^24 and one line per exact case."""
import pytest
import torch

import hyper_ref
import test_gpu_conv_exact as cx
import test_gpu_hyper as th
from test_gpu_fp32_step_kernels import report
from test_gpu_hyper import engine, vxm  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -24
LIMIT = 2 ** 24
TILE = 1024                       # columns per CTA of the weight backward (hyper.cu kHypTile)


def vec_width(N, tensors):
    """the load width (floats) hyper.cu's hyp_vec picks: 4 or 2 when N and every row-streamed pointer allow, else 1"""
    for vec in (4, 2):
        if N % vec == 0 and all(t.data_ptr() % (4 * vec) == 0 for t in tensors):
            return vec
    return 1


def fwd_width(N, A, a, W):
    return vec_width(N, (A, a, W))


def bwd_width(N, A, gA):
    return vec_width(N, (A, gA))


def _n_of(vxm, feats):
    return vxm.layers.hyper_layout(th._shapes(vxm, feats))[1]


# ---- A. the weight kernels at every width -----------------------------------------------------------------------------

WEIGHT_CASES = [("default", U) for U in (1, 7, 37, 128, 256)] + [("doubled", 128)] + \
               [(n, U) for n in (1, 1023, 1024, 1025, 4 * 1024 + 2) for U in (1, 7, 37, 256)]


def _size(vxm, n):
    return {"default": lambda: _n_of(vxm, th.DEFAULT_FEATS), "doubled": lambda: _n_of(vxm, cx.DOUBLED)}.get(n, lambda: n)()


class Slots:
    """A (U, N), a, W, grad_A, grad_a (N) as views at one float offset into buffers 4 floats longer"""

    def __init__(self, U, N, cuda):
        self.U, self.N = U, N
        self.bufs = {k: torch.empty(n + 4, device=cuda) for k, n in
                     (("A", U * N), ("a", N), ("W", N), ("gA", U * N), ("ga", N))}

    def at(self, off):
        v = {k: b[off:off + b.numel() - 4] for k, b in self.bufs.items()}
        v["A"], v["gA"] = v["A"].view(self.U, self.N), v["gA"].view(self.U, self.N)
        return v


def _fwd(lib, h, v, U, N):
    from voxelmorph_b200 import _lib
    _lib.check(lib.vxm_hyper_weights_fwd(_lib.ptr(h), _lib.ptr(v["A"]), _lib.ptr(v["a"]), _lib.ptr(v["W"]), U, N,
                                         _lib.stream_ptr()), "vxm_hyper_weights_fwd")


def _bwd(lib, h, v, dW, U, N, accumulate):
    """dh; the partial workspace starts as NaN, so a partial the kernel never wrote shows"""
    from voxelmorph_b200 import _lib
    dh = torch.full((U,), float("nan"), device=dW.device)
    work = torch.full((int(lib.vxm_hyper_workspace_bytes(U, N)),), 0xFF, dtype=torch.uint8, device=dW.device)
    _lib.check(lib.vxm_hyper_weights_bwd(_lib.ptr(h), _lib.ptr(v["A"]), _lib.ptr(dW), _lib.ptr(v["gA"]), _lib.ptr(v["ga"]),
                                         _lib.ptr(dh), _lib.ptr(work), U, N, accumulate, _lib.stream_ptr()),
               "vxm_hyper_weights_bwd")
    return dh


def _grid(shape, lim, unit, g):
    return torch.randint(-lim, lim + 1, shape, generator=g, device=g.device).float() * unit


@pytest.mark.parametrize("n,U", WEIGHT_CASES, ids=["%s-U%d" % c for c in WEIGHT_CASES])
def test_weight_kernels_exact_at_every_width(vxm, cuda, n, U):
    """h in {-1, 0, 1} 2^-3, A = 2^-6 k (|k| <= 8), a = 2^-9 j (|j| <= 64), dW in {-1, 0, 1} 2^-4 (nonzero with
    probability 1/8), prior gradients 2^-7 m (|m| <= 16).  Units: the forward's chain 2^-9 (every h A product and a),
    gA 2^-7, the dh chains 2^-10 (every A dW product).  Each partial sum is bounded by the sum of its terms' magnitudes:
    a column's |a| + sum_k |h A| for the forward, a (row, 1024-column tile) sum of |A dW| for a lane's chain and the warp
    tree, a row's sum of |A dW| for dh (summed in fp64, rounded once).  Below 2^24 units every one is exact, so Wflat, gA,
    ga and dh equal fp64 at every offset, fresh and accumulating."""
    lib = vxm._lib.load()
    N = _size(vxm, n)
    g = torch.Generator(device=cuda).manual_seed(7 + U + N % 97)
    h = cx.ternary((U,), g, torch.float32) * 2.0 ** -3
    A, a = _grid((U, N), 8, 2.0 ** -6, g), _grid((N,), 64, 2.0 ** -9, g)
    dW = (torch.randint(0, 8, (N,), generator=g, device=cuda) == 0).float() \
        * (2 * torch.randint(0, 2, (N,), generator=g, device=cuda).float() - 1) * 2.0 ** -4
    dW[0], dW[-1] = 2.0 ** -4, -2.0 ** -4          # the first and last tiles contribute to dh
    pA, pa = _grid((U, N), 16, 2.0 ** -7, g), _grid((N,), 16, 2.0 ** -7, g)
    hd, Ad, ad, dWd = h.double(), A.double(), a.double(), dW.double()
    want_W = ad + hd @ Ad
    want_dh = Ad @ dWd
    absAdW = Ad.abs() * dWd.abs()
    tiles = torch.nn.functional.pad(absAdW, (0, -N % TILE)).view(U, -1, TILE).sum(-1)
    units = {"forward chain": float((ad.abs() + hd.abs() @ Ad.abs()).max()) / 2.0 ** -9,
             "dh lane chain + warp tree (tile)": float(tiles.max()) / 2.0 ** -10,
             "dh (fp64 tile sum, rounded once)": float(absAdW.sum(1).max()) / 2.0 ** -10,
             "gA accumulated": float((pA.double().abs() + torch.outer(hd.abs(), dWd.abs())).max()) / 2.0 ** -7}
    del absAdW, tiles
    assert all(u < LIMIT and u == int(u) for u in units.values()), units
    slots = Slots(U, N, cuda)
    widths = {"fwd": set(), "bwd": set()}
    for off in range(4):
        v = slots.at(off)
        widths["fwd"].add(fwd_width(N, v["A"], v["a"], v["W"]))
        widths["bwd"].add(bwd_width(N, v["A"], v["gA"]))
        v["A"].copy_(A)
        v["a"].copy_(a)
        v["W"].fill_(float("nan"))
        _fwd(lib, h, v, U, N)
        assert torch.equal(v["W"].double(), want_W), ("Wflat", off)
        for acc in (0, 1):
            if acc:
                v["gA"].copy_(pA)
                v["ga"].copy_(pa)
            else:
                v["gA"].fill_(float("nan"))
                v["ga"].fill_(float("nan"))
            dh = _bwd(lib, h, v, dW, U, N, acc)
            want_gA = torch.outer(hd, dWd) + (pA.double() if acc else 0)
            assert torch.equal(v["gA"].double(), want_gA), ("grad A", off, acc)
            assert torch.equal(v["ga"].double(), dWd + (pa.double() if acc else 0)), ("grad a", off, acc)
            assert torch.equal(dh.double(), want_dh), ("dh", off, acc, (dh.double() - want_dh).abs().max())
    expect = {4, 2, 1} if N % 4 == 0 else {2, 1} if N % 2 == 0 else {1}
    print("\n[hyper weights exact N=%d U=%d] widths fwd %s bwd %s | largest partial sums in units (limit 2^24 = %d): %s"
          % (N, U, sorted(widths["fwd"]), sorted(widths["bwd"]), LIMIT, {k: int(u) for k, u in units.items()}))
    assert widths["fwd"] == widths["bwd"] == expect, widths


@pytest.mark.parametrize("n,U", [("default", 37), ("default", 128), ("doubled", 128), (4 * 1024 + 2, 7), (1025, 256)])
def test_weight_kernels_randn_same_at_every_width(vxm, cuda, n, U):
    """ordinary operands: Wflat, gA and ga bit-identical at every offset (the elementwise fma and add chains do not depend
    on the width), dh within the counted bound of test_gpu_hyper (a lane's 32-term chain, the 5-level warp tree, the fp64
    tile sum's rounding)"""
    lib = vxm._lib.load()
    N = _size(vxm, n)
    g = torch.Generator(device=cuda).manual_seed(11 + U)
    h, A, a, dW = (torch.randn(s, generator=g, device=cuda) for s in ((U,), (U, N), (N,), (N,)))
    pA, pa = torch.randn((U, N), generator=g, device=cuda), torch.randn((N,), generator=g, device=cuda)
    want_dh = A.double() @ dW.double()
    s_dh = A.double().abs() @ dW.double().abs()
    slots = Slots(U, N, cuda)
    first, widths, worst = None, set(), 0.0
    for off in range(4):
        v = slots.at(off)
        widths.add((fwd_width(N, v["A"], v["a"], v["W"]), bwd_width(N, v["A"], v["gA"])))
        v["A"].copy_(A)
        v["a"].copy_(a)
        _fwd(lib, h, v, U, N)
        out = [v["W"].clone()]
        for acc in (0, 1):
            if acc:
                v["gA"].copy_(pA)
                v["ga"].copy_(pa)
            dh = _bwd(lib, h, v, dW, U, N, acc)
            out += [v["gA"].clone(), v["ga"].clone()]
            worst = max(worst, float(((dh.double() - want_dh).abs() / s_dh.clamp_min(1e-300)).max()))
        if first is None:
            first = out
        bad = [i for i, (x, y) in enumerate(zip(first, out)) if not torch.equal(x, y)]
        assert not bad, ("offset %d: outputs (Wflat, gA, ga, gA acc, ga acc) differ from offset 0" % off, bad)
    print("\n[hyper weights randn N=%d U=%d] widths (fwd, bwd) %s: Wflat, gA, ga bit-identical" % (N, U, sorted(widths)))
    report("[hyper weights randn N=%d U=%d] dh, every width" % (N, U), worst, (32 + 5 + 2) * U32)


# ---- B. the hypernetwork at its limits ---------------------------------------------------------------------------------

LIMIT_CASES = {"p16-l%d-u%d" % (L, U): ("default", 16, U, L) for L in (1, 8) for U in (1, 7, 37, 200)}


def _limit_module(vxm, cuda, name):
    """test_gpu_hyper's construction; the first seed whose h has a positive unit, so the MLP's gradients are not all zero"""
    for seed in range(16):
        mod, hyp, dW = th._hyper_module(vxm, cuda, name, seed=seed, cases=LIMIT_CASES)
        with torch.no_grad():
            mlp = [(lin.weight.double(), lin.bias.double()) for lin in mod.hypernet]
            live = float(hyper_ref.hypernet(hyp.double(), mlp).max()) > 0
        if live:
            return mod, hyp, dW
    raise AssertionError("no seed gives a live hypernetwork")


def _in_flat(mod, opt):
    """every parameter's .grad is a view of the optimizer's flat gradient buffer"""
    base = opt.fp.grad.data_ptr()
    return all(base <= p.grad.data_ptr() < base + 4 * opt.fp.numel for p in mod.parameters())


def _flat_run(mod, hyp, dW, opt):
    opt.zero_grad()
    w = mod(hyp)
    w.backward(dW)
    return [w.detach().clone()] + [p.grad.clone() for p in mod.parameters()]


@pytest.mark.parametrize("name", sorted(LIMIT_CASES))
def test_hypernetwork_limits_vs_fp64(vxm, cuda, name):
    """fresh outputs (autograd) and FusedAdam's aligned flat views: both within the counted bounds, and equal"""
    mod, hyp, dW = _limit_module(vxm, cuda, name)
    fresh = th._run(mod, hyp, dW)
    th.check_vs_fp64(mod, hyp, dW, fresh, name + " fresh")
    opt = vxm.optim.FusedAdam(mod.parameters(), lr=1e-3)
    flat = _flat_run(mod, hyp, dW, opt)
    assert _in_flat(mod, opt)
    th.check_vs_fp64(mod, hyp, dW, flat, name + " flat")
    assert all(torch.equal(x, y) for x, y in zip(fresh, flat))


@pytest.mark.parametrize("pad,none_grad", [(1, False), (2, False), (3, False), (3, True)],
                         ids=["pad1", "pad2", "pad3", "pad3-one-grad-none"])
def test_hypernetwork_on_unaligned_flat_views(vxm, cuda, pad, none_grad):
    """a pad parameter of 1, 2 or 3 floats ahead of the module in FusedAdam's buffer: the accumulate path over unaligned
    A, a, gA and ga; with one .grad set to None, fresh outputs over the unaligned A that autograd adds into the views"""
    name = "p16-l8-u37"
    mod, hyp, dW = _limit_module(vxm, cuda, name)
    fresh = th._run(mod, hyp, dW)
    pad_p = torch.nn.Parameter(torch.zeros(pad, device=cuda))
    opt = vxm.optim.FusedAdam([pad_p] + list(mod.parameters()), lr=1e-3)
    opt.zero_grad()
    if none_grad:
        mod.hypernet[3].bias.grad = None
    w = mod(hyp)
    w.backward(dW)
    got = [w.detach().clone()] + [p.grad.clone() for p in mod.parameters()]
    A, a = mod.hyper_kernel, mod.hyper_bias
    U, N = A.shape
    widths = (fwd_width(N, A, a, mod.wflat), bwd_width(N, A, A.grad if not none_grad else torch.empty_like(A)))
    print("\n[hyper pad %d%s] hyper_kernel at byte %d mod 16; widths (fwd, bwd) %s"
          % (pad, ", one grad None" if none_grad else "", A.data_ptr() % 16, widths))
    assert A.data_ptr() % 16 != 0 and widths[0] == (2 if pad == 2 else 1)
    assert none_grad or _in_flat(mod, opt)
    th.check_vs_fp64(mod, hyp, dW, got, "%s pad %d%s" % (name, pad, " none-grad" if none_grad else ""))
    # Wflat, grad A and grad a as with 16-byte loads; dh (and with it the hypernetwork's gradients) sums each lane's
    # columns in another grouping, so those are held to the fp64 bounds above
    assert all(torch.equal(x, y) for x, y in zip(fresh[:3], got[:3]))
    assert not bool(pad_p.grad.any())


# ---- C. the step on FusedAdam's flat buffer ----------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["3d", "2d"])
@pytest.mark.parametrize("eng_name", ["f32", "bf16x3", "bf16"])
def test_hyper_step_on_flat_params_vs_oracle(vxm, cuda, engine, eng_name, name):  # noqa: F811
    """test_gpu_hyper's step check with FusedAdam built first: hyper_kernel sits after the flow head in the flat buffer,
    unaligned, and every gradient is read from the flat views"""
    model, opt = th.check_step_vs_oracle(vxm, cuda, engine, eng_name, name, flat=True)
    hw = model.hyper
    A, a = hw.hyper_kernel, hw.hyper_bias
    assert _in_flat(model, opt)
    U, N = A.shape
    print("[hyper flat step %s %s] hyper_kernel at float %d of the flat buffer (byte %d mod 16): widths fwd %d, bwd %d"
          % (eng_name, name, (A.data_ptr() - opt.fp.flat.data_ptr()) // 4, A.data_ptr() % 16, fwd_width(N, A, a, hw.wflat),
             bwd_width(N, A, A.grad)))
    assert A.data_ptr() % 16 != 0


# ---- D. generated weight gradients on every U-Net shape ---------------------------------------------------------------

GEN_NAMES = [n for n in sorted(cx.MODELS) if not cx.MODELS[n].probs]
GEN_CASES = [(n, e) for n in GEN_NAMES for e in ("bf16", "bf16x3")] + [(n, "f32") for n in ("2d", "doubled", "2d_doubled")]


@pytest.mark.parametrize("name,eng_name", GEN_CASES, ids=["%s-%s" % c for c in GEN_CASES])
def test_generated_grads_equal_vxmdense(vxm, cuda, monkeypatch, name, eng_name):
    """hyper_kernel = 0, hyper_bias = a VxmDense's U-Net parameters, the same flow head: the U-Net and head forward, then
    backward with one fixed flow gradient (no VecInt or warp atomics).  Flow, dW (hyper_bias.grad) against the VxmDense's
    concatenated U-Net gradients, the head's gradients and (default) the source image's gradient bit-identical; again
    with both models' parameters in FusedAdam's zeroed flat views.  3-D tensor-core cases under both polyphase / kd-fold
    settings."""
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", eng_name)
    kw, B = cx.MODELS[name].kw, cx.MODELS[name].B
    inshape = tuple(kw["inshape"])
    torch.manual_seed(60 + len(name))
    plain = vxm.networks.VxmDense(**kw).to(cuda).train()
    hyper = vxm.networks.HyperVxmDense(**kw).to(cuda).train()
    unet = list(plain.unet_model.parameters())
    assert hyper.hyper.shapes == [tuple(p.shape) for p in unet[0::2]]
    g = torch.Generator(device=cuda).manual_seed(61 + len(name))
    with torch.no_grad():
        plain.flow.weight.copy_(torch.randn(plain.flow.weight.shape, generator=g, device=cuda) * 0.05)
        hyper.hyper.hyper_kernel.zero_()
        hyper.hyper.hyper_bias.copy_(torch.cat([p.reshape(-1) for p in unet]))
        hyper.flow.weight.copy_(plain.flow.weight)
        hyper.flow.bias.copy_(plain.flow.bias)
    S = torch.rand((B, kw.get("src_feats", 1)) + inshape, generator=g, device=cuda)
    T = torch.rand((B, kw.get("trg_feats", 1)) + inshape, generator=g, device=cuda)
    hyp = torch.tensor([[0.37]], device=cuda)
    image_grad = name == "default"
    opts, gflow = {}, []

    def run(model, flat):
        if flat:
            if model not in opts:
                opts[model] = vxm.optim.FusedAdam(model.parameters(), lr=1e-3)
            opts[model].zero_grad()
        else:
            for p in model.parameters():
                p.grad = None
        src = S.clone().requires_grad_(image_grad)
        if model is hyper:
            hyper._assign(hyper.hyper(hyp))
        out = model._head(src, T)
        if not gflow:                     # the field's shape (half resolution for unet_half_res)
            gflow.append(torch.randn(out.shape, generator=g, device=cuda))
        out.backward(gflow[0])
        if model is hyper:
            hyper._assign(hyper.hyper.wflat)
        dW = hyper.hyper.hyper_bias.grad if model is hyper else torch.cat([p.grad.reshape(-1) for p in unet])
        return [out.detach().clone(), dW.clone(), model.flow.weight.grad.clone(), model.flow.bias.grad.clone(), src.grad]

    three_d = len(inshape) == 3 and eng_name != "f32"
    settings = [("1", "polyphase+kdfold"), ("0", "split+unfolded")] if three_d else [(None, "")]
    forms = []
    for env, label in settings:
        if env is not None:
            monkeypatch.setenv("VXM_B200_POLYPHASE", env)
            monkeypatch.setenv("VXM_B200_KDFOLD", env)
            for m in (plain, hyper):      # the plan caches the forms: build it again under the new setting
                m.__dict__.pop("_vxm_pack_plan", None)
        for flat in (False, True):
            want, got = run(plain, flat), run(hyper, flat)
            assert bool(want[1].any()) and (want[4] is not None) == image_grad
            what = ["flow", "dW", "flow.weight grad", "flow.bias grad", "source grad"]
            bad = [(w, int((x != y).sum())) for w, x, y in zip(what, want, got) if x is not None and not torch.equal(x, y)]
            assert not bad, (name, eng_name, label, "flat" if flat else "autograd", bad)
        if env is not None:
            forms.append([(L.fwd, L.dgrad) for L in hyper.__dict__["_vxm_pack_plan"].layers])
        print("\n[hyper generated %s %s%s] B=%d N=%d: flow, dW, head gradients%s bit-identical to VxmDense (autograd and "
              "flat views)" % (name, eng_name, " " + label if label else "", B, hyper.hyper.hyper_bias.numel(),
                               ", source gradient" if image_grad else ""))
    assert len(forms) != 2 or forms[0] != forms[1], "the two settings ran the same layer forms"
