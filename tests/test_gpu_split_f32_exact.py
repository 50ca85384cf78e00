"""The two engines `import voxelmorph` runs ('tc': bf16x3 for the U-Nets the tensor-core engine supports, f32 for the
others), checked exactly at the step's own sizes, and the bf16x3 backward's routing of MaxPool gradients.

bf16x3 forward: every launch of the split-precision plan (three passes x_lo w_hi + x_hi w_lo + x_hi w_hi, single
launches, channel blocks with their fp32 accumulator, the flow head's fp32 planar output) against the fp64 sum
sum x_hi w_hi + x_lo w_hi + x_hi w_lo (the lo * lo term is dropped by design), with the out_mode 3 epilogue (bias,
LeakyReLU, hi = bf16(x), lo = bf16(x - hi)) emulated in fp32.  Operands: activations hi in {-1, 0, 1}, lo in
2^-9 {-1, 0, 1}; weights 2^-6 k + 2^-15 j (|k| <= 2, j in {-1, 0, 1}, j = 0 where k = 0), so that w_hi = 2^-6 k and
w_lo = 2^-15 j exactly.  Every product is then a multiple of 2^-15 and every partial sum is below 2^22 of those units
(asserted, printed as the margin over 2^24).

f32 engine (conv3d_f32.cu): forward, masked dgrad, weight gradient accumulated onto an integer-valued prior and bias
gradient of every layer shape of the default model at 160x192x224 and of the doubled model at 64x96x112.  Those kernels
apply the LeakyReLU derivative to the output gradient as they load it, before the sums, so these tests use the slope
2^-2: with the model's 0.2 the masked products would round and no fp64 sum would be exact.

Run with -s to print every launch's mismatch count next to its margin."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import conv_exact_ref as ref
from test_gpu_conv_exact import CAPS, MODELS, _children, _unchildren, build_model, check_head_plan, check_resolves, mism, plan_sizes, ternary

pytestmark = pytest.mark.gpu

SLOPE = 0.2                      # the model's LeakyReLU slope (bf16x3 epilogue: applied once to an exact fp32 sum)
SLOPE_F32 = 0.25                 # the f32 tests' slope: exact products when the mask is applied on load
LO = 2.0 ** -9                   # activation lo parts: {-1, 0, 1} * LO
FULL = (160, 192, 224)


@pytest.fixture(scope="module")
def vx(cuda):
    import voxelmorph_b200 as vxm
    from voxelmorph_b200 import engine_bf16, tc
    vxm._lib.load()
    return vxm, engine_bf16, tc


def _report(title, rows, limit=0.25):
    """rows (launch, form, mismatches, margin): every mismatch count must be 0 and every margin below `limit`"""
    print("\n[%s] launch | form | mismatches (expected 0) | margin" % title)
    for name, form, n, margin in rows:
        print("  %-34s %-26s %8d   %.2e" % (name, form, n, margin))
    bad = [r for r in rows if r[2] or r[3] >= limit]
    assert not bad, bad


def sparse_ternary(shape, g, dtype=torch.float32, den=2):
    """{-1, 0, 1}, each nonzero with probability 1 / den"""
    nz = torch.randint(0, den, shape, generator=g, device=g.device) == 0
    return (nz * (2 * torch.randint(0, 2, shape, generator=g, device=g.device) - 1)).to(dtype)


def split_pair(shape, g):
    """(hi, lo) bf16 activations: hi in {-1, 0, 1}, lo in LO {-1, 0, 1}, drawn independently"""
    return ternary(shape, g), (ternary(shape, g).float() * LO).to(torch.bfloat16)


def split_weight(shape, g):
    """(w, k, j): w = 2^-6 k + 2^-15 j with |k| <= 2, j in {-1, 0, 1} and j = 0 where k = 0 (a lone 2^-15 j would be
    its own bf16 hi part); bf16(w) = 2^-6 k exactly: the round-to-nearest-even ties at k = +-1 go to 2^-6 k"""
    k = torch.randint(-2, 3, shape, generator=g, device=g.device).float()
    j = torch.randint(-1, 2, shape, generator=g, device=g.device).float() * (k != 0)
    return k * 2.0 ** -6 + j * 2.0 ** -15, k, j


def split_epilogue(y, bias, slope):
    """out_mode 3 of conv_tcs_kernel on an exact fp64 sum y: fp32 x = y + bias, x >= 0 ? x : x * slope, then
    hi = RNE bf16(x), lo = RNE bf16(x - hi)"""
    x = y.float() + bias.float()
    if slope is not None:
        x = torch.where(x >= 0, x, x * torch.tensor(slope, dtype=torch.float32, device=x.device))
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def torch_split(x):
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def _split_margin(cin, unit_terms, bias_units):
    """bound over 2^24 of a split-precision forward's partial sums: 27 taps x cin channels x (the three products' bounds in
    units) plus the bias"""
    return (27 * cin * unit_terms + bias_units) / 2 ** 24


# ---- 1. the bf16x3 forward, exactly, at the plan's own size -----------------------------------------------------------

@pytest.mark.parametrize("name", sorted(MODELS))
def test_split_forward_exact(vx, cuda, monkeypatch, name):
    """Every layer of the bf16x3 plan through _run(L.fwd_x3, L.pk_hi, ..., lo=(xa_lo, xb_lo, L.pk_lo)), as forward_tape
    runs it; the first layer on the output of planar_to_ndhwc8_split.  Every model of the exact tier's matrix (of a
    probabilistic one, the 2 nd-output head, whose hi / lo parts come from the concatenated fp32 head)."""
    vxm, eng, tc = vx
    kw, B = MODELS[name].kw, MODELS[name].B
    g = torch.Generator(device=cuda).manual_seed(11 + len(name))
    model = build_model(vxm, name).to(cuda)
    kj = {}
    with torch.no_grad():
        for p in model.parameters():
            w, k, j = split_weight(p.shape, g)
            p.copy_(w)
            kj[p] = (k, j)
    check_resolves(vxm, monkeypatch, name, model)
    plan = eng._plan_of(model, True)
    layers = plan.layers
    nd, kd = plan.nd, (3 if plan.nd == 3 else 1)
    if MODELS[name].probs:
        check_head_plan(model, plan)
        fw, _, lw, _ = layers[-1].srcs
        kj[layers[-1].w] = tuple(torch.cat([a, b]) for a, b in zip(kj[fw], kj[lw]))
    for L in layers:
        k, j = kj[L.w]
        assert torch.equal(L.w_hi, k * 2.0 ** -6) and torch.equal(L.w_lo, j * 2.0 ** -15)
    size, chans = plan_sizes(eng, plan, kw["inshape"])
    first, flow = layers[0], layers[-1]
    # image planes (a + b 2^-9) / 16, b = 0 where a = 0: hi = a / 16 and lo = b 2^-13 exactly (the tie at a = 1, b = -1
    # rounds to even, 2^-4), so the first layer's products are multiples of 2^-19 that fit 24 bits with the bias
    planes = []
    for _ in range(first.cin):
        a = ternary((B, 1) + size[0], g, torch.float32)
        planes.append((a + ternary((B, 1) + size[0], g, torch.float32) * (a != 0) * 2.0 ** -9) / 16)
    XH, XL = {}, {}
    XH[0], XL[0] = tc.planar_to_ndhwc8_split(planes)
    images = torch.cat(planes, 1).permute(0, 2, 3, 4, 1)
    img_hi, img_lo = torch_split(images)
    assert torch.equal(img_hi.float(), (images * 16).round() / 16)
    n_glue = (mism(XH[0][..., :first.cin], img_hi) + mism(XL[0][..., :first.cin], img_lo)
              + int(XH[0][..., first.cin:].count_nonzero()) + int(XL[0][..., first.cin:].count_nonzero()))
    for i, c in chans.items():
        if i != flow.out:
            XH[i], XL[i] = split_pair((B,) + size[i] + (c,), g)

    def lname(i, L):
        return "%02d %s (%d%s+%d)->%d %s" % (i, L.role, L.ca, "^" if L.up else "", L.cb, L.cout, "x".join(map(str, size[L.out])))

    rows = [("00 images", "planar_to_ndhwc8_split", n_glue, 0.0)]
    for i, L in enumerate(layers):
        if MODELS[name].probs and L is not flow:
            continue
        bias, D = L.bias.detach(), size[L.out][0]
        out = eng._run(L.fwd_x3, L.pk_hi, XH[L.a], XH.get(L.b), L.cout, kd, bias, lo=(XL[L.a], XL.get(L.b), L.pk_lo),
                       up=L.up, slope=L.slope, out_fp32_planar=L is flow)
        if L is first:
            hs, ls = [(img_hi, False)], [(img_lo, False)]
            margin = _split_margin(L.cin, 2 ** 10 + 2 + 1, 2 ** 14 + 2 ** 4)       # units of 2^-19
        else:
            hs = [(XH[L.a], L.up)] + ([(XH[L.b], False)] if L.b is not None else [])
            ls = [(XL[L.a], L.up)] + ([(XL[L.b], False)] if L.b is not None else [])
            margin = _split_margin(L.cin, 2 ** 10 + 2 + 1, 2 ** 10 + 1)            # units of 2^-15
        w3 = torch.cat([L.w_hi, L.w_hi, L.w_lo], 1).view(L.cout, 3 * L.cin, kd, 3, 3)      # [hi, lo, hi] sources
        if L is flow:
            res = out.permute(0, 2, 3, 4, 1)
            n = sum(ref.conv(hs + ls + hs, w3, D, nd=nd, finish=lambda y, d0, d1: mism(res[:, d0:d1], ref.epilogue(y, bias, bf16=False))))
        else:
            oh, ol = out

            def fin(y, d0, d1):
                h, lo = split_epilogue(y, bias, L.slope)
                return mism(oh[:, d0:d1], h) + mism(ol[:, d0:d1], lo)
            n = sum(ref.conv(hs + ls + hs, w3, D, nd=nd, finish=fin))
        kind = "one launch" if len(L.fwd_x3[0]) == len(L.fwd_x3[1]) == 1 else "%dx%d blocks" % (len(L.fwd_x3[0]), len(L.fwd_x3[1]))
        rows.append((lname(i, L), "fwd x3 " + kind + (" fp32 planar" if L is flow else ""), n, margin))
        del out
    assert any(len(L.fwd_x3[0]) * len(L.fwd_x3[1]) > 1 for L in layers) == MODELS[name].blocked
    _report("bf16x3 forward exact %s" % name, rows)


# ---- 2. the split glue, exactly, at full resolution -------------------------------------------------------------------

@pytest.mark.parametrize("nplanes", [2, 3, 8])
def test_planar_to_ndhwc8_split_exact(vx, cuda, nplanes):
    """hi = bf16(x), lo = bf16(x - hi) bit for bit, B = 2, planes sliced out of one (B, n, D, H, W) tensor (batch stride
    n * D * H * W, as forward_tape slices the images) and separate contiguous planes"""
    _, _, tc = vx
    g = torch.Generator(device=cuda).manual_seed(30 + nplanes)
    x = torch.randn((2, nplanes) + FULL, generator=g, device=cuda) * torch.exp2(torch.randint(-12, 13, (2, nplanes) + FULL, generator=g, device=cuda).float())
    # exact ties of the hi rounding (1 + 2^-8 (2m + 1) lies halfway between two bf16 neighbours), zeros and signs
    tie = (1 + 2.0 ** -8 * (2 * torch.randint(0, 64, x.shape, generator=g, device=cuda) + 1)) * (2 * torch.randint(0, 2, x.shape, generator=g, device=cuda) - 1)
    pick = torch.randint(0, 4, x.shape, generator=g, device=cuda)
    x = torch.where(pick == 0, tie.float(), torch.where(pick == 1, torch.zeros_like(x), x))
    rh, rl = torch_split(x.permute(0, 2, 3, 4, 1))
    counts = {}
    for kind, planes in (("strided", [x[:, i:i + 1] for i in range(nplanes)]), ("contiguous", [x[:, i:i + 1].contiguous() for i in range(nplanes)])):
        assert (planes[0].stride(0) == nplanes * planes[0][0].numel()) == (kind == "strided")
        hi, lo = tc.planar_to_ndhwc8_split(planes)
        counts[kind] = (mism(hi[..., :nplanes], rh) + mism(lo[..., :nplanes], rl) + int(hi[..., nplanes:].count_nonzero())
                        + int(lo[..., nplanes:].count_nonzero()))
    print("\n[planar_to_ndhwc8_split, %d planes, B = 2, full size] mismatches %s" % (nplanes, counts))
    assert all(n == 0 for n in counts.values()), counts


def _split_argmax(hi, lo, nd):
    """one-hot (.., nchild, C) of the first child with the largest hi + lo (fp32 add), and of the first with the largest hi"""
    ch, cl = _children(hi, nd).float(), _children(lo, nd).float()
    v = ch + cl
    one_hot = []
    for t in (v, ch):
        is_max = t == t.max(-2, keepdim=True).values
        one_hot.append(is_max & (is_max.cumsum(-2) == 1))
    return one_hot


@pytest.mark.parametrize("nd", [3, 2])
def test_pool_split_exact(vx, cuda, nd):
    """MaxPool(2) of (hi, lo) pairs at (1, 160, 192, 224, 16) (2-D: the 160 slices as the batch): the pooled pair is the
    pair of the first child with the largest hi + lo.  Many children tie on hi and differ in lo, some tie on both."""
    _, _, tc = vx
    g = torch.Generator(device=cuda).manual_seed(40 + nd)
    shape = (1,) + FULL + (16,) if nd == 3 else (FULL[0], 1) + FULL[1:] + (16,)
    hi, lo = ternary(shape, g), (ternary(shape, g).float() * LO).to(torch.bfloat16)
    yh, yl = tc.pool_split((hi, lo), nd)
    first, first_hi = _split_argmax(hi, lo, nd)
    rh = (_children(hi, nd).float() * first).sum(-2)
    rl = (_children(lo, nd).float() * first).sum(-2)
    differ = int((first != first_hi).any(-2).sum())
    v = _children(hi, nd).float() + _children(lo, nd).float()
    both = int(((v == v.max(-2, keepdim=True).values).sum(-2) > 1).sum())
    n = mism(yh, rh) + mism(yl, rl)
    print("\n[pool_split %d-D, full size] mismatches %d; pooled outputs whose hi argmax differs from the hi + lo one %d, "
          "with a tie on both %d" % (nd, n, differ, both))
    assert n == 0 and differ > 0 and both > 0


# ---- 3. the bf16x3 launches under the decomposition sweep ---------------------------------------------------------------

def _split_ops(kind, quantised, cuda):
    g = torch.Generator(device=cuda).manual_seed(200 + len(kind) + quantised)

    def act(s):
        return split_pair(s, g) if quantised else torch_split(torch.randn(s, generator=g, device=cuda))

    def wt(s):
        return split_weight(s, g)[0] if quantised else torch.randn(s, generator=g, device=cuda) * 0.05
    if kind == "concat_up":
        return dict(xa=act((2, 5, 11, 33, 32)), xb=act((2, 10, 22, 66, 16)), w=wt((32, 48, 3, 3, 3)), b=wt((32,)))
    assert kind == "blocked64"
    return dict(xa=act((2, 7, 13, 37, 64)), xb=None, w=wt((64, 64, 3, 3, 3)), b=wt((64,)))


def _split_launch(vx, kind, o):
    _, _, tc = vx
    cin, cout = o["w"].shape[1], o["w"].shape[0]
    if kind == "concat_up":
        assert tc.conv_blocks(32, 16, 32, 3) is None
        blocks = tc.one_block(cin, cout)
    else:
        blocks = tc.conv_blocks(64, 0, 64, 3)
        assert blocks is not None
    w_hi, w_lo = torch_split(o["w"])
    ph, pl = tc.pack_weights_blocks(w_hi.float(), False, blocks), tc.pack_weights_blocks(w_lo.float(), False, blocks)
    xb = o["xb"] or (None, None)
    return tc.conv_fwd_blocked(o["xa"][0], xb[0], blocks, ph, o["b"], cout, 3, up=kind == "concat_up", slope=SLOPE,
                               lo=(o["xa"][1], xb[1], pl))


def _split_reference(kind, o):
    w_hi, w_lo = (t.float() for t in torch_split(o["w"]))
    assert torch.equal(w_hi + w_lo, o["w"])
    up = kind == "concat_up"
    hs = [(o["xa"][0], up)] + ([(o["xb"][0], False)] if o["xb"] else [])
    ls = [(o["xa"][1], up)] + ([(o["xb"][1], False)] if o["xb"] else [])
    D = (o["xb"] or o["xa"])[0].shape[1]
    return split_epilogue(ref.conv(hs + ls + hs, torch.cat([w_hi, w_hi, w_lo], 1), D), o["b"], SLOPE)


@pytest.mark.parametrize("kind", ["concat_up", "blocked64"])
def test_split_decomposition_sweep(vx, cuda, monkeypatch, kind):
    """The split-precision forward (a single-launch concatenation 32^ + 16 -> 32 and a blocked 64 -> 64, ragged shapes,
    B = 2) with the persistent grid capped at 1, 2, 5 and 13 CTAs and uncapped.  Quantised operands: both outputs equal
    the fp64 reference at every cap.  Ordinary operands: both outputs are bit-identical across caps."""
    def run(o, cap):
        if cap is None:
            monkeypatch.delenv("VXM_B200_CONV_CTAS", raising=False)
        else:
            monkeypatch.setenv("VXM_B200_CONV_CTAS", cap)
        res = [t.clone() for t in _split_launch(vx, kind, o)]
        torch.cuda.synchronize()
        return res

    o = _split_ops(kind, True, cuda)
    refs = _split_reference(kind, o)
    counts = {cap: [mism(a, r) for a, r in zip(run(o, cap), refs)] for cap in CAPS}
    print("\n[split sweep %s, quantised] (hi, lo) mismatches by VXM_B200_CONV_CTAS: %s; margin %.2e"
          % (kind, counts, _split_margin(o["w"].shape[1], 2 ** 10 + 2 + 1, 2 ** 10 + 1)))
    assert all(n == 0 for c in counts.values() for n in c), counts
    o = _split_ops(kind, False, cuda)
    outs = {cap: run(o, cap) for cap in CAPS}
    for cap in CAPS:
        assert all(torch.equal(a, b) for a, b in zip(outs[cap], outs[None])), cap


# ---- 4. the bf16x3 backward routes each pool gradient to the child the forward chose -----------------------------------

def _expected_unpool(e_hi, e_lo, g_skip, g_pool, nd, slope):
    """unpool_combine after a split-precision pool: the skip gradient at every child plus the pool gradient at the first
    child with the largest hi + lo, times the LeakyReLU derivative (e_hi < 0), in fp32, rounded to bf16.  Also returns the
    number of pooled outputs whose hi argmax differs from that child."""
    first, first_hi = _split_argmax(e_hi, e_lo, nd)
    r = first.float() * g_pool.float().unsqueeze(-2)
    if g_skip is not None:
        r = r + _children(g_skip, nd).float()
    r = torch.where(_children(e_hi, nd) < 0, r * torch.tensor(slope, dtype=torch.float32, device=r.device), r)
    return _unchildren(r, nd).to(torch.bfloat16), int((first != first_hi).any(-2).sum())


def _record_pools(monkeypatch, eng, tc):
    """wraps the engine's split pool and its backward's unpool_combine; returns the list of records
    [(e_hi, e_lo, g_skip, g_pool, nd, slope, out)] filled as the backward runs"""
    lows, calls = {}, []
    pool_split, unpool = tc.pool_split, eng._unpool_combine

    def pool_rec(x, nd):
        lows[x[0].data_ptr()] = x
        return pool_split(x, nd)

    def unpool_rec(e_fine, g_skip, g_pool, nd, slope, *rest):
        out = unpool(e_fine, g_skip, g_pool, nd, slope, *rest)
        hi, lo = lows[e_fine.data_ptr()]
        assert hi is e_fine
        calls.append((hi, lo, g_skip, g_pool, nd, slope, out))
        return out
    monkeypatch.setattr(tc, "pool_split", pool_rec)
    monkeypatch.setattr(eng, "_unpool_combine", unpool_rec)
    return calls


def _check_routing(title, calls):
    rows, total = [], 0
    for i, (hi, lo, gs, gp, nd, slope, out) in enumerate(calls):
        exp, differ = _expected_unpool(hi, lo, gs, gp, nd, slope)
        n = mism(out, exp)
        rows.append((n, differ))
        total += differ
        print("  unpool %d %-22s mismatches %9d   pooled outputs with hi argmax != (hi + lo) argmax %9d"
              % (i, "x".join(map(str, hi.shape[1:])), n, differ))
    print("[%s] %d pooled outputs in all with a hi argmax that differs from the hi + lo one" % (title, total))
    return rows


def test_split_pool_routing_deterministic(vx, cuda, monkeypatch):
    """A first layer that copies image plane 0 (centre tap 1, every other weight and the bias 0) on images 1 + ~2^-10
    noise: every child of the first pool has hi = 1 and lo alone decides which child the forward takes.  The backward
    must send each pooled gradient to that child.  A 3-D model (8 children), then a 2-D one with B = 2 (4 children)."""
    vxm, eng, tc = vx
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "bf16x3")
    for shape, B, seed in (((32, 48, 64), 1, 50), ((96, 128), 2, 54)):
        nd = len(shape)
        g = torch.Generator(device=cuda).manual_seed(seed)
        torch.manual_seed(seed + 3)
        model = vxm.networks.VxmDense(inshape=shape).to(cuda)
        conv0 = model.unet_model.encoder[0][0].main
        with torch.no_grad():
            conv0.weight.zero_()
            conv0.bias.zero_()
            conv0.weight[(slice(None), 0) + (1,) * nd] = 1.0
        src = 1 + (torch.rand((B, 1) + shape, generator=g, device=cuda) - 0.5) * 2.0 ** -9
        trg = torch.rand((B, 1) + shape, generator=g, device=cuda)
        with monkeypatch.context() as m:
            calls = _record_pools(m, eng, tc)
            _, flow = model(src, trg)
            (flow * torch.randn(flow.shape, generator=g, device=cuda)).sum().backward()
            torch.cuda.synchronize()
        hi0 = calls[-1][0]                       # the backward runs the first pool last
        assert bool((hi0 == 1).all()) and all(c[4] == nd for c in calls)
        rows = _check_routing("routing, %d-D first layer copies 1 + noise, B = %d" % (nd, B), calls)
        assert rows[-1][1] > 0
        assert all(n == 0 for n, _ in rows), rows


def test_split_pool_routing_full_size_step(vx, cuda, monkeypatch):
    """A bf16x3 training step of the default model at 160x192x224 on smooth images: every unpool_combine output equals
    the emulation that routes the pool gradient to the forward's (hi + lo) argmax.  Prints how many pooled outputs have a
    hi argmax that differs from it."""
    vxm, eng, tc = vx
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "bf16x3")
    g = torch.Generator(device=cuda).manual_seed(51)

    def smooth():
        x = F.interpolate(torch.randn((1, 1, 10, 12, 14), generator=g, device=cuda), size=FULL, mode="trilinear", align_corners=False)
        return (x - x.min()) / (x.max() - x.min())
    src, trg = smooth(), smooth()
    torch.manual_seed(52)
    model = vxm.networks.VxmDense(inshape=FULL).to(cuda)
    calls = _record_pools(monkeypatch, eng, tc)
    y, flow = model(src, trg)
    loss = vxm.losses.NCC().loss(trg, y) + 0.01 * vxm.losses.Grad("l2", loss_mult=2).loss(None, flow)
    loss.backward()
    torch.cuda.synchronize()
    assert len(calls) == 4
    rows = _check_routing("routing, full-size bf16x3 step", calls)
    assert all(n == 0 for n, _ in rows), rows


# ---- 5. the fp32 engine, exactly, at the step's sizes ---------------------------------------------------------------------

# models VXM_B200_CONV_ENGINE=tc runs on f32: feature counts the tensor cores lack, more than 8 image planes
F32_MODELS = {"ragged": dict(inshape=(96, 112, 128), nb_unet_features=[[16, 24, 24, 24], [24, 24, 24, 24, 24, 12, 12]]),
              "planes9": dict(inshape=(64, 96, 112), src_feats=5, trg_feats=4)}


def _model_convs(name):
    """Every convolution of the model MODELS[name] or F32_MODELS[name] in execution order, from the model's own modules:
    (label, cin, cout, (D, H, W) it runs at (D = 1 in 2-D), B, activation, model name).  Encoder level i runs at
    inshape / 2^i, decoder level j at inshape / 2^(levels - 1 - j) (its convolutions precede the upsampling), the
    remaining convolutions and the flow head at full size (half size in a half-resolution U-Net, which skips the last
    upsampling)."""
    import voxelmorph_b200 as vxm
    kw, B = (MODELS[name].kw, MODELS[name].B) if name in MODELS else (F32_MODELS[name], 1)
    inshape = tuple(kw["inshape"])
    model = vxm.networks.VxmDense(**kw)
    unet = model.unet_model
    top = 1 if unet.half_res else 0
    levels = [(i, convs) for i, convs in enumerate(unet.encoder)] + \
             [(unet.nb_levels - 1 - j, convs) for j, convs in enumerate(unet.decoder)] + [(top, unet.remaining)]
    out = []
    for level, convs in levels:
        for blk in convs:
            out.append((level, blk.main, True))
    out.append((top, model.flow, False))
    return [("%s %02d %d->%d %s" % (name, i, m.in_channels, m.out_channels, "x".join(str(v >> level) for v in inshape)),
             m.in_channels, m.out_channels, (1,) * (3 - len(inshape)) + tuple(v >> level for v in inshape), B, act, name)
            for i, (level, m, act) in enumerate(out)]


# (cin, cout, shape (D, H, W; D = 1 for 2-D), B, activation): channel counts that end the kernels' blocks early.  Forward
# output blocks COB 8 / 16 / 32 by cout (dgrad: by cin), input stages CCK 4; weight gradient blocks WCO 16 x WCI 8.
# H and W are not multiples of the 32 x 16 (forward) and 32 x 8 (weight gradient) tiles.
RAGGED = [
    (1, 8, (11, 37, 45), 3, True),        # CCK stage of 1; dgrad: COB 8 of 1; WCI of 1; WCO cut at 8
    (3, 12, (1, 75, 101), 1, True),       # 2-D; partial COB 16, CCK stage of 3; dgrad: COB 8 of 3
    (5, 40, (13, 29, 70), 1, True),       # second COB 32 block of 8; WCI of 5; WCO: 16 + 16 + 8
    (9, 48, (1, 150, 203), 3, True),      # 2-D; second COB 32 block of 16; CCK 4 + 4 + 1; WCI 8 + 1; dgrad: COB 16 of 9
    (24, 2, (9, 45, 77), 3, True),        # COB 8 of 2; dgrad: COB 32 of 24, CCK stage of 2; WCO cut at 2
    (40, 24, (1, 83, 99), 1, True),       # 2-D; COB 32 of 24; dgrad: second COB 32 block of 8; WCO 16 + 8
    (24, 48, (7, 21, 53), 1, True),       # dgrad: COB 32 of 24; WCI 8 x 3; WCO 16 x 3
    (40, 12, (1, 61, 133), 3, True),      # 2-D; partial COB 16; dgrad: second COB 32 block of 8; WCI 8 x 5
    (9, 24, (5, 39, 66), 3, True),        # WCI 8 + 1, WCO 16 + 8; dgrad: COB 16 of 9 over a CCK of 24
    (5, 2, (1, 37, 45), 3, True),         # 2-D; COB 8 of 2, CCK stage of 1 after a full one; dgrad: COB 8 of 5
    (16, 2, (1, 192, 224), 3, False),     # the 2-D flow head
]


# ConditionalTemplateCreation's generator convolutions (extra_convs F -> F, atlas_gen F -> atlas_feats, no activation, at
# full resolution): (inshape, B, conv_nb_features F, atlas_feats).  F = 32 is the default, F = 4 the setting of
# tools/cond_template_step.py
COND_GEN = [((160, 192, 224), 1, 32, 1), ((160, 192, 224), 1, 4, 1), ((192, 224), 8, 32, 2)]


def _cond_gen_convs():
    """the generator convolutions, read off a ConditionalTemplateCreation's own modules (built at a small size of the same
    dimensionality: channel counts do not depend on it, and the phenotype decoder holds prod(inshape) F weights per
    attribute).  The extra convolutions are identical, so the first one stands for all of them."""
    import voxelmorph_b200 as vxm
    out = []
    for inshape, B, F, af in COND_GEN:
        m = vxm.networks.ConditionalTemplateCreation((16,) * len(inshape), (1,), conv_nb_features=F, atlas_feats=af)
        assert len({(c.in_channels, c.out_channels) for c in m.extra_convs}) == 1
        shape = (1,) * (3 - len(inshape)) + tuple(inshape)
        for what, c in (("extra_convs", m.extra_convs[0]), ("atlas_gen", m.atlas_gen)):
            out.append(("cond F=%d %s %d->%d %s B=%d" % (F, what, c.in_channels, c.out_channels, "x".join(map(str, inshape)), B),
                        c.in_channels, c.out_channels, shape, B, False, None))
    return out


def _f32_cases():
    # (label, cin, cout, shape (D, H, W; D = 1 with kd = 1 for 2-D), B, activation, model or None)
    return (_model_convs("default") + _model_convs("doubled") + [("2-D 32->16 B=2", 32, 16, (1, 192, 224), 2, True, None)]
            + _model_convs("2d_halfres") + _model_convs("ragged") + _model_convs("planes9") + _cond_gen_convs()
            + [("%s %d->%d %s B=%d" % ("2-D" if D == 1 else "3-D", cin, cout, "x".join(map(str, (D, H, W) if D > 1 else (H, W))), B),
                cin, cout, (D, H, W), B, act, None) for cin, cout, (D, H, W), B, act in RAGGED])


@pytest.mark.parametrize("case", _f32_cases(), ids=lambda c: c[0].replace(" ", "_"))
def test_f32_conv_exact(vx, cuda, monkeypatch, case):
    """vxm_conv3d_fwd_f32 / vxm_conv3d_bwd_f32 through the C ABI: forward (bias, LeakyReLU), dgrad with the LeakyReLU
    mask of a saved activation, weight and bias gradients accumulated onto integer-valued priors (split_reduce_kernel
    adds its 2 * SM split-K partials with +=), all equal to fp64.  Operands: x in {-1, 0, 1} (first layer: / 16),
    weights and bias 2^-6 k with |k| <= 8, output gradient in {-1, 0, 1} with nonzeros at probability 1/8 (at 1/2 the
    full-size bias gradient's partial sums would reach a third of 2^24 units)."""
    vxm, _, _ = vx
    lib = vxm._lib.load()
    name, cin, cout, shape, B, act, model = case
    if model in F32_MODELS:
        monkeypatch.setenv("VXM_B200_CONV_ENGINE", "tc")
        assert vxm.ops.resolve_engine(vxm.networks.VxmDense(**F32_MODELS[model])) == "f32"
    D, H, W = shape
    kd = 1 if D == 1 else 3
    first = cin <= 8
    slope = SLOPE_F32 if act else -1.0
    g = torch.Generator(device=cuda).manual_seed(300 + cin + cout + D)
    xunit = 2.0 ** -4 if first else 1.0
    x = sparse_ternary((B, cin, D, H, W), g) * xunit
    w = torch.randint(-8, 9, (cout, cin, kd, 3, 3), generator=g, device=cuda).float() * 2.0 ** -6
    b = torch.randint(-8, 9, (cout,), generator=g, device=cuda).float() * 2.0 ** -6
    y = torch.empty((B, cout, D, H, W), device=cuda)
    P = vxm._lib.ptr
    st = vxm._lib.stream_ptr()
    vxm._lib.check(lib.vxm_conv3d_fwd_f32(P(x), P(w), P(b), P(y), B, cin, cout, D, H, W, kd, ctypes.c_float(slope), st), "fwd")
    gy = sparse_ternary((B, cout, D, H, W), g, den=8)
    mask = sparse_ternary((B, cout, D, H, W), g)          # the saved activation: only its sign is read
    prior_w = torch.randint(-4, 5, w.shape, generator=g, device=cuda).float()
    prior_b = torch.randint(-4, 5, b.shape, generator=g, device=cuda).float()
    gx, gw, gb = torch.empty_like(x), prior_w.clone(), prior_b.clone()
    work = torch.empty(int(lib.vxm_conv3d_bwd_workspace_bytes(B, cin, cout, D, H, W, kd)), dtype=torch.uint8, device=cuda)
    vxm._lib.check(lib.vxm_conv3d_bwd_f32(P(gy), P(mask) if act else None, P(x), P(w), P(gx), P(gw), P(gb), P(work), B, cin, cout,
                                          D, H, W, kd, ctypes.c_float(slope), st), "bwd")
    torch.cuda.synchronize()

    def cl(t):                # (B, C, D, H, W) -> channels-last view
        return t.permute(0, 2, 3, 4, 1)
    gm = cl(torch.where(mask < 0, gy * SLOPE_F32, gy) if act else gy)
    rows = []
    n = sum(ref.conv([(cl(x), False)], w, D, finish=lambda r, d0, d1: mism(cl(y)[:, d0:d1], ref.epilogue(
        r, b, SLOPE_F32 if act else None, bf16=False))))
    rows.append((name, "fwd", n, (27 * cin * 8 + 8 / xunit) / 2 ** 24))               # units of 2^-6 * xunit
    n = sum(ref.conv([(gm, False)], ref.dgrad_weight(w), D, finish=lambda r, d0, d1: mism(cl(gx)[:, d0:d1], r.float())))
    rows.append((name, "dgrad" + (" masked" if act else ""), n, 27 * cout * 32 / 2 ** 24))  # |g| <= 4, |w| <= 8 units of 2^-8
    rw, rb = ref.wgrad([(cl(x), False)], gm, kd)
    aw, ab = ref.wgrad([(cl(x), False)], gm, kd, absolute=True)
    gunit = SLOPE_F32 if act else 1.0
    rows.append((name, "wgrad accumulated", mism(gw, prior_w + rw.float()),
                 (float(aw.max()) + 4) / (xunit * gunit) / 2 ** 24))
    rows.append((name, "bias grad accumulated", mism(gb, prior_b + rb.float()), (float(ab.max()) + 4) / gunit / 2 ** 24))
    _report("f32 exact %s" % name, rows)


def test_f32_pool_upcat_exact(vx, cuda):
    """maxpool2 (forward and backward: the gradient to the first maximal child) and upsample2_cat (forward and backward)
    of unet_ops.cu against torch at full resolution, with ternary inputs so that ties are frequent: 3-D (1, C, 160, 192,
    224) and 2-D (8, C, 192, 224), the f32 engine's planar layout."""
    vxm, _, _ = vx
    from voxelmorph_b200 import ops
    for nd, B, fine, seed in ((3, 1, FULL, 60), (2, 8, FULL[1:], 61)):
        g = torch.Generator(device=cuda).manual_seed(seed)
        coarse = tuple(v // 2 for v in fine)

        def cl(t):            # (B, C, [D,] H, W) -> channels-last (B, D, H, W, C), D = 1 in 2-D
            return t.permute(0, 2, 3, 4, 1) if nd == 3 else t.permute(0, 2, 3, 1)[:, None]

        def planar(t):        # the inverse of cl
            return t.permute(0, 4, 1, 2, 3) if nd == 3 else t[:, 0].permute(0, 3, 1, 2)
        x = ternary((B, 16) + fine, g, torch.float32).requires_grad_(True)
        y = ops.maxpool2(x)
        gy = ternary(y.shape, g, torch.float32)
        y.backward(gy)
        ch = _children(cl(x.detach()), nd)
        is_max = ch == ch.max(4, keepdim=True).values
        first = is_max & (is_max.cumsum(4) == 1)
        assert bool((is_max.sum(4) > 1).any())
        n_pool = mism(y.detach(), (F.max_pool3d if nd == 3 else F.max_pool2d)(x.detach(), 2))
        n_pool_bwd = mism(x.grad, planar(_unchildren(first.float() * cl(gy).unsqueeze(4), nd)))
        a = ternary((B, 32) + coarse, g, torch.float32).requires_grad_(True)
        skip = ternary((B, 16) + fine, g, torch.float32).requires_grad_(True)
        out = ops.upsample2_cat(a, skip)
        go = ternary(out.shape, g, torch.float32)
        out.backward(go)
        up = planar(ref.upsample2(cl(a.detach()), nd))
        n_up = mism(out.detach(), torch.cat([up, skip.detach()], 1))
        n_up_bwd = mism(a.grad, planar(ref.children_sum(cl(go[:, :32]).double(), nd).float())) + mism(skip.grad, go[:, 32:])
        print("\n[f32 glue, full size, %d-D, B = %d] maxpool2 %d | its backward %d | upsample2_cat %d | its backward %d mismatches"
              % (nd, B, n_pool, n_pool_bwd, n_up, n_up_bwd))
        assert n_pool == n_pool_bwd == n_up == n_up_bwd == 0
