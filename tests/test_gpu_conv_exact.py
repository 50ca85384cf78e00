"""Every tensor-core convolution launch of the training step, checked exactly at the step's own size for a matrix of U-Nets
(3-D and 2-D, half-resolution, two convolutions per level, all-16-feature, 3 image planes, B > 1), and the persistent
kernels' item loops checked under every decomposition a GPU with 1, 2, 5 or 13 SMs would run (VXM_B200_CONV_CTAS).

Operands are chosen so that every fp32 sum the kernels form is exact, whatever the MMA or reduction order: activations
and gradients in {-1, 0, 1} (each nonzero with probability 1/2), weights and biases 2^-6 k with |k| <= 8 (merged polyphase
taps |k| <= 32, still bf16-exact), image and flow-gradient planes in {-1, 0, 1} / 16.  Every product and partial sum is
then an integer multiple of one power of two below 2^24 of those units; the test asserts the bounds (printed as the
margin: the bound over 2^24) rather than assuming them.  The kernels' results must equal the fp64 tap sums of
conv_exact_ref.py, with the epilogue (bias add, LeakyReLU or its derivative with the model's slope 0.2, bf16 rounding)
emulated in fp32: any dropped, doubled or misplaced contribution fails.  Run with -s to print every launch's mismatch
count next to its margin."""
import collections

import pytest
import torch

import conv_exact_ref as ref

pytestmark = pytest.mark.gpu

SLOPE = 0.2                      # the model's LeakyReLU slope: its fp32 products round, as in the step
PLANE = 2.0 ** -4                # image and flow-gradient planes: {-1, 0, 1} * PLANE
DOUBLED = [[32, 64, 64, 64], [64, 64, 64, 64, 64, 32, 32]]
F16 = [[16, 16, 16, 16], [16, 16, 16, 16, 16, 16, 16]]
CAPS = ["1", "2", "5", "13", None]


@pytest.fixture(scope="module")
def vx(cuda):
    import voxelmorph_b200 as vxm
    from voxelmorph_b200 import engine_bf16, tc
    vxm._lib.load()
    return vxm, engine_bf16, tc


def ternary(shape, g, dtype=torch.bfloat16):
    """{-1, 0, 1}, each nonzero with probability 1/2"""
    nz = torch.randint(0, 2, shape, generator=g, device=g.device)
    return (nz * (2 * torch.randint(0, 2, shape, generator=g, device=g.device) - 1)).to(dtype)


def qweight(shape, g):
    return torch.randint(-8, 9, shape, generator=g, device=g.device).float() * 2.0 ** -6


def mism(a, b):
    assert a.shape == b.shape, (a.shape, b.shape)
    return int((a != b.to(a.dtype)).sum())


def _margin(cin, children=1):
    """bound on |partial sums| of a forward / dgrad over 2^24, in units of (operand unit) x 2^-6: 27 taps x cin channels x
    |x| <= 1 unit x |w| <= 8 units (merged taps partition the same terms), x 8 for a sum over upsampled children, plus a bias
    of <= 8 units of 2^-6 (128 units of the image planes' 2^-10)"""
    return (27 * cin * 8 * children + 128) / 2 ** 24


def _form_name(f, split=False):
    if f == "fold":
        return "kd-folded"
    if f[0] == "poly":
        return "polyphase %s" % ("forward" if f[1] == 1 else "coarse")
    kind = "one launch" if len(f[0]) == len(f[1]) == 1 else "%dx%d blocks" % (len(f[0]), len(f[1]))
    return kind + (" split" if split else "")


def _report(title, rows):
    """rows (launch, form, mismatches, margin): every mismatch count must be 0 and every margin below 1/4"""
    print("\n[%s] launch | form | mismatches (expected 0) | margin" % title)
    for name, form, n, margin in rows:
        print("  %-34s %-26s %8d   %.2e" % (name, form, n, margin))
    bad = [r for r in rows if r[2] or r[3] >= 0.25]
    assert not bad, bad


# ---- a. every convolution of the plan, exactly, at the plan's own size -------------------------------------------------

# kw: the VxmDense arguments (every size divisible by 2^levels); B: the batch; tc: the engine VXM_B200_CONV_ENGINE=tc runs
# the model on; blocked: whether its bf16x3 plan has channel-blocked launches.  "doubled" (64 channels) runs on f32 under
# 'tc' and is checked here for VXM_B200_CONV_ENGINE=bf16 / bf16x3 set explicitly.
# probs: a VxmDenseProbabilistic, whose head is one 2 nd-output convolution (flow, then log_sigma); its U-Net layers are those of
# the VxmDense case of the same arguments, so only the head is checked
Case = collections.namedtuple("Case", "kw B tc blocked probs", defaults=(False,))
MODELS = {
    "default": Case(dict(inshape=(160, 192, 224)), 1, "bf16x3", False),
    "doubled": Case(dict(inshape=(64, 96, 112), nb_unet_features=DOUBLED), 1, "f32", True),
    "default_b2": Case(dict(inshape=(96, 128, 160)), 2, "bf16x3", False),
    "halfres": Case(dict(inshape=(160, 192, 224), unet_half_res=True), 1, "bf16x3", False),
    "ncpl2": Case(dict(inshape=(84, 100, 132), nb_unet_features=16, nb_unet_levels=3, nb_unet_conv_per_level=2), 1, "bf16x3", False),
    "feat16": Case(dict(inshape=(64, 96, 112), nb_unet_features=F16), 2, "bf16x3", False),
    "planes3": Case(dict(inshape=(64, 96, 112), src_feats=2, trg_feats=1), 1, "bf16x3", False),
    "2d": Case(dict(inshape=(192, 224)), 8, "bf16x3", False),
    "2d_doubled": Case(dict(inshape=(160, 192), nb_unet_features=DOUBLED), 2, "f32", True),
    "2d_halfres": Case(dict(inshape=(176, 240), unet_half_res=True), 3, "bf16x3", False),
    "probs": Case(dict(inshape=(160, 192, 224)), 1, "bf16x3", False, True),
    "probs_2d": Case(dict(inshape=(192, 224)), 8, "bf16x3", False, True),
    "probs_halfres": Case(dict(inshape=(160, 192, 224), unet_half_res=True), 2, "bf16x3", False, True),
}


def build_model(vxm, name):
    cls = vxm.networks.VxmDenseProbabilistic if MODELS[name].probs else vxm.networks.VxmDense
    return cls(**MODELS[name].kw)


def plan_sizes(eng, plan, inshape):
    """(D, H, W) and channels of every tensor id of the plan: 0 = the images (D = 1 in 2-D), a pool halves d (3-D only), h
    and w, a convolution after an upsample works at its skip's (twice its source's) size"""
    size, chans = {0: tuple(inshape) if plan.nd == 3 else (1,) + tuple(inshape)}, {}
    for op in plan.ops:
        if isinstance(op, eng._Layer):
            size[op.out], chans[op.out] = size[op.b if op.b is not None else op.a], op.cout
        else:
            _, s, d = op
            D, H, W = size[s]
            size[d], chans[d] = (D // 2 if plan.nd == 3 else D, H // 2, W // 2), chans[s]
    return size, chans


def check_resolves(vxm, monkeypatch, name, model):
    """the engine `import voxelmorph` ('tc') runs the model on is the one the case states"""
    monkeypatch.setenv("VXM_B200_CONV_ENGINE", "tc")
    assert vxm.ops.resolve_engine(model) == MODELS[name].tc
    monkeypatch.delenv("VXM_B200_CONV_ENGINE")


def quantise(model, g):
    with torch.no_grad():
        for p in model.parameters():
            p.copy_(qweight(p.shape, g))


def tape_operands(eng, tc, plan, inshape, B, g):
    """The exact tier's operands of a plan: image planes (B, 1, D, H, W) and their channels-last cat, the ternary bf16
    tensor X[i] of every tensor id but the flow's (X[0]: the images as the first convolution reads them), the ternary
    output gradient G of every convolution but the head, and the head's gradient planes with their channels-last cat"""
    size, chans = plan_sizes(eng, plan, inshape)
    first, flow = plan.layers[0], plan.layers[-1]
    planes = [ternary((B, 1) + size[0], g, torch.float32) * PLANE for _ in range(first.cin)]
    images = torch.cat(planes, 1).permute(0, 2, 3, 4, 1)
    X = {i: ternary((B,) + size[i] + (c,), g) for i, c in chans.items() if i != flow.out}
    X[0] = tc.planar_fold_kd(planes, 8) if first.fwd == "fold" else tc.planar_to_ndhwc8(planes)
    G = {L.out: ternary((B,) + size[L.out] + (L.cout,), g) for L in plan.layers if L is not flow}
    gplanes = [ternary((B, 1) + size[flow.out], g, torch.float32) * PLANE for _ in range(flow.cout)]
    gflow = torch.cat(gplanes, 1).permute(0, 2, 3, 4, 1)
    return size, planes, images, X, G, gplanes, gflow


def check_head_plan(model, plan):
    """the plan facts of a probabilistic model's head: one 2 nd-output convolution that is never kd-folded, derived from
    four parameters, whose persistent operands are cat(flow, log_sigma) bit for bit"""
    flow = plan.layers[-1]
    assert flow.role == "flow" and flow.cout == 2 * plan.nd and flow.dgrad != "fold"
    assert len(flow.srcs) == 4 and flow.srcs[0] is model.flow.weight and flow.srcs[3] is model.log_sigma.bias
    assert torch.equal(flow.w, torch.cat([model.flow.weight.detach(), model.log_sigma.weight.detach()]))
    assert torch.equal(flow.bias, torch.cat([model.flow.bias.detach(), model.log_sigma.bias.detach()]))


# "split+unfolded" changes a form only in 3-D (polyphase and kd folding are 3-D forms); a probabilistic head runs the same
# form in both settings, and its U-Net layers are checked by the VxmDense cases
@pytest.mark.parametrize("name,forms", [(n, f) for n in sorted(MODELS) for f in ("polyphase+kdfold", "split+unfolded")
                                        if f == "polyphase+kdfold" or (len(MODELS[n].kw["inshape"]) == 3 and not MODELS[n].probs)])
def test_plan_launches_exact(vx, cuda, monkeypatch, name, forms):
    """Forward, dgrad and weight gradient of every layer of the plan through the engine's own calls (_run, WgradBatch), with
    the arguments forward_tape / backward_tape pass.  "split+unfolded" (VXM_B200_POLYPHASE=0, VXM_B200_KDFOLD=0) runs the
    layers whose form that changes.  A probabilistic model: its 2 nd-output head only."""
    vxm, eng, tc = vx
    kw, B = MODELS[name].kw, MODELS[name].B
    g = torch.Generator(device=cuda).manual_seed(1 + len(name))
    model = build_model(vxm, name).to(cuda)
    quantise(model, g)
    check_resolves(vxm, monkeypatch, name, model)
    monkeypatch.setenv("VXM_B200_POLYPHASE", "1")
    monkeypatch.setenv("VXM_B200_KDFOLD", "1")
    base = [L for L in eng._walk(model) if isinstance(L, eng._Layer)]
    if forms == "split+unfolded":
        monkeypatch.setenv("VXM_B200_POLYPHASE", "0")
        monkeypatch.setenv("VXM_B200_KDFOLD", "0")
    plan = eng._plan_of(model, False)
    layers = plan.layers
    nd, kd = plan.nd, (3 if plan.nd == 3 else 1)
    if MODELS[name].probs:
        check_head_plan(model, plan)
        only = {len(layers) - 1}
    else:
        only = {i for i, (L, L0) in enumerate(zip(layers, base)) if forms == "polyphase+kdfold" or L.fwd != L0.fwd or L.dgrad != L0.dgrad}
    assert only
    if forms == "polyphase+kdfold":
        assert (layers[0].fwd == "fold") == (nd == 3 and layers[0].cin == 2)
        if name == "default":
            assert sum(1 for L in layers if L.dgrad_skip is not None) == 4 and layers[-1].dgrad == "fold"
    first, flow = layers[0], layers[-1]
    size, planes, images, X, G, gplanes, gflow = tape_operands(eng, tc, plan, kw["inshape"], B, g)
    for L in layers:
        assert bool(((L.w * 64).abs() <= 8).all()) and bool(((L.bias * 64).abs() <= 8).all())

    def srcs(L):
        return [(images, False)] if L is first else [(X[L.a], L.up)] + ([(X[L.b], False)] if L.b is not None else [])

    def coarse(t, d0, d1):
        """the slices of an upsampled source under fine output slices d0 .. d1 - 1"""
        return t[:, d0 // 2:d1 // 2] if nd == 3 else t[:, d0:d1]

    def lname(i, L):
        return "%02d %s (%d%s+%d)->%d %s" % (i, L.role, L.ca, "^" if L.up else "", L.cb, L.cout, "x".join(map(str, size[L.out])))

    rows = []
    for i, L in enumerate(layers):
        if i not in only:
            continue
        w, bias, D = L.w.detach().view(L.cout, L.cin, kd, 3, 3), L.bias.detach(), size[L.out][0]
        # ---- forward ----
        out = eng._run(L.fwd, L.pk_fwd, X[0] if L is first else X[L.a], X.get(L.b), L.cout, kd, bias, up=L.up, slope=L.slope,
                       out_fp32_planar=L is flow)
        if L is flow:
            out = out.permute(0, 2, 3, 4, 1)
        n = sum(ref.conv(srcs(L), w, D, nd=nd, finish=lambda y, d0, d1: mism(out[:, d0:d1], ref.epilogue(y, bias, L.slope, bf16=L is not flow))))
        rows.append((lname(i, L), "fwd " + _form_name(L.fwd), n, _margin(L.cin)))
        # ---- dgrad, in the plan's form ----
        if L.dgrad is None:
            continue
        wt = ref.dgrad_weight(w)
        if L is flow:
            g_in = tc.planar_fold_kd(gplanes, 16) if L.dgrad == "fold" else tc.planar_to_ndhwc8(gplanes)
            sl, mask = plan.slope[L.a], X[L.a]
            res = eng._run(L.dgrad, L.pk_dgrad, g_in, None, L.cin, kd, slope=sl, mask=mask)
            n = sum(ref.conv([(gflow, False)], wt, D, finish=lambda y, d0, d1: mism(res[:, d0:d1], ref.epilogue(y, slope=sl, mask=mask[:, d0:d1]))))
            rows.append((lname(i, L), "dgrad " + _form_name(L.dgrad), n, _margin(L.cout)))
        elif L.b is None:
            sl = plan.slope.get(L.a)        # None: a pooling output, no activation to differentiate
            mask = None if sl is None else X[L.a]
            res = eng._run(L.dgrad, L.pk_dgrad, G[L.out], None, L.cin, kd, slope=sl, mask=mask)
            n = sum(ref.conv([(G[L.out], False)], wt, D, finish=lambda y, d0, d1: mism(
                res[:, d0:d1], ref.epilogue(y, slope=sl, mask=None if mask is None else mask[:, d0:d1]))))
            rows.append((lname(i, L), "dgrad " + _form_name(L.dgrad) + (" masked" if mask is not None else ""), n, _margin(L.cout)))
        elif L.dgrad_skip is not None:
            sl, act = plan.slope[L.a], X[L.a]
            coarse = eng._run(L.dgrad, L.pk_dgrad, G[L.out], None, L.ca, 3, mask=act, slope=sl)
            skip = eng._run(L.dgrad_skip, L.pk_dgrad_skip, G[L.out], None, L.cb, 3)
            ns = ref.conv([(G[L.out], False)], wt, D, finish=lambda y, d0, d1: (
                mism(coarse[:, d0 // 2:d1 // 2], ref.epilogue(ref.children_sum(y[..., :L.ca]), slope=sl, mask=act[:, d0 // 2:d1 // 2])),
                mism(skip[:, d0:d1], ref.epilogue(y[..., L.ca:]))))
            rows.append((lname(i, L), "dgrad " + _form_name(L.dgrad), sum(a for a, _ in ns), _margin(L.cout, 8)))
            rows.append((lname(i, L), "dgrad skip " + _form_name(L.dgrad_skip), sum(b for _, b in ns), _margin(L.cout)))
        else:
            sl, act = plan.slope[L.a], X[L.a]
            g_up, g_sk = eng._run(L.dgrad, L.pk_dgrad, G[L.out], None, L.cin, kd, split=L.ca)
            gzc = eng._sumpool_mask(g_up, act, nd, sl)

            def fin(y, d0, d1):
                up = ref.epilogue(y[..., :L.ca])
                return (mism(g_up[:, d0:d1], up), mism(g_sk[:, d0:d1], ref.epilogue(y[..., L.ca:])),
                        mism(coarse(gzc, d0, d1), ref.epilogue(ref.children_sum(up.double(), nd), slope=sl, mask=coarse(act, d0, d1))))
            ns = ref.conv([(G[L.out], False)], wt, D, finish=fin)
            rows.append((lname(i, L), "dgrad " + _form_name(L.dgrad, True), sum(a + b for a, b, _ in ns), _margin(L.cout)))
            rows.append((lname(i, L), "sumpool_mask", sum(c for _, _, c in ns), _margin(L.cout, 2 ** nd)))
        del out
    # ---- weight gradients: every layer into one WgradBatch in backward_tape's order, one flush; fresh, then accumulated ----
    refs = {}
    for i, L in enumerate(layers):
        if i in only:
            gz = gflow if L is flow else G[L.out]
            wunit, bunit = (PLANE if L is first or L is flow else 1.0), (PLANE if L is flow else 1.0)    # x * gz, gz
            gw, gb = ref.wgrad(srcs(L), gz, kd, nd=nd)
            aw, ab = ref.wgrad(srcs(L), gz, kd, absolute=True, nd=nd)
            margin = max(float(aw.max()) / wunit, float(ab.max()) / bunit / 2) / 2 ** 24    # weights < 2^22, biases < 2^23 units
            refs[i] = (gw.float().view(L.w.shape), gb.float(), margin)
    for accumulate in (False, True):
        batch = tc.WgradBatch.get(cuda)
        batch.reset()
        got = []
        for i, L in reversed(list(enumerate(layers))):
            if i not in only:
                continue
            if L is flow and L.dgrad == "fold":
                gwf = torch.empty((9, L.cin, 1, 3, 3), device=cuda)
                gbf = torch.empty(9, device=cuda)
                batch.add_khm(X[L.a], tc.planar_fold_kd(gplanes, 16), gwf, gbf, L.cin, 9)
                got.append((i, "wgrad kd-folded (kh in M)", lambda gwf=gwf, gbf=gbf, L=L: eng.unfold_grad_flow(gwf, gbf, 3, L.cin), None))
            elif L is first and L.fwd == "fold":
                gwf = torch.empty((L.cout, 3 * L.cin, 1, 3, 3), device=cuda)
                gbf = torch.empty(L.cout, device=cuda)
                if L.khm:
                    batch.add_khm(X[0], G[L.out], gwf, gbf, 3 * L.cin, L.cout)
                else:
                    batch.add(X[0], None, G[L.out], gwf, gbf, 3 * L.cin, L.cout, 1, False, False)
                got.append((i, "wgrad kd-folded" + (" (kh in M)" if L.khm else ""),
                            lambda gwf=gwf, gbf=gbf, L=L: (eng.unfold_grad_first(gwf, L.cout, L.cin), gbf), None))
            else:
                g_in = tc.planar_to_ndhwc8(gplanes) if L is flow else G[L.out]
                xa = X[0] if L is first else X[L.a]
                prior = None
                if accumulate:         # the flat-gradient path: integer-valued prior content
                    prior = (torch.randint(-4, 5, L.w.shape, generator=g, device=cuda).float(),
                             torch.randint(-4, 5, L.bias.shape, generator=g, device=cuda).float())
                    gw, gb = tc.conv_wgrad(xa, X.get(L.b), g_in, L.cin, L.cout, kd, up=L.up, out_w=prior[0].clone(),
                                           out_b=prior[1].clone(), batch=batch)
                else:
                    gw, gb = tc.conv_wgrad(xa, X.get(L.b), g_in, L.cin, L.cout, kd, up=L.up, batch=batch)
                got.append((i, "wgrad" + (" accumulated" if accumulate else ""), lambda gw=gw, gb=gb: (gw, gb), prior))
        batch.flush()
        for i, form, res, prior in got:
            gw, gb = res()
            rw, rb, margin = refs[i]
            if prior is not None:
                rw, rb = prior[0] + rw, prior[1] + rb
            rows.append((lname(i, layers[i]), form, mism(gw.reshape(rw.shape), rw) + mism(gb, rb), margin))
    _report("exact %s %s" % (name, forms), rows)


@pytest.mark.parametrize("name", ["probs", "probs_2d"])
def test_head_split_exact(vx, cuda, monkeypatch, name):
    """backward_tape over the exact tier's operands and a quantised head gradient: the 2 nd-output head's weight and bias
    gradients reach flow.weight, flow.bias, log_sigma.weight and log_sigma.bias as the [:nd] / [nd:] slices of the fp64
    sums, through autograd's dict; with the parameters re-pointed into FlatParams, into the four .grad views on top of
    integer-valued priors, and autograd gets nothing for them."""
    vxm, eng, tc = vx
    kw, B = MODELS[name].kw, MODELS[name].B
    g = torch.Generator(device=cuda).manual_seed(70 + len(name))
    model = build_model(vxm, name).to(cuda)
    quantise(model, g)
    plan = eng._plan_of(model, False)
    check_head_plan(model, plan)
    nd, kd = plan.nd, (3 if plan.nd == 3 else 1)
    flow = plan.layers[-1]
    _, _, _, X, _, gplanes, gflow = tape_operands(eng, tc, plan, kw["inshape"], B, g)
    g_flow = torch.cat(gplanes, 1)
    if nd == 2:
        g_flow = g_flow.squeeze(2)         # as forward_tape returns a 2-D flow
    gw, gb = ref.wgrad([(X[flow.a], False)], gflow, kd, nd=nd)
    aw, ab = ref.wgrad([(X[flow.a], False)], gflow, kd, absolute=True, nd=nd)
    margin = max(float(aw.max()) / PLANE, float(ab.max()) / PLANE / 2) / 2 ** 24
    heads = [model.flow.weight, model.flow.bias, model.log_sigma.weight, model.log_sigma.bias]
    want = [gw[:nd].float(), gb[:nd].float(), gw[nd:].float(), gb[nd:].float()]
    want = [w.reshape(p.shape) for w, p in zip(want, heads)]
    rows = []
    grads = eng.backward_tape(dict(plan=plan, tensors=X, split=False, pool_lows={}), g_flow)
    for p, w, what in zip(heads, want, ("flow.weight", "flow.bias", "log_sigma.weight", "log_sigma.bias")):
        rows.append((what, "head split", mism(grads[p], w), margin))
    fp = vxm.optim.FlatParams(list(model.parameters()))
    fp.grad.copy_(torch.randint(-4, 5, (fp.numel,), generator=g, device=cuda).float())
    priors = [p.grad.clone() for p in heads]
    views = [p.grad for p in heads]
    grads = eng.backward_tape(dict(plan=plan, tensors=X, split=False, pool_lows={}), g_flow)
    assert not any(p in grads for p in heads)
    assert all(p.grad is v for p, v in zip(heads, views))
    for p, w, prior, what in zip(heads, want, priors, ("flow.weight", "flow.bias", "log_sigma.weight", "log_sigma.bias")):
        rows.append((what, "flat view accumulated", mism(p.grad, prior + w), margin))
    _report("head split %s" % name, rows)


# every model of the matrix, both engines; "default" with source.requires_grad, so that the image dgrad runs as well
FLAT_CASES = [(n, s) for n in sorted(MODELS) for s in (False, True)]


@pytest.mark.parametrize("name,split", FLAT_CASES, ids=["%s-%s" % (n, "bf16x3" if s else "bf16") for n, s in FLAT_CASES])
def test_flat_grads_equal_autograd(vx, cuda, name, split):
    """unet_flow on ordinary weights and images, backward with one fixed flow gradient (no VecInt or warp atomics), once
    with plain parameters (autograd) and once with FusedAdam's FlatParams views zeroed by zero_grad: every parameter's
    gradient bit-identical, written in place into the flat buffer (the kd-folded first layer and flow head through their
    unfolded views, the 2 nd-output head through its split, 2-D layers through the squeeze), and the image gradient
    unchanged."""
    vxm, eng, _ = vx
    kw, B = MODELS[name].kw, MODELS[name].B
    torch.manual_seed(90 + len(name))
    model = build_model(vxm, name).to(cuda)
    g = torch.Generator(device=cuda).manual_seed(91 + len(name))
    with torch.no_grad():
        for m in (model.flow, getattr(model, "log_sigma", None)):
            if m is not None:
                m.weight.copy_(torch.randn(m.weight.shape, generator=g, device=cuda) * 0.05)
    inshape = tuple(kw["inshape"])
    S = torch.rand((B, kw.get("src_feats", 1)) + inshape, generator=g, device=cuda)
    T = torch.rand((B, kw.get("trg_feats", 1)) + inshape, generator=g, device=cuda)
    image_grad = name == "default"
    params = list(model.parameters())
    gflow = []

    def run():
        src = S.clone().requires_grad_(image_grad)
        out = eng.unet_flow(model, src, T, split=split)
        if not gflow:
            gflow.append(torch.randn(out.shape, generator=g, device=cuda))
        out.backward(gflow[0])
        return out.detach(), [p.grad.clone() for p in params], src.grad

    f1, g1, s1 = run()
    assert all(bool(t.any()) for t in g1)
    fp = vxm.optim.FlatParams(params)
    fp.zero_grad()
    views = [p.grad for p in params]
    f2, g2, s2 = run()
    assert all(p.grad is v for p, v in zip(params, views))         # accumulated in place: autograd got nothing
    assert torch.equal(f1, f2)
    bad = [n for (n, _), a, b in zip(model.named_parameters(), g1, g2) if not torch.equal(a, b)]
    assert not bad, bad
    assert (s1 is None) == (not image_grad) and (s1 is None or torch.equal(s1, s2))


# ---- b. the glue kernels of the full-size backward ------------------------------------------------------------------

def _children(x, nd=3):
    """(B, D, H, W, C) -> (B, Dc, Hc, Wc, nchild, C): the 8 (3-D) or 4 (2-D, Dc = D) children of every coarse voxel, in the
    kernels' (kd, kh, kw) order"""
    B, D, H, W, C = x.shape
    if nd == 2:
        return x.reshape(B, D, H // 2, 2, W // 2, 2, C).permute(0, 1, 2, 4, 3, 5, 6).reshape(B, D, H // 2, W // 2, 4, C)
    return x.reshape(B, D // 2, 2, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4, 6, 7).reshape(B, D // 2, H // 2, W // 2, 8, C)


def _unchildren(c, nd=3):
    B, Dc, Hc, Wc, _, C = c.shape
    if nd == 2:
        return c.reshape(B, Dc, Hc, Wc, 2, 2, C).permute(0, 1, 2, 4, 3, 5, 6).reshape(B, Dc, 2 * Hc, 2 * Wc, C)
    return c.reshape(B, Dc, Hc, Wc, 2, 2, 2, C).permute(0, 1, 4, 2, 5, 3, 6, 7).reshape(B, 2 * Dc, 2 * Hc, 2 * Wc, C)


# the full-resolution activations of the default model: 3-D (B = 1), and 2-D (B = 8, held as (B, 1, H, W, C))
GLUE_SHAPES = {3: (1, 160, 192, 224), 2: (8, 1, 192, 224)}


@pytest.mark.parametrize("nd,with_skip", [(3, True), (3, False), (2, True), (2, False)], ids=["True", "False", "2d-True", "2d-False"])
def test_glue_kernels_exact_at_full_size(vx, cuda, nd, with_skip):
    """pool, unpool_combine (gradient to the FIRST maximal child, ties frequent with ternary activations) and sumpool_mask
    at the full-resolution shapes of the default model, 3-D and 2-D, against fp64 / fp32 emulations."""
    _, eng, _ = vx
    g = torch.Generator(device=cuda).manual_seed(9 + (nd == 2))
    s32 = torch.tensor(SLOPE, dtype=torch.float32, device=cuda)
    fine = GLUE_SHAPES[nd]
    B, D, H, W = fine
    x = ternary(fine + (16,), g)
    y = eng._pool(x, nd)
    ch = _children(x, nd).double()
    mx = ch.max(4, keepdim=True).values
    assert mism(y, mx.squeeze(4)) == 0
    is_max = ch == mx
    first = is_max & (is_max.cumsum(4) == 1)
    assert bool((first.sum(4) == 1).all()) and bool((is_max.sum(4) > 1).any())
    gs = ternary(x.shape, g) if with_skip else None
    gp = ternary(y.shape, g)
    out = eng._unpool_combine(x, gs, gp, nd, SLOPE)
    r = first.float() * gp.float().unsqueeze(4) + (_children(gs, nd).float() if with_skip else 0)
    r = torch.where(ch < 0, r * s32, r)
    n_unpool = mism(out, _unchildren(r, nd).to(torch.bfloat16))
    gf = ternary(fine + (32,), g)
    act = ternary((B, D // 2 if nd == 3 else D, H // 2, W // 2, 32), g)
    sp = eng._sumpool_mask(gf, act, nd, SLOPE)
    s = ref.children_sum(gf.double(), nd).float()
    n_sum = mism(sp, torch.where(act < 0, s * s32, s).to(torch.bfloat16))
    print("\n[glue, full size, %d-D, B = %d] pool 0 | unpool_combine%s %d | sumpool_mask %d mismatches"
          % (nd, B, "" if with_skip else " (no skip)", n_unpool, n_sum))
    assert n_unpool == 0 and n_sum == 0


# ---- c. the decomposition sweep: VXM_B200_CONV_CTAS caps the persistent grid ------------------------------------------

def _ops(kind, quantised, cuda):
    """operands of one sweep launch: ragged shapes (partial w tiles, H not a multiple of the tile height, odd depth, B = 2;
    the 2-D kinds, held as (B, 1, H, W, C), with B = 3)"""
    g = torch.Generator(device=cuda).manual_seed(100 + len(kind) + quantised)
    act = (lambda s: ternary(s, g)) if quantised else (lambda s: torch.randn(s, generator=g, device=cuda).to(torch.bfloat16))
    wt = (lambda s: qweight(s, g)) if quantised else (lambda s: torch.randn(s, generator=g, device=cuda) * 0.05)
    plane = (lambda s: ternary(s, g, torch.float32) * PLANE) if quantised else (lambda s: torch.randn(s, generator=g, device=cuda))
    if kind == "plain":
        return dict(x=act((2, 11, 21, 67, 16)), w=wt((32, 16, 3, 3, 3)), b=wt((32,)))
    if kind == "masked_dgrad":
        return dict(gz=act((2, 11, 21, 67, 32)), w=wt((32, 16, 3, 3, 3)), act=act((2, 11, 21, 67, 16)))
    if kind == "concat_up":
        return dict(xa=act((2, 5, 11, 33, 32)), xb=act((2, 10, 22, 66, 32)), w=wt((32, 64, 3, 3, 3)), b=wt((32,)))
    if kind == "polyphase":
        return dict(xa=act((2, 7, 11, 33, 32)), xb=act((2, 14, 22, 66, 16)), w=wt((32, 48, 3, 3, 3)), b=wt((32,)),
                    gz=act((2, 14, 22, 66, 32)), act=act((2, 7, 11, 33, 32)))
    if kind == "blocked64":
        return dict(x=act((2, 7, 13, 37, 64)), w=wt((64, 64, 3, 3, 3)), b=wt((64,)))
    if kind == "plain_2d":
        return dict(x=act((3, 1, 21, 67, 16)), w=wt((32, 16, 1, 3, 3)), b=wt((32,)))
    if kind == "masked_dgrad_2d":
        return dict(gz=act((3, 1, 21, 67, 32)), w=wt((32, 16, 1, 3, 3)), act=act((3, 1, 21, 67, 16)))
    if kind == "concat_up_2d":
        return dict(xa=act((3, 1, 11, 33, 32)), xb=act((3, 1, 22, 66, 16)), w=wt((32, 48, 1, 3, 3)), b=wt((32,)))
    if kind == "wgrad_2d":
        return dict(xa=act((3, 1, 11, 33, 32)), xb=act((3, 1, 22, 66, 16)), gz=act((3, 1, 22, 66, 32)),   # 32^ + 16 -> 32
                    x=act((3, 1, 21, 67, 16)), g=act((3, 1, 21, 67, 32)))                                   # 16 -> 32
    assert kind == "wgrad"
    return dict(xa=act((2, 7, 11, 33, 32)), xb=act((2, 14, 22, 66, 16)), gz=act((2, 14, 22, 66, 32)),      # rem0: 32^ + 16 -> 32
                x64=act((1, 9, 14, 40, 64)), g64=act((1, 9, 14, 40, 64)),                                # 64 x 64 slices
                planes=[plane((2, 1, 11, 21, 67)) for _ in range(2)], g16=act((2, 11, 21, 67, 16)))       # kd-folded, kh in M


def _launch(vx, kind, o):
    _, eng, tc = vx
    kd = 1 if kind.endswith("_2d") else 3
    if kind.startswith("plain"):
        wpk, cp = tc.pack_weights_t(o["w"], variant="s")
        return (tc.conv_fwd_t(o["x"], None, wpk, cp, o["b"], 32, kd, slope=SLOPE),)
    if kind.startswith("masked_dgrad"):
        wpk, cp = tc.pack_weights_t(o["w"], transposed=True, variant="s")
        return (tc.conv_fwd_t(o["gz"], None, wpk, cp, None, 16, kd, slope=SLOPE, mask=o["act"]),)
    if kind.startswith("concat_up"):
        assert tc.conv_blocks(32, o["xb"].shape[-1], 32, kd) is None
        wpk, cp = tc.pack_weights_t(o["w"], variant="s")
        return (tc.conv_fwd_t(o["xa"], o["xb"], wpk, cp, o["b"], 32, kd, up=True, slope=SLOPE),)
    if kind == "polyphase":
        fwd = tc.conv_fwd_poly(o["xa"], o["xb"], tc.pack_weights_poly(o["w"], 1, 32), o["b"], 32, SLOPE)
        return fwd, tc.dgrad_poly(o["gz"], tc.pack_weights_poly(o["w"], 2, 32), o["act"], SLOPE)
    if kind == "blocked64":
        blocks = tc.conv_blocks(64, 0, 64, 3)
        assert blocks is not None
        return (tc.conv_fwd_blocked(o["x"], None, blocks, tc.pack_weights_blocks(o["w"], False, blocks), o["b"], 64, 3, slope=SLOPE),)
    batch = tc.WgradBatch.get(o["gz"].device)
    batch.reset()
    if kind == "wgrad_2d":          # KD = 1 partials (no kh in M), one flush
        w1, b1 = tc.conv_wgrad(o["xa"], o["xb"], o["gz"], 48, 32, 1, up=True, batch=batch)
        w2, b2 = tc.conv_wgrad(o["x"], None, o["g"], 16, 32, 1, batch=batch)
        batch.flush()
        return w1, b1, w2, b2
    w1, b1 = tc.conv_wgrad(o["xa"], o["xb"], o["gz"], 48, 32, 3, up=True, batch=batch)
    w2, b2 = tc.conv_wgrad(o["x64"], None, o["g64"], 64, 64, 3, batch=batch)
    gwf = torch.empty((16, 6, 1, 3, 3), device=o["gz"].device)
    gbf = torch.empty(16, device=o["gz"].device)
    batch.add_khm(tc.planar_fold_kd(o["planes"], 8), o["g16"], gwf, gbf, 6, 16)
    batch.flush()
    return w1, b1, w2, b2, gwf, gbf


def _reference(vx, kind, o):
    _, eng, _ = vx
    nd = 2 if kind.endswith("_2d") else 3
    if kind.startswith("plain"):
        return (torch.cat(ref.conv([(o["x"], False)], o["w"], o["x"].shape[1], finish=lambda y, *_: ref.epilogue(y, o["b"], SLOPE)), 1),)
    if kind.startswith("masked_dgrad"):
        return (torch.cat(ref.conv([(o["gz"], False)], ref.dgrad_weight(o["w"]), o["gz"].shape[1],
                                   finish=lambda y, d0, d1: ref.epilogue(y, slope=SLOPE, mask=o["act"][:, d0:d1])), 1),)
    if kind.startswith("concat_up"):
        return (ref.epilogue(ref.conv([(o["xa"], True), (o["xb"], False)], o["w"], o["xb"].shape[1], nd=nd), o["b"], SLOPE),)
    if kind == "polyphase":
        fwd = ref.epilogue(ref.conv([(o["xa"], True), (o["xb"], False)], o["w"], 14), o["b"], SLOPE)
        y = ref.conv([(o["gz"], False)], ref.dgrad_weight(o["w"]), 14)[..., :32]
        return fwd, ref.epilogue(ref.children_sum(y), slope=SLOPE, mask=o["act"])
    if kind == "blocked64":
        return (ref.epilogue(ref.conv([(o["x"], False)], o["w"], 7), o["b"], SLOPE),)
    if kind == "wgrad_2d":        # (sources, output gradient, kd, nd, unit of x)
        ws = (([(o["xa"], True), (o["xb"], False)], o["gz"], 1, 2, 1), ([(o["x"], False)], o["g"], 1, 2, 1))
    else:
        ws = (([(o["xa"], True), (o["xb"], False)], o["gz"], 3, 3, 1), ([(o["x64"], False)], o["g64"], 3, 3, 1),
              ([(eng.fold_planes(o["planes"]), False)], o["g16"], 1, 3, PLANE))
    out = []
    for srcs, gz, kd, nd, unit in ws:
        gw, gb = ref.wgrad(srcs, gz, kd, nd=nd)
        aw, ab = ref.wgrad(srcs, gz, kd, absolute=True, nd=nd)
        assert float(aw.max()) < 2 ** 22 * unit and float(ab.max()) < 2 ** 23
        out += [gw.float(), gb.float()]
    return tuple(out)


@pytest.mark.parametrize("kind", ["plain", "masked_dgrad", "concat_up", "polyphase", "blocked64", "wgrad",
                                  "plain_2d", "masked_dgrad_2d", "concat_up_2d", "wgrad_2d"])
def test_decomposition_sweep(vx, cuda, monkeypatch, kind):
    """Each launch kind with its persistent grid capped at 1, 2, 5 and 13 CTAs (many items per CTA, partial last waves,
    other depth chunkings) and uncapped.  Quantised operands: every cap equals fp64 exactly.  Ordinary operands: the
    forward and dgrad outputs are bit-identical across caps (one CTA writes each output tile, in a fixed MMA order); the
    weight gradient is bit-identical between two runs at the same cap, and the cap does change its per-CTA partition."""
    def run(o, cap):
        if cap is None:
            monkeypatch.delenv("VXM_B200_CONV_CTAS", raising=False)
        else:
            monkeypatch.setenv("VXM_B200_CONV_CTAS", cap)
        res = [t.clone() for t in _launch(vx, kind, o)]
        torch.cuda.synchronize()
        return res

    o = _ops(kind, True, cuda)
    refs = _reference(vx, kind, o)
    counts = {cap: [mism(a, r) for a, r in zip(run(o, cap), refs)] for cap in CAPS}
    print("\n[sweep %s, quantised] mismatches per output by VXM_B200_CONV_CTAS: %s" % (kind, counts))
    assert all(n == 0 for c in counts.values() for n in c), counts
    o = _ops(kind, False, cuda)
    outs = {cap: run(o, cap) for cap in CAPS}
    if kind.startswith("wgrad"):
        for cap in CAPS:
            assert all(torch.equal(a, b) for a, b in zip(outs[cap], run(o, cap))), cap
        assert not all(torch.equal(a, b) for a, b in zip(outs["1"], outs[None]))
    else:
        for cap in CAPS:
            assert all(torch.equal(a, b) for a, b in zip(outs[cap], outs[None])), cap
