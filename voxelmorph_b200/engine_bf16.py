"""The tensor-core (bf16 operands / fp32 accumulation) execution engine of Unet + flow head.

`unet_flow(model, source, target)` computes `model.flow(model.unet_model(cat(source, target)))`
(reference voxelmorph/torch/networks.py:253-257) entirely with the wgmma convolution kernels and the
channels-last bf16 glue kernels: every activation between the fp32 input images and the fp32 flow field is a
bf16 (B,D,H,W,C) tensor, the concat / upsample / bias / LeakyReLU / LeakyReLU-derivative are fused into the
convolution kernels, and the backward pass (dgrad, wgrad, pooling and skip routing) is written out by hand —
torch autograd only sees one node.  Parameters stay the module's own fp32 `nn.Parameter`s, except in a model whose U-Net
weights are generated (HyperVxmDense): its convolutions hold plain views of one persistent flat buffer, and the backward
returns their gradient as one flat tensor of the same layout.
"""
import torch

from . import _lib, tc

_weights_epoch = 0


def bump_weights_epoch():
    """Called by optimizers that update parameters behind torch's back (FusedAdam) so packed copies refresh."""
    global _weights_epoch
    _weights_epoch += 1


class _Layer:
    """One convolution of a model's plan: its parameters, its inputs (tensor ids of the walk: 0 = the images, then every
    convolution and pooling output in execution order) and how it runs.  `fwd` / `dgrad`: the execution form of the
    forward and of the dgrad (see _run); `fwd_x3`: the block grid of the split-precision forward; `dgrad_skip`: with a
    polyphase dgrad, the form of the skip part (the dgrad's own form then yields the upsampled part only); `dgrad_img`
    (first convolution only): the form of the dgrad into the image planes, which runs only when an image asks for its
    gradient (_Plan.image_dgrad_packs).  `srcs`: the parameters the layer's operands are derived from — its own weight, or
    for the head of a probabilistic model the weights and biases of `flow` and `log_sigma`, which the plan concatenates
    into the persistent `w` / `bias` of one 2 nd-output convolution."""
    __slots__ = ("w", "bias", "slope", "role", "a", "b", "out", "up", "ca", "cb", "cin", "cout", "fwd", "fwd_x3", "dgrad", "khm",
                 "dgrad_skip", "dgrad_img", "pk_fwd", "pk_dgrad", "pk_dgrad_skip", "pk_hi", "pk_lo", "w_hi", "w_lo", "srcs")


def _refuse(what):
    raise _lib.VxmError("bf16 tensor-core engine: %s (use VXM_B200_CONV_ENGINE=f32 for other U-Net shapes)" % what)


def _form(ca, cb, nout, kd, kw, split=None):
    """Execution form of a convolution on the swizzled kw-stacked kernel: its channel blocks (tc.conv_blocks), or the 1 x 1
    grid of one launch (kw: input channels of the weight operand).  Refuses a shape one of whose launches the kernel lacks."""
    blocks = tc.conv_blocks(ca, cb, nout, kd, split)
    launches = [(ca, cb, nout)] if blocks is None else \
        [((ca, cb) if src == 2 else (kb, 0)) + (nb,) for src, _, kb in blocks[0] for _, nb, _, _ in blocks[1]]
    for c0, c1, n in launches:
        if not _lib.load().vxm_conv3d_tcs_supported(c0, c1, n):
            _refuse("no tensor-core kernel takes a (%d + %d) -> %d convolution" % (c0, c1, n))
    return blocks if blocks is not None else tc.one_block(kw, nout)


def _walk(model):
    """The U-Net and flow head of `model` (a VxmDense) in execution order: _Layer and ("pool", in_id, out_id) entries with
    shapes and execution forms only (allocates nothing).  Refuses a model some convolution of which no engine path runs.
    A model with a `log_sigma` module (VxmDenseProbabilistic) has a head of 2 nd outputs: `flow` then `log_sigma`, one
    forward, one dgrad and one weight gradient."""
    unet = model.unet_model
    w0 = unet.encoder[0][0].main.weight
    if w0.dim() not in (4, 5):
        _refuse("2-D or 3-D convolutions only")
    kd = 3 if w0.dim() == 5 else 1
    fold = kd == 3 and tc.kdfold_enabled()
    poly = kd == 3 and tc.polyphase_enabled()
    ops = []
    chans = [8]           # channels of every tensor id: the images enter as one bf16 channels-last tensor of 8 channels
    cur, pending_up, skips = 0, None, [None]

    def conv(m, slope, role="inner", extra=None):
        nonlocal cur, pending_up
        L = _Layer()
        L.w, L.bias, L.slope, L.role = m.weight, m.bias, slope, role
        if not isinstance(m.weight, torch.nn.Parameter):
            # a generated weight (a view of the model's flat buffer): the plan keeps no autograd history of it
            L.w, L.bias = m.weight.detach(), m.bias.detach()
        L.srcs = (L.w,) if extra is None else (m.weight, m.bias, extra.weight, extra.bias)
        # a convolution after an upsample reads the upsampled previous output, then the skip (a fused upsample + concat)
        L.a, L.b = pending_up if pending_up is not None else (cur, None)
        L.up, pending_up = pending_up is not None, None
        L.ca, L.cb = chans[L.a], (0 if L.b is None else chans[L.b])
        L.cout, L.cin = m.weight.shape[0] + (0 if extra is None else extra.weight.shape[0]), m.weight.shape[1]
        if m.weight.dim() != w0.dim():
            _refuse("convolutions of different dimensionality")
        if role == "first":
            if L.cin > 8:
                _refuse("the first convolution takes at most 8 input feature planes (src_feats + trg_feats)")
        elif L.ca + L.cb != L.cin or L.cin % 16 or L.cin > (64 if role == "flow" else 128):
            _refuse("unsupported convolution input channels %d (+%d); need a multiple of 16, at most 128 (64 into the flow "
                    "head)" % (L.ca, L.cb))
        if role == "flow" and L.cout > 8:
            _refuse("the flow head has %d components" % L.cout)
        if role != "flow" and L.cout not in (8, 16, 32, 64):
            _refuse("a U-Net convolution has %d output channels; supported feature counts are 8, 16, 32 and 64" % L.cout)
        L.fwd = L.fwd_x3 = _form(L.ca, L.cb, L.cout, kd, L.cin)
        # kd folded into the channels of the layers with 2 / 3 real channels on one side (3 instead of 9 MMA steps per
        # tile): the forward of the first convolution (bf16), the dgrad of the flow head
        if role == "first" and fold and 3 * L.cin <= 8 and L.cout in (8, 16, 32):
            L.fwd = "fold"
        L.dgrad_img = None
        if role == "first":
            # no dgrad in the step's own launch sequence: the images of a training step need no gradient.  When one does
            # (_UnetFlowFn), the masked output gradient (cout channels) is convolved with the transposed weights into
            # cin <= 8 fp32 planes: the shape of the flow head's forward, and its launch
            L.dgrad = None
            L.dgrad_img = _form(L.cout, 0, L.cin, kd, L.cout)
        elif role == "flow" and fold and L.b is None and L.cin in (8, 16) and 3 * L.cout <= 16:
            L.dgrad = "fold"
        else:                             # the flow gradient enters as 8 channels; a concatenation's dgrad splits its output
            L.dgrad = _form(8 if role == "flow" else L.cout, 0, L.cin, kd, L.cout, L.ca if L.b is not None else None)
        # polyphase forms of a concatenation with a 32-channel upsampled source (taps that read the same coarse voxel
        # merged): the forward of 32 + 16 -> 32 (kd), and the dgrad as a coarse launch for the upsampled source (kd, kh;
        # LeakyReLU derivative included) plus a fine launch for the skip channels
        L.dgrad_skip = None
        if poly and L.up and L.b is not None and L.ca == 32 and L.cout == 32:
            if L.cb == 16:
                L.fwd = ("poly", 1, L.ca)
            L.dgrad = ("poly", 2, L.ca)
            L.dgrad_skip = (((2, 0, L.cout),), ((L.ca, L.cb, 0, 0),))
            _form(L.cout, 0, L.cb, kd, L.cout)          # (refuses a skip width no launch takes)
        L.khm = L.cout <= 16              # weight gradient of the folded first layer: kh-in-M takes at most 16 outputs
        L.out = cur = len(chans)
        chans.append(L.cout)
        ops.append(L)

    def pool():
        nonlocal cur
        ops.append(("pool", cur, len(chans)))
        cur = len(chans)
        chans.append(chans[ops[-1][1]])

    for convs in unet.encoder:
        for blk in convs:
            conv(blk.main, blk.activation.negative_slope, "first" if cur == 0 else "inner")
        skips.append(cur)
        pool()
    for level, convs in enumerate(unet.decoder):
        for blk in convs:
            conv(blk.main, blk.activation.negative_slope)
        if not unet.half_res or level < (unet.nb_levels - 2):
            pending_up = (cur, skips.pop())
    for blk in unet.remaining:
        conv(blk.main, blk.activation.negative_slope)
    conv(model.flow, None, "flow", getattr(model, "log_sigma", None))        # no activation, fp32 planar output
    return ops


def supports(model):
    """True when the tensor-core engine runs every convolution of `model` (a VxmDense) in one launch per layer with feature
    counts in {8, 16, 32} and inputs of at most 64 channels: what VXM_B200_CONV_ENGINE=tc selects the tensor cores for.
    VXM_B200_CONV_ENGINE=bf16 | bf16x3 run every model _walk accepts, U-Nets with 64-channel layers and concatenations of
    up to 128 channels included (in channel blocks)."""
    try:
        ops = _walk(model)
    except (AttributeError, _lib.VxmError):
        return False
    return all(L.role == "flow" or (L.cout in (8, 16, 32) and L.ca + L.cb <= 64) for L in ops if isinstance(L, _Layer))


class _Plan:
    """A model's walk (_walk) with every packed operand it runs on.  The bf16 operands (forward and transposed copy of
    every convolution: whole, in channel blocks or kd-folded) are refreshed by ONE pack launch per step.  The bf16x3
    forward operands, the bf16 hi and lo parts of every weight in the block grid of tc.conv_fwd_blocked, are packed from
    persistent fp32 buffers by one more launch, so that their refresh stays graph-capturable."""

    def __init__(self, model):
        self.ops = _walk(model)
        self.layers = [L for L in self.ops if isinstance(L, _Layer)]
        self.nd = self.layers[0].w.dim() - 2
        for L in self.layers:
            if len(L.srcs) > 1:           # the 2 nd-output head: persistent operands, refilled by refresh
                L.w = torch.empty((L.cout,) + tuple(L.w.shape[1:]), dtype=torch.float32, device=L.w.device)
                L.bias = torch.empty(L.cout, dtype=torch.float32, device=L.w.device)
        self.slope = {L.out: float(L.slope) for L in self.layers if L.slope is not None}     # convolution output id -> slope
        bf16, x3 = [], []
        for L in self.layers:
            w = L.w.detach()
            L.w_hi, L.w_lo = torch.empty_like(w), torch.empty_like(w)
            bf16 += [(w, False, L.fwd)] + ([(w, True, L.dgrad)] if L.dgrad is not None else []) + \
                    ([(w, True, L.dgrad_skip)] if L.dgrad_skip is not None else [])
            x3 += [(L.w_hi, False, L.fwd_x3), (L.w_lo, False, L.fwd_x3)]
        self.bf16, self.x3 = tc.PackTable(bf16), tc.PackTable(x3)
        packs, packs3 = iter(self.bf16.packs), iter(self.x3.packs)
        for L in self.layers:
            L.pk_fwd, L.pk_dgrad = next(packs), (next(packs) if L.dgrad is not None else None)
            L.pk_dgrad_skip = next(packs) if L.dgrad_skip is not None else None
            L.pk_hi, L.pk_lo = next(packs3), next(packs3)
        self.ptrs = self.weight_ptrs()
        self.stamps = [None, None]
        self.img_table, self.img_stamp = None, None
        self.gen_ptr = None               # the generated weights' buffer (_plan_of)

    def weight_ptrs(self):
        return tuple(p.data_ptr() for L in self.layers for p in L.srcs)

    def refresh(self, split):
        stamp = (_weights_epoch, tuple(p._version for L in self.layers for p in L.srcs))
        if stamp != self.stamps[0]:
            for L in self.layers:
                if len(L.srcs) > 1:       # device copies: graph-capturable like the pack launch
                    fw, fb, lw, lb = L.srcs
                    torch.cat([fw.detach(), lw.detach()], out=L.w)
                    torch.cat([fb.detach(), lb.detach()], out=L.bias)
            self.bf16.refresh()
            self.stamps[0] = stamp
        if split and stamp != self.stamps[1]:
            for L in self.layers:         # hi = bf16(w), lo = w - hi
                w = L.w.detach()
                L.w_hi.copy_(w.to(torch.bfloat16))
                torch.sub(w, L.w_hi, out=L.w_lo)
            self.x3.refresh()
            self.stamps[1] = stamp

    def image_dgrad_packs(self):
        """The transposed operand of the first convolution (its dgrad into the image planes), refreshed.  It lives in a
        table of its own, built on first use and repacked by one launch of its own per weight update: the pack launch
        of a step whose images need no gradient keeps its descriptors and its size.  (Build it in an eager step — the
        warm-up of a graph capture — since the descriptor upload is a host-to-device copy.)"""
        first = self.layers[0]
        if self.img_table is None:
            self.img_table = tc.PackTable([(first.w.detach(), True, first.dgrad_img)])
        stamp = (_weights_epoch, first.w._version)
        if stamp != self.img_stamp:
            self.img_table.refresh()
            self.img_stamp = stamp
        return self.img_table.packs[0]


def _plan_of(model, split, generated=None):
    """The model's plan with its operands refreshed (built lazily; rebuilt when the parameters moved, e.g. after
    .to(device) or FlatParams, or when `generated`, the flat buffer the U-Net's weights are views of, did).  The
    refresh stamp counts bump_weights_epoch calls, which the weight generation makes: generated weights repack on every
    step, and a captured step records the pack launch."""
    plan = model.__dict__.get("_vxm_pack_plan")
    gen_ptr = None if generated is None else generated.data_ptr()
    if plan is None or plan.ptrs != plan.weight_ptrs() or plan.gen_ptr != gen_ptr:
        plan = _Plan(model)
        plan.gen_ptr = gen_ptr
        object.__setattr__(model, "_vxm_pack_plan", plan)
    plan.refresh(split)
    return plan


def _pool(x, nd):
    lib = _lib.load()
    B, D, H, W, C = x.shape
    Dc = D // 2 if nd == 3 else D
    y = torch.empty((B, Dc, H // 2, W // 2, C), dtype=torch.bfloat16, device=x.device)
    if (nd == 3 and D % 2) or H % 2 or W % 2:
        raise _lib.VxmError("bf16 engine: odd sizes cannot be pooled (U-Net shapes must be divisible by 2 per level)")
    _lib.check(lib.vxm_pool2_ndhwc_bf16(_lib.ptr(x), _lib.ptr(y), B, Dc, H // 2, W // 2, C, nd, _lib.stream_ptr()), "vxm_pool2_ndhwc_bf16")
    return y


def _sumpool_mask(g_fine, act_coarse, nd, slope):
    lib = _lib.load()
    B, Dc, Hc, Wc, C = act_coarse.shape
    out = torch.empty_like(act_coarse)
    _lib.check(lib.vxm_sumpool_mask_ndhwc_bf16(_lib.ptr(g_fine), _lib.ptr(act_coarse), _lib.ptr(out), B, Dc, Hc, Wc, C, nd, slope,
                                               _lib.stream_ptr()), "vxm_sumpool_mask_ndhwc_bf16")
    return out


def _unpool_combine(e_fine, g_skip, g_pool, nd, slope, e_lo=None):
    """Gradient through MaxPool(2) plus the skip gradient, times the LeakyReLU derivative.  e_lo: the lo parts of a
    split-precision forward, whose pool chose the child on hi + lo; the gradient then goes to that child."""
    lib = _lib.load()
    B, D, H, W, C = e_fine.shape
    Dc = D // 2 if nd == 3 else D
    out = torch.empty_like(e_fine)
    if e_lo is None:
        _lib.check(lib.vxm_unpool_combine_ndhwc_bf16(_lib.ptr(e_fine), _lib.ptr(g_skip), _lib.ptr(g_pool), _lib.ptr(out), B, Dc, H // 2,
                                                     W // 2, C, nd, slope, _lib.stream_ptr()), "vxm_unpool_combine_ndhwc_bf16")
    else:
        _lib.check(lib.vxm_unpool_combine_split_ndhwc_bf16(_lib.ptr(e_fine), _lib.ptr(e_lo), _lib.ptr(g_skip), _lib.ptr(g_pool),
                                                           _lib.ptr(out), B, Dc, H // 2, W // 2, C, nd, slope, _lib.stream_ptr()),
                   "vxm_unpool_combine_split_ndhwc_bf16")
    return out


def _run(form, packs, xa, xb, nout, kd, bias=None, lo=None, **kw):
    """The engine's one kernel selection: runs a convolution of the plan (a forward, or a dgrad on the transposed operand) in
    its execution form.  "fold": one 2-D launch over kd-folded channels; a 1 x 1 grid: one launch of the swizzled
    kw-stacked kernel (tc.conv_fwd_t); ("poly", mode, ca): a polyphase launch (tc.conv_fwd_poly; tc.dgrad_poly, whose
    `mask` is the coarse activation); channel blocks, and every split-precision forward (lo): tc.conv_fwd_blocked."""
    if form[0] == "poly":
        wpk = packs[0, 0][0]
        return tc.conv_fwd_poly(xa, xb, wpk, bias, nout, kw["slope"]) if form[1] == 1 else tc.dgrad_poly(xa, wpk, kw["mask"], kw["slope"])
    if form == "fold" or (lo is None and len(form[0]) == len(form[1]) == 1):
        wpk, coutp = packs[0, 0]
        return tc.conv_fwd_t(xa, xb, wpk, (coutp, "s"), bias, nout, 1 if form == "fold" else kd, **kw)
    return tc.conv_fwd_blocked(xa, xb, form, packs, bias, nout, kd, lo=lo, **kw)


def _flat_grads(L):
    """True when every parameter of L has a contiguous .grad view of FusedAdam's flat gradient buffer (optim.FlatParams
    marks them): the weight gradients are then accumulated into it directly, and autograd receives none for them."""
    return all(getattr(p, "_vxm_flat_grad", False) and p.grad is not None and p.grad.is_contiguous()
               for p in (L.w, L.bias) if p is not None)


def forward_tape(model, source, target, split=False, generated=None):
    """Runs Unet + flow head, returns (flow fp32 (B,nd,*vol), tape).  `split`: split-precision (bf16x3) forward — every
    activation is a (hi, lo) bf16 pair and every layer three tensor-core passes; the tape keeps the hi parts, which is
    what the (bf16-operand) backward reads, and the lo parts of the pool inputs, so that the backward routes each pool
    gradient to the child the pool chose on hi + lo.  `generated`: the flat buffer the U-Net's weights are views of
    (HyperVxmDense), whose gradient backward_tape then returns under the key "generated"."""
    nd = source.dim() - 2
    kd = 3 if nd == 3 else 1
    _lib.require_cuda(source, target, what="VxmDense")
    source, target = _lib.contig(source), _lib.contig(target)
    plan = _plan_of(model, split, generated)
    planes = [source[:, i:i + 1] for i in range(source.shape[1])] + [target[:, i:i + 1] for i in range(target.shape[1])]
    first = plan.layers[0]
    if nd != plan.nd or len(planes) != first.cin:
        raise _lib.VxmError("bf16 engine: the model takes %d %d-D image planes (src_feats + trg_feats), got %d %d-D"
                            % (first.cin, plan.nd, len(planes), nd))
    tensors = {}         # tensor id -> bf16 NDHWC tensor
    lows = {}            # tensor id -> lo part (split precision only)
    pool_lows = {}       # pool input id -> lo part, kept on the tape
    if split:
        tensors[0], lows[0] = tc.planar_to_ndhwc8_split(planes)
    elif first.fwd == "fold":
        tensors[0] = tc.planar_fold_kd(planes, 8)      # (kd, plane) channels: the first convolution runs as 2-D
    else:
        tensors[0] = tc.planar_to_ndhwc8(planes)
    for L in plan.ops:
        if not isinstance(L, _Layer):
            _, src, dst = L
            if split:
                tensors[dst], lows[dst] = tc.pool_split((tensors[src], lows[src]), nd)
                pool_lows[src] = lows[src]
            else:
                tensors[dst] = _pool(tensors[src], nd)
            continue
        bias = None if L.bias is None else L.bias.detach()
        kw = dict(up=L.up, slope=L.slope, out_fp32_planar=L.role == "flow")
        if split:
            out = _run(L.fwd_x3, L.pk_hi, tensors[L.a], tensors.get(L.b), L.cout, kd, bias, lo=(lows[L.a], lows.get(L.b), L.pk_lo), **kw)
        else:
            out = _run(L.fwd, L.pk_fwd, tensors[L.a], tensors.get(L.b), L.cout, kd, bias, **kw)
        if L.role == "flow":
            flow = out
        elif split:
            tensors[L.out], lows[L.out] = out
        else:
            tensors[L.out] = out
    if nd == 2:
        flow = flow.squeeze(2)
    return flow, dict(plan=plan, tensors=tensors, split=split, pool_lows=pool_lows,
                      generated=None if generated is None else generated.detach())


def backward_tape(ctx, g_flow, image_grad=False):
    """Hand-written backward over the plan.  Returns {param: grad}; with `image_grad`, the fp32 planar gradient w.r.t. the
    image planes (B, src_feats + trg_feats, D, H, W) (D = 1 for a 2-D model) under the key "images" as well."""
    plan, tensors = ctx["plan"], ctx["tensors"]
    nd = plan.nd
    kd = 3 if nd == 3 else 1
    g_flow = _lib.contig(g_flow.float())
    if nd == 2:
        g_flow = g_flow.unsqueeze(2)
    dev = g_flow.device
    batch = tc.WgradBatch.get(dev)
    batch.reset()
    gz = {}       # conv-output id -> masked gradient (bf16 NDHWC)
    graw = {}     # pool-output id -> raw gradient
    gskip = {}    # encoder-output id -> raw skip gradient
    grads = {}
    folded = []   # (layer, gw2d, gb2d): 2-D weight gradients of the kd-folded layers, mapped back after the flush
    heads = []    # (layer, gw, gb): weight gradient of a 2 nd-output head, split between its modules after the flush
    base = ctx.get("generated")
    dW = None if base is None else torch.zeros(base.numel(), dtype=torch.float32, device=dev)
    gen = {}      # layer -> (weight, bias) views of dW at the layer's place in the generated layout
    if dW is not None:
        for L in plan.layers:
            if L.role != "flow":
                ow, ob = [(t.data_ptr() - base.data_ptr()) // base.element_size() for t in (L.w, L.bias)]
                gen[L] = (dW[ow:ow + L.w.numel()].view(L.w.shape), dW[ob:ob + L.cout])
        grads["generated"] = dW
    for L in reversed(plan.ops):
        if not isinstance(L, _Layer):
            _, src, dst = L
            gz[src] = _unpool_combine(tensors[src], gskip.pop(src, None), graw.pop(dst), nd, plan.slope[src], ctx["pool_lows"].pop(src, None))
            continue
        xa, xb = tensors[L.a], tensors.get(L.b)
        if L.role == "flow":
            # the fp32 planar flow gradient becomes a bf16 channels-last tensor: 8 channels, or kd-folded (kd', component) =
            # 9 of 16 channels
            planes = [g_flow[:, i:i + 1] for i in range(g_flow.shape[1])]
            g_in = tc.planar_fold_kd(planes, 16) if L.dgrad == "fold" else tc.planar_to_ndhwc8(planes)
        else:
            g_in = gz.pop(L.out)
        # ---- weight gradient ----
        if L.dgrad == "fold":
            gwf = torch.empty((3 * nd, L.cin, 1, 3, 3), dtype=torch.float32, device=dev)
            gbf = torch.empty(3 * nd, dtype=torch.float32, device=dev) if L.bias is not None else None
            batch.add_khm(xa, g_in, gwf, gbf, L.cin, 3 * nd)
            folded.append((L, gwf, gbf))
        elif L.fwd == "fold" and not ctx["split"]:
            # first layer over the kd-folded images: a 2-D weight gradient
            gwf = torch.empty((L.cout, 3 * L.cin, 1, 3, 3), dtype=torch.float32, device=dev)
            gbf = torch.empty(L.cout, dtype=torch.float32, device=dev) if L.bias is not None else None
            if L.khm:
                batch.add_khm(xa, g_in, gwf, gbf, 3 * L.cin, L.cout)
            else:
                batch.add(xa, None, g_in, gwf, gbf, 3 * L.cin, L.cout, 1, False, False)
            folded.append((L, gwf, gbf))
        elif L in gen:
            # generated weights: accumulated into the zeroed flat gradient at their own place, no per-layer tensors
            tc.conv_wgrad(xa, xb, g_in, L.cin, L.cout, kd, up=L.up, out_w=gen[L][0], out_b=gen[L][1], batch=batch)
        elif len(L.srcs) > 1:
            heads.append((L,) + tc.conv_wgrad(xa, xb, g_in, L.cin, L.cout, kd, up=L.up, batch=batch))
        elif _flat_grads(L):
            tc.conv_wgrad(xa, xb, g_in, L.cin, L.cout, kd, up=L.up, out_w=L.w.grad, out_b=None if L.bias is None else L.bias.grad,
                          batch=batch)
        else:
            gw, gb = tc.conv_wgrad(xa, xb, g_in, L.cin, L.cout, kd, up=L.up, batch=batch)
            grads[L.w] = gw.squeeze(2) if nd == 2 else gw
            if L.bias is not None:
                grads[L.bias] = gb
        # ---- dgrad ----
        if L.dgrad is None:
            if image_grad and L.role == "first":
                # bf16 operands as in every other dgrad; no bias, activation or mask (the images are the leaves), and the
                # layer's input is not read, so a kd-folded image tensor on the tape does not matter
                grads["images"] = _run(L.dgrad_img, plan.image_dgrad_packs(), g_in, None, L.cin, kd, out_fp32_planar=True)
            continue
        t = L.a
        if L.b is None:
            sl = plan.slope.get(t)         # None: a pooling output, no activation to differentiate
            res = _run(L.dgrad, L.pk_dgrad, g_in, None, L.cin, kd, slope=sl, mask=None if sl is None else tensors[t])
            (graw if sl is None else gz)[t] = res
        elif L.dgrad_skip is not None:
            # polyphase: the coarse source's gradient (its 8 children summed, LeakyReLU derivative applied) in one launch
            gz[t] = _run(L.dgrad, L.pk_dgrad, g_in, None, L.ca, kd, mask=tensors[t], slope=plan.slope[t])
            gskip[L.b] = _run(L.dgrad_skip, L.pk_dgrad_skip, g_in, None, L.cb, kd)
        else:
            # single dgrad pass over the whole concat input: N = Ca + Cb output channels, split on store
            g_up, g_sk = _run(L.dgrad, L.pk_dgrad, g_in, None, L.cin, kd, split=L.ca)
            gz[t] = _sumpool_mask(g_up, tensors[t], nd, plan.slope[t])   # grad wrt upsample(a): sum children
            del g_up
            gskip[L.b] = g_sk
    batch.flush()     # one launch reduces every layer's per-CTA partials (fixed order: deterministic)
    for L, gwf, gbf in folded:
        gw, gb = (unfold_grad_first(gwf, L.cout, L.cin), gbf) if L.role == "first" else unfold_grad_flow(gwf, gbf, nd, L.cin)
        if L in gen:
            gen[L][0].add_(gw)
            gen[L][1].add_(gb)
        elif _flat_grads(L):
            L.w.grad.add_(gw)
            if L.bias is not None:
                L.bias.grad.add_(gb)
        else:
            grads[L.w] = gw.contiguous()
            if L.bias is not None:
                grads[L.bias] = gb.contiguous()
    for L, gw, gb in heads:
        fw, fb, lw, lb = L.srcs
        k = fw.shape[0]
        gw = gw.squeeze(2) if nd == 2 else gw
        for p, g in ((fw, gw[:k]), (fb, gb[:k]), (lw, gw[k:]), (lb, gb[k:])):
            if getattr(p, "_vxm_flat_grad", False) and p.grad is not None and p.grad.is_contiguous():
                p.grad.add_(g)
            else:
                grads[p] = g.contiguous()
    return grads


# ---- index algebra of the kd-folded layers (pure tensor views; checked on CPU against torch's own 3-D convolution in
# tests/test_kdfold_algebra.py, on the GPU against the kernels in tests/test_gpu_tc.py) ----------------------------------------

def fold_planes(planes):
    """Reference (torch) form of csrc/ndhwc_ops.cu:planar_fold_kd_kernel: [(B,1,D,H,W)] * n -> (B, D, H, W, 3n), channel
    kd * n + p = plane p at slice d + kd - 1, zero outside the volume."""
    x = torch.cat(planes, dim=1)                                   # (B, n, D, H, W)
    xp = torch.nn.functional.pad(x, (0, 0, 0, 0, 1, 1))            # one zero slice on either side of D
    D = x.shape[2]
    return torch.cat([xp[:, :, kd:kd + D] for kd in range(3)], dim=1).permute(0, 2, 3, 4, 1).contiguous()


def fold_weight_first(w):
    """3-D weight (Cout, P, 3, 3, 3) of the first convolution -> the 2-D weight (Cout, 3P, 3, 3) the folded tensor is convolved
    with: input channel kd * P + p <-> (tap kd, plane p).  (What vxm_conv3d_tcs_pack_desc_fold packs, transposed = 0.)"""
    co, p = w.shape[0], w.shape[1]
    return w.permute(0, 2, 1, 3, 4).reshape(co, 3 * p, 3, 3)


def fold_weight_flow_dgrad(w):
    """3-D weight (C, Cin, 3, 3, 3) of the flow head -> the 2-D cross-correlation kernel (Cin, 3C, 3, 3) that turns the folded flow
    gradient (channel kd' * C + c = component c at slice d + kd' - 1) into the gradient w.r.t. the head's input:
    K[ci][kd' * C + c][kh][kw] = w[c][ci][2 - kd'][2 - kh][2 - kw].  (vxm_conv3d_tcs_pack_desc_fold, transposed = 1.)"""
    c, ci = w.shape[0], w.shape[1]
    return w.flip(2, 3, 4).permute(1, 2, 0, 3, 4).reshape(ci, 3 * c, 3, 3)


def unfold_grad_first(gwf, cout, cin):
    """2-D weight gradient (Cout, 3 Cin, 1, 3, 3) of the folded first layer -> (Cout, Cin, 3, 3, 3): gwf[co][kd * P + p] = gw[co][p][kd]."""
    return gwf.view(cout, 3, cin, 3, 3).permute(0, 2, 1, 3, 4)


def unfold_grad_flow(gwf, gbf, nd, cin):
    """2-D weight gradient (3 nd, Cin, 1, 3, 3) of the flow head against the folded flow gradient -> (nd, Cin, 3, 3, 3):
    gwf[kd' * nd + c][ci][kh][kw] = gw[c][ci][2 - kd'][kh][kw]  (x at slice d pairs with the flow gradient at d + kd' - 1, i.e.
    the gradient at v with x at v + 1 - kd').  The bias gradient is the channel sum of the unshifted copy (kd' = 1)."""
    gw = gwf.view(3, nd, cin, 3, 3).flip(0).permute(1, 2, 0, 3, 4)
    return gw, (None if gbf is None else gbf[nd:2 * nd])


class _UnetFlowFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, source, target, split, generated, *params):
        flow, tape = forward_tape(model, source, target, split=split, generated=generated)
        ctx.tape = tape
        ctx.params = params
        ctx.model_ref = model
        # (source, target) that ask for their gradient, and how the image planes split between them
        ctx.image_grads = tuple(ctx.needs_input_grad[1:3])
        ctx.src_feats = source.shape[1]
        return flow

    @staticmethod
    def backward(ctx, g_flow):
        dp = getattr(ctx.model_ref, "_dp", None)
        if dp is not None:
            dp.schedule()      # gradients written straight into .grad views bypass the parameter hooks
        grads = backward_tape(ctx.tape, g_flow, image_grad=any(ctx.image_grads))
        ctx.tape = None
        g_source = g_target = None
        if any(ctx.image_grads):
            g_img = grads.pop("images")
            if g_flow.dim() == 4:         # 2-D: drop the depth axis, as forward_tape does for the flow
                g_img = g_img.squeeze(2)
            if ctx.image_grads[0]:
                g_source = g_img[:, :ctx.src_feats]
            if ctx.image_grads[1]:
                g_target = g_img[:, ctx.src_feats:]
        return (None, g_source, g_target, None, grads.get("generated")) + tuple(grads.get(p) for p in ctx.params)


def unet_flow(model, source, target, split=False, generated=None):
    """flow = model.flow(model.unet_model(cat(source, target))) on the tensor-core engine (for a model with `log_sigma`:
    cat(flow(x), log_sigma(x)), the probabilistic model's flow_params).  split=False: bf16 operands
    (throughput mode); split=True: bf16x3 split precision in the forward (flow within 1e-4 of the fp32 reference), the
    backward uses bf16 operands in both modes.  `generated` (HyperVxmDense): the flat tensor the U-Net's weights are
    views of; its gradient is formed as one flat tensor of the same layout."""
    head = [model.flow] + ([model.log_sigma] if hasattr(model, "log_sigma") else [])
    params = list(model.unet_model.parameters()) + [p for m in head for p in m.parameters()]
    return _UnetFlowFn.apply(model, source, target, bool(split), generated, *params)
