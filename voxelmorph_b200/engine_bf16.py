"""The tensor-core (bf16 operands / fp32 accumulation) execution engine of Unet + flow head.

`unet_flow(model, source, target)` computes `model.flow(model.unet_model(cat(source, target)))`
(reference voxelmorph/torch/networks.py:253-257) entirely with the wgmma convolution kernels and the
channels-last bf16 glue kernels: every activation between the fp32 input images and the fp32 flow field is a
bf16 (B,D,H,W,C) tensor, the concat / upsample / bias / LeakyReLU / LeakyReLU-derivative are fused into the
convolution kernels, and the backward pass (dgrad, wgrad, pooling and skip routing) is written out by hand —
torch autograd only sees one node.  Parameters stay the module's own fp32 `nn.Parameter`s.
"""
import torch

from . import _lib, tc

_weights_epoch = 0


def bump_weights_epoch():
    """Called by optimizers that update parameters behind torch's back (FusedAdam) so packed copies refresh."""
    global _weights_epoch
    _weights_epoch += 1


class _PackCache:
    """Packed (bf16, MMA-ordered) copies of the convolution weights.  The copies live ON the parameter object
    (attribute `_vxm_packs`), so they die with it: a table keyed by id()/data_ptr would hand a new model the packed
    weights of a freed one whenever Python and the caching allocator both reuse the address."""

    def get(self, w, key, fn):
        packs = getattr(w, "_vxm_packs", None)
        if packs is None:
            packs = {}
            w._vxm_packs = packs
        stamp = (w.data_ptr(), w._version, _weights_epoch, tuple(w.shape), tc._variant())
        hit = packs.get(key)
        if hit is None or hit[0] != stamp:
            hit = (stamp, fn())
            packs[key] = hit
        return hit[1]


_cache = _PackCache()


class _PackPlan:
    """Every packed operand of a model (forward + transposed copy of each convolution, swizzled kw-stacked format) refreshed
    by ONE kernel launch (tc.vxm_conv3d_tcs_pack_multi) instead of one launch per operand (23 per training step)."""

    def __init__(self, model):
        import ctypes
        lib = _lib.load()
        unet = model.unet_model
        convs = [b.main for lvl in unet.encoder for b in lvl] + [b.main for lvl in unet.decoder for b in lvl] + \
                [b.main for b in unet.remaining] + [model.flow]
        self.params = [c.weight for c in convs]
        dev = self.params[0].device
        dsz = int(lib.vxm_conv3d_tcs_pack_desc_bytes())
        host = ctypes.create_string_buffer(dsz * (16 * len(convs) + 2))      # <= 2 K x 4 N blocks per operand
        self.table = {}
        self.keep = []
        n, begin = 0, 0
        # kd-folded 2-D operands (tc.planar_fold_kd): forward of the first convolution, dgrad of the flow head
        for w, transposed in ((self.params[0], False), (self.params[-1], True)):
            if w.dim() != 5 or w.shape[2] != 3:
                continue
            Cout, Cin = w.shape[0], w.shape[1]
            real_in, nout = (Cout, Cin) if transposed else (Cin, Cout)
            if 3 * real_in > (16 if transposed else 8) or nout not in (8, 16, 32):
                continue
            coutp = 16 if nout <= 16 else 32
            out = torch.empty(int(lib.vxm_conv3d_tcs_packed_bytes(3 * real_in, coutp, 1)) // 2, dtype=torch.bfloat16, device=dev)
            cnt = lib.vxm_conv3d_tcs_pack_desc_fold(ctypes.cast(ctypes.addressof(host) + n * dsz, ctypes.c_void_p), _lib.ptr(w), _lib.ptr(out),
                                                    Cout, Cin, coutp, 1 if transposed else 0, begin)
            if cnt <= 0:
                continue
            self.table[(id(w), transposed, "fold")] = (out, (coutp, "s"))
            self.keep.append(out)
            begin += cnt
            n += 1
        for li, w in enumerate(self.params):
            w5 = w if w.dim() == 5 else w.unsqueeze(2)
            Cout, Cin, kd = w5.shape[0], w5.shape[1], w5.shape[2]
            # a concatenating layer (decoder, after an upsample) reads the previous layer's output first, then the skip
            ca = self.params[li - 1].shape[0] if li and Cin > self.params[li - 1].shape[0] else Cin
            for transposed in (False, True):
                if transposed and li == 0:
                    continue                      # the images need no gradient: no dgrad of the first layer
                cin_eff, nout = (Cout, Cin) if transposed else (Cin, Cout)
                if li and Cout <= 64 and ca <= 64 and Cin - ca <= 64:
                    blocks = tc.conv_blocks(Cout, 0, Cin, int(kd), ca if ca < Cin else None) if transposed else \
                        tc.conv_blocks(ca, Cin - ca, Cout, int(kd))
                    if blocks is not None:        # channel-blocked layer: one operand per (K block, N block)
                        packs, n, begin = tc.block_descs(w, transposed, blocks, host, n, begin, dsz)
                        self.table[(id(w), transposed, "blk")] = (blocks, packs)
                        self.keep.extend(p[0] for p in packs.values())
                        continue
                if nout > 64 or cin_eff > 64:
                    continue
                coutp = 16 if nout <= 16 else (32 if nout <= 32 else (48 if nout <= 48 else 64))
                nbytes = int(lib.vxm_conv3d_tcs_packed_bytes(cin_eff, coutp, kd))
                out = torch.empty(nbytes // 2, dtype=torch.bfloat16, device=dev)
                cnt = lib.vxm_conv3d_tcs_pack_desc(ctypes.cast(ctypes.addressof(host) + n * dsz, ctypes.c_void_p), _lib.ptr(w), _lib.ptr(out),
                                                   Cout, Cin, kd, coutp, 1 if transposed else 0, begin)
                if cnt <= 0:
                    continue
                self.table[(id(w), transposed)] = (out, (coutp, "s"))
                self.keep.append(out)
                begin += cnt
                n += 1
        self.ndesc, self.total = n, begin
        self.descs = torch.frombuffer(bytearray(host.raw[:max(1, n) * dsz]), dtype=torch.uint8).to(dev)
        self.ptrs = tuple(w.data_ptr() for w in self.params)
        self.stamp = None

    def valid_for(self, model):
        return self.ptrs == tuple(w.data_ptr() for w in self.params)

    def refresh(self):
        stamp = (_weights_epoch, tuple(w._version for w in self.params))
        if stamp != self.stamp and self.ndesc:
            _lib.check(_lib.load().vxm_conv3d_tcs_pack_multi(_lib.ptr(self.descs), self.ndesc, self.total, _lib.stream_ptr()),
                       "vxm_conv3d_tcs_pack_multi")
            self.stamp = stamp

    def lookup(self, w, transposed):
        return self.table.get((id(w), transposed))

    def lookup_blocks(self, w, transposed, blocks):
        """Block operands of `w` packed for `blocks` (tc.conv_blocks), or None."""
        hit = self.table.get((id(w), transposed, "blk"))
        return hit[1] if hit is not None and hit[0] == blocks else None

    def lookup_fold(self, w, transposed):
        return self.table.get((id(w), transposed, "fold"))


def _plan_of(model):
    """The model's pack plan (built lazily; rebuilt when the parameters moved, e.g. after .to(device) or FlatParams)."""
    if tc._variant() not in ("auto", "s"):
        return None
    plan = model.__dict__.get("_vxm_pack_plan")
    if plan is None or not plan.valid_for(model):
        plan = _PackPlan(model)
        object.__setattr__(model, "_vxm_pack_plan", plan)
    plan.refresh()
    return plan


def supports(model):
    """True when every convolution of `model` (a VxmDense) runs in one launch per layer on the tensor-core kernels: feature
    counts in {8, 16, 32}, concatenated inputs a multiple of 16 and at most 64 channels, at most 8 image planes.  This is
    what VXM_B200_CONV_ENGINE=tc selects the tensor cores for; VXM_B200_CONV_ENGINE=bf16 | bf16x3 also run U-Nets with
    64-channel layers and concatenations of up to 128 channels, in channel blocks (tc.conv_blocks)."""
    try:
        unet = model.unet_model
        convs = [b.main for lvl in unet.encoder for b in lvl] + [b.main for lvl in unet.decoder for b in lvl] + \
                [b.main for b in unet.remaining]
        first = convs[0]
        if first.weight.shape[1] > 8 or first.weight.dim() not in (4, 5):
            return False
        for i, c in enumerate(convs):
            co, ci = c.weight.shape[0], c.weight.shape[1]
            if co not in (8, 16, 32):
                return False
            if i > 0 and (ci % 16 or ci > 64):
                return False
        fl = model.flow
        return fl.weight.shape[1] % 16 == 0 and fl.weight.shape[1] <= 64 and fl.weight.shape[0] <= 8
    except AttributeError:
        return False


def _check_cout(c, what):
    if c not in (8, 16, 32, 64):
        raise _lib.VxmError("bf16 tensor-core engine: %s has %d channels; supported feature counts are 8, 16, 32 and 64 "
                            "(use VXM_B200_CONV_ENGINE=f32 for other U-Net shapes)" % (what, c))


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


def _unpool_combine(e_fine, g_skip, g_pool, nd, slope):
    lib = _lib.load()
    B, D, H, W, C = e_fine.shape
    Dc = D // 2 if nd == 3 else D
    out = torch.empty_like(e_fine)
    _lib.check(lib.vxm_unpool_combine_ndhwc_bf16(_lib.ptr(e_fine), _lib.ptr(g_skip), _lib.ptr(g_pool), _lib.ptr(out), B, Dc, H // 2,
                                                 W // 2, C, nd, slope, _lib.stream_ptr()), "vxm_unpool_combine_ndhwc_bf16")
    return out


class _Conv:
    """One convolution of the tape: inputs, output, parameters."""
    __slots__ = ("w", "b", "planar", "xa", "xb", "up", "out", "slope", "cin", "cout", "a_id", "b_id", "out_id", "planar_out",
                 "xa_lo", "xb_lo", "fold")


def _run_conv_split(cv, kd):
    """Forward of one tape entry in split precision (three tensor-core passes, see tc.conv_fwd_split).  Returns the
    (hi, lo) output pair, or the fp32 planar flow."""
    def packs():
        wh, wl = tc.split_weights(cv.w)
        return tc.pack_weights_t(wh, variant="s"), tc.pack_weights_t(wl, variant="s")
    blocks = None if cv.planar_out else tc.conv_blocks(_width(cv.xa), _width(cv.xb), cv.cout, kd)
    if blocks is not None:
        def block_packs():
            sp = getattr(cv.w, "_vxm_split_blocks", None)       # persistent buffers: the refresh stays graph-capturable
            if sp is None or sp.blocks != blocks:
                sp = tc.SplitBlockPacks(cv.w, blocks)
                cv.w._vxm_split_blocks = sp
            return sp.refresh(cv.w)
        sp = _cache.get(cv.w, "fwd_split_blk", block_packs)
        return tc.conv_fwd_blocked(cv.xa, cv.xb, blocks, sp.hi, cv.b.detach() if cv.b is not None else None, cv.cout, kd, up=cv.up,
                                   slope=cv.slope, lo=(cv.xa_lo, cv.xb_lo, sp.lo))
    pk = _cache.get(cv.w, "fwd_split", packs)
    xa = None if cv.xa is None else (cv.xa, cv.xa_lo)
    xb = None if cv.xb is None else (cv.xb, cv.xb_lo)
    return tc.conv_fwd_split(xa, xb, pk, cv.b.detach() if cv.b is not None else None, cv.cout, kd, up=cv.up,
                             out_fp32_planar=cv.planar_out, slope=cv.slope)


def _width(x):
    return 0 if x is None else x.shape[-1]


def _block_packs(plan, cv, transposed, blocks):
    packs = plan.lookup_blocks(cv.w, transposed, blocks) if plan is not None else None
    if packs is None:
        raise _lib.VxmError("bf16 engine: the %d -> %d convolution runs in channel blocks, which need the swizzled kw-stacked "
                            "kernel (VXM_B200_TC_KERNEL=auto|s)" % (cv.cin, cv.cout))
    return packs


def _run_conv(cv, kd, plan=None):
    """Forward of one tape entry."""
    ca = 0 if cv.xa is None else cv.xa.shape[-1]
    cb = 0 if cv.xb is None else cv.xb.shape[-1]
    blocks = None if (cv.planar is not None or cv.fold == "x" or cv.planar_out) else tc.conv_blocks(ca, cb, cv.cout, kd)
    if blocks is not None:
        return tc.conv_fwd_blocked(cv.xa, cv.xb, blocks, _block_packs(plan, cv, False, blocks), cv.b.detach() if cv.b is not None else None,
                                   cv.cout, kd, up=cv.up, slope=cv.slope)
    if cv.fold == "x":
        # kd folded into the input channels: a 2-D convolution per slice (3 instead of 9 MMA steps per tile)
        wpk, cp = plan.lookup_fold(cv.w, False)
        return tc.conv_fwd_t(cv.xa, None, wpk, cp, cv.b.detach() if cv.b is not None else None, cv.cout, 1, slope=cv.slope)
    if cv.planar is None and tc.use_t_kernel(ca, cb, cv.cout):
        hit = plan.lookup(cv.w, False) if (plan is not None and tc._use_s(ca, cb, cv.cout)) else None
        wpk, cp = hit if hit is not None else _cache.get(cv.w, "fwd_t", lambda: tc.pack_weights_t(cv.w.detach()))
        return tc.conv_fwd_t(cv.xa, cv.xb, wpk, cp, cv.b.detach() if cv.b is not None else None, cv.cout, kd, up=cv.up,
                             out_fp32_planar=cv.planar_out, slope=cv.slope)
    wpk, NP = _cache.get(cv.w, "fwd", lambda: tc.pack_weights(cv.w.detach()))
    return tc.conv_fwd(cv.xa, cv.xb, wpk, NP, cv.b.detach() if cv.b is not None else None, cv.cout, kd, up=cv.up, planar=cv.planar,
                       out_fp32_planar=cv.planar_out, slope=cv.slope)


def forward_tape(model, source, target, split=False):
    """Runs Unet + flow head, returns (flow fp32 (B,nd,*vol), tape).  `split`: split-precision (bf16x3) forward — every
    activation is a (hi, lo) bf16 pair and every layer three tensor-core passes; the tape keeps the hi parts, which is
    what the (bf16-operand) backward reads."""
    unet = model.unet_model
    nd = source.dim() - 2
    kd = 3 if nd == 3 else 1
    _lib.require_cuda(source, target, what="VxmDense")
    source, target = _lib.contig(source), _lib.contig(target)
    planes = [source[:, i:i + 1] for i in range(source.shape[1])] + [target[:, i:i + 1] for i in range(target.shape[1])]
    if len(planes) > 8:
        raise _lib.VxmError("bf16 engine: at most 8 input feature planes (src_feats + trg_feats)")
    tape = []            # list of ("conv", _Conv) / ("pool", in_id, out_id)
    tensors = {}         # id -> bf16 NDHWC tensor
    lows = {}            # id -> lo part (split precision only)
    plan = None if split else _plan_of(model)
    producer = {}        # id -> "conv" | "pool"
    next_id = [0]

    def new_id():
        next_id[0] += 1
        return next_id[0]

    def conv(block_main, slope, planar=None, a_id=None, b_id=None, up=False, planar_out=False):
        cv = _Conv()
        cv.w, cv.b = block_main.weight, block_main.bias
        cv.planar = planar
        cv.xa = tensors[a_id] if a_id is not None else None
        cv.xb = tensors[b_id] if b_id is not None else None
        cv.up, cv.slope, cv.planar_out = up, slope, planar_out
        cv.cout, cv.cin = cv.w.shape[0], cv.w.shape[1]
        cv.a_id, cv.b_id = a_id, b_id
        cv.xa_lo = lows.get(a_id) if split else None
        cv.xb_lo = lows.get(b_id) if split else None
        cv.fold = "x" if (a_id is not None and producer.get(a_id) == "input" and fold_first) else None
        if not planar_out:
            _check_cout(cv.cout, "a U-Net convolution output")
        if planar is None:
            ca = 0 if cv.xa is None else cv.xa.shape[-1]
            cb = 0 if cv.xb is None else cv.xb.shape[-1]
            first_layer = cv.xa is not None and producer.get(a_id) == "input"
            if first_layer:
                if ca != 8 or cb or cv.cin > 8 or (cv.fold == "x" and 3 * cv.cin > 8):
                    raise _lib.VxmError("bf16 engine: the first convolution takes at most 8 input feature planes")
            elif ca + cb != cv.cin or (ca + cb) % 16 or ca + cb > (64 if planar_out else 128):
                raise _lib.VxmError("bf16 engine: unsupported convolution input channels %d (+%d); need a multiple of 16, at most 128 "
                                    "(64 into the flow head) (use VXM_B200_CONV_ENGINE=f32 for other U-Net shapes)" % (ca, cb))
        out = _run_conv_split(cv, kd) if split else _run_conv(cv, kd, plan)
        cv.out_id = new_id()
        if split and not planar_out:
            out, lows[cv.out_id] = out
        cv.out = out
        cv.xa_lo = cv.xb_lo = None      # the backward reads the hi parts only
        if not planar_out:
            tensors[cv.out_id] = out
            producer[cv.out_id] = "conv"
        tape.append(("conv", cv))
        return cv.out_id

    def pool(in_id):
        oid = new_id()
        if split:
            y, lows[oid] = tc.pool_split((tensors[in_id], lows[in_id]), nd)
        else:
            y = _pool(tensors[in_id], nd)
        return _pool_done(y, in_id, oid)

    def _pool_done(y, in_id, oid):
        tensors[oid] = y
        producer[oid] = "pool"
        tape.append(("pool", in_id, oid))
        return oid

    # the fp32 images enter as one bf16 channels-last tensor with 8 channels (src planes, trg planes, zeros)
    cur = new_id()
    first_w = unet.encoder[0][0].main.weight
    fold_first = (not split and nd == 3 and tc.kdfold_enabled() and plan is not None and plan.lookup_fold(first_w, False) is not None
                  and first_w.shape[1] == len(planes) and tc._variant() in ("auto", "s"))
    if split:
        tensors[cur], lows[cur] = tc.planar_to_ndhwc8_split(planes)
    elif fold_first:
        tensors[cur] = tc.planar_fold_kd(planes, 8)      # (kd, plane) channels: the first convolution runs as 2-D
    else:
        tensors[cur] = tc.planar_to_ndhwc8(planes)
    producer[cur] = "input"
    skips = [None]
    for level, convs in enumerate(unet.encoder):
        for blk in convs:
            slope = blk.activation.negative_slope
            cur = conv(blk.main, slope, a_id=cur)
        skips.append(cur)
        cur = pool(cur)
    pending_up = None    # (a_id, skip_id) to be consumed by the next convolution as a fused upsample+concat
    for level, convs in enumerate(unet.decoder):
        for blk in convs:
            slope = blk.activation.negative_slope
            if pending_up is not None:
                cur = conv(blk.main, slope, a_id=pending_up[0], b_id=pending_up[1], up=True)
                pending_up = None
            else:
                cur = conv(blk.main, slope, a_id=cur)
        if not unet.half_res or level < (unet.nb_levels - 2):
            pending_up = (cur, skips.pop())
    for blk in unet.remaining:
        slope = blk.activation.negative_slope
        if pending_up is not None:
            cur = conv(blk.main, slope, a_id=pending_up[0], b_id=pending_up[1], up=True)
            pending_up = None
        else:
            cur = conv(blk.main, slope, a_id=cur)
    # flow head (no activation, fp32 planar output)
    if pending_up is not None:
        fid = conv(model.flow, None, a_id=pending_up[0], b_id=pending_up[1], up=True, planar_out=True)
    else:
        fid = conv(model.flow, None, a_id=cur, planar_out=True)
    flow = tape[-1][1].out
    if nd == 2:
        flow = flow.squeeze(2)
    return flow, dict(tape=tape, tensors=tensors, producer=producer, nd=nd, kd=kd, plan=_plan_of(model) if split else plan)


def backward_tape(ctx, g_flow):
    """Hand-written backward over the tape.  Returns {param: grad}."""
    lib = _lib.load()
    tape, tensors, producer, nd, kd = ctx["tape"], ctx["tensors"], ctx["producer"], ctx["nd"], ctx["kd"]
    plan = ctx.get("plan")
    g_flow = _lib.contig(g_flow.float())
    if nd == 2:
        g_flow = g_flow.unsqueeze(2)
    batch = tc.WgradBatch.get(g_flow.device)
    batch.reset()
    gz = {}       # conv-output id -> masked gradient (bf16 NDHWC)
    graw = {}     # pool-output id -> raw gradient
    gskip = {}    # encoder-output id -> raw skip gradient
    grads = {}
    dev = g_flow.device
    folded = []   # (conv, gw2d, gb2d, kind): 2-D weight gradients of the kd-folded layers, mapped back after the flush
    for entry in reversed(tape):
        if entry[0] == "pool":
            _, in_id, out_id = entry
            e = tensors[in_id]
            gz[in_id] = _unpool_combine(e, gskip.pop(in_id, None), graw.pop(out_id), nd, _slope_of(ctx, in_id))
            continue
        cv = entry[1]
        fold_g = (cv.planar_out and nd == 3 and tc.kdfold_enabled() and plan is not None and plan.lookup_fold(cv.w, True) is not None
                  and cv.xb is None and not cv.up and cv.xa is not None and cv.xa.shape[-1] in (8, 16) and cv.xa.shape[-1] == cv.cin
                  and producer.get(cv.a_id) == "conv" and tc._variant() in ("auto", "s"))
        if fold_g:
            # flow head, kd folded into the channels of the flow gradient: (kd', component) = 9 of 16 channels
            g_in = tc.planar_fold_kd([g_flow[:, i:i + 1] for i in range(g_flow.shape[1])], 16)
            gwf = torch.empty((3 * nd, cv.cin, 1, 3, 3), dtype=torch.float32, device=dev)
            gbf = torch.empty(3 * nd, dtype=torch.float32, device=dev) if cv.b is not None else None
            batch.add_khm(cv.xa, g_in, gwf, gbf, cv.cin, 3 * nd)
            folded.append((cv, gwf, gbf, "g"))
            t = cv.a_id
            wpk, cp = plan.lookup_fold(cv.w, True)
            gz[t] = tc.conv_fwd_t(g_in, None, wpk, cp, None, cv.cin, 1, slope=_slope_of(ctx, t), mask=tensors[t])
            continue
        if cv.planar_out:
            # flow head: the fp32 planar flow gradient becomes an 8-channel bf16 channels-last tensor
            g_in = tc.planar_to_ndhwc8([g_flow[:, i:i + 1] for i in range(g_flow.shape[1])])
        else:
            g_in = gz.pop(cv.out_id)
        if cv.fold == "x":
            # first layer over the kd-folded images: 2-D weight gradient with kh in M, no dgrad
            gwf = torch.empty((cv.cout, 3 * cv.cin, 1, 3, 3), dtype=torch.float32, device=dev)
            gbf = torch.empty(cv.cout, dtype=torch.float32, device=dev) if cv.b is not None else None
            if g_in.shape[-1] <= 16:
                batch.add_khm(cv.xa, g_in, gwf, gbf, 3 * cv.cin, cv.cout)
            else:      # kh-in-M takes at most 16 output channels: a wider first layer runs the plain 2-D kernel
                batch.add(cv.xa, None, g_in, gwf, gbf, 3 * cv.cin, cv.cout, 1, False, False)
            folded.append((cv, gwf, gbf, "x"))
            continue
        # parameters whose .grad is a view of FusedAdam's flat gradient buffer (optim.FlatParams marks them)
        # are accumulated into directly by the reduce kernel; autograd then receives no gradient for them
        direct = (getattr(cv.w, "_vxm_flat_grad", False) and cv.w.grad is not None and cv.w.grad.is_contiguous()
                  and (cv.b is None or (getattr(cv.b, "_vxm_flat_grad", False) and cv.b.grad is not None)))
        if direct:
            tc.conv_wgrad(cv.xa, cv.xb, g_in, cv.cin, cv.cout, kd, up=cv.up, planar_x=cv.planar,
                          out_w=cv.w.grad, out_b=None if cv.b is None else cv.b.grad, batch=batch)
        else:
            gw, gb = tc.conv_wgrad(cv.xa, cv.xb, g_in, cv.cin, cv.cout, kd, up=cv.up, planar_x=cv.planar, batch=batch)
            grads[cv.w] = gw.squeeze(2) if nd == 2 else gw
            if cv.b is not None:
                grads[cv.b] = gb
        g_in_planar = None
        # ---- dgrad ----
        if cv.planar is not None or producer.get(cv.a_id) == "input":
            continue       # first layer: the images need no gradient
        w = cv.w.detach()
        if cv.b_id is None:
            t = cv.a_id
            msk = tensors[t] if producer[t] == "conv" else None
            sl = _slope_of(ctx, t) if producer[t] == "conv" else None
            blocks = tc.conv_blocks(g_in.shape[-1], 0, cv.cin, kd)
            if blocks is not None:
                res = tc.conv_fwd_blocked(g_in, None, blocks, _block_packs(plan, cv, True, blocks), None, cv.cin, kd, slope=sl, mask=msk)
            elif tc.use_t_kernel(g_in.shape[-1], 0, cv.cin):
                hit = plan.lookup(cv.w, True) if (plan is not None and tc._use_s(g_in.shape[-1], 0, cv.cin)) else None
                wpk, cp = hit if hit is not None else _cache.get(cv.w, "dgrad_t", lambda: tc.pack_weights_t(w, transposed=True))
                res = tc.conv_fwd_t(g_in, None, wpk, cp, None, cv.cin, kd, slope=sl, mask=msk)
            else:
                wpk, NP = _cache.get(cv.w, "dgrad", lambda: tc.pack_weights(w, transposed=True))
                res = tc.conv_fwd(g_in, None, wpk, NP, None, cv.cin, kd, planar=g_in_planar, slope=sl, mask=msk)
            if producer[t] == "conv":
                gz[t] = res
            else:
                graw[t] = res
        else:
            ca = cv.xa.shape[-1]
            # single dgrad pass over the whole concat input: N = Ca + Cb output channels, split on store
            blocks = tc.conv_blocks(g_in.shape[-1], 0, cv.cin, kd, ca)
            if blocks is not None:
                g_up, g_sk = tc.conv_fwd_blocked(g_in, None, blocks, _block_packs(plan, cv, True, blocks), None, cv.cin, kd, split=ca)
            elif tc.use_t_kernel(g_in.shape[-1], 0, cv.cin):
                hit = plan.lookup(cv.w, True) if (plan is not None and tc._use_s(g_in.shape[-1], 0, cv.cin)) else None
                wpk, cp = hit if hit is not None else _cache.get(cv.w, "dgrad_t", lambda: tc.pack_weights_t(w, transposed=True))
                g_up, g_sk = tc.conv_fwd_t(g_in, None, wpk, cp, None, cv.cin, kd, split=ca)
            else:
                wpk, NP = _cache.get(cv.w, "dgrad", lambda: tc.pack_weights(w, transposed=True))
                g_up, g_sk = tc.conv_fwd(g_in, None, wpk, NP, None, cv.cin, kd, planar=g_in_planar, split=ca)
            gz[cv.a_id] = _sumpool_mask(g_up, tensors[cv.a_id], nd, _slope_of(ctx, cv.a_id))   # grad wrt upsample(a): sum children
            del g_up
            gskip[cv.b_id] = g_sk
    batch.flush()     # one launch reduces every layer's per-CTA partials (fixed order: deterministic)
    for cv, gwf, gbf, kind in folded:
        if kind == "x":
            gw, gb = unfold_grad_first(gwf, cv.cout, cv.cin), gbf
        else:
            gw, gb = unfold_grad_flow(gwf, gbf, nd, cv.cin)
        direct = (getattr(cv.w, "_vxm_flat_grad", False) and cv.w.grad is not None
                  and (cv.b is None or (getattr(cv.b, "_vxm_flat_grad", False) and cv.b.grad is not None)))
        if direct:
            cv.w.grad.add_(gw)
            if cv.b is not None:
                cv.b.grad.add_(gb)
        else:
            grads[cv.w] = gw.contiguous()
            if cv.b is not None:
                grads[cv.b] = gb.contiguous()
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


def _slope_of(ctx, tid):
    for entry in ctx["tape"]:
        if entry[0] == "conv" and entry[1].out_id == tid:
            s = entry[1].slope
            return -1.0 if s is None else float(s)
    return -1.0


class _UnetFlowFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, source, target, split, *params):
        flow, tape = forward_tape(model, source, target, split=split)
        ctx.tape = tape
        ctx.params = params
        ctx.model_ref = model
        return flow

    @staticmethod
    def backward(ctx, g_flow):
        dp = getattr(ctx.model_ref, "_dp", None)
        if dp is not None:
            dp.schedule()      # gradients written straight into .grad views bypass the parameter hooks
        grads = backward_tape(ctx.tape, g_flow)
        ctx.tape = None
        return (None, None, None, None) + tuple(grads.get(p) for p in ctx.params)


def unet_flow(model, source, target, split=False):
    """flow = model.flow(model.unet_model(cat(source, target))) on the tensor-core engine.  split=False: bf16 operands
    (throughput mode); split=True: bf16x3 split precision in the forward (flow within 1e-4 of the fp32 reference), the
    backward uses bf16 operands in both modes."""
    params = [p for p in list(model.unet_model.parameters()) + list(model.flow.parameters())]
    return _UnetFlowFn.apply(model, source, target, bool(split), *params)
