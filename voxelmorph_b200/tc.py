"""Host wrappers of the wgmma implicit-GEMM convolution engine (csrc/conv3d_tc.cu, csrc/conv3d_tc_wgrad.cu).

Activations of this engine are bf16, channels-last: a (B, C, D, H, W) logical tensor is held as a contiguous
(B, D, H, W, C) bf16 tensor (`ndhwc`).  Weights stay fp32 in the nn.Module (reference layout
(Cout, Cin, 3, 3, 3)); packed bf16 copies are refreshed whenever the parameter version changes.
"""
import ctypes
import functools
import threading

import torch

from . import _lib


def np_for(cout):
    """MMA N (16, 32, 48 or 64) for a launch with `cout` output channels (wider layers: conv_blocks)."""
    if cout <= 16:
        return 16
    if cout <= 32:
        return 32
    if cout <= 48:
        return 48
    if cout <= 64:
        return 64
    raise _lib.VxmError("tensor-core conv engine: at most 64 output channels per launch (got %d)" % cout)


def to_ndhwc_bf16(x):
    """(B,C,D,H,W) fp32 -> (B,D,H,W,C) bf16 contiguous (test / boundary helper; torch copy kernels)."""
    return x.permute(0, 2, 3, 4, 1).contiguous().to(torch.bfloat16)


def from_ndhwc(x):
    return x.permute(0, 4, 1, 2, 3).float().contiguous()


def pack_weights(w, transposed=False):
    """fp32 (Cout, Cin, kd, 3, 3) -> packed bf16 operand for vxm_conv3d_tc_fwd (dgrad operator if transposed)."""
    lib = _lib.load()
    if w.dim() == 4:
        w = w.unsqueeze(2)
    w = w.contiguous()
    Cout, Cin, kd = w.shape[0], w.shape[1], w.shape[2]
    cin_eff, nout = (Cout, Cin) if transposed else (Cin, Cout)
    NP = np_for(nout)
    nbytes = int(lib.vxm_conv3d_tc_packed_bytes(cin_eff, NP, kd))
    out = torch.empty(nbytes // 2, dtype=torch.bfloat16, device=w.device)
    _lib.check(lib.vxm_conv3d_tc_pack(_lib.ptr(w), _lib.ptr(out), Cout, Cin, kd, NP, 1 if transposed else 0,
                                      _lib.stream_ptr()), "vxm_conv3d_tc_pack")
    return out, NP


def conv_fwd(xa, xb, wpk, NP, bias, cout, kd, up=False, planar=None, out_fp32_planar=False, slope=None, mask=None, split=None):
    """Launch the tensor-core convolution.  xa / xb: bf16 NDHWC tensors (xa at half resolution when `up`);
    planar: list of <= 4 fp32 (B,1,D,H,W) tensors used instead of xa/xb.  Returns bf16 NDHWC (B,D,H,W,cout)
    or, with out_fp32_planar, fp32 (B,cout,D,H,W)."""
    lib = _lib.load()
    if planar is not None:
        ref = planar[0]
        B, D, H, W = ref.shape[0], ref.shape[-3] if ref.dim() == 5 else 1, ref.shape[-2], ref.shape[-1]
        arr_p = (ctypes.c_void_p * 4)(*([p.data_ptr() for p in planar] + [0] * (4 - len(planar))))
        arr_s = (ctypes.c_longlong * 4)(*([p.stride(0) for p in planar] + [0] * (4 - len(planar))))
        xf, xs, npl, Ca, Cb = arr_p, arr_s, len(planar), 0, 0
        dev = ref.device
    else:
        full = xb if xb is not None else xa
        B, D, H, W = full.shape[0], full.shape[1], full.shape[2], full.shape[3]
        if xb is None and up:
            D, H, W = (D * 2 if kd == 3 else D), H * 2, W * 2
        Ca = 0 if xa is None else xa.shape[-1]
        Cb = 0 if xb is None else xb.shape[-1]
        xf, xs, npl = None, None, 0
        dev = full.device
    out2 = None
    if out_fp32_planar:
        out = torch.empty((B, cout, D, H, W), dtype=torch.float32, device=dev)
    elif split:
        out = torch.empty((B, D, H, W, split), dtype=torch.bfloat16, device=dev)
        out2 = torch.empty((B, D, H, W, cout - split), dtype=torch.bfloat16, device=dev)
    else:
        out = torch.empty((B, D, H, W, cout), dtype=torch.bfloat16, device=dev)
    s = -1.0 if slope is None else float(slope)
    _lib.check(lib.vxm_conv3d_tc_fwd(_lib.ptr(xa), _lib.ptr(xb), xf, xs, npl, _lib.ptr(wpk), _lib.ptr(bias), _lib.ptr(out),
                                     _lib.ptr(mask), B, D, H, W, Ca, Cb, 1 if up else 0, cout, NP, kd,
                                     1 if out_fp32_planar else 0, s, _lib.ptr(out2), int(split or 0), _lib.stream_ptr()),
               "vxm_conv3d_tc_fwd")
    return (out, out2) if split else out


def _planar_args(planar):
    if planar is None:
        return None, None, 0
    arr_p = (ctypes.c_void_p * 4)(*([p.data_ptr() for p in planar] + [0] * (4 - len(planar))))
    arr_s = (ctypes.c_longlong * 4)(*([p.stride(0) for p in planar] + [0] * (4 - len(planar))))
    return arr_p, arr_s, len(planar)


_wgrad_ws = {}
_ws_lock = threading.Lock()      # workspace tables are shared by the per-GPU threads of nn.DataParallel


def conv_wgrad(xa, xb, gz, cin, cout, kd, up=False, planar_x=None, planar_g=None, need_bias=True, out_w=None, out_b=None, batch=None):
    """fp32 grad_w (cout, cin, kd, 3, 3) and grad_b (cout) from the layer input (xa/xb or planar_x) and gz.
    `batch` (a WgradBatch; channels-last sources only): only the wgmma partial-sum kernels are launched now, the reduction
    into gw / gb happens at `batch.flush()` together with every other layer's."""
    lib = _lib.load()
    ref = gz if gz is not None else planar_g[0]
    dev = ref.device
    # out_w / out_b: existing (contiguous fp32) gradient buffers to ACCUMULATE into instead of fresh tensors
    accumulate = out_w is not None
    gw = out_w if accumulate else torch.empty((cout, cin, kd, 3, 3), dtype=torch.float32, device=dev)
    gb = out_b if accumulate else (torch.empty(cout, dtype=torch.float32, device=dev) if need_bias else None)
    if batch is not None:
        batch.add(xa, xb, gz, gw, gb, cin, cout, kd, up, accumulate)
        return gw, gb
    if gz is not None:
        B, D, H, W, Cg = gz.shape
    else:
        B, D, H, W, Cg = ref.shape[0], (ref.shape[-3] if ref.dim() == 5 else 1), ref.shape[-2], ref.shape[-1], 8
    key = (dev.index, torch.cuda.current_stream(dev).cuda_stream, kd)
    work = _wgrad_ws.get(key)
    if work is None:
        with _ws_lock:
            work = _wgrad_ws.get(key)
            if work is None:
                work = torch.empty(int(lib.vxm_conv3d_tc_wgrad_workspace_bytes(kd)), dtype=torch.uint8, device=dev)
                _wgrad_ws[key] = work
    xf, xs, npx = _planar_args(planar_x)
    gf, gs, npg = _planar_args(planar_g)
    Ca = 0 if xa is None else xa.shape[-1]
    Cb = 0 if xb is None else xb.shape[-1]
    _lib.check(lib.vxm_conv3d_tc_wgrad(_lib.ptr(xa), _lib.ptr(xb), xf, xs, npx, _lib.ptr(gz), gf, gs, npg, _lib.ptr(gw),
                                       _lib.ptr(gb), _lib.ptr(work), B, D, H, W, Ca, Cb, 1 if up else 0, cin, Cg, cout, kd,
                                       1 if accumulate else 0, _lib.stream_ptr()), "vxm_conv3d_tc_wgrad")
    return gw, gb


def planar_to_ndhwc8(planes):
    """<= 8 planar fp32 (B,1,[D,]H,W) volumes -> one bf16 (B,D,H,W,8) tensor (unused channels zero)."""
    lib = _lib.load()
    ref = planes[0]
    B = ref.shape[0]
    D, H, W = (ref.shape[-3] if ref.dim() == 5 else 1), ref.shape[-2], ref.shape[-1]
    n = len(planes)
    arr_p = (ctypes.c_void_p * 8)(*([p.data_ptr() for p in planes] + [0] * (8 - n)))
    arr_s = (ctypes.c_longlong * 8)(*([p.stride(0) for p in planes] + [0] * (8 - n)))
    out = torch.empty((B, D, H, W, 8), dtype=torch.bfloat16, device=ref.device)
    _lib.check(lib.vxm_planar_to_ndhwc8_bf16(arr_p, arr_s, n, _lib.ptr(out), B, D * H * W, _lib.stream_ptr()),
               "vxm_planar_to_ndhwc8_bf16")
    return out


def kdfold_enabled():
    """kd-folded execution of the two layers with 2 / 3 real channels on one side (VXM_B200_KDFOLD=0: A/B switch)."""
    import os
    return os.environ.get("VXM_B200_KDFOLD", "1") != "0"


def polyphase_enabled():
    """Polyphase execution of the 3-D concat layers with a 32-channel upsampled source (VXM_B200_POLYPHASE=0: A/B
    switch back to the 27-tap forms over the duplicated slices)."""
    import os
    return os.environ.get("VXM_B200_POLYPHASE", "1") != "0"


def pack_weights_poly(w, mode, ca):
    """Packed polyphase operand (vxm_conv3d_tcs_pack_desc_poly) of the 3-D weight w (Cout, Cin, 3, 3, 3) of a concat
    layer whose first `ca` input channels are upsampled: mode 1 forward, 2 coarse dgrad.  Stand-alone helper (tests /
    tools); the engine packs through its model plan."""
    table = PackTable([(w.contiguous(), mode == 2, ("poly", mode, ca))])
    table.refresh()
    torch.cuda.current_stream(w.device).synchronize()       # the descriptor table must outlive the launch
    return table.packs[0][0, 0][0]


def conv_fwd_poly(xa, xb, wpk, bias, cout, slope):
    """Forward of a (32 upsampled + 16) -> 32 concat layer on its polyphase operand: xa the coarse source, xb the skip
    (B, D, H, W, 16); bias + LeakyReLU; returns bf16 (B, D, H, W, cout)."""
    lib = _lib.load()
    B, D, H, W = xb.shape[:4]
    out = torch.empty((B, D, H, W, cout), dtype=torch.bfloat16, device=xb.device)
    _lib.check(lib.vxm_conv3d_tcs_poly(_lib.ptr(xa), _lib.ptr(xb), _lib.ptr(wpk), _lib.ptr(bias), _lib.ptr(out), None, B, D, H, W,
                                       xa.shape[-1], xb.shape[-1], cout, 1, float(slope), _lib.stream_ptr()), "vxm_conv3d_tcs_poly")
    return out


def dgrad_poly(g, wpk, act, slope):
    """Coarse dgrad on the polyphase operand: g (B, D, H, W, 32) the layer's output gradient, act (B, D / 2, H / 2, W / 2, C)
    the upsampled source, a LeakyReLU activation of negative slope `slope` -> bf16 (B, D / 2, H / 2, W / 2, C), the gradient
    w.r.t. that source's pre-activation (sum over its 8 children, times the LeakyReLU derivative)."""
    lib = _lib.load()
    B, D, H, W, C = g.shape
    out = torch.empty_like(act)
    _lib.check(lib.vxm_conv3d_tcs_poly(_lib.ptr(g), None, _lib.ptr(wpk), None, _lib.ptr(out), _lib.ptr(act), B, D, H, W, C, 0,
                                       act.shape[-1], 2, float(slope), _lib.stream_ptr()), "vxm_conv3d_tcs_poly")
    return out


def planar_fold_kd(planes, cout):
    """<= cout/3 planar fp32 (B,1,D,H,W) volumes -> bf16 (B,D,H,W,cout) with channel kd * n + p = plane p at slice d + kd - 1
    (zero outside the volume): the kd taps of a 3-D convolution folded into the channels (csrc/ndhwc_ops.cu)."""
    lib = _lib.load()
    ref = planes[0]
    B, D, H, W = ref.shape[0], ref.shape[-3], ref.shape[-2], ref.shape[-1]
    n = len(planes)
    arr_p = (ctypes.c_void_p * 8)(*([p.data_ptr() for p in planes] + [0] * (8 - n)))
    arr_s = (ctypes.c_longlong * 8)(*([p.stride(0) for p in planes] + [0] * (8 - n)))
    out = torch.empty((B, D, H, W, cout), dtype=torch.bfloat16, device=ref.device)
    _lib.check(lib.vxm_planar_fold_kd_bf16(arr_p, arr_s, n, _lib.ptr(out), B, D, H * W, cout, _lib.stream_ptr()), "vxm_planar_fold_kd_bf16")
    return out


def pack_weights_fold(w, transposed=False):
    """Packed kd-folded 2-D operand of the 3-D weight w (Cout, Cin, 3, 3, 3) (see vxm_conv3d_tcs_pack_desc_fold).
    Returns (tensor, (coutp, "s")).  Stand-alone helper (tests / tools); the engine packs through its model plan."""
    table = PackTable([(w.contiguous(), transposed, "fold")])
    table.refresh()
    torch.cuda.current_stream(w.device).synchronize()       # the descriptor table must outlive the launch
    out, coutp = table.packs[0][0, 0]
    return out, (coutp, "s")


# ---- kw-stacked kernels: variant "s" (swizzled operands; what the engine runs) and "t" (SWIZZLE_NONE operands) ----------

def pack_weights_t(w, transposed=False, variant="s"):
    """Packed weights for a kw-stacked kernel.  Returns (tensor, (coutp, variant))."""
    lib = _lib.load()
    if w.dim() == 4:
        w = w.unsqueeze(2)
    w = w.contiguous()
    Cout, Cin, kd = w.shape[0], w.shape[1], w.shape[2]
    cin_eff, nout = (Cout, Cin) if transposed else (Cin, Cout)
    coutp = 16 if nout <= 16 else (32 if nout <= 32 else (48 if nout <= 48 else 64))
    fb, fp = (lib.vxm_conv3d_tcs_packed_bytes, lib.vxm_conv3d_tcs_pack) if variant == "s" else \
             (lib.vxm_conv3d_tct_packed_bytes, lib.vxm_conv3d_tct_pack)
    nbytes = int(fb(cin_eff, coutp, kd))
    out = torch.empty(nbytes // 2, dtype=torch.bfloat16, device=w.device)
    _lib.check(fp(_lib.ptr(w), _lib.ptr(out), Cout, Cin, kd, coutp, 1 if transposed else 0, _lib.stream_ptr()),
               "vxm_conv3d_tc%s_pack" % variant)
    return out, (coutp, variant)


def conv_fwd_t(xa, xb, wpk, coutp, bias, cout, kd, up=False, out_fp32_planar=False, slope=None, mask=None, split=None):
    lib = _lib.load()
    coutp, variant = coutp if isinstance(coutp, tuple) else (coutp, "t")
    fwd = lib.vxm_conv3d_tcs_fwd if variant == "s" else lib.vxm_conv3d_tct_fwd
    full = xb if xb is not None else xa
    B, D, H, W = full.shape[0], full.shape[1], full.shape[2], full.shape[3]
    if xb is None and up:
        D, H, W = (D * 2 if kd == 3 else D), H * 2, W * 2
    Ca = 0 if xa is None else xa.shape[-1]
    Cb = 0 if xb is None else xb.shape[-1]
    dev = full.device
    out2 = None
    if out_fp32_planar:
        out = torch.empty((B, cout, D, H, W), dtype=torch.float32, device=dev)
    elif split:
        out = torch.empty((B, D, H, W, split), dtype=torch.bfloat16, device=dev)
        out2 = torch.empty((B, D, H, W, cout - split), dtype=torch.bfloat16, device=dev)
    else:
        out = torch.empty((B, D, H, W, cout), dtype=torch.bfloat16, device=dev)
    s = -1.0 if slope is None else float(slope)
    _lib.check(fwd(_lib.ptr(xa), _lib.ptr(xb), _lib.ptr(wpk), _lib.ptr(bias), _lib.ptr(out), _lib.ptr(mask),
                   B, D, H, W, Ca, Cb, 1 if up else 0, cout, coutp, kd, 1 if out_fp32_planar else 0, s,
                   _lib.ptr(out2), int(split or 0), _lib.stream_ptr()), "vxm_conv3d_tc%s_fwd" % variant)
    return (out, out2) if split else out


# ---- channel-blocked execution of the layers one launch cannot hold (64 -> 64, 128 -> 64, ...) -------------------------

@functools.lru_cache(maxsize=None)
def conv_blocks(ca, cb, nout, kd, split=None):
    """Channel blocks of a convolution with inputs xa (ca channels) + xb (cb) and `nout` outputs (split: the first
    `split` outputs go to one tensor, the rest to another), or None when one launch of the kw-stacked kernel takes it.
    Returns (K blocks [(src, k0, kb)], N blocks [(n0, nb, dst, doff)]): src 0 = xa alone, 1 = xb alone, 2 = both; output
    channels [n0, n0 + nb) land in output `dst` at channel `doff`.  A concatenation over 64 channels is split at the
    source boundary (sources have at most 64 channels), the 64-channel source last: its launch runs the epilogue.  Output
    blocks are 64 channels wide where the packed weights of one leave room for the slab ring, else 32 (3-D, 64-channel K)."""
    lib = _lib.load()
    cin = ca + cb
    if cin <= 64 and nout <= 64 and lib.vxm_conv3d_tcs_fits(cin, np_for(nout), kd):
        return None
    if cin <= 64:
        ks = ((2, 0, cin),)
    else:
        ks = ((0, 0, ca), (1, ca, cb))
        if ca == 64 and cb != 64:
            ks = ks[::-1]
    nbmax = 64 if lib.vxm_conv3d_tcs_fits(max(k[2] for k in ks), 64, kd) else 32
    pieces = [(0, split, 0), (split, nout - split, 1)] if split else [(0, nout, 0)]
    return ks, tuple((p0 + j, min(nbmax, pn - j), dst, j) for p0, pn, dst in pieces for j in range(0, pn, nbmax))


def one_block(cin, nout):
    """The 1 x 1 block grid (see conv_blocks) of a convolution that runs as one launch per pass: `cin` input channels of
    the weight operand (the input tensor may pad them), `nout` outputs."""
    return ((2, 0, cin),), ((0, nout, 0, 0),)


class PackTable:
    """Packed bf16 operands of several weights, all refreshed by ONE vxm_conv3d_tcs_pack_multi launch.  `operands`:
    [(w, transposed, form)] with form "fold" (the kd-folded 2-D operand of a 3-D weight, see vxm_conv3d_tcs_pack_desc_fold),
    ("poly", mode, ca) (a polyphase operand, see vxm_conv3d_tcs_pack_desc_poly) or channel blocks (conv_blocks,
    one_block).  packs[i] = {(ki, ni): (tensor, coutp)} of operand i ((0, 0) for a folded or polyphase one).  The
    descriptor table is uploaded once and points at the (contiguous fp32) weights themselves, so `refresh` repacks their
    current values and can be captured in a CUDA graph."""

    def __init__(self, operands):
        lib = _lib.load()
        dsz = int(lib.vxm_conv3d_tcs_pack_desc_bytes())
        host = ctypes.create_string_buffer(dsz * sum(1 if f == "fold" or f[0] == "poly" else len(f[0]) * len(f[1]) for _, _, f in operands))
        self.packs, self.n, self.total = [], 0, 0
        for w, transposed, form in operands:
            w5 = w if w.dim() == 5 else w.unsqueeze(2)
            Cout, Cin, kd = w5.shape[0], w5.shape[1], w5.shape[2]
            t = 1 if transposed else 0
            packs = {}
            if form != "fold" and form[0] == "poly":
                _, mode, ca = form
                out = torch.empty(int(lib.vxm_conv3d_tcs_poly_packed_bytes(mode, Cout, Cin, ca)) // 2, dtype=torch.bfloat16, device=w.device)
                cnt = lib.vxm_conv3d_tcs_pack_desc_poly(self._slot(host, dsz), _lib.ptr(w5), _lib.ptr(out), Cout, Cin, ca, mode, self.total)
                self._add(packs, (0, 0), out, 32, cnt)
            elif form == "fold":
                real_in, nout = (Cout, Cin) if transposed else (Cin, Cout)
                coutp = 16 if nout <= 16 else 32
                out = torch.empty(int(lib.vxm_conv3d_tcs_packed_bytes(3 * real_in, coutp, 1)) // 2, dtype=torch.bfloat16, device=w.device)
                cnt = lib.vxm_conv3d_tcs_pack_desc_fold(self._slot(host, dsz), _lib.ptr(w5), _lib.ptr(out), Cout, Cin, coutp, t, self.total)
                self._add(packs, (0, 0), out, coutp, cnt)
            else:
                for ki, (_, k0, kb) in enumerate(form[0]):
                    for ni, (n0, nb, _, _) in enumerate(form[1]):
                        coutp = np_for(nb)
                        out = torch.empty(int(lib.vxm_conv3d_tcs_packed_bytes(kb, coutp, kd)) // 2, dtype=torch.bfloat16, device=w.device)
                        cnt = lib.vxm_conv3d_tcs_pack_desc_blk(self._slot(host, dsz), _lib.ptr(w5), _lib.ptr(out), Cout, Cin, kd, coutp, t,
                                                               n0, nb, k0, kb, self.total)
                        self._add(packs, (ki, ni), out, coutp, cnt)
            self.packs.append(packs)
        self.descs = torch.frombuffer(bytearray(host.raw), dtype=torch.uint8).to(operands[0][0].device)

    def _slot(self, host, dsz):
        return ctypes.cast(ctypes.addressof(host) + self.n * dsz, ctypes.c_void_p)

    def _add(self, packs, key, out, coutp, cnt):
        if cnt <= 0:
            raise _lib.VxmError("vxm_conv3d_tcs_pack_desc: %s" % _lib.last_error())
        packs[key] = (out, coutp)
        self.n, self.total = self.n + 1, self.total + cnt

    def refresh(self):
        _lib.check(_lib.load().vxm_conv3d_tcs_pack_multi(_lib.ptr(self.descs), self.n, self.total, _lib.stream_ptr()),
                   "vxm_conv3d_tcs_pack_multi")


def pack_weights_blocks(w, transposed, blocks):
    """Packed block operands of one weight (one launch).  Returns {(ki, ni): (tensor, coutp)}; the descriptor table stays
    referenced by the result (key None) until the launch has read it."""
    table = PackTable([(w.contiguous(), transposed, blocks)])
    table.refresh()
    packs = table.packs[0]
    packs[None] = table
    return packs


def _ptr_at(t, off):
    return None if t is None else ctypes.c_void_p(t.data_ptr() + off * t.element_size())


def conv_fwd_blocked(xa, xb, blocks, packs, bias, nout, kd, up=False, slope=None, mask=None, split=None, lo=None, out_fp32_planar=False):
    """One convolution in channel blocks (see conv_blocks); packs[(ki, ni)] = (operand, coutp) of K block ki, N block ni.
    Every N block accumulates its K blocks in an fp32 channels-last buffer (out_mode 2) and the last launch adds bias and
    activation (or the LeakyReLU-derivative mask) and stores its channels into the full-width bf16 output.
    lo = (xa_lo, xb_lo, packs_lo): split precision (bf16x3), three passes per K block, x_lo * w_hi + x_hi * w_lo +
    x_hi * w_hi (smallest terms first); returns the (hi, lo) pair, or with out_fp32_planar (one N block) the fp32 planar
    (B, nout, D, H, W) output.  A 1 x 1 grid (one_block) is the split-precision form of a layer that runs in one launch.
    split: returns the outputs [0, split) and [split, nout) as two tensors (dgrad of a concatenation)."""
    lib = _lib.load()
    ks, ns = blocks
    full = xb if xb is not None else xa
    B, D, H, W = full.shape[0], full.shape[1], full.shape[2], full.shape[3]
    if xb is None and up:
        D, H, W = (D * 2 if kd == 3 else D), H * 2, W * 2
    if mask is not None and split:
        raise _lib.VxmError("conv_fwd_blocked: a mask with a split output is not implemented")
    if out_fp32_planar and (split or len(ns) != 1):
        raise _lib.VxmError("conv_fwd_blocked: the fp32 planar output takes one N block")
    if out_fp32_planar:
        outs = [torch.empty((B, nout, D, H, W), dtype=torch.float32, device=full.device)]
    else:
        outs = [torch.empty((B, D, H, W, c), dtype=torch.bfloat16, device=full.device) for c in ([split, nout - split] if split else [nout])]
    outs_lo = [torch.empty_like(o) for o in outs] if lo is not None and not out_fp32_planar else [None] * len(outs)
    s = -1.0 if slope is None else float(slope)
    ca = 0 if xa is None else xa.shape[-1]
    cb = 0 if xb is None else xb.shape[-1]
    for ni, (n0, nb, dst, doff) in enumerate(ns):
        out, pitch = outs[dst], outs[dst].shape[-1]
        passes = [(ki, 0, False) for ki in range(len(ks))] if lo is None else \
                 [p for ki in range(len(ks)) for p in ((ki, 1, False), (ki, 0, True), (ki, 0, False))]   # x_lo w_hi, x_hi w_lo, x_hi w_hi
        acc = None
        for pi, (ki, xlo, wlo) in enumerate(passes):
            src, _, kb = ks[ki]
            pa = xa if not xlo else lo[0]
            pb = xb if not xlo else lo[1]
            if src == 0:
                x0, x1, c0, c1, u = pa, None, kb, 0, up
            elif src == 1:
                x0, x1, c0, c1, u = pb, None, kb, 0, False
            else:
                x0, x1, c0, c1, u = pa, pb, ca, cb, up
            wpk, coutp = (lo[2] if wlo else packs)[(ki, ni)]
            if pi + 1 < len(passes):
                ain = acc
                if acc is None:
                    acc = torch.empty((B, D, H, W, coutp), dtype=torch.float32, device=full.device)
                o, olo, m, mode, op, bptr = _lib.ptr(acc), None, None, 2, 0, None
            elif out_fp32_planar:        # + bias -> fp32 planar (the flow head), an entry point without an output pitch
                _lib.check(lib.vxm_conv3d_tcs_fwd_acc(_lib.ptr(x0), _lib.ptr(x1), _lib.ptr(wpk), _lib.ptr(bias), _lib.ptr(out), None,
                                                      _lib.ptr(acc), B, D, H, W, c0, c1, 1 if u else 0, nb, coutp, kd, 1, s,
                                                      _lib.stream_ptr()), "vxm_conv3d_tcs_fwd_acc")
                continue
            else:
                ain = acc
                o, olo, m = _ptr_at(out, doff), _ptr_at(outs_lo[dst], doff), _ptr_at(mask, n0)
                mode, op, bptr = (3 if lo is not None else 0), pitch, _ptr_at(bias, n0)
            _lib.check(lib.vxm_conv3d_tcs_fwd_blk(_lib.ptr(x0), _lib.ptr(x1), _lib.ptr(wpk), bptr, o, olo, m, _lib.ptr(ain),
                                                  B, D, H, W, c0, c1, 1 if u else 0, nb, coutp, kd, mode, s, op, _lib.stream_ptr()),
                       "vxm_conv3d_tcs_fwd_blk")
    if out_fp32_planar:
        return outs[0]
    if lo is not None:
        return outs[0], outs_lo[0]
    return tuple(outs) if split else outs[0]


# ---- split-precision (bf16x3) glue ------------------------------------------------------------------------------------

def planar_to_ndhwc8_split(planes):
    """<= 8 planar fp32 volumes -> (hi, lo) bf16 (B,D,H,W,8) tensors with hi + lo = x to 16 mantissa bits."""
    lib = _lib.load()
    ref = planes[0]
    B = ref.shape[0]
    D, H, W = (ref.shape[-3] if ref.dim() == 5 else 1), ref.shape[-2], ref.shape[-1]
    n = len(planes)
    arr_p = (ctypes.c_void_p * 8)(*([p.data_ptr() for p in planes] + [0] * (8 - n)))
    arr_s = (ctypes.c_longlong * 8)(*([p.stride(0) for p in planes] + [0] * (8 - n)))
    hi = torch.empty((B, D, H, W, 8), dtype=torch.bfloat16, device=ref.device)
    lo = torch.empty_like(hi)
    _lib.check(lib.vxm_planar_to_ndhwc8_split_bf16(arr_p, arr_s, n, _lib.ptr(hi), _lib.ptr(lo), B, D * H * W, _lib.stream_ptr()),
               "vxm_planar_to_ndhwc8_split_bf16")
    return hi, lo


def pool_split(x, nd):
    lib = _lib.load()
    xh, xl = x
    B, D, H, W, C = xh.shape
    Dc = D // 2 if nd == 3 else D
    yh = torch.empty((B, Dc, H // 2, W // 2, C), dtype=torch.bfloat16, device=xh.device)
    yl = torch.empty_like(yh)
    _lib.check(lib.vxm_pool2_split_ndhwc_bf16(_lib.ptr(xh), _lib.ptr(xl), _lib.ptr(yh), _lib.ptr(yl), B, Dc, H // 2, W // 2, C, nd,
                                              _lib.stream_ptr()), "vxm_pool2_split_ndhwc_bf16")
    return yh, yl


# ---- deferred weight-gradient reduction: every layer's partials reduced by ONE launch at the end of the backward pass ----

class WgradBatch:
    """Collects the pending reductions of the wgmma weight-gradient kernels of one backward pass
    (vxm_conv3d_tc_wgrad2_partial) and reduces them all in one launch (`flush`).  One instance per (device, stream);
    the workspace is persistent (512 MB: the default 3-D U-Net at 160x192x224 needs ~200 MB of per-CTA partials)."""

    _cache = {}
    WORK_BYTES = 512 << 20

    @classmethod
    def get(cls, device):
        key = (device.index, torch.cuda.current_stream(device).cuda_stream)
        b = cls._cache.get(key)
        if b is None:
            with _ws_lock:
                b = cls._cache.get(key)
                if b is None:
                    b = cls._cache[key] = cls(device)
        return b

    def __init__(self, device):
        lib = _lib.load()
        self.dev = device
        self.dsz = int(lib.vxm_conv3d_tc_wgrad2_desc_bytes())
        self.maxn = int(lib.vxm_conv3d_tc_wgrad2_max_pending())
        self.host = ctypes.create_string_buffer(self.dsz * self.maxn)
        self.n = ctypes.c_int(0)
        self.used = ctypes.c_size_t(0)
        self.off = 0
        self.work = torch.empty(self.WORK_BYTES, dtype=torch.uint8, device=device)

    def add(self, xa, xb, gz, gw, gb, cin, cout, kd, up, accumulate):
        lib = _lib.load()
        B, D, H, W, Cg = gz.shape
        Ca = 0 if xa is None else xa.shape[-1]
        Cb = 0 if xb is None else xb.shape[-1]
        # 64-channel operands run as 32-channel slices: one pending reduction per slice pair, partial_bytes per two pairs
        nsub = ((Ca + 31) // 32 + (Cb + 31) // 32) * ((Cg + 31) // 32)
        need = int(lib.vxm_conv3d_tc_wgrad2_partial_bytes(kd)) * ((nsub + 1) // 2)
        if self.off + need > self.WORK_BYTES or self.n.value + max(2, nsub) > self.maxn:
            self.flush()
        _lib.check(lib.vxm_conv3d_tc_wgrad2_partial(_lib.ptr(xa), _lib.ptr(xb), _lib.ptr(gz), _lib.ptr(gw), _lib.ptr(gb),
                                                    ctypes.c_void_p(self.work.data_ptr() + self.off), self.WORK_BYTES - self.off,
                                                    ctypes.byref(self.used), ctypes.cast(self.host, ctypes.c_void_p), ctypes.byref(self.n),
                                                    B, D, H, W, Ca, Cb, 1 if up else 0, cin, Cg, cout, kd, 1 if accumulate else 0,
                                                    _lib.stream_ptr()), "vxm_conv3d_tc_wgrad2_partial")
        self.off += int(self.used.value)

    def add_khm(self, x, gz, gw2d, gb, cin_real, cout_real):
        """Weight gradient of a kd-folded layer: x (B,D,H,W,Cx) against gz (B,D,H,W,Cg) -> gw2d (cout_real, cin_real, 1, 3, 3)
        (overwritten at flush), gb (cout_real) or None."""
        lib = _lib.load()
        need = int(lib.vxm_conv3d_tc_wgrad2_partial_bytes(1))
        if self.off + need > self.WORK_BYTES or self.n.value + 1 > self.maxn:
            self.flush()
        B, D, H, W, Cg = gz.shape
        _lib.check(lib.vxm_conv3d_tc_wgrad2_partial_khm(_lib.ptr(x), _lib.ptr(gz), _lib.ptr(gw2d), _lib.ptr(gb),
                                                        ctypes.c_void_p(self.work.data_ptr() + self.off), self.WORK_BYTES - self.off,
                                                        ctypes.byref(self.used), ctypes.cast(self.host, ctypes.c_void_p), ctypes.byref(self.n),
                                                        B, D, H, W, x.shape[-1], cin_real, Cg, cout_real, 0, _lib.stream_ptr()),
                   "vxm_conv3d_tc_wgrad2_partial_khm")
        self.off += int(self.used.value)

    def reset(self):
        """Drop pending reductions (after an error mid-backward)."""
        self.n.value = 0
        self.off = 0

    def flush(self):
        if self.n.value:
            _lib.check(_lib.load().vxm_conv3d_tc_wgrad2_flush(ctypes.cast(self.host, ctypes.c_void_p), self.n.value, _lib.stream_ptr()),
                       "vxm_conv3d_tc_wgrad2_flush")
        self.n.value = 0
        self.off = 0
