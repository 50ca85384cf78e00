"""ctypes binding of the C-ABI library (include/vxm_b200.h -> libvxm_b200.so).

The product path has no CPU or torch fallback: if the library is missing, or a tensor is
not a CUDA float32 tensor, the call fails loudly.
"""
import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvxm_b200.so")

c_f = ctypes.c_void_p        # device pointers travel as void*
c_i = ctypes.c_int
c_sz = ctypes.c_size_t
c_fl = ctypes.c_float
c_d = ctypes.c_double

# name -> (restype, argtypes); mirrors include/vxm_b200.h declaration by declaration
SIGNATURES = {
    "vxm_last_error": (ctypes.c_char_p, []),
    "vxm_version": (ctypes.c_char_p, []),
    "vxm_launch_count": (ctypes.c_uint64, []),
    "vxm_warp_fwd": (c_i, [c_f, c_f, c_f] + [c_i] * 9 + [c_i, c_i, c_f]),
    "vxm_warp_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f] + [c_i] * 9 + [c_i, c_i, c_f]),
    "vxm_vecint_workspace_bytes": (c_sz, [c_i] * 6),
    "vxm_vecint_fwd": (c_i, [c_f, c_f, c_f, c_f] + [c_i] * 7 + [c_f]),
    "vxm_vecint_bwd": (c_i, [c_f, c_f, c_f, c_f] + [c_i] * 7 + [c_f]),
    "vxm_vecint_fast_states_bytes": (c_sz, [c_i] * 5),
    "vxm_vecint_fast_work_bytes": (c_sz, [c_i] * 5),
    "vxm_debug_gridsync": (c_i, [c_i, c_i, c_f]),
    "vxm_resize_fwd": (c_i, [c_f, c_f] + [c_i] * 8 + [c_fl, c_fl, c_f]),
    "vxm_resize_bwd": (c_i, [c_f, c_f] + [c_i] * 8 + [c_fl, c_fl, c_f]),
    "vxm_ncc_fwd": (c_i, [c_f, c_f, c_f, c_f, c_f] + [c_i] * 7 + [c_f]),
    "vxm_ncc_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f] + [c_i] * 7 + [c_f]),
    "vxm_ncc_fwd2": (c_i, [c_f, c_f, c_f, c_f, c_f] + [c_i] * 8 + [c_f]),
    "vxm_ncc_bwd2": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f] + [c_i] * 8 + [c_f]),
    "vxm_jacdet": (c_i, [c_f, c_f, c_f] + [c_i] * 5 + [c_f]),
    "vxm_reduce_workspace_bytes": (c_sz, []),
    "vxm_gradloss_fwd": (c_i, [c_f, c_f, c_f] + [c_i] * 7 + [c_fl, c_f]),
    "vxm_gradloss_bwd": (c_i, [c_f, c_f, c_f] + [c_i] * 7 + [c_fl, c_f]),
    "vxm_mse_fwd": (c_i, [c_f, c_f, c_f, c_f, c_sz, c_f]),
    "vxm_mse_bwd": (c_i, [c_f, c_f, c_f, c_f, c_sz, c_f]),
    "vxm_mse_scaled_fwd": (c_i, [c_f, c_f, c_f, c_f, c_sz, c_d, c_f]),
    "vxm_mse_scaled_bwd": (c_i, [c_f, c_f, c_f, c_f, c_sz, c_d, c_f]),
    "vxm_kl_fwd": (c_i, [c_f, c_f, c_f] + [c_i] * 5 + [c_fl, c_f]),
    "vxm_kl_bwd": (c_i, [c_f, c_f, c_f] + [c_i] * 5 + [c_fl, c_f]),
    "vxm_dice_workspace_bytes": (c_sz, [c_i]),
    "vxm_dice_fwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_i, c_sz, c_f]),
    "vxm_dice_bwd": (c_i, [c_f, c_f, c_f, c_f, c_i, c_sz, c_f]),
    "vxm_conv3d_fwd_f32": (c_i, [c_f, c_f, c_f, c_f] + [c_i] * 7 + [c_fl, c_f]),
    "vxm_conv3d_bwd_workspace_bytes": (c_sz, [c_i] * 7),
    "vxm_conv3d_bwd_f32": (c_i, [c_f] * 8 + [c_i] * 7 + [c_fl, c_f]),
    "vxm_conv3d_tc_packed_bytes": (c_sz, [c_i] * 3),
    "vxm_conv3d_tc_pack": (c_i, [c_f, c_f] + [c_i] * 5 + [c_f]),
    "vxm_conv3d_tc_fwd": (c_i, [c_f, c_f, c_f, c_f, c_i, c_f, c_f, c_f, c_f] + [c_i] * 11 + [c_fl, c_f, c_i, c_f]),
    "vxm_conv3d_tct_packed_bytes": (c_sz, [c_i] * 3),
    "vxm_conv3d_tct_pack": (c_i, [c_f, c_f] + [c_i] * 5 + [c_f]),
    "vxm_conv3d_tct_supported": (c_i, [c_i] * 3),
    "vxm_conv3d_tct_fwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f] + [c_i] * 11 + [c_fl, c_f, c_i, c_f]),
    "vxm_conv3d_tcs_packed_bytes": (c_sz, [c_i] * 3),
    "vxm_conv3d_tcs_pack": (c_i, [c_f, c_f] + [c_i] * 5 + [c_f]),
    "vxm_conv3d_tcs_supported": (c_i, [c_i] * 3),
    "vxm_conv3d_tcs_pack_desc_bytes": (c_sz, []),
    "vxm_conv3d_tcs_pack_desc": (c_i, [c_f, c_f, c_f] + [c_i] * 6),
    "vxm_conv3d_tcs_pack_desc_blk": (c_i, [c_f, c_f, c_f] + [c_i] * 10),
    "vxm_conv3d_tcs_pack_desc_fold": (c_i, [c_f, c_f, c_f] + [c_i] * 5),
    "vxm_conv3d_tcs_pack_multi": (c_i, [c_f, c_i, c_i, c_f]),
    "vxm_conv3d_tcs_fwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f] + [c_i] * 11 + [c_fl, c_f, c_i, c_f]),
    "vxm_conv3d_tcs_fwd_acc": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f] + [c_i] * 11 + [c_fl, c_f]),
    "vxm_conv3d_tcs_fits": (c_i, [c_i] * 3),
    "vxm_conv3d_tcs_fwd_blk": (c_i, [c_f] * 8 + [c_i] * 11 + [c_fl, c_i, c_f]),
    "vxm_conv3d_tcs_poly_packed_bytes": (c_sz, [c_i] * 4),
    "vxm_conv3d_tcs_pack_desc_poly": (c_i, [c_f, c_f, c_f] + [c_i] * 5),
    "vxm_conv3d_tcs_poly": (c_i, [c_f] * 6 + [c_i] * 8 + [c_fl, c_f]),
    "vxm_conv3d_tc_wgrad_workspace_bytes": (c_sz, [c_i]),
    "vxm_conv3d_tc_wgrad": (c_i, [c_f, c_f, c_f, c_f, c_i, c_f, c_f, c_f, c_i, c_f, c_f, c_f] + [c_i] * 12 + [c_f]),
    "vxm_conv3d_tc_wgrad2_desc_bytes": (c_sz, []),
    "vxm_conv3d_tc_wgrad2_max_pending": (c_i, []),
    "vxm_conv3d_tc_wgrad2_partial_bytes": (c_sz, [c_i]),
    "vxm_conv3d_tc_wgrad2_partial": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_sz, c_f, c_f, c_f] + [c_i] * 12 + [c_f]),
    "vxm_conv3d_tc_wgrad2_flush": (c_i, [c_f, c_i, c_f]),
    "vxm_conv3d_tc_wgrad2_partial_khm": (c_i, [c_f, c_f, c_f, c_f, c_f, c_sz, c_f, c_f, c_f] + [c_i] * 9 + [c_f]),
    "vxm_pool2_ndhwc_bf16": (c_i, [c_f, c_f] + [c_i] * 6 + [c_f]),
    "vxm_sumpool_mask_ndhwc_bf16": (c_i, [c_f, c_f, c_f] + [c_i] * 6 + [c_fl, c_f]),
    "vxm_unpool_combine_ndhwc_bf16": (c_i, [c_f, c_f, c_f, c_f] + [c_i] * 6 + [c_fl, c_f]),
    "vxm_planar_to_ndhwc8_bf16": (c_i, [c_f, c_f, c_i, c_f, c_i, c_sz, c_f]),
    "vxm_planar_to_ndhwc8_split_bf16": (c_i, [c_f, c_f, c_i, c_f, c_f, c_i, c_sz, c_f]),
    "vxm_planar_fold_kd_bf16": (c_i, [c_f, c_f, c_i, c_f, c_i, c_i, c_sz, c_i, c_f]),
    "vxm_pool2_split_ndhwc_bf16": (c_i, [c_f, c_f, c_f, c_f] + [c_i] * 6 + [c_f]),
    "vxm_unpool_combine_split_ndhwc_bf16": (c_i, [c_f, c_f, c_f, c_f, c_f] + [c_i] * 6 + [c_fl, c_f]),
    "vxm_maxpool2_fwd": (c_i, [c_f, c_f, c_f] + [c_i] * 6 + [c_f]),
    "vxm_maxpool2_bwd": (c_i, [c_f, c_f, c_f] + [c_i] * 6 + [c_f]),
    "vxm_upcat_fwd": (c_i, [c_f, c_f, c_f] + [c_i] * 7 + [c_f]),
    "vxm_upcat_bwd": (c_i, [c_f, c_f, c_f] + [c_i] * 7 + [c_f]),
    "vxm_adam_step": (c_i, [c_f, c_f, c_f, c_f, c_sz, c_i] + [c_fl] * 6 + [c_f]),
    "vxm_adam_step_dev": (c_i, [c_f, c_f, c_f, c_f, c_sz, c_f] + [c_fl] * 6 + [c_f]),
    "vxm_mean_stream_fwd": (c_i, [c_f] * 6 + [c_i, c_sz, c_fl, c_i, c_f]),
    "vxm_mean_stream_bwd": (c_i, [c_f, c_f, c_f, c_i, c_sz, c_sz, c_f]),
    "vxm_sample_normal_logvar_fwd": (c_i, [c_f] * 5 + [c_i, c_i, c_sz, c_f]),
    "vxm_sample_normal_logvar_bwd": (c_i, [c_f] * 5 + [c_i, c_i, c_sz, c_f]),
    "vxm_pheno_decoder_workspace_bytes": (c_sz, [c_i]),
    "vxm_pheno_decoder_fwd": (c_i, [c_f] * 6 + [c_i, c_i, c_i, c_sz, c_f]),
    "vxm_pheno_decoder_bwd": (c_i, [c_f] * 10 + [c_i, c_i, c_i, c_sz, c_i, c_f]),
    "vxm_hyper_workspace_bytes": (c_sz, [c_i, c_sz]),
    "vxm_hyper_mlp_fwd": (c_i, [c_f] * 5 + [c_i, c_i, c_i, c_f]),
    "vxm_hyper_mlp_bwd": (c_i, [c_f] * 6 + [c_i, c_i, c_i, c_i, c_f]),
    "vxm_hyper_weights_fwd": (c_i, [c_f] * 4 + [c_i, c_sz, c_f]),
    "vxm_hyper_weights_bwd": (c_i, [c_f] * 7 + [c_i, c_sz, c_i, c_f]),
    "vxm_mi_workspace_bytes": (c_sz, [c_i, c_sz, c_i]),
    "vxm_mi_fwd": (c_i, [c_f] * 6 + [c_i, c_sz, c_i, c_fl, c_fl, c_fl, c_f]),
    "vxm_mi_bwd": (c_i, [c_f] * 7 + [c_i, c_sz, c_i, c_fl, c_fl, c_fl, c_f]),
    "vxm_point_warp_workspace_bytes": (c_sz, [c_i] * 6),
    "vxm_point_warp_fwd": (c_i, [c_f] * 3 + [c_i] * 6 + [c_fl, c_f]),
    "vxm_point_warp_bwd": (c_i, [c_f] * 4 + [c_sz] + [c_i] * 6 + [c_fl, c_f]),
    "vxm_value_at_fwd": (c_i, [c_f] * 3 + [c_i] * 7 + [c_f]),
    "vxm_value_at_bwd": (c_i, [c_f] * 4 + [c_i] * 7 + [c_f]),
}

_lib = None
_lock = threading.Lock()


class VxmError(RuntimeError):
    pass


def load():
    """dlopen the library (idempotent).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            raise VxmError(
                "voxelmorph_b200: %s not found — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C voxelmorph_b200/csrc`).  There is no CPU / torch fallback." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def last_error():
    return load().vxm_last_error().decode("utf-8", "replace")


def check(rc, what):
    if rc != 0:
        raise VxmError("%s failed (%d): %s" % (what, rc, last_error()))


def launch_count():
    return int(load().vxm_launch_count())


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(*tensors, what="voxelmorph_b200"):
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise VxmError("%s: CUDA tensors are required (the GPU path has no CPU fallback); got a %s tensor"
                           % (what, t.device))
        if t.dtype != torch.float32:
            raise VxmError("%s: float32 tensors are required at the module boundary; got %s" % (what, t.dtype))


def contig(t):
    return t if t.is_contiguous() else t.contiguous()


# ---- small persistent workspaces (zero-initialised once; kernels leave them zeroed) ----------
_reduce_ws = {}


def reduce_workspace(device):
    """Per (device, stream) scratch for the deterministic two-stage reductions."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    ws = _reduce_ws.get(key)
    if ws is None:
        lib = load()     # (takes the same lock: resolve the library first)
        with _lock:      # nn.DataParallel (train.py:151-154) calls the replicas from one thread per GPU
            ws = _reduce_ws.get(key)
            if ws is None:
                nbytes = int(lib.vxm_reduce_workspace_bytes())
                ws = torch.zeros(nbytes, dtype=torch.uint8, device=device)
                _reduce_ws[key] = ws
    return ws
