"""ctypes binding of libcocos_b200.so (include/cocos_b200.h).

There is deliberately NO fallback: if the shared library is missing or an
entry point is absent, importing/using the ops raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcocos_b200.so")

_c_int, _c_float, _c_ll, _vp = ctypes.c_int, ctypes.c_float, ctypes.c_longlong, ctypes.c_void_p

# name -> argtypes (restype is int unless noted); mirrors include/cocos_b200.h
SIGNATURES = {
    "cocos_abi_version": [],
    "cocos_last_error": [],
    "cocos_pack_rows_f16": [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _vp, _vp],
    "cocos_pack_v_f16": [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _vp],
    "cocos_corr_warp_fwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int,
                            _c_float, _vp],
    "cocos_corr_warp_bwd_ds": [_vp] * 10 + [_c_int] * 8 + [_c_float, _vp],
    "cocos_spade_mod_fwd": [_vp] * 5 + [_c_int] * 5 + [_c_float, _c_float, _c_int, _vp],
    "cocos_spade_mod_bwd": [_vp] * 7 + [_c_int] * 5 + [_c_float, _c_int, _vp],
    "cocos_cast_pitch": [_vp, _vp, ctypes.c_longlong] + [_c_int] * 6 + [_vp],
    "cocos_conv_wgrad": [_vp, _vp, _vp] + [_c_int] * 11 + [_vp, _vp, _vp],
    "cocos_conv_fwd": [_vp, _vp, _vp, _vp] + [_c_int] * 10 + [_vp],
    "cocos_normalize_pack": [_vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_float, _vp],
    "cocos_normalize_pack_bwd": [_vp] * 7 + [_c_int] * 5 + [_vp],
    "cocos_transpose_f16_bf16": [_vp, _vp, _c_int, _c_int, _c_int, _vp],
    "cocos_inst_act_fwd": [_vp] * 4 + [_c_int, _c_int, _c_float, _c_float, _vp],
    "cocos_inst_act_bwd": [_vp] * 5 + [_c_int, _c_int, _c_float, _vp],
    "cocos_tapconv": [_vp, _vp],
    "cocos_tapwgrad": [_vp, _vp],
    "cocos_tapwgrad_workspace": [_vp, _vp],
    "cocos_pack_w": [_vp, _c_int, _c_int, _c_int, _vp, _c_int, _c_int, _c_int, _c_int, _vp, _vp, _vp, _c_int, _c_int, _vp],
    "cocos_spade_mod_nhwc_fwd": [_vp, _c_int, _c_int, _vp, _c_int, _c_int, _vp, _c_int, _c_int, _vp, _vp] + [_c_int] * 5
                                + [_c_float, _c_float, _vp],
    "cocos_spade_mod_nhwc_bwd": [_vp, _c_int, _vp, _c_int, _c_int, _vp, _c_int, _c_int, _c_int, _vp, _vp, _vp, _c_int,
                                 _c_int, _vp, _c_int] + [_c_int] * 5 + [_c_float, _vp],
    "cocos_ctx_rows_fwd": [_vp, _vp, _c_int, _c_int, _c_float, _c_float, _vp],
    "cocos_ctx_rows_bwd": [_vp, _vp, _vp, _c_int, _c_int, _c_int, _c_float, _c_float, _vp],
    "cocos_sn_power_iter": [_vp, _c_int, _c_int, _c_int, _vp, _vp, _vp, _c_float, _c_int, _vp],
    "cocos_pono_stats_nhwc": [_vp, _c_int, _c_int, _c_int, _c_ll, _c_float, _vp, _vp, _vp],
    "cocos_in_stats_nhwc": [_vp, _c_int, _c_int, _c_int, _c_int, _c_int, _vp, _vp, _vp, _vp],
    "cocos_inst_act_nhwc_fwd": [_vp, _c_int, _c_int, _vp, _vp, _c_int, _c_int, _vp, _c_float, _vp, _c_int, _c_int,
                                _c_int, _c_int, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_float, _vp, _c_int, _c_int,
                                _c_int, _vp],
    "cocos_inst_act_nhwc_bwd": [_vp, _c_int, _c_int, _vp, _c_int, _vp, _c_int, _c_int, _vp, _vp, _c_int, _c_int, _vp,
                                _c_float, _vp, _vp, _vp, _c_int, _c_int, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                _c_int, _c_float, _vp, _c_int, _c_int, _vp, _c_int, _c_int, _c_int, _c_int, _vp, _vp,
                                _vp],
    "cocos_act_bwd_nhwc": [_vp, _c_int, _vp, _c_int, _c_int, _c_int, _vp, _c_int] + [_c_int] * 5 + [_c_float, _vp],
    "cocos_nhwc_pack": [_vp, _vp] + [_c_int] * 13 + [_vp],
    "cocos_pair_loss_nhwc_fwd": [_vp, _c_int, _vp, _c_int, _vp, _c_int, _c_ll, _c_int, _c_float, _c_int, _vp, _vp, _vp,
                                 _vp],
    "cocos_pair_loss_nhwc_bwd": [_vp, _c_int, _vp, _c_int, _vp, _c_int, _c_ll, _c_int, _c_float, _c_int, _vp, _vp, _c_int,
                                 _c_int, _vp],
    "cocos_cast_op_bf16": [_vp, _c_int, _c_int, _vp, _c_int, _c_ll, _vp],
    "cocos_maxpool2_nhwc_fwd": [_vp, _vp] + [_c_int] * 4 + [_vp],
    "cocos_maxpool2_nhwc_bwd": [_vp, _vp, _vp] + [_c_int] * 4 + [_vp],
    "cocos_nhwc_unpack": [_vp] + [_c_int] * 8 + [_vp] + [_c_int] * 6 + [_vp],
    "cocos_colsum_nhwc": [_vp, _c_int, _c_int, _c_int, _c_ll, _vp, _vp, _vp, _vp],
    "cocos_gemm_f16": [_vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_ll, _c_ll, _c_ll,
                       _c_float, _c_int, _c_int, _vp],
    "cocos_se_nhwc_fwd": [_vp, _c_int, _c_int, _vp, _c_int, _c_int, _vp, _vp, _vp, _c_int, _c_int, _vp, _vp, _vp]
                         + [_c_int] * 4 + [_vp, _vp, _vp],
    "cocos_se_nhwc_bwd": [_vp, _c_int, _vp, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _vp, _vp]
                         + [_c_int] * 4 + [_vp, _vp, _vp],
    "cocos_nhwc_to_op": [_vp, _c_int, _c_int, _vp, _c_int, _c_int, _c_ll, _vp],
    "cocos_attn_pack_nhwc": [_vp] + [_c_int] * 8 + [_vp, _vp, _vp, _c_int, _c_int, _vp, _c_int, _vp, _c_int, _vp, _vp],
    "cocos_attn_do_rows": [_vp] + [_c_int] * 4 + [_vp, _c_int, _vp, _vp, _c_int, _vp],
    "cocos_attn_grad_unpack": [_vp] * 4 + [_c_int] * 7 + [_vp, _c_int, _vp],
}

_lib = None
LAUNCHES = 0  # kernels enqueued through the C-ABI (bench.py reports it)


class CocosError(RuntimeError):
    pass


def build():
    """Compile the extension in-tree (nvcc, sm_90a)."""
    import subprocess
    subprocess.check_call(["bash", os.path.join(_HERE, "csrc", "build.sh")])


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CocosError(
            "libcocos_b200.so not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "or cocosnet_b200/csrc/build.sh. There is no CPU/PyTorch fallback for the hot path." % LIB_PATH)
    h = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(h, name)  # AttributeError if the symbol is missing
        fn.argtypes = argtypes
        fn.restype = ctypes.c_char_p if name == "cocos_last_error" else ctypes.c_int
    _lib = h
    return h


def call_with_workspace(fn, args, stream, what, kernels=1):
    """fn(*args, ws, &ws_floats, stream) under the C-ABI workspace protocol: a size query (nothing launched), then the
    call with a workspace from torch's caching allocator (stream-ordered, usable under CUDA-graph capture)."""
    import torch
    need = ctypes.c_longlong(0)
    check(fn(*args, None, ctypes.byref(need), stream), what, kernels=0)
    ws = torch.empty((max(need.value, 1),), dtype=torch.float32, device="cuda")
    need.value = ws.numel()
    check(fn(*args, ws.data_ptr(), ctypes.byref(need), stream), what, kernels=kernels)


def check(rc, what, kernels=1):
    global LAUNCHES
    LAUNCHES += kernels
    if rc != 0:
        msg = lib().cocos_last_error()
        raise CocosError("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else "?"))
