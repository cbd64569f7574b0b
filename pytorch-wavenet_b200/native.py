"""ctypes binding of libwavenet_b200.so (the C ABI declared in include/wavenet_b200.h).

There is no fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
Build the library with ``make -C pytorch-wavenet_b200/csrc`` (or ``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libwavenet_b200.so")

c_float_p = C.POINTER(C.c_float)
c_void_pp = C.POINTER(C.c_void_p)


class BlockArgs(C.Structure):
    _fields_ = [("d_h_in", C.c_void_p), ("d_h_out", C.c_void_p), ("d_skip", C.c_void_p),
                ("d_wfg_t", C.c_void_p), ("d_bfg", C.c_void_p), ("d_wrs_t", C.c_void_p), ("d_brs", C.c_void_p),
                ("B", C.c_int), ("L", C.c_int), ("R", C.c_int), ("D", C.c_int), ("S", C.c_int), ("k", C.c_int),
                ("dilation", C.c_int), ("in_start", C.c_int), ("out_start", C.c_int), ("skip_start", C.c_int),
                ("skip_init", C.c_int), ("mode", C.c_int), ("d_fg_save", C.c_void_p)]


class BlockBwdArgs(C.Structure):
    _fields_ = [("d_dh_out", C.c_void_p), ("d_dskip", C.c_void_p), ("d_fg", C.c_void_p),
                ("d_dfg", C.c_void_p), ("d_z", C.c_void_p), ("d_dh_in", C.c_void_p),
                ("d_wrs_rows", C.c_void_p), ("d_wfg_bwd", C.c_void_p),
                ("B", C.c_int), ("L", C.c_int), ("R", C.c_int), ("D", C.c_int), ("S", C.c_int), ("k", C.c_int),
                ("dilation", C.c_int), ("in_start", C.c_int), ("out_start", C.c_int),
                ("gs_out", C.c_int), ("ds_start", C.c_int), ("gz", C.c_int), ("gs_in", C.c_int)]


class HeadBwdArgs(C.Structure):
    _fields_ = [("d_dlogits", C.c_void_p), ("d_skip", C.c_void_p),
                ("d_y1", C.c_void_p), ("d_dy1", C.c_void_p), ("d_dskip", C.c_void_p),
                ("d_w1_t", C.c_void_p), ("d_b1", C.c_void_p), ("d_w2_rows", C.c_void_p), ("d_w1_rows", C.c_void_p),
                ("B", C.c_int), ("L", C.c_int), ("S", C.c_int), ("E", C.c_int), ("classes", C.c_int),
                ("skip_start", C.c_int), ("out_len", C.c_int)]


class WgradArgs(C.Structure):
    _fields_ = [("d_g", C.c_void_p), ("d_x", C.c_void_p), ("d_dw", C.c_void_p), ("d_work", C.c_void_p),
                ("g_seq_stride", C.c_longlong), ("x_seq_stride", C.c_longlong),
                ("dw_n_stride", C.c_longlong), ("dw_c_stride", C.c_longlong),
                ("ldg", C.c_int), ("ldx", C.c_int), ("B", C.c_int), ("rows", C.c_int), ("N", C.c_int), ("C", C.c_int)]


class TcBlockArgs(C.Structure):
    _fields_ = [("d_h_in", C.c_void_p), ("d_h_out", C.c_void_p), ("d_skip", C.c_void_p), ("d_z", C.c_void_p),
                ("d_wa", C.c_void_p), ("d_ba", C.c_void_p), ("d_wb", C.c_void_p), ("d_bb", C.c_void_p),
                ("B", C.c_int), ("L", C.c_int), ("R", C.c_int), ("D", C.c_int), ("S", C.c_int), ("k", C.c_int),
                ("dilation", C.c_int), ("in_start", C.c_int), ("out_start", C.c_int), ("skip_start", C.c_int),
                ("skip_init", C.c_int), ("d_fg_save", C.c_void_p)]


PREC_BF16, PREC_BF16_PAIRS = 1, 2        # WN_PREC_* of include/wavenet_b200.h
GEN_SRC_FRAMES, GEN_SRC_PAIRS = 0, 1     # WN_GEN_SRC_* (wn_gen_prefill_layer)


class TbBlockArgs(C.Structure):
    _fields_ = [("d_h_in", C.c_void_p), ("d_h_out", C.c_void_p), ("d_skip", C.c_void_p),
                ("d_w_all", C.c_void_p), ("d_bias4", C.c_void_p), ("layer", C.c_int), ("n_layers", C.c_int),
                ("channels", C.c_int), ("precision", C.c_int),
                ("B", C.c_int), ("L", C.c_int), ("dilation", C.c_int),
                ("in_start", C.c_int), ("out_start", C.c_int), ("skip_start", C.c_int), ("skip_init", C.c_int),
                ("d_fg_save", C.c_void_p)]


class TbStackArgs(C.Structure):
    _fields_ = [("h_ptrs", c_void_pp), ("d_skip", C.c_void_p), ("d_w_all", C.c_void_p), ("d_bias_all", C.c_void_p),
                ("d_fg_all", C.c_void_p), ("d_desc", C.c_void_p), ("d_flags", C.c_void_p),
                ("n_layers", C.c_int), ("channels", C.c_int), ("precision", C.c_int), ("B", C.c_int), ("L", C.c_int),
                ("skip_start", C.c_int), ("dilations", C.POINTER(C.c_int)), ("in_start", C.POINTER(C.c_int)),
                ("out_start", C.POINTER(C.c_int))]


class TbBwdArgs(C.Structure):
    _fields_ = [("d_dh_out", C.c_void_p), ("d_dskip", C.c_void_p), ("d_fg", C.c_void_p),
                ("d_dfg", C.c_void_p), ("d_z", C.c_void_p), ("d_dh_in", C.c_void_p), ("d_wb_all", C.c_void_p),
                ("layer", C.c_int), ("n_layers", C.c_int), ("channels", C.c_int), ("precision", C.c_int),
                ("B", C.c_int), ("L", C.c_int), ("dilation", C.c_int),
                ("in_start", C.c_int), ("out_start", C.c_int),
                ("gs_out", C.c_int), ("ds_start", C.c_int), ("gz", C.c_int), ("gs_in", C.c_int)]


class TbWgradArgs(C.Structure):
    _fields_ = [("d_dskip", C.c_void_p), ("d_dh_out", C.c_void_p), ("d_dfg", C.c_void_p), ("d_z", C.c_void_p),
                ("d_h_in", C.c_void_p), ("d_gws", C.c_void_p), ("d_gwr", C.c_void_p), ("d_gwf", C.c_void_p),
                ("d_gwg", C.c_void_p), ("d_work", C.c_void_p), ("channels", C.c_int), ("precision", C.c_int),
                ("B", C.c_int), ("L", C.c_int), ("dilation", C.c_int),
                ("in_start", C.c_int), ("ds_start", C.c_int), ("id_start", C.c_int), ("gz", C.c_int)]


class HeadArgs(C.Structure):
    _fields_ = [("d_skip", C.c_void_p), ("d_logits", C.c_void_p),
                ("d_w1_t", C.c_void_p), ("d_b1", C.c_void_p), ("d_w2_t", C.c_void_p), ("d_b2", C.c_void_p),
                ("B", C.c_int), ("L", C.c_int), ("S", C.c_int), ("E", C.c_int), ("classes", C.c_int),
                ("skip_start", C.c_int), ("out_len", C.c_int), ("mode", C.c_int)]


class GenWeights(C.Structure):
    _fields_ = [("d_start_w", C.c_void_p), ("d_start_b", C.c_void_p),
                ("d_wf", c_void_pp), ("d_bf", c_void_pp), ("d_wg", c_void_pp), ("d_bg", c_void_pp),
                ("d_wr", c_void_pp), ("d_br", c_void_pp), ("d_ws", c_void_pp), ("d_bs", c_void_pp),
                ("d_end1_w", C.c_void_p), ("d_end1_b", C.c_void_p), ("d_end2_w", C.c_void_p), ("d_end2_b", C.c_void_p)]


class GenShape(C.Structure):
    _fields_ = [("n_layers", C.c_int), ("k", C.c_int), ("R", C.c_int), ("D", C.c_int), ("S", C.c_int),
                ("E", C.c_int), ("classes", C.c_int), ("n_streams", C.c_int), ("dilations", C.POINTER(C.c_int))]


class GenStreamParams(C.Structure):
    _fields_ = [("n_given", C.c_int), ("top_k", C.c_int), ("temperature", C.c_float), ("regularize", C.c_float),
                ("top_p", C.c_double)]


class GenStreamPos(C.Structure):
    _fields_ = [("origin", C.c_int), ("sample0", C.c_int), ("first0", C.c_int)]


class GenRunArgs(C.Structure):
    _fields_ = [("d_first", C.c_void_p), ("n_given", C.c_int),
                ("d_forced", C.c_void_p), ("d_uniforms", C.c_void_p),
                ("d_out_idx", C.c_void_p), ("d_out_logits", C.c_void_p),
                ("n_samples", C.c_int), ("t0", C.c_int), ("n_evals", C.c_int),
                ("temperature", C.c_float), ("regularize", C.c_float)]


# every exported symbol of include/wavenet_b200.h: name -> (restype, argtypes)
SIGNATURES = {
    "wn_version": (C.c_int, []),
    "wn_last_error_string": (C.c_char_p, []),
    "wn_device_info": (C.c_int, [C.POINTER(C.c_int)] * 5),
    "wn_n1p": (C.c_int, [C.c_int]),
    "wn_n2p": (C.c_int, [C.c_int]),
    "wn_pack_gate_weights": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 3 + [C.c_void_p] * 3),
    "wn_pack_res_skip_weights": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 3 + [C.c_void_p] * 3),
    "wn_pack_1x1_weights": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 2 + [C.c_void_p] * 3),
    "wn_start_fwd_dense": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p]),
    "wn_start_fwd_index_u8": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p]),
    "wn_start_fwd_index_i64": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p]),
    "wn_block_fwd": (C.c_int, [C.POINTER(BlockArgs), C.c_void_p]),
    "wn_head_fwd": (C.c_int, [C.POINTER(HeadArgs), C.c_void_p]),
    "wn_tc_supported": (C.c_int, [C.c_int] * 4),
    "wn_tc_pack_block_weights": (C.c_int, [C.c_void_p] * 8 + [C.c_int] * 4 + [C.c_void_p] * 5),
    "wn_tc_block_fwd": (C.c_int, [C.POINTER(TcBlockArgs), C.c_void_p]),
    "wn_tc_read_trace": (C.c_int, [C.POINTER(C.c_longlong), C.c_int]),
    "wn_tb_supported": (C.c_int, [C.c_int] * 4),
    "wn_tb_precision_supported": (C.c_int, [C.c_int] * 2),
    "wn_tb_weight_bytes_per_layer": (C.c_size_t, [C.c_int] * 2),
    "wn_tb_pack_all_weights": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wn_tb_start_index_u8": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p] * 2),
    "wn_tb_start_index_i64": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p] * 2),
    "wn_pair_from_frames": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 4 + [C.c_void_p]),
    "wn_frames_from_pair": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 4 + [C.c_void_p]),
    "wn_frames_from_chunks4": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 5 + [C.c_void_p]),
    "wn_tb_block_fwd": (C.c_int, [C.POINTER(TbBlockArgs), C.c_void_p]),
    "wn_tb_stack_desc_bytes": (C.c_size_t, []),
    "wn_tb_stack_items": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "wn_tb_stack_fwd": (C.c_int, [C.POINTER(TbStackArgs), C.c_void_p]),
    "wn_tb_bwd_weight_bytes_per_layer": (C.c_size_t, [C.c_int] * 2),
    "wn_tb_pack_all_bwd_weights": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "wn_tb_block_bwd_data": (C.c_int, [C.POINTER(TbBwdArgs), C.c_void_p]),
    "wn_tb_wgrad_workspace_bytes": (C.c_size_t, []),
    "wn_tb_wgrad": (C.c_int, [C.POINTER(TbWgradArgs), C.c_void_p]),
    "wn_block_bwd_data": (C.c_int, [C.POINTER(BlockBwdArgs), C.c_void_p]),
    "wn_head_bwd_data": (C.c_int, [C.POINTER(HeadBwdArgs), C.c_void_p]),
    "wn_cond_table": (C.c_int, [C.c_void_p] + [C.c_int] * 3 + [C.c_void_p, C.c_int] + [C.c_void_p] * 2),
    "wn_block_fwd_cond": (C.c_int, [C.POINTER(BlockArgs), C.c_void_p, C.c_void_p]),
    "wn_tb_block_fwd_cond": (C.c_int, [C.POINTER(TbBlockArgs), C.c_void_p, C.c_void_p]),
    "wn_tb_stack_fwd_cond": (C.c_int, [C.POINTER(TbStackArgs), C.c_void_p, C.c_void_p]),
    "wn_cond_frame_sums": (C.c_int, [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p] * 2),
    "wn_cond_table_frames": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 2 + [C.c_void_p, C.c_int, C.c_void_p] + [C.c_int] * 3
                             + [C.c_void_p] * 2),
    "wn_block_fwd_cond_frames": (C.c_int, [C.POINTER(BlockArgs), C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "wn_tb_block_fwd_cond_frames": (C.c_int, [C.POINTER(TbBlockArgs), C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "wn_tb_stack_fwd_cond_frames": (C.c_int, [C.POINTER(TbStackArgs), C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "wn_cond_segment_sums": (C.c_int, [C.c_void_p] + [C.c_int] * 7 + [C.c_void_p] * 2),
    "wn_tb_local_padded_channels": (C.c_int, [C.c_int] * 2),
    "wn_tb_local_weight_bytes_per_layer": (C.c_size_t, [C.c_int] * 3),
    "wn_tb_local_from_channels": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 4 + [C.c_void_p]),
    "wn_tb_pack_local_weights": (C.c_int, [C.c_void_p] + [C.c_int] * 4 + [C.c_void_p] * 2),
    "wn_tb_block_fwd_local": (C.c_int, [C.POINTER(TbBlockArgs), C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "wn_tb_stack_fwd_local": (C.c_int, [C.POINTER(TbStackArgs), C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "wn_local_weight_grad_workspace_bytes": (C.c_size_t, [C.c_int] * 2),
    "wn_local_weight_grad": (C.c_int, [C.c_void_p] + [C.c_int] * 4 + [C.c_void_p, C.c_int] + [C.c_void_p] * 3),
    "wn_local_data_grad_add": (C.c_int, [C.c_void_p] + [C.c_int] * 4 + [C.c_void_p, C.c_int] + [C.c_void_p] * 2),
    "wn_wgrad_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "wn_wgrad": (C.c_int, [C.POINTER(WgradArgs), C.c_void_p]),
    "wn_tc_wgrad_supported": (C.c_int, [C.c_int, C.c_int]),
    "wn_tc_wgrad": (C.c_int, [C.POINTER(WgradArgs), C.c_void_p]),
    "wn_tc_bwd_supported": (C.c_int, [C.c_int] * 4),
    "wn_tc_pack_block_bwd_weights": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p] * 3),
    "wn_tc_block_bwd_data": (C.c_int, [C.POINTER(BlockBwdArgs), C.c_void_p, C.c_void_p, C.c_void_p]),
    "wn_ce_workspace_bytes": (C.c_size_t, []),
    "wn_ce_fwd_bwd": (C.c_int, [C.c_void_p] * 6 + [C.c_int] * 2 + [C.c_void_p]),
    "wn_adam_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int] + [C.c_float] * 5 + [C.c_int, C.c_void_p]),
    "wn_adam_step_f64": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int] + [C.c_double] * 5 + [C.c_int, C.c_void_p]),
    "wn_scatter_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int] * 5 + [C.c_void_p]),

    "wn_colsum_workspace_bytes": (C.c_size_t, [C.c_longlong, C.c_int]),
    "wn_colsum": (C.c_int, [C.c_void_p] * 3 + [C.c_longlong, C.c_int, C.c_int, C.c_void_p]),
    "wn_relu_copy": (C.c_int, [C.c_void_p] * 2 + [C.c_longlong, C.c_void_p]),
    "wn_scale_by": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]),
    "wn_gen_workspace_bytes": (C.c_int, [C.POINTER(GenShape), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "wn_gen_create": (C.c_int, [C.POINTER(GenShape), C.POINTER(GenWeights), C.c_void_p, C.c_void_p,
                                C.POINTER(C.c_void_p)]),
    "wn_gen_reset": (C.c_int, [C.c_void_p, C.c_void_p]),
    "wn_gen_prefill_layer": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p] + [C.c_int] * 4 + [C.c_void_p]),
    "wn_gen_prefill_commit": (C.c_int, [C.c_void_p, C.c_int]),
    "wn_gen_run": (C.c_int, [C.c_void_p, C.POINTER(GenRunArgs), C.c_void_p]),
    "wn_gen_destroy": (C.c_int, [C.c_void_p]),
    "wn_gen_set_mode": (C.c_int, [C.c_void_p, C.c_int]),
    "wn_gen_weights_changed": (C.c_int, [C.c_void_p]),
    "wn_gen_set_condition": (C.c_int, [C.c_void_p, C.c_void_p]),
    "wn_gen_set_condition_frames": (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_int] * 3),
    "wn_gen_set_condition_stream_frames": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int]),
    "wn_gen_set_truncation": (C.c_int, [C.c_void_p, C.c_int, C.c_double]),
    "wn_gen_set_stream_params": (C.c_int, [C.c_void_p, C.POINTER(GenStreamParams)]),
    "wn_gen_set_stream_positions": (C.c_int, [C.c_void_p, C.POINTER(GenStreamPos)]),
    "wn_gen_seat_layer": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]
                          + [C.c_int] * 3 + [C.c_void_p]),
    "wn_gen_set_time": (C.c_int, [C.c_void_p, C.c_int]),
    "wn_gen_kernel_id": (C.c_int, [C.c_void_p]),
    "wn_gen_check": (C.c_int, [C.c_void_p, C.c_void_p]),
    "wn_gen_read_trace": (C.c_int, [C.c_void_p, C.POINTER(C.c_longlong), C.c_int, C.c_void_p]),
    "wn_gen_launch_info": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 3),
}

_lib: Optional[C.CDLL] = None


def lib() -> C.CDLL:
    """The loaded library; raises (never falls back) when it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"wavenet_b200: {LIB_PATH} is missing -- build it with `make -C {os.path.join(_HERE, 'csrc')}` "
                "(there is no CPU or eager fallback)")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)          # AttributeError here == header and library disagree
            fn.restype, fn.argtypes = res, args
        if handle.wn_version() != 3:
            raise RuntimeError("wavenet_b200: ABI version mismatch between native.py and libwavenet_b200.so")
        _lib = handle
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().wn_last_error_string().decode("utf-8", "replace")
        raise RuntimeError(f"wavenet_b200 native call failed ({what}, code {rc}): {msg}")


def ptr(t) -> Optional[int]:
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def ptr_array(tensors):
    """ctypes array of device pointers (None entries -> NULL); keep the return value alive during the call."""
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = None if t is None else t.data_ptr()
    return arr


def device_info():
    vals = [C.c_int() for _ in range(5)]
    check(lib().wn_device_info(*[C.byref(v) for v in vals]), "wn_device_info")
    keys = ("sm_count", "cc_major", "cc_minor", "smem_optin", "l2_bytes")
    return {k: v.value for k, v in zip(keys, vals)}
