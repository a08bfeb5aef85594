"""ctypes binding of libds2_b200.so (the C-ABI declared in include/ds2_b200.h).

There is no fallback: if the shared library is missing or a call fails, an exception is raised.
"""
import contextlib
import ctypes as C
import os

import torch  # also loads libcudart.so.12, which the library links against

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libds2_b200.so")

RNN_LSTM, RNN_GRU, RNN_TANH = 0, 1, 2
PREC_FP32, PREC_TF32, PREC_F16 = 0, 1, 2

vp, i32, i64, f32, sz = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t


class RnnDesc(C.Structure):
    _fields_ = [("rnn_type", i32), ("bidirectional", i32), ("T", i32), ("B", i32), ("In", i32), ("H", i32),
                ("training", i32), ("bn_momentum", f32), ("bn_eps", f32), ("deferred_dw", i32)]


# name -> (restype, argtypes); must list every symbol of include/ds2_b200.h (tests check this)
PROTOTYPES = {
    "ds2_version": (C.c_char_p, []),
    "ds2_last_error": (C.c_char_p, []),
    "ds2_device_check": (i32, [C.POINTER(i32)] * 3),
    "ds2_set_precision": (i32, [i32]),
    "ds2_get_precision": (i32, []),
    "ds2_launch_count": (i64, [i32]),
    "ds2_fallback_count": (i64, [i32]),
    "ds2_set_side_stream": (i32, [vp]),
    "ds2_join_side_stream": (i32, [vp]),
    "ds2_prof_enable": (i32, [i32]),
    "ds2_prof_report": (i32, [C.c_char_p, sz]),
    "ds2_seq_lens_host": (i32, [vp, i32, vp]),
    "ds2_conv_frontend_workspace_bytes": (sz, [i32, i32]),
    "ds2_conv_frontend_fwd": (i32, [i32, i32] + [vp] * 14 + [i32, f32, f32] + [vp] * 6 + [sz, vp]),
    "ds2_conv_frontend_bwd": (i32, [i32, i32] + [vp] * 22 + [sz, vp]),
    "ds2_rnn_reserve_floats": (sz, [C.POINTER(RnnDesc)]),
    "ds2_rnn_workspace_bytes": (sz, [C.POINTER(RnnDesc)]),
    "ds2_rnn_layer_fwd": (i32, [C.POINTER(RnnDesc)] + [vp] * 17 + [sz, vp]),
    "ds2_rnn_layer_bwd": (i32, [C.POINTER(RnnDesc)] + [vp] * 18 + [sz, vp]),
    "ds2_lookahead_fwd": (i32, [i32] * 4 + [vp] * 4),
    "ds2_lookahead_bwd": (i32, [i32] * 4 + [vp] * 7),
    "ds2_fc_head_workspace_bytes": (sz, [i32, i32, i32]),
    "ds2_fc_head_fwd": (i32, [i32, i32, i32] + [vp] * 6 + [i32, f32, f32, i32] + [vp] * 4 + [sz, vp]),
    "ds2_fc_head_bwd": (i32, [i32, i32, i32] + [vp] * 11 + [sz, vp]),
    "ds2_ctc_workspace_bytes": (sz, [i32, i32, i32, i32]),
    "ds2_ctc_loss_fwd_bwd": (i32, [i32, i32, i32] + [vp] * 4 + [i32, i32] + [vp] * 3 + [sz, vp]),
    "ds2_ctc_align_workspace_bytes": (sz, [i32, i32, i32, i32]),
    "ds2_ctc_align": (i32, [i32, i32, i32, vp, i32] + [vp] * 3 + [i32, i32] + [vp] * 5 + [sz, vp]),
    "ds2_greedy_decode": (i32, [i32, i32, i32, vp, vp, i32, vp, vp, vp, vp]),
    "ds2_greedy_decode_stream": (i32, [i32, i32, vp, vp, vp, i32, vp, vp, vp]),
    "ds2_beam_decode_workspace_bytes": (sz, [i32] * 4),
    "ds2_beam_decode": (i32, [i32, i32, i32, vp, vp, i32, i32, i32, f32] + [vp] * 6 + [sz, vp]),
    "ds2_lm_bytes": (sz, [i32, vp, i64]),
    "ds2_lm_build": (i32, [i32, vp, vp, vp, vp, i32, i32, i64, vp, vp, vp, vp, sz, vp]),
    "ds2_beam_decode_lm_workspace_bytes": (sz, [i32] * 4),
    "ds2_beam_decode_lm": (i32, [i32, i32, i32, vp, vp, i32, i32, i32, f32, vp, i32, C.c_double, C.c_double, i32]
                           + [vp] * 6 + [sz, vp]),
    "ds2_beam_decode_lm_grid_workspace_bytes": (sz, [i32] * 5),
    "ds2_beam_decode_lm_grid": (i32, [i32, i32, i32, vp, vp, i32, i32, i32, f32, vp, i32, i32, vp, i32]
                                + [vp] * 3 + [sz, vp]),
    "ds2_beam_decode_stream_state_bytes": (sz, [i32] * 3),
    "ds2_beam_decode_lm_stream_state_bytes": (sz, [i32] * 3),
    "ds2_beam_decode_stream": (i32, [i32, i32, vp, vp, i32, i32, i32, f32, i32, i32, i32] + [vp] * 6 + [sz, vp]),
    "ds2_beam_decode_lm_stream": (i32, [i32, i32, vp, vp, i32, i32, i32, f32, vp, i32, C.c_double, C.c_double, i32,
                                        i32, i32, i32] + [vp] * 6 + [sz, vp]),
    "ds2_error_counts_workspace_bytes": (sz, [i32, i32, i64, i32]),
    "ds2_error_counts": (i32, [i32, i32, i32, vp, vp, vp, i64, vp, i32, i32, i32] + [vp] * 3 + [sz, vp]),
    "ds2_spectrogram_workspace_bytes": (sz, [i32]),
    "ds2_spectrogram_batch": (i32, [i32, vp, vp, vp, i32, i32, i32, vp, i32, i32, vp, i32, vp, sz, vp]),
    "ds2_spectrogram_stream_state_bytes": (sz, [i32]),
    "ds2_spectrogram_stream_workspace_bytes": (sz, [i32, i32]),
    "ds2_spectrogram_stream": (i32, [i32, vp, vp, i32, i32, i32, vp, vp, i32, vp, vp, sz, vp]),
    "ds2_spec_augment_workspace_bytes": (sz, [i32]),
    "ds2_spec_augment": (i32, [i32, i32, i32] + [vp] * 5 + [sz, vp]),
    "ds2_optim_workspace_bytes": (sz, []),
    "ds2_adamw_step": (i32, [i64] + [vp] * 4 + [f32] * 5 + [i32, f32, f32, vp, vp, vp]),
    "ds2_sgd_nesterov_step": (i32, [i64] + [vp] * 3 + [f32] * 3 + [i32, f32, f32, vp, vp, vp]),
    "ds2_gemm_workspace_bytes": (sz, [i32] * 5),
    "ds2_gemm": (i32, [i32] * 5 + [f32, vp, i32, vp, i32, f32, vp, i32, vp, sz, vp]),
    "ds2_gemm_f16": (i32, [i32] * 3 + [f32, vp, i32, vp, i32, f32, vp, i32, vp]),
    "ds2_gemm_f16_scaled": (i32, [i32] * 3 + [f32, vp, i32, vp, i32, f32, vp, i32, vp, vp]),
}

_lib = None


class Ds2Error(RuntimeError):
    pass


def get_lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Ds2Error(f"{LIB_PATH} not found: build it with `make -C deepspeech.pytorch_b200/csrc` "
                           "(or __graft_entry__.build()); there is no CPU / eager fallback")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = get_lib().ds2_last_error().decode(errors="replace")
        raise Ds2Error(f"{what} failed with code {rc}: {msg}")


def current_stream():
    """the `stream` argument of the C-ABI: the current stream of the CURRENT device, so callers make the tensors'
    device current first (kernels, TMA descriptors and the per-device shared-memory opt-ins all bind to it)"""
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@contextlib.contextmanager
def precision_mode(code):
    """run the block in the library's precision mode `code` (PREC_*) and restore the mode it found on exit, also on
    an exception; `None` leaves the mode alone"""
    if code is None:
        yield
        return
    lib = get_lib()
    saved = lib.ds2_get_precision()
    if saved != code:
        check(lib.ds2_set_precision(code), "ds2_set_precision")
    try:
        yield
    finally:
        lib.ds2_set_precision(saved)


def autocast(precision):
    """the reference's autocast around a forward at the model's `precision`: 16 selects the fp16 mode for the block,
    any other value leaves the process-wide mode (`set_precision`) alone"""
    return precision_mode(PREC_F16 if precision == 16 else None)


def ptr(t):
    """device (or host) pointer of a tensor, None -> NULL"""
    return None if t is None else C.c_void_p(t.data_ptr())


def ptr_array(tensors):
    arr = (C.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])
    return arr
