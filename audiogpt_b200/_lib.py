"""ctypes binding of libagpt_b200.so (include/agpt_b200.h).

The product path has NO CPU fallback: if the library is missing or there is no
CUDA device, the first call raises.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libagpt_b200.so")

AGPT_MAX_UPS = 8
AGPT_MAX_RBK = 8
AGPT_MAX_DIL = 8
AGPT_MAX_LEVELS = 8


class HifiganCfg(C.Structure):
    _fields_ = [
        ("n_mels", C.c_int), ("c_out", C.c_int), ("upsample_initial_channel", C.c_int),
        ("num_upsamples", C.c_int),
        ("upsample_rates", C.c_int * AGPT_MAX_UPS),
        ("upsample_kernel_sizes", C.c_int * AGPT_MAX_UPS),
        ("resblock_type", C.c_int), ("num_kernels", C.c_int),
        ("resblock_kernel_sizes", C.c_int * AGPT_MAX_RBK),
        ("resblock_num_dilations", C.c_int * AGPT_MAX_RBK),
        ("resblock_dilations", (C.c_int * AGPT_MAX_DIL) * AGPT_MAX_RBK),
        ("use_nsf", C.c_int), ("activation", C.c_int), ("snake_logscale", C.c_int),
    ]


class DiffnetCfg(C.Structure):
    _fields_ = [("in_dims", C.c_int), ("hidden_size", C.c_int), ("residual_layers", C.c_int),
                ("residual_channels", C.c_int), ("dilation_cycle_length", C.c_int)]


class UnetCfg(C.Structure):
    _fields_ = [("in_channels", C.c_int), ("out_channels", C.c_int), ("model_channels", C.c_int),
                ("num_res_blocks", C.c_int), ("num_levels", C.c_int),
                ("channel_mult", C.c_int * AGPT_MAX_LEVELS),
                ("attn_at_level", C.c_int * AGPT_MAX_LEVELS),
                ("num_heads", C.c_int), ("num_head_channels", C.c_int),
                ("transformer_depth", C.c_int), ("context_dim", C.c_int)]


class VaeCfg(C.Structure):
    _fields_ = [("embed_dim", C.c_int), ("z_channels", C.c_int), ("ch", C.c_int), ("out_ch", C.c_int),
                ("num_levels", C.c_int), ("ch_mult", C.c_int * AGPT_MAX_LEVELS), ("num_res_blocks", C.c_int),
                ("attn_at_level", C.c_int * AGPT_MAX_LEVELS)]


class PeCfg(C.Structure):
    _fields_ = [("n_mel_bins", C.c_int), ("hidden_size", C.c_int), ("conv_layers", C.c_int),
                ("predictor_hidden", C.c_int), ("predictor_layers", C.c_int), ("predictor_kernel", C.c_int)]


class Fs2Cfg(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "hidden_size", "num_heads", "enc_layers", "dec_layers", "enc_ffn_kernel", "dec_ffn_kernel", "n_tokens", "out_dims",
        "predictor_hidden", "dur_predictor_layers", "dur_predictor_kernel", "predictor_layers", "predictor_kernel",
        "use_pos_embed", "rel_pos", "pitch_type", "use_energy_embed", "use_midi")]


_lock = threading.Lock()
_lib = None


def lib() -> C.CDLL:
    """Load the library once.  Raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -m audiogpt_b200.build` "
                "(audiogpt_b200 has no CPU/PyTorch fallback)")
        L = C.CDLL(LIB_PATH)
        L.agpt_last_error.restype = C.c_char_p
        L.agpt_launch_count.restype = C.c_longlong
        L.agpt_destroy.argtypes = [C.c_void_p]
        L.agpt_destroy.restype = None
        L.agpt_vae_encoder_create.argtypes = [C.POINTER(VaeCfg), C.c_int, C.POINTER(C.POINTER(C.c_float)), C.c_int, C.c_int,
                                              C.POINTER(C.c_void_p)]
        L.agpt_vae_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _lib = L
        return L


def check(rc: int):
    if rc != 0:
        raise RuntimeError("libagpt_b200: " + lib().agpt_last_error().decode("utf-8", "replace"))


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("audiogpt_b200 needs a CUDA device (H100 / sm_90a); there is no CPU fallback")


def host_weight_array(tensors):
    """tensors: list of torch tensors -> (ctypes float** array, keepalive list of numpy arrays)."""
    keep = [np.ascontiguousarray(t.detach().to("cpu", torch.float32).numpy()) for t in tensors]
    arr = (C.POINTER(C.c_float) * len(keep))()
    for i, a in enumerate(keep):
        arr[i] = a.ctypes.data_as(C.POINTER(C.c_float))
    return arr, keep


def fptr(t: torch.Tensor):
    return C.c_void_p(t.data_ptr())


def cur_stream(device=None):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def launch_count() -> int:
    return int(lib().agpt_launch_count())


class HandleOwner:
    """Owns an agpt_handle; destroyed with the Python object."""

    def __init__(self):
        self._h = C.c_void_p(None)

    def _destroy(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                lib().agpt_destroy(h)
            except Exception:   # interpreter shutdown: module globals may already be gone
                pass
            try:
                h.value = None
            except Exception:
                pass

    def __del__(self):
        self._destroy()
