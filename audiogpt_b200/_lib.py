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
AGPT_W2V_MAX_CONV = 8


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
                ("transformer_depth", C.c_int), ("context_dim", C.c_int),
                ("use_spatial_transformer", C.c_int), ("resblock_updown", C.c_int), ("attention_order", C.c_int)]


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


class GsConfig(C.Structure):
    """agpt_gs_cfg (a tagged struct in the header, like agpt_clap_cfg; the create entry point takes a plain pointer)."""
    _fields_ = [("fs2", Fs2Cfg)] + [(n, C.c_int) for n in (
        "n_vq", "glow_hidden", "glow_kernel", "glow_blocks", "glow_layers", "share_wn_layers")]


class GsTaps(C.Structure):
    """agpt_gs_taps (a tagged struct in the header: optional stage outputs of agpt_gs_forward)."""
    _fields_ = [("mel_pre_flow", C.c_void_p), ("prosody", C.c_void_p * 3), ("vq_idx", C.c_void_p * 3)]


class ClapConfig(C.Structure):
    """agpt_clap_cfg: the one config struct with float fields (a tagged struct in the header; the create entry point
    takes it as a plain pointer)."""
    _fields_ = [(n, C.c_int) for n in (
        "vocab_size", "max_position_embeddings", "type_vocab_size", "hidden_size", "num_layers", "num_heads",
        "intermediate_size", "d_proj")] + [("layer_norm_eps", C.c_float), ("proj_layer_norm_eps", C.c_float)]


class Cnn14Config(C.Structure):
    """agpt_cnn14_cfg (a tagged struct in the header, like agpt_clap_cfg; the create entry point takes a plain pointer)."""
    _fields_ = [(n, C.c_int) for n in ("window_size", "hop_size", "mel_bins", "out_emb", "d_proj")]


class LassConfig(C.Structure):
    """agpt_lass_cfg (a tagged struct in the header, like agpt_clap_cfg; the create entry point takes a plain pointer)."""
    _fields_ = [(n, C.c_int) for n in (
        "vocab_size", "max_position_embeddings", "type_vocab_size", "hidden_size", "num_layers", "num_heads",
        "intermediate_size")] + [("layer_norm_eps", C.c_float)]


class PvtConfig(C.Structure):
    """agpt_pvt_cfg (a tagged struct in the header, like agpt_clap_cfg; the create entry point takes a plain pointer)."""
    _fields_ = [(n, C.c_int) for n in ("window_size", "hop_size", "mel_bins", "classes_num")] + [
        (n, C.c_int * 4) for n in ("embed_dims", "depths", "num_heads", "mlp_ratios", "sr_ratios")] + [
        ("interpolate_ratio", C.c_int), ("layer_norm_eps", C.c_float), ("embed_norm_eps", C.c_float)]


class TsdConfig(C.Structure):
    """agpt_tsd_cfg (a tagged struct in the header, like agpt_clap_cfg; the create entry point takes a plain pointer)."""
    _fields_ = [(n, C.c_int) for n in ("time_resolution", "att_pool", "enhancement", "top")] + [
        ("tao", C.c_float), ("mel_bins", C.c_int), ("outputdim", C.c_int)]


class BinauralConfig(C.Structure):
    """agpt_binaural_cfg (the create entry point takes a plain pointer)."""
    _fields_ = [("layers", C.c_int), ("channels", C.c_int)]


class BinauralRow(C.Structure):
    """agpt_binaural_row: one BinauralNetwork forward (a batch item or a chunk of the tool's loop)."""
    _fields_ = [(n, C.c_int64) for n in ("mono_off", "T", "view_off", "view_stride", "K", "keep", "out_off", "out_stride")]


class W2vConfig(C.Structure):
    """agpt_w2v_cfg (a tagged struct in the header, like agpt_clap_cfg; the create entry point takes a plain pointer)."""
    _fields_ = [("conv_layers", C.c_int), ("conv_dim", C.c_int), ("conv_kernel", C.c_int * AGPT_W2V_MAX_CONV),
                ("conv_stride", C.c_int * AGPT_W2V_MAX_CONV)] + [(n, C.c_int) for n in (
        "hidden_size", "num_layers", "num_heads", "intermediate_size", "num_conv_pos_embeddings",
        "num_conv_pos_embedding_groups", "vocab_size")] + [("layer_norm_eps", C.c_float)]


class EmoConfig(C.Structure):
    """agpt_emo_cfg (a tagged struct in the header, like agpt_clap_cfg; the create entry point takes a plain pointer)."""
    _fields_ = [(n, C.c_int) for n in ("input_size", "hidden_size", "num_layers", "embedding_size")]


class TapconvProbeArgs(C.Structure):
    """agpt_tapconv_probe_args (a tagged struct in the header: it carries pointers and floats)."""
    _fields_ = [(n, C.c_int) for n in ("kind", "Cin", "Cout", "K", "dil", "Wreal", "strip_w", "u", "pad", "g")] + [
        ("w", C.c_void_p), ("b", C.c_void_p), ("G", C.c_int), ("L", C.c_int),
        ("inp", C.c_void_p), ("in_gstride", C.c_long), ("in_pitch", C.c_int),
        ("out", C.c_void_p), ("out_gstride", C.c_long), ("out_pitch", C.c_int),
        ("res", C.c_void_p), ("res_gstride", C.c_long), ("res_pitch", C.c_int),
        ("out2", C.c_void_p), ("out2_gstride", C.c_long), ("out2_pitch", C.c_int),
        ("pro", C.c_int), ("slope", C.c_float), ("pvec", C.c_void_p), ("pvec_gstride", C.c_int),
        ("epi", C.c_int), ("scale", C.c_float), ("accumulate", C.c_int), ("csplit", C.c_int),
        ("evec", C.c_void_p), ("evec_gstride", C.c_int),
        ("tc_tall", C.c_int), ("plane_in", C.c_int),
        ("po_hi", C.c_void_p), ("po_lo", C.c_void_p), ("po_slope", C.c_float),
        ("pl_hi", C.c_void_p), ("pl_lo", C.c_void_p), ("pl_pitch", C.c_int),
        ("fma", C.c_int), ("pair", C.c_int),
        ("w2", C.c_void_p), ("b2", C.c_void_p), ("K2", C.c_int), ("dil2", C.c_int)]


class TapconvPipes(C.Structure):
    """agpt_tapconv_pipes: the pipeline switches of agpt_tapconv_probe_pipes."""
    _fields_ = [(n, C.c_int) for n in ("tc_dual", "tc_pipe", "tc_narrow_pipe", "tc_conv_pipe")]


# ran[4] of agpt_tapconv_probe_pipes, in the header's enum order (AGPT_TC_KERN_<name>)
TC_KERNS = ("TILE", "DUAL", "PAIR_PIPE", "NARROW_PIPE", "CONV_PIPE")


# agpt_nn_probe_args.op, in the header's enum order (AGPT_NN_<name>)
NN_OPS = ("GROUPNORM", "LAYERNORM", "SOFTMAX_ROWS", "TRANSPOSE_PAD", "COPY_PAD_ROWS", "CONCAT", "UPSAMPLE2", "AVGPOOL2",
          "IM2COL_S2", "CF_TO_CL_PAD", "TIMESTEP", "TIMESTEP_DEV", "DDIM_TAB", "CONV_OUT_DDIM")


class NnProbeArgs(C.Structure):
    """agpt_nn_probe_args (a tagged struct in the header: it carries pointers and floats)."""
    _fields_ = [("op", C.c_int)] + [(n, C.c_void_p) for n in (
        "x", "x2", "y", "y2", "gamma", "beta", "w", "b", "table", "step", "sel_table", "sel_out")] + [
        ("sel_cols", C.c_int), ("t", C.c_void_p)] + [(n, C.c_int) for n in (
        "N", "H", "W", "C", "C2", "G", "act", "pad", "Nsrc", "single")] + [
        ("rows", C.c_long), ("cols", C.c_int), ("pitch", C.c_int), ("rows_pad", C.c_int),
        ("eps", C.c_float), ("scale", C.c_float)]


# agpt_fs_probe_args.op, in the header's enum order (AGPT_FS_<name>)
FS_OPS = ("EMBED_TOKENS", "ROWMASK", "DUR", "LR_SCAN", "LR_FILL", "GATHER", "AFFINE_MASK", "POSITIONS", "POSEMB_ADD",
          "PITCH_FRAME", "PITCH_PH", "ENERGY", "EMBED_ADD", "GS_SUM", "GS_ACCUM", "GS_REFMASK", "GS_WN_GATE", "GS_SEGMEAN",
          "GS_VQ", "GS_CATPOS", "GS_KPM", "GS_PITCH", "GS_COND_CAT", "GS_SQUEEZE", "GS_FLOW_STEP", "PE_MASK", "PE_DENORM")


class FsProbeArgs(C.Structure):
    """agpt_fs_probe_args (a tagged struct in the header: it carries pointers, ints and floats)."""
    _fields_ = [("op", C.c_int)] + [(n, C.c_void_p) for n in (
        "tok", "midi", "slur", "idx", "idx2", "idx3", "mel2ph", "x", "x2", "x3", "x4", "x5", "E", "E2", "E3", "w", "b",
        "y", "y2", "y3", "iy", "iy2", "kpm")] + [(n, C.c_int) for n in (
        "B", "T", "T2", "H", "C", "M", "nseg", "ntok", "pos_mode", "use_uv", "norm", "first")] + [
        ("rows", C.c_long)] + [(n, C.c_float) for n in ("escale", "neg_emb", "xscale", "alpha", "mean", "std_")]


# agpt_audio_probe_args.op, in the header's enum order (AGPT_AU_<name>)
AU_OPS = ("FRAMES", "LOGMEL", "POWMEL", "STFT_ROWS", "MAGPHASE", "ISTFT_FRAMES", "ISTFT_FINISH", "RESAMPLE", "CNN14_HEAD",
          "L2NORM2", "SIMILARITY", "LASS_INPUT", "LASS_HEAD", "W2V_STEM")


class AudioProbeArgs(C.Structure):
    """agpt_audio_probe_args (a tagged struct in the header: it carries pointers, ints, longs and floats)."""
    _fields_ = [("op", C.c_int)] + [(n, C.c_void_p) for n in (
        "x", "x2", "w", "g", "b", "starts", "y", "y2", "part", "stat", "cnt")] + [(n, C.c_int) for n in (
        "B", "T", "F", "C", "D", "W", "n", "hop", "nb", "nm", "ch", "pitch", "Na", "Nt", "k0", "s0", "s1", "orig", "nw",
        "width", "clip")] + [(n, C.c_long) for n in ("rows", "N", "R", "sb", "stt", "sf")] + [
        (n, C.c_float) for n in ("scale", "shift", "eps")]


# agpt_voc_probe_args.op, in the header's enum order (AGPT_VC_<name>)
VC_OPS = ("CF_TO_CL", "CONV_POST", "AA_SNAKE", "NSF_ADD", "STEP_EMBED", "STEP_EMBED_DEV", "P_SAMPLE_TAB")


class VocProbeArgs(C.Structure):
    """agpt_voc_probe_args (a tagged struct in the header: it carries pointers, ints, longs and a float)."""
    _fields_ = [("op", C.c_int)] + [(n, C.c_void_p) for n in (
        "x", "w", "b", "a", "inv_b", "taps", "t", "ctr", "noises_pp", "y", "ran")] + [(n, C.c_int) for n in (
        "B", "L", "C", "c_out", "Lh", "K", "st", "pad", "nsteps", "clip")] + [
        (n, C.c_long) for n in ("n", "noise_stride")] + [("slope", C.c_float)]


# agpt_an_probe_args.op, in the header's enum order (AGPT_AN_<name>)
AN_OPS = ("LASS_AFFINE", "LASS_UPCOL", "LASS_SHUFFLE", "LASS_FILM", "LASS_FILM_VEC", "LASS_UP", "TSD_PAD4", "TSD_FUSE",
          "TSD_REFEMB", "TSD_HEAD", "TSD_MIX_INTERP", "CLAP_EMBED", "CLAP_EMBED_TYPED", "CLAP_GELU", "EMO_MEAN_NORM",
          "EMO_LINEAR_NORM")


class AnProbeArgs(C.Structure):
    """agpt_an_probe_args (a tagged struct in the header: it carries a handle, pointers, ints and longs)."""
    _fields_ = [("op", C.c_int)] + [(n, C.c_void_p) for n in (
        "h", "x", "x2", "s", "t", "w", "b", "w2", "b2", "vec", "alpha", "beta", "ids", "type_ids", "mask", "woff", "hoff",
        "nin", "dst", "ja", "jb", "y", "y2", "scratch", "kpm", "info")] + [(n, C.c_int) for n in (
        "B", "C", "hh", "ww", "level", "nj", "hid_len", "vec_len", "vec_off", "Td", "T", "O", "n", "att_pool", "N", "L", "H",
        "E", "vocab", "ntypes", "max_blocks")] + [(n, C.c_long) for n in ("rows", "rows_per_sample")]


# (restype, argtypes) of every entry point of include/agpt_b200.h.  Every data pointer and stream is a c_void_p, which
# takes fptr(t), ndarray.ctypes.data_as(...), ctypes arrays, string buffers, byref(...) and None alike.
_I, _L, _F, _D, _P = C.c_int, C.c_long, C.c_float, C.c_double, C.c_void_p
_W = C.POINTER(C.POINTER(C.c_float))     # const float* const* host_weights
_OUT = C.POINTER(C.c_void_p)             # agpt_handle* out
PROTOTYPES = {
    "agpt_last_error": (C.c_char_p, []),
    "agpt_version": (_I, []),
    "agpt_launch_count": (C.c_longlong, []),
    "agpt_destroy": (None, [_P]),
    "agpt_profile_enable": (_I, [_I]),
    "agpt_profile_collect": (_I, [_P, _P, _P, _P]),
    "agpt_profile_tall_launches": (C.c_longlong, []),
    "agpt_profile_plane_launches": (C.c_longlong, []),
    "agpt_profile_dual_launches": (C.c_longlong, []),
    "agpt_profile_pipe_launches": (C.c_longlong, []),
    "agpt_profile_narrow_pipe_launches": (C.c_longlong, []),
    "agpt_profile_conv_pipe_launches": (C.c_longlong, []),
    "agpt_profile_dump": (_L, [_P, _L]),
    "agpt_fma_peak_tflops": (_D, []),
    "agpt_set_tensor_cores": (_I, [_I]),
    "agpt_attention": (_I, [_P, _I, _P, _I, _P, _I, _P, _I, _I, _I, _I, _I, _I, _P]),
    "agpt_set_attention_tc": (_I, [_I]),
    "agpt_attention_masked": (_I, [_P, _I, _P, _I, _P, _I, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "agpt_tapconv_probe": (_I, [_P, _P, _P]),
    "agpt_tapconv_probe_pipes": (_I, [_P, _P, _P, _P]),
    "agpt_nn_probe": (_I, [_P, _P]),
    "agpt_fs_probe": (_I, [_P, _P]),
    "agpt_audio_probe": (_I, [_P, _P]),
    "agpt_voc_probe": (_I, [_P, _P]),
    "agpt_an_probe": (_I, [_P, _P]),
    "agpt_hifigan_create": (_I, [C.POINTER(HifiganCfg), _W, _I, _I, _OUT]),
    "agpt_hifigan_forward": (_I, [_P, _P, _P, _I, _I, _P, _P]),
    "agpt_hifigan_vocode_host": (_I, [_P, _P, _P, _I, _I, _P]),
    "agpt_nsf_source": (_I, [_P, _I, _I, _I, _F, _P, _F, _P, _P, _F, _F, _F, _P, _P]),
    "agpt_diffnet_create": (_I, [C.POINTER(DiffnetCfg), _W, _I, _I, _OUT]),
    "agpt_diffnet_set_cond": (_I, [_P, _P, _I, _I, _P]),
    "agpt_diffnet_eps": (_I, [_P, _P, _P, _P, _P]),
    "agpt_gd_p_sample": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _L, _P, _P]),
    "agpt_gd_sample_loop": (_I, [_P, _P, _I, _I, _P, _P, _L, _I, _P]),
    "agpt_diffnet_launches_per_step": (_L, [_P]),
    "agpt_axpby5": (_I, [_P, _P, _P, _P, _P, _P, _I, _L, _P, _P]),
    "agpt_unet_create": (_I, [C.POINTER(UnetCfg), _W, _I, _I, _OUT]),
    "agpt_unet_set_context": (_I, [_P, _P, _I, _I, _P]),
    "agpt_unet_set_concat": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "agpt_unet_forward": (_I, [_P, _P, _P, _I, _I, _I, _P, _P]),
    "agpt_ddim_update": (_I, [_P, _P, _I, _F, _F, _F, _F, _F, _P, _F, _I, _L, _P, _P, _P]),
    "agpt_unet_ddim_sample": (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _F, _P, _P, _P]),
    "agpt_unet_launches_per_step": (_L, [_P]),
    "agpt_vae_create": (_I, [C.POINTER(VaeCfg), _W, _I, _I, _OUT]),
    "agpt_vae_decode": (_I, [_P, _P, _I, _I, _I, _P, _P]),
    "agpt_vae_encoder_create": (_I, [C.POINTER(VaeCfg), _I, _W, _I, _I, _OUT]),
    "agpt_vae_encode": (_I, [_P, _P, _I, _I, _I, _P, _P]),
    "agpt_pe_create": (_I, [C.POINTER(PeCfg), _W, _I, _I, _OUT]),
    "agpt_pe_forward": (_I, [_P, _P, _I, _I, _P, _P, _I, _I, _F, _F, _P]),
    "agpt_fs2_create": (_I, [C.POINTER(Fs2Cfg), _W, _I, _I, _OUT]),
    "agpt_fs2_encode": (_I, [_P, _P, _I, _I, _P, _P, _P, _I, _P, _P, _P, _P]),
    "agpt_fs2_decode": (_I, [_P, _I, _P, _P, _P, _P, _P, _I, _I, _F, _F, _P, _P, _P, _P, _P, _P, _P]),
    "agpt_gs_create": (_I, [_P, _W, _I, _I, _OUT]),
    "agpt_gs_encode": (_I, [_P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _P, _P, _P]),
    "agpt_gs_forward": (_I, [_P, _I, _P, _P, _P, _I, _P, _I, _P, _I, _P, _F, _F, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "agpt_clap_create": (_I, [_P, _W, _I, _I, _OUT]),
    "agpt_clap_encode": (_I, [_P, _P, _I, _I, _P, _P]),
    "agpt_clap_encode_cls": (_I, [_P, _P, _P, _P, _I, _I, _P, _P]),
    "agpt_clap_similarity": (_I, [_P, _I, _P, _I, _I, _F, _P, _P]),
    "agpt_cnn14_create": (_I, [_P, _W, _I, _I, _OUT]),
    "agpt_cnn14_set_resample": (_I, [_P, _I, _I, _I, _P, _I]),
    "agpt_cnn14_embed": (_I, [_P, _P, _L, _I, _P, _P, _P]),
    "agpt_lass_create": (_I, [_P, _W, _I, _I, _OUT]),
    "agpt_lass_text": (_I, [_P, _P, _P, _I, _I, _P, _P]),
    "agpt_lass_mask": (_I, [_P, _P, _I, _I, _I, _L, _L, _L, _P, _P, _P, _P]),
    "agpt_stft_create": (_I, [_I, _I, _W, _I, _I, _OUT]),
    "agpt_stft_transform": (_I, [_P, _P, _I, _L, _P, _P, _P]),
    "agpt_stft_inverse": (_I, [_P, _P, _P, _I, _I, _P, _P]),
    "agpt_pvt_create": (_I, [_P, _W, _I, _I, _OUT]),
    "agpt_pvt_frames": (_I, [_P, _L, _P]),
    "agpt_pvt_forward": (_I, [_P, _P, _I, _L, _P, _P, _P, _P]),
    "agpt_pvt_dwconv_gelu": (_I, [_P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P]),
    "agpt_pvt_patch7": (_I, [_P, _P, _P, _P, _P, _F, _I, _I, _I, _I, _P, _P]),
    "agpt_pvt_sr_gather": (_I, [_P, _I, _I, _I, _I, _I, _P, _P]),
    "agpt_pvt_head": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P]),
    "agpt_tsd_create": (_I, [_P, _W, _I, _I, _OUT]),
    "agpt_tsd_frames": (_I, [_P, _I, _I, _P]),
    "agpt_tsd_forward": (_I, [_P, _P, _P, _I, _I, _I, _P, _P, _P]),
    "agpt_tsd_stage_events": (_I, [_P, _P, _I]),
    "agpt_tsd_stem": (_I, [_P, _P, _P, _I, _I, _I, _P, _P]),
    "agpt_tsd_avgpool": (_I, [_P, _I, _I, _I, _I, _I, _I, _P, _P]),
    "agpt_tsd_gru": (_I, [_P, _P, _P, _I, _I, _P, _P]),
    "agpt_tsd_enhance": (_I, [_P, _I, _I, _I, _P, _I, _P, _I, _F, _W, _P, _P, _P, _P, _P]),
    "agpt_binaural_create": (_I, [_P, _W, _I, _I, _OUT]),
    "agpt_binaural_forward": (_I, [_P, _P, _P, _P, _I, _P, _I, _P]),
    "agpt_binaural_frames": (_I, [_P, _P, _P, _I, _P, _P]),
    "agpt_binaural_warp": (_I, [_P, _P, _P, _P, _I, _P, _I, _P]),
    "agpt_w2v_create": (_I, [_P, _W, _I, _I, _OUT]),
    "agpt_w2v_frames": (_I, [_P, _L, _P]),
    "agpt_w2v_logits": (_I, [_P, _P, _I, _L, _P, _P]),
    "agpt_w2v_features": (_I, [_P, _P, _I, _L, _P, _P]),
    "agpt_w2v_pos_conv": (_I, [_P, _P, _I, _I, _P, _P]),
    "agpt_emo_create": (_I, [_P, _W, _I, _I, _OUT]),
    "agpt_emo_partials": (_I, [_L, _I, _D, _D, _P, _P, _P]),
    "agpt_emo_embed": (_I, [_P, _P, _L, _I, _D, _D, _P, _P, _P]),
    "agpt_emo_hidden": (_I, [_P, _P, _I, _I, _P, _P]),
    "agpt_emo_forward": (_I, [_P, _P, _I, _I, _P, _P]),
    "agpt_emo_mel": (_I, [_P, _P, _L, _P, _P]),
    "agpt_emo_lstm": (_I, [_P, _P, _I, _I, _L, _P, _P, _P]),
}

_lock = threading.Lock()
_lib = None


def lib() -> C.CDLL:
    """Load the library once and declare every prototype.  Raises if it has not been built (no fallback)."""
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
        for name, (restype, argtypes) in PROTOTYPES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = restype, argtypes
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


def call(name: str, device, *args):
    """agpt_<name>(*args, stream) on ``device``'s current stream; raises on a non-zero return."""
    with torch.cuda.device(device):
        check(getattr(lib(), "agpt_" + name)(*args, cur_stream(device)))


class Engine:
    """One agpt_handle built by ``create`` (an agpt_*_create entry point) from a module's weights; destroyed with the
    Python object."""

    def __init__(self, create: str):
        self.create = create
        self.h = C.c_void_p()
        self.sig = None

    def destroy(self):
        if self.h.value:
            try:
                lib().agpt_destroy(self.h)
            except Exception:   # interpreter shutdown: module globals may already be gone
                pass
            self.h.value = None
        self.sig = None

    def __del__(self):
        self.destroy()

    def ensure(self, device: torch.device, sources, build) -> bool:
        """Build the handle on ``device`` unless it was built there from ``sources`` as they are now: the same
        (data_ptr, _version, device.type) of every tensor.  ``build()`` returns (the create call's leading arguments,
        the weight tensors in the C ABI's order).  Returns True when it (re)built the handle."""
        require_cuda()
        idx = device.index if device.index is not None else torch.cuda.current_device()
        sig = (tuple((t.data_ptr(), t._version, t.device.type) for t in sources), idx)
        if self.h.value and sig == self.sig:
            return False
        self.destroy()
        args, weights = build()
        arr, keep = host_weight_array(weights)
        h = C.c_void_p()
        check(getattr(lib(), self.create)(*args, arr, len(keep), idx, C.byref(h)))
        self.h, self.sig = h, sig
        return True

    def call(self, name: str, device, *args):
        """agpt_<name>(handle, *args, stream) on ``device``'s current stream."""
        call(name, device, self.h, *args)


# ``_h = _lib.engine_handle`` in a class body: the handle of the instance's ``_engine`` (bench.py and the samplers
# pass it to the entry points that take a model handle)
engine_handle = property(lambda self: self._engine.h)
