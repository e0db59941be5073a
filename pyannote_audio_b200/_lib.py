"""ctypes binding of libb200diar.so (C ABI declared in include/b200diar.h).

There is NO CPU fallback: if the CUDA library is missing or cannot be loaded, importing a product op raises.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libb200diar.so")

c_float_p = C.POINTER(C.c_float)


class SegWeights(C.Structure):
    _fields_ = [
        ("wav_norm_weight", C.c_float), ("wav_norm_bias", C.c_float),
        ("sinc_filters", c_float_p),
        ("norm_weight", c_float_p * 3), ("norm_bias", c_float_p * 3),
        ("conv_weight", c_float_p * 2), ("conv_bias", c_float_p * 2),
        ("lstm_layers", C.c_int32),
        ("lstm_w_ih", c_float_p * 8), ("lstm_w_hh", c_float_p * 8),
        ("lstm_b_ih", c_float_p * 8), ("lstm_b_hh", c_float_p * 8),
        ("linear_weight", c_float_p * 2), ("linear_bias", c_float_p * 2),
        ("classifier_weight", c_float_p), ("classifier_bias", c_float_p),
    ]


class SegCapture(C.Structure):
    _fields_ = [
        ("af_wav", C.c_void_p), ("P0", C.c_void_p), ("af0", C.c_void_p), ("P1", C.c_void_p), ("af1", C.c_void_p),
        ("P2", C.c_void_p), ("af2", C.c_void_p), ("x0", C.c_void_p),
        ("gx", C.c_void_p * 4), ("y", C.c_void_p * 4), ("y_hi", C.c_void_p * 4), ("y_lo", C.c_void_p * 4),
        ("z1", C.c_void_p), ("z1_hi", C.c_void_p), ("z1_lo", C.c_void_p), ("z2", C.c_void_p),
        ("cls", C.c_void_p), ("logp", C.c_void_p), ("scores", C.c_void_p), ("max_scores", C.c_void_p),
    ]


class ConvBN(C.Structure):
    _fields_ = [("conv_weight", c_float_p), ("bn_weight", c_float_p), ("bn_bias", c_float_p),
                ("bn_mean", c_float_p), ("bn_var", c_float_p)]


class EmbWeights(C.Structure):
    _fields_ = [("stem", ConvBN), ("block_conv1", ConvBN * 16), ("block_conv2", ConvBN * 16),
                ("block_shortcut", ConvBN * 16), ("seg1_weight", c_float_p), ("seg1_bias", c_float_p)]


class EmbBottleneckWeights(C.Structure):
    _fields_ = [("num_blocks", C.c_int32 * 4), ("stem", ConvBN), ("block_conv1", C.POINTER(ConvBN)),
                ("block_conv2", C.POINTER(ConvBN)), ("block_conv3", C.POINTER(ConvBN)),
                ("block_shortcut", C.POINTER(ConvBN)), ("seg1_weight", c_float_p), ("seg1_bias", c_float_p)]


class XvecWeights(C.Structure):
    _fields_ = [
        ("wav_norm_weight", C.c_float), ("wav_norm_bias", C.c_float),
        ("sinc_filters", c_float_p),
        ("norm_weight", c_float_p * 3), ("norm_bias", c_float_p * 3),
        ("conv_weight", c_float_p * 2), ("conv_bias", c_float_p * 2),
        ("tdnn_weight", c_float_p * 5), ("tdnn_bias", c_float_p * 5),
        ("bn_weight", c_float_p * 5), ("bn_bias", c_float_p * 5), ("bn_mean", c_float_p * 5), ("bn_var", c_float_p * 5),
        ("dimension", C.c_int32), ("embedding_weight", c_float_p), ("embedding_bias", c_float_p),
    ]


class XvecMfccWeights(C.Structure):
    _fields_ = [
        ("dct_mat", c_float_p), ("window", c_float_p), ("mel_fb", c_float_p),
        ("tdnn_weight", c_float_p * 5), ("tdnn_bias", c_float_p * 5),
        ("bn_weight", c_float_p * 5), ("bn_bias", c_float_p * 5), ("bn_mean", c_float_p * 5), ("bn_var", c_float_p * 5),
        ("dimension", C.c_int32), ("embedding_weight", c_float_p), ("embedding_bias", c_float_p),
    ]


class SslLayerWeights(C.Structure):
    _fields_ = [(name, c_float_p) for name in (
        "in_proj_weight", "in_proj_bias", "out_proj_weight", "out_proj_bias", "gru_weight", "gru_bias", "gru_const",
        "layer_norm_weight", "layer_norm_bias", "ff1_weight", "ff1_bias", "ff2_weight", "ff2_bias",
        "final_layer_norm_weight", "final_layer_norm_bias")]


class SslWeights(C.Structure):
    _fields_ = [
        ("conv0_weight", c_float_p), ("conv0_norm_weight", c_float_p), ("conv0_norm_bias", c_float_p),
        ("conv_weight", c_float_p * 6),
        ("proj_norm_weight", c_float_p), ("proj_norm_bias", c_float_p), ("proj_weight", c_float_p),
        ("proj_bias", c_float_p), ("pos_conv_weight", c_float_p), ("pos_conv_bias", c_float_p),
        ("encoder_norm_weight", c_float_p), ("encoder_norm_bias", c_float_p),
        ("rel_attn_embed", c_float_p), ("rel_bucket", C.POINTER(C.c_int32)),
        ("num_layers", C.c_int32), ("layer", SslLayerWeights * 12), ("layer_weights", c_float_p),
        ("lstm_layers", C.c_int32),
        ("lstm_w_ih", c_float_p * 8), ("lstm_w_hh", c_float_p * 8),
        ("lstm_b_ih", c_float_p * 8), ("lstm_b_hh", c_float_p * 8),
        ("linear_weight", c_float_p * 2), ("linear_bias", c_float_p * 2),
        ("classifier_weight", c_float_p), ("classifier_bias", c_float_p),
    ]


class B200Error(RuntimeError):
    pass


_lib = None

_PROTOS = {
    "b200_last_error": (C.c_char_p, []),
    "b200_version": (C.c_int, []),
    "b200_ctx_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    "b200_ctx_destroy": (C.c_int, [C.c_void_p]),
    "b200_ctx_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64]),
    "b200_ctx_launch_count": (C.c_int64, [C.c_void_p]),
    "b200_ctx_timer": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
    "b200_seg_load": (C.c_int, [C.c_void_p, C.POINTER(SegWeights)]),
    "b200_seg_load_head": (C.c_int, [C.c_void_p, C.POINTER(SegWeights), C.c_int32, C.c_int32]),
    "b200_emb_load": (C.c_int, [C.c_void_p, C.POINTER(EmbWeights)]),
    "b200_emb_load_bottleneck": (C.c_int, [C.c_void_p, C.POINTER(EmbBottleneckWeights)]),
    "b200_xvec_load": (C.c_int, [C.c_void_p, C.POINTER(XvecWeights)]),
    "b200_xvec_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                                    C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_xvec_mfcc_load": (C.c_int, [C.c_void_p, C.POINTER(XvecMfccWeights)]),
    "b200_xvec_mfcc_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                         C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_xvec_mfcc_features": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                          C.c_void_p]),
    "b200_ssl_load": (C.c_int, [C.c_void_p, C.POINTER(SslWeights), C.c_int32, C.c_int32]),
    "b200_ssl_forward_window": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_ssl_forward_scores": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_ssl_features": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                    C.c_void_p]),
    "b200_seg_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    "b200_seg_forward_window": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_seg_forward_scores": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_seg_stages": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                  C.POINTER(SegCapture), C.c_void_p]),
    "b200_seg_head_stages": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(SegCapture),
                                       C.c_void_p]),
    "b200_sincnet_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                       C.c_void_p]),
    "b200_powerset_to_multilabel": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "b200_powerset_to_multilabel_generic": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                                      C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_emb_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    "b200_emb_forward_push": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_int32, C.c_void_p]),
    "b200_push": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p]),
    "b200_emb_fbank": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_emb_trunk": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_emb_trunk_stage": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_void_p]),
    "b200_emb_forward_utt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                                       C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_emb_forward_embedding": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                             C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_stats_pool": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_int32, C.c_int32, C.c_void_p]),
    "b200_speaker_count": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_reconstruct": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                   C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_frame_transitions": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                        C.c_void_p]),
    "b200_clean_frames": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_linkage_centroid": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                        C.c_void_p]),
    "b200_linkage_centroid_batched": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                                C.c_void_p, C.c_void_p]),
    "b200_linkage_bytes": (C.c_int64, [C.c_void_p, C.c_int32, C.c_int32]),
    "b200_vbx_batched": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                   C.c_double, C.c_double, C.c_int32, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    "b200_fcluster_distance": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_void_p]),
    "b200_cdist_cosine": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                    C.c_void_p]),
    "b200_vbx": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double,
                           C.c_int32, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_audio_num_frames": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32]),
    "b200_emb_fbank_plan": (C.c_int64, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_audio_ingest": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int32,
                                    C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]),
    "b200_aggregate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                 C.c_void_p, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "b200_aggregate_window": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_int32, C.c_float, C.c_float, C.c_void_p,
                                        C.c_void_p]),
    "b200_powerset_speech": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "b200_powerset_speech_generic": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                               C.c_void_p, C.c_void_p]),
    "b200_plda_transform": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_weighted_centroids": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                          C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200_assign": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
}

# symbols that every build must export (tests/test_abi.py checks the header against the .so)
def load():
    """Load the shared library (once). Raises B200Error with a clear message when it is not there."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200Error(
            f"{LIB_PATH} not found: build it with `python -m pyannote_audio_b200._build` "
            "(or __graft_entry__.build()). pyannote_audio_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _PROTOS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int):
    if rc == 0:
        return
    msg = load().b200_last_error().decode("utf-8", "replace")
    if rc == -1:
        raise ValueError(msg)
    if rc == -3:
        raise MemoryError(msg)
    raise B200Error(f"[b200 status {rc}] {msg}")
