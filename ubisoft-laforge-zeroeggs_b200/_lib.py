"""ctypes binding of libzeggs_b200.so (include/zeggs_b200.h).  Fails loudly when the library is
missing: there is no CPU or PyTorch fallback for the compute path."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libzeggs_b200.so")

c_float_p = C.c_void_p  # raw device pointers are passed as integers (tensor.data_ptr())


class MelArgs(C.Structure):
    _fields_ = [("n_clips", C.c_int), ("n_samples", C.c_int), ("n_fft", C.c_int), ("hop", C.c_int),
                ("n_mels", C.c_int), ("anim_length", C.c_int), ("min_amp", C.c_float),
                ("frames_per_anim", C.c_double),
                ("wav", C.c_void_p), ("window", C.c_void_p), ("twiddle", C.c_void_p),
                ("fb_start", C.c_void_p), ("fb_len", C.c_void_p), ("fb_off", C.c_void_p), ("fb_w", C.c_void_p),
                ("mel_out", C.c_void_p), ("feat_out", C.c_void_p), ("fb_total", C.c_int),
                ("gain", C.c_void_p), ("wav_i16", C.c_void_p)]


GATHER_MAX = 12


class GatherArgs(C.Structure):
    _fields_ = [("B", C.c_int), ("T", C.c_int), ("n_arrays", C.c_int), ("src", C.c_void_p * GATHER_MAX), ("dst", C.c_void_p * GATHER_MAX),
                ("width", C.c_int * GATHER_MAX), ("start", C.c_void_p), ("ex_out", C.c_void_p), ("L", C.c_int), ("ex_width", C.c_int),
                ("n_ex", C.c_int), ("ex_src", C.c_int * GATHER_MAX), ("ex_start", C.c_void_p), ("ex_n", C.c_void_p)]


class PosePostArgs(C.Structure):
    _fields_ = [("N", C.c_int), ("T", C.c_int), ("J", C.c_int), ("rebase", C.c_int), ("start_pos", C.c_float * 3),
                ("start_rot", C.c_float * 4), ("root_pos", C.c_void_p), ("root_rot", C.c_void_p), ("lpos", C.c_void_p),
                ("ltxy", C.c_void_p), ("positions", C.c_void_p), ("euler_deg", C.c_void_p), ("lrot", C.c_void_p)]


class LoudnessArgs(C.Structure):
    _fields_ = [("n_clips", C.c_int), ("n_samples", C.c_int), ("n_seg", C.c_int), ("n_blocks", C.c_int), ("warm", C.c_int),
                ("coef", C.c_double * 10), ("inv_block_len", C.c_double), ("target_lufs", C.c_double),
                ("wav", C.c_void_p), ("wav_i16", C.c_void_p), ("seg_bounds", C.c_void_p), ("blk_seg_lo", C.c_void_p),
                ("blk_seg_hi", C.c_void_p), ("gain_out", C.c_void_p), ("lufs_out", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


class Ctx(C.Structure):
    """zeggs_ctx: per-call GEMM context (scratch buffer, GEMM mode, single-pass weight gradients)."""
    _fields_ = [("scratch", C.c_void_p), ("scratch_bytes", C.c_size_t), ("gemm_mode", C.c_int), ("fast_wgrad", C.c_int)]


class DecoderFwdArgs(C.Structure):
    _fields_ = ([("B", C.c_int), ("T", C.c_int), ("H", C.c_int), ("S", C.c_int), ("Z", C.c_int), ("dt", C.c_float)] +
                [(n, C.c_void_p) for n in (
                    "W0", "b0", "W_ih0", "b_ih0", "W_hh0", "b_hh0", "W_ih1", "b_ih1", "W_hh1", "b_hh1", "W2", "b2",
                    "Wc0", "bc0", "Wc1", "bc1", "Wc2", "bc2", "packed",
                    "in_mean", "in_std", "out_mean", "out_std",
                    "root_pos0", "root_rot0", "pose0", "gaze_pos", "speech", "style",
                    "Y", "root_pos", "root_rot", "workspace")] +
                [("workspace_bytes", C.c_size_t), ("save_for_backward", C.c_int), ("engine", C.c_int),
                 ("packed_tc", C.c_void_p), ("workspace_tc", C.c_void_p), ("ctx", C.c_void_p)])


class DecoderBwdArgs(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in (
        "dY", "dRootPos", "dRootRot", "packed_bwd",
        "dW0", "db0", "dW_ih0", "db_ih0", "dW_hh0", "db_hh0", "dW_ih1", "db_ih1", "dW_hh1", "db_hh1", "dW2", "db2",
        "dWc0", "dbc0", "dWc1", "dbc1", "dWc2", "dbc2", "dSpeech", "dStyle", "workspace")] +
        [("workspace_bytes", C.c_size_t), ("packed_bwd_tc", C.c_void_p), ("workspace_tc", C.c_void_p), ("phase", C.c_int)])


class DecoderFilmFwdArgs(C.Structure):
    _fields_ = [("dec", DecoderFwdArgs)] + [(n, C.c_void_p) for n in ("Wm", "bm", "Wg", "bg", "Wb", "bb")]


class DecoderFilmBwdArgs(C.Structure):
    _fields_ = [("dec", DecoderBwdArgs)] + [(n, C.c_void_p) for n in ("dWm", "dbm", "dWg", "dbg", "dWb", "dbb")]


def _struct(name, ints=(), floats=(), ptrs=(), tail=()):
    fields = [(n, C.c_int) for n in ints] + [(n, C.c_float) for n in floats] + [(n, C.c_void_p) for n in ptrs] + list(tail)
    return type(name, (C.Structure,), {"_fields_": fields})


SpeechEncArgs = _struct("SpeechEncArgs", ints=("B", "T", "C_in", "H", "O"),
                        ptrs=("W0", "b0", "W1", "b1", "W2", "b2", "x", "mask0", "mask1", "y", "workspace"),
                        tail=[("workspace_bytes", C.c_size_t), ("ctx", C.c_void_p)])
SpeechEncGrads = _struct("SpeechEncGrads", ptrs=("dy", "dW0", "db0", "dW1", "db1", "dW2", "db2"))
STYLE_W = ("Wc1", "bc1", "ln1_g", "ln1_b", "Wc2", "bc2", "ln2_g", "ln2_b", "Win", "bin", "Wout", "bout", "ln3_g", "ln3_b",
           "Wf1", "bf1", "Wf2", "bf2", "ln4_g", "ln4_b")
StyleEncArgs = _struct("StyleEncArgs", ints=("B", "T", "C_in", "H", "E", "nheads"), floats=("temperature",),
                       ptrs=STYLE_W + ("x", "eps", "pe", "mask_c1", "mask_c2", "mask_attn", "mask_ao", "mask_ff",
                                       "z", "mu", "logvar", "workspace"),
                       tail=[("workspace_bytes", C.c_size_t), ("ctx", C.c_void_p)])
StyleEncGrads = _struct("StyleEncGrads", ptrs=("dz", "dmu", "dlogvar") + tuple("d" + n for n in STYLE_W))
STYLE_GRU_W = ("Wc1", "bc1", "Wc2", "bc2", "W_ih", "W_hh", "b_ih", "b_hh", "W_ih_r", "W_hh_r", "b_ih_r", "b_hh_r", "Wp", "bp")
StyleEncGruArgs = _struct("StyleEncGruArgs", ints=("B", "T", "C_in", "H", "E"), floats=("temperature",),
                          ptrs=STYLE_GRU_W + ("x", "eps", "z", "mu", "logvar", "workspace"),
                          tail=[("workspace_bytes", C.c_size_t), ("ctx", C.c_void_p)])
StyleEncGruGrads = _struct("StyleEncGruGrads", ptrs=("dz", "dmu", "dlogvar") + tuple("d" + n for n in STYLE_GRU_W))


LossArgs = _struct("LossArgs", ints=("B", "T", "Z"), floats=("dt", "kl_weight"),
                   ptrs=("Y", "root_pos", "root_rot", "WY", "W_root_pos", "W_root_rot", "gaze_pos", "parents", "mu", "logvar",
                         "losses", "dY", "dRootPos", "dRootRot", "dmu", "dlogvar", "workspace"),
                   tail=[("workspace_bytes", C.c_size_t), ("kl_weight_dev", C.c_void_p)])

AnimFeaturesArgs = _struct("AnimFeaturesArgs", ints=("T", "J"),
                           tail=[("order", C.c_int * 3), ("spine2", C.c_int), ("hips", C.c_int), ("head", C.c_int), ("dt", C.c_double)] +
                           [(n, C.c_void_p) for n in ("rotations", "positions", "parents", "root_pos", "root_rot", "root_vel", "root_vrt",
                                                      "lpos", "ltxy", "lvel", "lvrt", "gaze_pos", "gaze_dir", "quat_out", "workspace")] +
                           [("workspace_bytes", C.c_size_t)])
SplineArgs = _struct("SplineArgs", tail=[("n", C.c_longlong), ("m", C.c_longlong), ("C", C.c_int), ("in_f64", C.c_int), ("x", C.c_void_p),
                                         ("y", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)])
MOMENTS_MAX_GROUPS = 8
MomentsArgs = _struct("MomentsArgs", ints=("n_groups",),
                      tail=[("src", C.c_void_p * MOMENTS_MAX_GROUPS), ("width", C.c_int * MOMENTS_MAX_GROUPS), ("rows", C.c_void_p),
                            ("n_sel", C.c_longlong), ("mean", C.c_void_p), ("std", C.c_void_p), ("group_std", C.c_void_p),
                            ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)])
ResampleArgs = _struct("ResampleArgs", tail=[("n_in", C.c_longlong), ("n_out", C.c_longlong), ("channels", C.c_int), ("dtype", C.c_int),
                                             ("L", C.c_int), ("M", C.c_int), ("K4", C.c_int), ("delay", C.c_longlong), ("pcm", C.c_void_p),
                                             ("taps", C.c_void_p), ("out", C.c_void_p)])
BvhParseArgs = _struct("BvhParseArgs", tail=[("n_bytes", C.c_longlong), ("n_frames", C.c_int), ("C", C.c_int), ("max_flagged", C.c_int),
                                             ("text", C.c_void_p), ("out", C.c_void_p), ("flagged", C.c_void_p), ("status", C.c_void_p),
                                             ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)])
BvhFormatArgs = _struct("BvhFormatArgs", ints=("T", "J", "in_f64", "max_flagged"),
                        tail=[("positions", C.c_void_p), ("rotations", C.c_void_p), ("seq", C.c_void_p), ("out", C.c_void_p),
                              ("out_capacity", C.c_longlong), ("row_start", C.c_void_p), ("flagged", C.c_void_p), ("status", C.c_void_p),
                              ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)])
EMBED_MAX_GROUPS = 128
EMBED_MAX_Z = 16384
EmbeddingMomentsArgs = _struct("EmbeddingMomentsArgs", tail=[("N", C.c_longlong), ("Z", C.c_int), ("G", C.c_int), ("X", C.c_void_p),
                                                             ("group", C.c_void_p), ("mean", C.c_void_p), ("cov", C.c_void_p),
                                                             ("group_sum", C.c_void_p), ("group_count", C.c_void_p),
                                                             ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)])


# every symbol include/zeggs_b200.h declares: (name, restype, argtypes)
# C struct name -> ctypes mirror (checked against the library's sizeof at test time: tests/test_abi_cpu.py)
def struct_mirrors():
    return {"zeggs_ctx": Ctx, "zeggs_mel_args": MelArgs, "zeggs_loudness_args": LoudnessArgs, "zeggs_decoder_fwd_args": DecoderFwdArgs,
            "zeggs_decoder_bwd_args": DecoderBwdArgs, "zeggs_speech_enc_args": SpeechEncArgs, "zeggs_speech_enc_grads": SpeechEncGrads,
            "zeggs_style_enc_args": StyleEncArgs, "zeggs_style_enc_grads": StyleEncGrads,
            "zeggs_loss_args": LossArgs, "zeggs_pose_post_args": PosePostArgs, "zeggs_gather_args": GatherArgs,
            "zeggs_style_enc_gru_args": StyleEncGruArgs, "zeggs_style_enc_gru_grads": StyleEncGruGrads,
            "zeggs_anim_features_args": AnimFeaturesArgs, "zeggs_spline_args": SplineArgs, "zeggs_moments_args": MomentsArgs,
            "zeggs_resample_args": ResampleArgs, "zeggs_decoder_film_fwd_args": DecoderFilmFwdArgs,
            "zeggs_decoder_film_bwd_args": DecoderFilmBwdArgs, "zeggs_bvh_parse_args": BvhParseArgs,
            "zeggs_bvh_format_args": BvhFormatArgs, "zeggs_embedding_moments_args": EmbeddingMomentsArgs}


SYMBOLS = [
    ("zeggs_last_error", C.c_char_p, []),
    ("zeggs_version", C.c_int, []),
    ("zeggs_struct_size", C.c_size_t, [C.c_char_p]),
    ("zeggs_launch_count", C.c_longlong, []),
    ("zeggs_timing_enable", None, [C.c_int]),
    ("zeggs_timing_reset", None, []),
    ("zeggs_timing_read", C.c_int, [C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    ("zeggs_mel_num_frames", C.c_int, [C.c_int, C.c_int, C.c_int]),
    ("zeggs_mel_forward", C.c_int, [C.POINTER(MelArgs), C.c_void_p]),
    ("zeggs_window_gather", C.c_int, [C.POINTER(GatherArgs), C.c_void_p]),
    ("zeggs_normalize_rows", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]),
    ("zeggs_pose_to_bvh_channels", C.c_int, [C.POINTER(PosePostArgs), C.c_void_p]),
    ("zeggs_loudness_workspace_bytes", C.c_size_t, [C.c_int, C.c_int]),
    ("zeggs_loudness_gain", C.c_int, [C.POINTER(LoudnessArgs), C.c_void_p]),
    ("zeggs_decoder_packed_bytes", C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    ("zeggs_decoder_pack_weights", C.c_int, [C.POINTER(DecoderFwdArgs), C.c_void_p, C.c_void_p]),
    ("zeggs_decoder_workspace_bytes", C.c_size_t, [C.c_int] * 6),
    ("zeggs_decoder_window_fwd", C.c_int, [C.POINTER(DecoderFwdArgs), C.c_void_p]),
    ("zeggs_decoder_packed_tc_bytes", C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    ("zeggs_decoder_tc_workspace_bytes", C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    ("zeggs_decoder_pack_weights_tc", C.c_int, [C.POINTER(DecoderFwdArgs), C.c_void_p, C.c_void_p]),
    ("zeggs_debug_set_tc_trace", None, [C.c_void_p]),
    ("zeggs_decoder_packed_bwd_bytes", C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    ("zeggs_decoder_pack_weights_bwd", C.c_int, [C.POINTER(DecoderFwdArgs), C.c_void_p, C.c_void_p]),
    ("zeggs_decoder_bwd_workspace_bytes", C.c_size_t, [C.c_int] * 5),
    ("zeggs_decoder_window_bwd", C.c_int, [C.POINTER(DecoderFwdArgs), C.POINTER(DecoderBwdArgs), C.c_void_p]),
    ("zeggs_decoder_packed_bwd_tc_bytes", C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    ("zeggs_decoder_bwd_tc_workspace_bytes", C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    ("zeggs_decoder_pack_weights_bwd_tc", C.c_int, [C.POINTER(DecoderFwdArgs), C.c_void_p, C.c_void_p]),
    ("zeggs_decoder_packed_film_bytes", C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    ("zeggs_decoder_pack_weights_film", C.c_int, [C.POINTER(DecoderFilmFwdArgs), C.c_void_p, C.c_void_p]),
    ("zeggs_decoder_film_workspace_bytes", C.c_size_t, [C.c_int] * 6),
    ("zeggs_decoder_film_window_fwd", C.c_int, [C.POINTER(DecoderFilmFwdArgs), C.c_void_p]),
    ("zeggs_decoder_packed_bwd_film_bytes", C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    ("zeggs_decoder_pack_weights_bwd_film", C.c_int, [C.POINTER(DecoderFilmFwdArgs), C.c_void_p, C.c_void_p]),
    ("zeggs_decoder_film_bwd_workspace_bytes", C.c_size_t, [C.c_int] * 5),
    ("zeggs_decoder_film_window_bwd", C.c_int, [C.POINTER(DecoderFilmFwdArgs), C.POINTER(DecoderFilmBwdArgs), C.c_void_p]),
    ("zeggs_speech_enc_workspace_bytes", C.c_size_t, [C.c_int] * 5),
    ("zeggs_speech_enc_fwd", C.c_int, [C.POINTER(SpeechEncArgs), C.c_void_p]),
    ("zeggs_speech_enc_bwd", C.c_int, [C.POINTER(SpeechEncArgs), C.POINTER(SpeechEncGrads), C.c_void_p]),
    ("zeggs_style_enc_workspace_bytes", C.c_size_t, [C.c_int] * 6),
    ("zeggs_style_enc_fwd", C.c_int, [C.POINTER(StyleEncArgs), C.c_void_p]),
    ("zeggs_style_enc_bwd", C.c_int, [C.POINTER(StyleEncArgs), C.POINTER(StyleEncGrads), C.c_void_p]),
    ("zeggs_style_enc_gru_workspace_bytes", C.c_size_t, [C.c_int] * 6),
    ("zeggs_style_enc_gru_fwd", C.c_int, [C.POINTER(StyleEncGruArgs), C.c_void_p]),
    ("zeggs_style_enc_gru_bwd", C.c_int, [C.POINTER(StyleEncGruArgs), C.POINTER(StyleEncGruGrads), C.c_void_p]),
    ("zeggs_loss_workspace_bytes", C.c_size_t, [C.c_int, C.c_int]),
    ("zeggs_loss_fwd_bwd", C.c_int, [C.POINTER(LossArgs), C.c_void_p]),
    ("zeggs_dropout_mask", C.c_int, [C.c_void_p, C.c_size_t, C.c_float, C.c_ulonglong, C.c_void_p]),
    ("zeggs_dropout_mask_dev", C.c_int, [C.c_void_p, C.c_size_t, C.c_float, C.c_void_p, C.c_ulonglong, C.c_void_p]),
    ("zeggs_randn_dev", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_ulonglong, C.c_void_p]),
    ("zeggs_radam_step_dev", C.c_int, [C.c_void_p] * 4 + [C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("zeggs_sgemm", C.c_int, [C.c_int] * 4 + [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                               C.c_int, C.c_int, C.c_int, C.c_void_p]),
    ("zeggs_tc_gemm_bf16", C.c_int, [C.c_int] * 3 + [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    ("zeggs_gemm_f32_ctx", C.c_int, [C.c_void_p] + [C.c_int] * 4 + [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_int, C.c_int, C.c_void_p]),
    ("zeggs_split_bf16", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    ("zeggs_anim_features_workspace_bytes", C.c_size_t, [C.c_int, C.c_int]),
    ("zeggs_anim_features", C.c_int, [C.POINTER(AnimFeaturesArgs), C.c_void_p]),
    ("zeggs_quat_to_euler_deg", C.c_int, [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]),
    ("zeggs_spline_resample_workspace_bytes", C.c_size_t, [C.c_longlong, C.c_int]),
    ("zeggs_spline_resample", C.c_int, [C.POINTER(SplineArgs), C.c_void_p]),
    ("zeggs_masked_moments_workspace_bytes", C.c_size_t, [C.c_longlong, C.c_int]),
    ("zeggs_masked_moments", C.c_int, [C.POINTER(MomentsArgs), C.c_void_p]),
    ("zeggs_embedding_moments_workspace_size", C.c_size_t, [C.c_longlong, C.c_int, C.c_int]),
    ("zeggs_embedding_moments", C.c_int, [C.POINTER(EmbeddingMomentsArgs), C.c_void_p]),
    ("zeggs_resample", C.c_int, [C.POINTER(ResampleArgs), C.c_void_p]),
    ("zeggs_bvh_parse_motion_workspace_size", C.c_size_t, [C.c_longlong, C.c_int]),
    ("zeggs_bvh_parse_motion", C.c_int, [C.POINTER(BvhParseArgs), C.c_void_p]),
    ("zeggs_bvh_format_motion_max_size", C.c_longlong, [C.c_int, C.c_int]),
    ("zeggs_bvh_format_motion_workspace_size", C.c_size_t, [C.c_int, C.c_int]),
    ("zeggs_bvh_format_motion", C.c_int, [C.POINTER(BvhFormatArgs), C.c_void_p]),
]

_lib = None


class ZeggsError(RuntimeError):
    pass


def lib():
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ZeggsError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                "zeggs_b200 has no CPU fallback.")
        l = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(l, name)  # AttributeError if the ABI and the header drift apart
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().zeggs_last_error()
        raise ZeggsError(f"{what} failed (rc={rc}): {msg.decode() if msg else ''}")


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device pointer of a contiguous float32/int32 CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise ZeggsError("zeggs_b200 kernels take CUDA tensors (no CPU path)")
    if not t.is_contiguous():
        raise ZeggsError("tensor must be contiguous")
    return t.data_ptr()
