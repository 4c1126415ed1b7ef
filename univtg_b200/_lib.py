"""ctypes binding of include/univtg_b200.h (the C-ABI of the CUDA library).

There is no CPU fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# UNIVTG_LIB: A/B-test another build of the same ABI (profiling only)
LIB_PATH = os.environ.get("UNIVTG_LIB") or os.path.join(_HERE, "lib", "libunivtg_b200.so")
_lib = None

c_int = ctypes.c_int32
c_void_p = ctypes.c_void_p
c_size_t = ctypes.c_size_t
c_float = ctypes.c_float


class Config(ctypes.Structure):
    """univtg_config (include/univtg_b200.h)."""

    _fields_ = [
        ("hidden_dim", c_int),
        ("nheads", c_int),
        ("dim_feedforward", c_int),
        ("enc_layers", c_int),
        ("n_input_proj", c_int),
        ("v_feat_dim", c_int),
        ("t_feat_dim", c_int),
        ("operand_format", c_int),
    ]


class Shape(ctypes.Structure):
    """univtg_shape."""

    _fields_ = [("batch", c_int), ("l_vid", c_int), ("l_txt", c_int), ("training", c_int)]


class Rng(ctypes.Structure):
    """univtg_rng."""

    _fields_ = [("seed", ctypes.c_uint64), ("input_dropout", c_float), ("droppath", c_float)]


class TxtPos(ctypes.Structure):
    """univtg_txt_pos."""

    _fields_ = [("table", c_void_p), ("max_q_l", c_int), ("ln_weight", c_void_p), ("ln_bias", c_void_p), ("drop_mul", c_void_p),
                ("scratch", c_void_p)]


class GemmProblem(ctypes.Structure):
    """univtg_gemm_problem (one problem of univtg_op_gemm_group)."""

    _fields_ = [("a", c_void_p), ("lda", c_int), ("a_mn", c_int), ("b", c_void_p), ("ldb", c_int), ("b_mn", c_int), ("M", c_int),
                ("N", c_int), ("K", c_int), ("ksplit", c_int), ("a_fmt", c_int), ("b_fmt", c_int), ("out_fmt", c_int), ("conv", c_int),
                ("tap", c_int), ("bias", c_void_p), ("act", c_int), ("alpha", c_float), ("row_scale", c_void_p), ("rps_in", c_int),
                ("rps_out", c_int), ("row_off", c_int), ("zero_sep", c_int), ("skip_sep", c_int), ("resid", c_void_p),
                ("ld_resid", c_int), ("addtab", c_void_p), ("ld_addtab", c_int), ("out32", c_void_p), ("ld32", c_int),
                ("out32_id", c_void_p), ("ld32_id", c_int), ("out16", c_void_p), ("out16p", c_void_p), ("ld16", c_int),
                ("accumulate", c_int), ("mask16", c_void_p), ("ld_mask", c_int), ("mask_mul", c_int), ("dact16", c_void_p),
                ("ld_dact", c_int), ("colsum", c_void_p), ("colsum_scale", c_float), ("vec_ok", c_int)]


class LnBwd(ctypes.Structure):
    """univtg_ln_bwd."""

    _fields_ = [("dout", c_void_p), ("ld_dout", c_int), ("y", c_void_p), ("ld_y", c_int), ("y16", c_void_p), ("y_fmt", c_int),
                ("mean", c_void_p), ("rstd", c_void_p), ("gamma", c_void_p), ("rows", c_int), ("d", c_int), ("row_scale", c_void_p),
                ("L", c_int), ("relu_mask_y", c_int), ("dy32", c_void_p), ("dbr16", c_void_p), ("ld16", c_int), ("fmt16", c_int),
                ("dgamma", c_void_p), ("dbeta", c_void_p), ("colsum", c_void_p), ("pgrad_scale", c_float), ("dout_mul", c_void_p)]


class HeadFinalBwd(ctypes.Structure):
    """univtg_head_final_bwd."""

    _fields_ = [(n, c_void_p) for n in ("g_logits", "g_spans", "pred_logits", "pred_spans", "h_cls", "h_span", "w_cls", "w_span", "dz",
                                        "dh_cls", "dh_span", "gw_cls", "gb_cls", "gw_span", "gb_span", "cs_cls", "cs_span")] + \
        [("in_scale", c_float), ("pgrad_scale", c_float), ("B", c_int), ("Lv", c_int), ("d", c_int), ("fmt_act", c_int), ("fmt_grad", c_int)]


class TxtPosBwd(ctypes.Structure):
    """univtg_txt_pos_bwd."""

    _fields_ = [(n, c_void_p) for n in ("dpos", "xt", "table", "gamma", "mean", "rstd", "mul32", "dx", "dtable", "dgamma", "dbeta")] + \
        [("pgrad_scale", c_float), ("B", c_int), ("Lt", c_int), ("L", c_int), ("Lv", c_int), ("d", c_int)]


class LnFwd(ctypes.Structure):
    """univtg_ln_fwd."""

    _fields_ = [("in_", c_void_p), ("in16", c_void_p), ("in_fmt", c_int), ("ld_in", c_int), ("add16", c_void_p), ("ld_add16", c_int),
                ("sum_out", c_void_p), ("rows", c_int), ("d", c_int), ("gamma", c_void_p), ("beta", c_void_p), ("eps", c_float),
                ("fmt", c_int), ("lo", ctypes.c_int64), ("L", c_int), ("Lv", c_int), ("out32", c_void_p), ("out16", c_void_p),
                ("out16p", c_void_p), ("ld16", c_int), ("pos", c_void_p), ("pos_txt", c_void_p), ("outc", c_void_p), ("mul32", c_void_p),
                ("mean_out", c_void_p), ("rstd_out", c_void_p)]


class TxtPosFwd(ctypes.Structure):
    """univtg_txt_pos_fwd."""

    _fields_ = [(n, c_void_p) for n in ("xt", "table", "gamma", "beta", "mul32", "pos", "mean_out", "rstd_out", "xpos16")] + \
        [(n, c_int) for n in ("B", "Lt", "L", "Lv", "d", "fmt")] + [("lo", ctypes.c_int64)]


class AttnFwd(ctypes.Structure):
    """univtg_attn_fwd."""

    _fields_ = [("qkv", c_void_p), ("key_mask", c_void_p), ("out", c_void_p), ("lse", c_void_p)] + \
        [(n, c_int) for n in ("B", "L", "H", "dh", "fmt", "impl", "causal")]


class AttnBwd(ctypes.Structure):
    """univtg_attn_bwd."""

    _fields_ = [(n, c_void_p) for n in ("qkv", "dO", "key_mask", "lse", "delta", "dqkv32", "dqkv16")] + \
        [(n, c_int) for n in ("B", "L", "H", "dh", "fmt", "impl")]


class ClipConfig(ctypes.Structure):
    """univtg_clip_config."""

    _fields_ = [(n, c_int) for n in ("embed_dim", "vision_width", "vision_layers", "patch_size", "image_resolution", "text_width",
                                     "text_layers", "context_length", "vocab_size", "operand_format")]


# symbol -> (restype, argtypes); every symbol declared in include/univtg_b200.h must be listed here
SIGNATURES = {
    "univtg_last_error": (ctypes.c_char_p, []),
    "univtg_abi_version": (c_int, []),
    "univtg_num_params": (c_int, [ctypes.POINTER(Config)]),
    "univtg_packed_bytes": (c_size_t, [ctypes.POINTER(Config)]),
    "univtg_pack_weights": (c_int, [ctypes.POINTER(Config), ctypes.POINTER(c_void_p), c_int, c_void_p, c_void_p]),
    "univtg_workspace_bytes": (c_size_t, [ctypes.POINTER(Config), ctypes.POINTER(Shape)]),
    "univtg_prepare_workspace": (c_int, [ctypes.POINTER(Config), ctypes.POINTER(Shape), c_void_p, c_int, c_void_p]),
    "univtg_plan_create": (c_int, [ctypes.POINTER(Config), ctypes.POINTER(Shape), c_void_p, c_void_p, c_void_p, c_void_p,
                                   ctypes.POINTER(c_void_p)]),
    "univtg_plan_destroy": (None, [c_void_p]),
    "univtg_forward": (c_int, [c_void_p] * 12),
    "univtg_forward_num_launches": (c_int, [c_void_p]),
    "univtg_launch_count": (ctypes.c_int64, []),
    "univtg_host_register": (c_int, [c_void_p, c_size_t, c_int]),
    "univtg_h2d_gather_batch": (c_int, [c_void_p] * 11 + [c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "univtg_host_assemble_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_int, c_int, c_int, c_int, c_int, c_int]),
    "univtg_train_workspace_bytes": (c_size_t, [ctypes.POINTER(Config), ctypes.POINTER(Shape)]),
    "univtg_forward_train": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     ctypes.POINTER(c_void_p), ctypes.POINTER(Rng), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p]),
    "univtg_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(c_void_p), ctypes.POINTER(Rng),
                                c_void_p, c_void_p, c_void_p, c_void_p, c_float, ctypes.POINTER(c_void_p), c_int, c_void_p]),
    "univtg_dropout_mask": (c_int, [ctypes.POINTER(Rng), c_int, c_size_t, c_size_t, c_void_p, c_void_p]),
    "univtg_droppath_scales": (c_int, [ctypes.POINTER(Rng), c_int, c_int, c_void_p, c_void_p]),
    "univtg_plan_set_attention_dropout": (c_int, [c_void_p, c_float]),
    "univtg_plan_set_txt_pos": (c_int, [c_void_p, ctypes.POINTER(TxtPos)]),
    "univtg_txt_pos_scratch_bytes": (c_size_t, [ctypes.POINTER(Config), ctypes.POINTER(Shape)]),
    "univtg_attention_dropout_mask": (c_int, [ctypes.POINTER(Rng), c_float, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "univtg_loss_scratch_bytes": (c_size_t, [c_int, c_int]),
    "univtg_loss_forward": (c_int, [c_void_p] * 10 + [c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p, c_void_p]),
    "univtg_loss_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p]),
    "univtg_qfvs_loss_forward": (c_int, [c_void_p] * 6 + [c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "univtg_qfvs_loss_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p]),
    "univtg_backward_stages":(c_int, [ctypes.POINTER(Config), c_void_p, c_int]),
    "univtg_plan_set_grad_events": (c_int, [c_void_p, ctypes.POINTER(c_void_p), c_int]),
    "univtg_plan_set_backward_sm_budget": (c_int, [c_void_p, c_int]),
    "univtg_decode_mr": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                 c_void_p]),
    "univtg_temporal_nms": (c_int, [c_void_p, c_int, c_int, c_int, ctypes.c_double, c_int, c_void_p, c_void_p, c_void_p]),
    "univtg_eval_mr": (c_int, [c_void_p] * 4 + [c_int, c_int] + [c_void_p] * 5),
    "univtg_eval_hl": (c_int, [c_void_p] * 4 + [c_int, c_int, c_int] + [c_void_p] * 4),
    "univtg_eval_hl_topk": (c_int, [c_void_p] * 5 + [c_int] * 5 + [c_void_p, c_void_p]),
    "univtg_qfvs_match": (c_int, [c_void_p] * 4 + [c_int, c_int, c_void_p, c_void_p]),
    "univtg_adamw_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_size_t, c_float, c_float, c_float, c_float,
                                  c_float, c_int, c_float, c_int, c_void_p, ctypes.POINTER(Config), c_void_p, c_void_p]),
    "univtg_pack_vectors": (c_int, [ctypes.POINTER(Config), ctypes.POINTER(c_void_p), c_int, c_void_p, c_void_p]),
    "univtg_plan_set_profiling": (c_int, [c_void_p, c_int]),
    "univtg_plan_set_input_format": (c_int, [c_void_p, c_int]),
    "univtg_plan_read_profile": (c_int, [c_void_p, c_void_p, c_void_p, c_int]),
    "univtg_op_gemm": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int,
                               c_float, c_void_p, c_void_p, c_void_p]),
    "univtg_op_gemm_cluster": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int,
                                       c_float, c_void_p, c_void_p, c_void_p]),
    "univtg_op_gemm_group": (c_int, [ctypes.POINTER(GemmProblem), c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "univtg_op_layernorm_bwd": (c_int, [ctypes.POINTER(LnBwd), ctypes.POINTER(Rng), c_int, c_void_p, c_void_p]),
    "univtg_op_head_final_bwd": (c_int, [ctypes.POINTER(HeadFinalBwd), c_void_p]),
    "univtg_op_colsum16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_float, c_void_p, c_int, c_int, c_int, c_void_p]),
    "univtg_op_cvt16_colsum": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_float, c_void_p, c_int, c_int,
                                       c_int, c_void_p]),
    "univtg_op_stream_gather": (c_int, [c_void_p, c_int, c_int, c_void_p, c_float, c_void_p, c_void_p, c_float, c_int, c_int, c_int,
                                        c_int, c_void_p]),
    "univtg_op_pool_bwd": (c_int, [c_void_p] * 6 + [c_float, c_int, c_int, c_int, c_void_p]),
    "univtg_op_txt_pos_bwd": (c_int, [ctypes.POINTER(TxtPosBwd), ctypes.POINTER(Rng), c_int, c_void_p]),
    "univtg_debug_gemm_timeline": (c_int, [c_void_p]),
    "univtg_debug_choose_tile": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "univtg_op_layernorm": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_float, c_int, c_void_p, c_void_p, c_int,
                                    c_void_p]),
    "univtg_op_attention": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                    c_void_p]),
    "univtg_op_attention_bwd": (c_int, [c_void_p] * 7 + [c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "univtg_op_attn_delta": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "univtg_op_attention_bwd_full": (c_int, [ctypes.POINTER(AttnBwd), ctypes.POINTER(Rng), c_float, c_int, c_void_p, c_void_p,
                                             c_void_p]),
    "univtg_op_layernorm_fwd": (c_int, [ctypes.POINTER(LnFwd), ctypes.POINTER(Rng), c_int, c_void_p, c_void_p]),
    "univtg_op_txt_pos": (c_int, [ctypes.POINTER(TxtPosFwd), ctypes.POINTER(Rng), c_int, c_void_p]),
    "univtg_op_sine_pos": (c_int, [c_void_p] * 5 + [c_int, c_int, c_int, c_int, ctypes.POINTER(Rng), c_int, c_void_p, c_void_p]),
    "univtg_op_pool_saliency": (c_int, [c_void_p] * 9 + [c_int, c_int, c_int, c_int, c_void_p]),
    "univtg_op_conv_head_final": (c_int, [c_void_p] * 8 + [c_int, c_int, c_int, c_int, c_void_p]),
    "univtg_op_attention_fwd": (c_int, [ctypes.POINTER(AttnFwd), ctypes.POINTER(Rng), c_float, c_int, c_void_p, c_void_p]),
    "univtg_clip_num_params": (c_int, [ctypes.POINTER(ClipConfig)]),
    "univtg_clip_packed_bytes": (c_size_t, [ctypes.POINTER(ClipConfig)]),
    "univtg_clip_pack_weights": (c_int, [ctypes.POINTER(ClipConfig), ctypes.POINTER(c_void_p), c_int, c_int, c_void_p, c_void_p]),
    "univtg_clip_workspace_bytes": (c_size_t, [ctypes.POINTER(ClipConfig), c_int, c_int, c_int]),
    "univtg_clip_encode_image": (c_int, [ctypes.POINTER(ClipConfig), c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p,
                                         c_void_p]),
    "univtg_clip_encode_text": (c_int, [ctypes.POINTER(ClipConfig), c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p,
                                        c_void_p, c_void_p]),
    "univtg_clip_num_launches": (c_int, [ctypes.POINTER(ClipConfig), c_int, c_int]),
    "univtg_teacher_class_bytes": (c_size_t, [c_int, c_int]),
    "univtg_teacher_prepare_classes": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "univtg_teacher_chunk_bytes": (c_size_t, [c_int, ctypes.c_int64, c_int, c_int]),
    "univtg_teacher_label": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, ctypes.c_int64, c_int,
                                     ctypes.c_double, c_void_p, c_size_t, c_void_p, c_void_p]),
    "univtg_debug_py_floordiv": (c_int, [c_void_p, ctypes.c_int64, ctypes.c_double, c_void_p]),
}


def load_library():
    """Load libunivtg_b200.so and attach signatures.  Raises if the library was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "univtg_b200 has no CPU or PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    if lib.univtg_abi_version() != 2:
        raise RuntimeError("univtg_b200: ABI version mismatch between header and library")
    _lib = lib
    return lib


def last_error():
    lib = load_library()
    msg = lib.univtg_last_error()
    return msg.decode() if msg else ""


def check(rc, what):
    if rc != 0:
        raise RuntimeError(f"univtg_b200: {what} failed (rc={rc}): {last_error()}")


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    return c_void_p(t.data_ptr())


def stream_ptr():
    import torch

    return c_void_p(torch.cuda.current_stream().cuda_stream)
