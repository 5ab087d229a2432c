"""ctypes binding of libmsam_b200.so (include/msam_b200.h).  There is NO CPU fallback: if the library is missing or
no sm_90 device is present, calls raise."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmsam_b200.so")


class MsamConfig(ctypes.Structure):
    _fields_ = [
        ("embed_dim", c_int32), ("depth", c_int32), ("num_heads", c_int32), ("global_attn", c_int32 * 8),
        ("window_size", c_int32), ("image_size", c_int32), ("patch_size", c_int32), ("out_chans", c_int32),
        ("max_batch", c_int32), ("max_prompts", c_int32),
    ]


_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(micro_sam_b200 has no CPU / PyTorch fallback)."
            )
        L = ctypes.CDLL(LIB_PATH)
        L.msam_last_error.restype = c_char_p
        L.msam_launch_count.restype = c_int64
        L.msam_create.argtypes = [POINTER(MsamConfig), c_int, POINTER(c_void_p)]
        L.msam_destroy.argtypes = [c_void_p]
        L.msam_load_weight.argtypes = [c_void_p, c_char_p, c_void_p, POINTER(c_int64), c_int]
        L.msam_finalize_weights.argtypes = [c_void_p]
        L.msam_encode_f32.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_void_p]
        L.msam_encode_u8.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]
        L.msam_op_gemm.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                   c_int, c_void_p]
        L.msam_op_gemm_tn.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]
        L.msam_op_gemm_nn.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]
        L.msam_op_layernorm.argtypes = [c_void_p, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int, c_void_p]
        L.msam_op_attention.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p]
        L.msam_op_dec_t2i.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p]
        L.msam_op_dec_i2t.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]
        L.msam_op_dec_upscale.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p]
        L.msam_set_image_embedding.argtypes = [c_void_p, c_void_p, c_void_p]
        L.msam_decode.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]
        L.msam_decode_ex.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                     c_void_p]
        L.msam_prompt_encode.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                         c_void_p]
        L.msam_get_dense_pe.argtypes = [c_void_p, c_void_p, c_void_p]
        L.msam_mask_decode.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]
        L.msam_mask_stats.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p,
                                      c_void_p, c_void_p]
        L.msam_mask_stats_lazy.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p, c_float,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
        L.msam_remove_small_regions.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]
        L.msam_mask_boxes.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]
        L.msam_local_otsu_threshold.argtypes = [c_void_p, c_int, c_void_p, c_void_p]
        L.msam_mask_stats_ex.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_float, c_void_p, c_void_p,
                                         c_void_p, c_void_p]
        L.msam_upsample_masks_ex.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                             c_void_p, c_void_p]
        L.msam_paint_ex.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int,
                                    c_void_p, c_int, c_void_p]
        L.msam_upsample_masks.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p,
                                          c_void_p, c_void_p]
        L.msam_paint.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_int,
                                 c_void_p, c_int, c_void_p]
        L.msam_amg_filter_nms.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_float, c_float,
                                          POINTER(c_int32), POINTER(c_int32), c_void_p, c_void_p, c_void_p]
        L.msam_mask_loss_stats.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]
        L.msam_to_image.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]
        L.msam_paint_min_area.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                          c_float, c_void_p, c_int, c_void_p]
        L.msam_finish_segmentation.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]
        L.msam_paint_canvas.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                        c_float, c_int, c_int, c_void_p, c_int, c_void_p]
        L.msam_canvas_to_label.argtypes = [c_void_p, c_int64, c_void_p, c_void_p]
        L.msam_mask_nms.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_int, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p]
        L.msam_profile.argtypes = [c_int]
        L.msam_profile_report.argtypes = [ctypes.c_char_p, c_int]
        L.msam_encode_u8_blocks.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]
        L.msam_encode_train.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_void_p]
        L.msam_encode_backward.argtypes = [c_void_p, c_void_p, c_void_p]
        L.msam_encoder_grad.argtypes = [c_void_p, c_char_p, c_void_p, c_int64, c_void_p]
        L.msam_op_bgemm.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int64, c_int64, c_int64,
                                    c_int64, c_int, c_int, c_void_p, c_int, c_int64, c_int64, c_float, c_int, c_void_p]
        L.msam_op_layernorm_bwd.argtypes = [c_void_p, c_int, c_int, c_void_p, c_float, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                            c_void_p, c_void_p]
        L.msam_debug_attn_trace.argtypes = [c_void_p]
        L.msam_decoder_train_forward.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                                 c_void_p]
        L.msam_decoder_train_forward_ex.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p,
                                                    c_void_p, c_void_p]
        L.msam_op_mask_downscaling_train.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
        L.msam_decoder_train_backward.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
        L.msam_decoder_grad.argtypes = [c_void_p, c_char_p, c_void_p, c_int64, c_void_p]
        L.msam_decoder_zero_grads.argtypes = [c_void_p, c_void_p]
        L.msam_optimizer_step.argtypes = [c_void_p, c_float, c_float, c_float, c_float, c_float, c_void_p]
        L.msam_train_param.argtypes = [c_void_p, c_char_p, c_void_p, c_int64, c_void_p]
        L.msam_train_tensor_count.argtypes = [c_void_p]
        L.msam_train_tensor_info.argtypes = [c_void_p, c_int, ctypes.c_char_p, c_int, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_int64)]
        L.msam_mask_loss_backward.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]
        L.msam_prompt_targets.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_double, c_uint64, c_void_p,
                                          c_void_p, c_void_p, c_void_p]
        L.msam_prompt_sample_points.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                                c_uint64, c_void_p, c_void_p, c_void_p, c_void_p]
        L.msam_prompt_iterative.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_uint64,
                                            c_void_p, c_void_p, c_void_p]
        _lib = L
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError("libmsam_b200: " + lib().msam_last_error().decode())


def profile_report():
    """Per-kernel CUDA-event times since msam_profile(1): list of {"name", "ms", "n", "flops", "bytes"}."""
    import json
    buf = ctypes.create_string_buffer(1 << 16)
    n = lib().msam_profile_report(buf, len(buf))
    if n < 0:
        raise RuntimeError("libmsam_b200: " + lib().msam_last_error().decode())
    return json.loads(buf.value.decode())


def launch_count() -> int:
    return int(lib().msam_launch_count())


def ptr(t):
    """device/host pointer of a contiguous torch tensor (or None)."""
    if t is None:
        return None
    assert t.is_contiguous(), "tensor must be contiguous"
    return c_void_p(t.data_ptr())


def cur_stream():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)
