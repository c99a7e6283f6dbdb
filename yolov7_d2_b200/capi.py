"""ctypes binding of libyb200.so -- the only way Python reaches the CUDA kernels.

There is no fallback: if the library is missing or a symbol is absent, importing the hot path fails loudly.
Every wrapper takes torch tensors only to read `data_ptr()` / shapes and the current CUDA stream; the C ABI
itself (include/yb200.h) sees plain pointers and integers.
"""
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libyb200.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "yb200.h")

c_int = ctypes.c_int
c_i64 = ctypes.c_int64
c_void_p = ctypes.c_void_p
c_float = ctypes.c_float


class Yb200Error(RuntimeError):
    pass


ERR_INVALID, ERR_UNSUPPORTED, ERR_CUDA = -1, -2, -3  # yb200_status (include/yb200.h)


class Act(ctypes.Structure):
    """mirror of `yb200_act` (include/yb200.h)"""

    _fields_ = [
        ("ptr", c_void_p),
        ("n", ctypes.c_int32),
        ("h", ctypes.c_int32),
        ("w", ctypes.c_int32),
        ("c", ctypes.c_int32),
        ("c_pitch", ctypes.c_int32),
        ("c_off", ctypes.c_int32),
    ]


class PackDesc(ctypes.Structure):
    """mirror of `yb200_pack_desc` (include/yb200.h)"""

    _fields_ = [("w_oihw", c_void_p), ("w_fwd", c_void_p), ("w_dgrad", c_void_p), ("cout", ctypes.c_int32), ("cin", ctypes.c_int32),
                ("ksize", ctypes.c_int32), ("cout_pad", ctypes.c_int32), ("cin_pad", ctypes.c_int32), ("reserved", ctypes.c_int32)]


MOSAIC_MAX_SOURCES = 5  # four tiles and the mixup source


class MosaicDesc(ctypes.Structure):
    """mirror of `yb200_mosaic_desc` (include/yb200.h)"""

    _fields_ = [("src_off", c_i64 * MOSAIC_MAX_SOURCES), ("out_off", c_i64), ("minv", ctypes.c_double * 6),
                ("src_h", ctypes.c_int32 * MOSAIC_MAX_SOURCES), ("src_w", ctypes.c_int32 * MOSAIC_MAX_SOURCES),
                ("tile_h", ctypes.c_int32 * 4), ("tile_w", ctypes.c_int32 * 4), ("rect", ctypes.c_int32 * 16), ("pad", ctypes.c_int32 * 8),
                ("in_h", ctypes.c_int32), ("in_w", ctypes.c_int32), ("out_h", ctypes.c_int32), ("out_w", ctypes.c_int32),
                ("mode", ctypes.c_int32), ("mix", ctypes.c_int32), ("mix_h", ctypes.c_int32), ("mix_w", ctypes.c_int32),
                ("jit_h", ctypes.c_int32), ("jit_w", ctypes.c_int32), ("flip", ctypes.c_int32), ("x_off", ctypes.c_int32),
                ("y_off", ctypes.c_int32), ("reserved", ctypes.c_int32)]


def declared_symbols(header_path=HEADER_PATH):
    """Every function the public header declares (used by the CPU test that checks the exports)."""
    with open(header_path) as fh:
        src = fh.read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(yb200_[a-z0-9_]+)\s*\(", src)))


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Yb200Error(
                f"{LIB_PATH} not found: build it with `python -m yolov7_d2_b200.build` (needs nvcc). "
                "The hot path has no CPU / PyTorch fallback."
            )
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.yb200_last_error.restype = ctypes.c_char_p
        _lib.yb200_conv2d_wgrad_workspace.restype = c_i64
        _lib.yb200_simota_workspace.restype = c_i64
        _lib.yb200_nms_workspace.restype = c_i64
        _lib.yb200_grad_norm_workspace.restype = c_i64
        for _n in ("yb200_dwconv7_wgrad_workspace", "yb200_layernorm_bwd_workspace", "yb200_colsum_workspace", "yb200_attention_bwd_workspace"):
            getattr(_lib, _n).restype = c_i64
        for name in declared_symbols():
            if not hasattr(_lib, name):
                raise Yb200Error(f"libyb200.so does not export {name} declared in include/yb200.h")
    return _lib


def check(rc, what):
    if rc != 0:
        raise Yb200Error(f"{what} failed ({rc}): {lib().yb200_last_error().decode()}")


def stream_ptr():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return c_void_p(t.data_ptr()) if t is not None else c_void_p(0)


def act(t, c_off=0, c=None):
    """View of an NHWC bf16 tensor [N,H,W,Cpitch] (contiguous) restricted to channels [c_off, c_off+c)."""
    assert t.dtype in (torch.bfloat16, torch.float16) and t.dim() == 4 and t.is_contiguous(), (t.dtype, t.shape, t.stride())
    n, h, w, cp = t.shape
    return Act(t.data_ptr(), n, h, w, cp - c_off if c is None else c, cp, c_off)


def _f32(t):
    assert t.dtype == torch.float32 and t.is_contiguous(), (t.dtype, t.shape)
    return ptr(t)


def _i32(t):
    assert t.dtype == torch.int32 and t.is_contiguous(), (t.dtype, t.shape)
    return ptr(t)


def detr_match_cost(logits, boxes, labels, target_boxes, offsets, num_targets, w_class, w_bbox, w_giou, cost):
    """yb200_detr_match_cost on the current stream: logits [L, B, Q, K1], boxes [L, B, Q, 4] -> cost (L*Q*G floats + the status word)"""
    L, B, Q, K1 = logits.shape
    check(lib().yb200_detr_match_cost(_f32(logits), _f32(boxes), _i32(labels), _f32(target_boxes), _i32(offsets), L, B, Q, K1, num_targets,
                                      c_float(w_class), c_float(w_bbox), c_float(w_giou), _f32(cost), stream_ptr()), "detr_match_cost")


def detr_set_loss(logits, boxes, match, labels, target_boxes, offsets, eos_coef, num_boxes, out):
    """yb200_detr_set_loss on the current stream: out [L, 5] = (loss_ce, loss_bbox, loss_giou, cardinality_error, class_error) per layer"""
    L, B, Q, K1 = logits.shape
    check(lib().yb200_detr_set_loss(_f32(logits), _f32(boxes), _i32(match), _i32(labels), _f32(target_boxes), _i32(offsets), L, B, Q, K1,
                                    c_float(eos_coef), c_float(num_boxes), _f32(out), stream_ptr()), "detr_set_loss")


def detr_set_loss_bwd(logits, boxes, match, labels, target_boxes, offsets, eos_coef, num_boxes, grad, dlogits, dboxes):
    """yb200_detr_set_loss_bwd on the current stream: grad [L, 3] (device) -> dlogits, dboxes shaped like logits, boxes"""
    L, B, Q, K1 = logits.shape
    check(lib().yb200_detr_set_loss_bwd(_f32(logits), _f32(boxes), _i32(match), _i32(labels), _f32(target_boxes), _i32(offsets), L, B, Q, K1,
                                        c_float(eos_coef), c_float(num_boxes), _f32(grad), _f32(dlogits), _f32(dboxes), stream_ptr()),
          "detr_set_loss_bwd")


def sparseinst_target_masks(masks, table, num_targets, input_shape, size, out, tsq):
    """yb200_sparseinst_target_masks on the current stream: packed uint8 masks + int64 [G, 3] table -> out [G, H, W], tsq [G]"""
    assert masks.dtype == torch.uint8 and table.dtype == torch.int64 and table.is_contiguous()
    check(lib().yb200_sparseinst_target_masks(ptr(masks), ptr(table), num_targets, int(input_shape[0]), int(input_shape[1]), int(size[0]), int(size[1]),
                                              _f32(out), _f32(tsq), stream_ptr()), "sparseinst_target_masks")


def sparseinst_match_cost(logits, masks, labels, offsets, tmasks, tsq, num_targets, alpha, beta, cost):
    """yb200_sparseinst_match_cost on the current stream: logits [B, N, K], masks [B, N, H, W] -> cost (N*G floats + the status word)"""
    B, N, K = logits.shape
    check(lib().yb200_sparseinst_match_cost(_f32(logits), _f32(masks), _i32(labels), _i32(offsets), _f32(tmasks), _f32(tsq), B, N, K,
                                            masks.shape[-2] * masks.shape[-1], num_targets, c_float(alpha), c_float(beta), _f32(cost), stream_ptr()),
          "sparseinst_match_cost")


def sparseinst_set_loss(logits, masks, scores, match, labels, offsets, tmasks, tsq, num_pairs, weights, num_instances, save, out):
    """yb200_sparseinst_set_loss on the current stream: out [4] = weighted (loss_ce, loss_objectness, loss_dice, loss_mask); save [B, N, 8]"""
    B, N, K = logits.shape
    w_ce, w_obj, w_dice, w_mask = (c_float(w) for w in weights)
    check(lib().yb200_sparseinst_set_loss(_f32(logits), _f32(masks), _f32(scores), _i32(match), _i32(labels), _i32(offsets), _f32(tmasks), _f32(tsq), B, N,
                                          K, masks.shape[-2] * masks.shape[-1], num_pairs, w_ce, w_obj, w_dice, w_mask, c_float(num_instances),
                                          _f32(save), _f32(out), stream_ptr()), "sparseinst_set_loss")


def sparseinst_set_loss_bwd(logits, masks, scores, match, labels, offsets, tmasks, tsq, save, num_pairs, weights, num_instances, grad, dlogits, dmasks,
                            dscores):
    """yb200_sparseinst_set_loss_bwd on the current stream: grad [4] (device) -> dlogits, dmasks, dscores shaped like logits, masks, scores"""
    B, N, K = logits.shape
    w_ce, w_obj, w_dice, w_mask = (c_float(w) for w in weights)
    check(lib().yb200_sparseinst_set_loss_bwd(_f32(logits), _f32(masks), _f32(scores), _i32(match), _i32(labels), _i32(offsets), _f32(tmasks), _f32(tsq),
                                              _f32(save), B, N, K, masks.shape[-2] * masks.shape[-1], num_pairs, w_ce, w_obj, w_dice, w_mask,
                                              c_float(num_instances), _f32(grad), _f32(dlogits), _f32(dmasks), _f32(dscores), stream_ptr()),
          "sparseinst_set_loss_bwd")
