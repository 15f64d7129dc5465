"""ctypes binding of libwaternet_b200.so (the C ABI in include/waternet_b200.h).

There is no CPU implementation behind this module: if the shared library is
missing or was not built, importing callers get a RuntimeError that says how to
build it.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int16, c_int64, c_size_t, c_uint8, c_uint16, c_uint64, c_void_p

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, "libwaternet_b200.so")

MODE_FP32_SIMT = 0
MODE_BF16X3 = 1
MODE_BF16_FP8 = 2
MODE_DEFAULT = -1
MODE_BF16 = 3          # WN_MODE_BF16: single-pass bf16 training (wn_set_train_mode)
NUM_PARAMS = 34
VGG_NUM_PARAMS = 32     # WN_VGG_NUM_PARAMS: weight and bias of VGG19's 16 convolutions
NUM_TIMING_SLOTS = 23
DEBUG_BACKWARD_BUFFERS = 25  # WN_DEBUG_BACKWARD_BUFFERS
ABI_VERSION = 11
PEER_HANDLE_BYTES = 64  # WN_PEER_HANDLE_BYTES
MAX_PEERS = 15          # WN_MAX_PEERS


class RaggedImage(ctypes.Structure):
    """wn_ragged_image: one image of a ragged batch (device pointers)."""
    _fields_ = [("rgb", c_void_p), ("out_u8", c_void_p), ("out_f32", c_void_p), ("height", c_int), ("width", c_int)]


class RaggedTensors(ctypes.Structure):
    """wn_ragged_tensors: the four fp32 inputs of one image of a ragged batch, their element strides (sN, sC, sH, sW
    each), its fp32 contiguous (1,3,H,W) output and its size (device pointers)."""
    _fields_ = [("x", c_void_p), ("wb", c_void_p), ("he", c_void_p), ("gc", c_void_p), ("in_strides", c_int64 * 16),
                ("out", c_void_p), ("height", c_int), ("width", c_int)]


RAGGED_TENSORS_BYTES = 176  # sizeof(wn_ragged_tensors), asserted in csrc/api.cu


class QualityImage(ctypes.Structure):
    """wn_quality_image: one (out, ref) pair of a wn_quality call, fp32 contiguous (3,H,W) device pointers, its size
    and its group (the images sharing SSIM's data range)."""
    _fields_ = [("out", c_void_p), ("ref", c_void_p), ("height", c_int), ("width", c_int), ("group", c_int)]


QUALITY_STATS = 7  # WN_QUALITY_STATS: float64 statistics per image of wn_quality


class SSIMGradImage(ctypes.Structure):
    """wn_ssim_grad_image: one (out, ref) pair of a wn_ssim_grad call and the gradient it receives, fp32 contiguous
    (3,H,W) device pointers, its size, its group and the weight of its SSIM in the differentiated sum."""
    _fields_ = [("out", c_void_p), ("ref", c_void_p), ("grad", c_void_p), ("height", c_int), ("width", c_int),
                ("group", c_int), ("scale", ctypes.c_double)]


# name -> (restype, argtypes); mirrors include/waternet_b200.h one to one
_SIGNATURES = {
    "wn_abi_version": (c_int, []),
    "wn_last_error": (c_char_p, []),
    "wn_create": (c_int, [c_int, POINTER(c_void_p)]),
    "wn_destroy": (None, [c_void_p]),
    "wn_build_tables_host": (c_int, [POINTER(c_uint16), POINTER(c_uint16), POINTER(c_int16), POINTER(c_int16),
                                     POINTER(c_uint8), POINTER(c_uint8), POINTER(c_float)]),
    "wn_pack_weights": (c_int, [c_void_p, POINTER(c_void_p), c_void_p]),
    "wn_forward_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "wn_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_void_p,
                           c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "wn_preprocess_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "wn_preprocess_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "wn_white_balance_gray_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "wn_white_balance_gray_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "wn_resize_u8": (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_int), POINTER(c_int), c_int, c_void_p, c_int, c_int,
                             c_int, c_void_p]),
    "wn_postprocess_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "wn_enhance_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "wn_enhance_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                              c_void_p, c_size_t, c_void_p]),
    "wn_enhance_u8_peers": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_void_p), c_int, c_int, c_int, c_int,
                                    c_int, c_void_p, c_size_t, c_void_p]),
    "wn_enhance_tiled_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong, c_int]),
    "wn_enhance_u8_tiled": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                    ctypes.c_longlong, c_int, c_void_p, c_size_t, c_void_p]),
    "wn_enhance_ragged_workspace_bytes": (c_size_t, [POINTER(c_int), POINTER(c_int), c_int, c_int, c_int,
                                                     ctypes.c_longlong, c_int]),
    "wn_enhance_u8_ragged": (c_int, [c_void_p, POINTER(RaggedImage), c_int, c_int, c_int, ctypes.c_longlong, c_int,
                                     c_void_p, c_size_t, c_void_p]),
    "wn_launch_count": (c_uint64, [c_void_p]),
    "wn_submodule_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "wn_confidence_maps": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_void_p,
                                   c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "wn_refine": (c_int, [c_void_p, c_int, c_void_p, c_void_p, POINTER(c_int64), c_void_p, c_int, c_int, c_int,
                          c_int, c_void_p, c_size_t, c_void_p]),
    "wn_forward_tiled_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong, c_int]),
    "wn_forward_tiled": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_void_p,
                                 c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong, c_int, c_void_p, c_size_t,
                                 c_void_p]),
    "wn_submodule_tiled_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong, c_int]),
    "wn_confidence_maps_tiled": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64),
                                         c_void_p, c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong, c_int,
                                         c_void_p, c_size_t, c_void_p]),
    "wn_refine_tiled": (c_int, [c_void_p, c_int, c_void_p, c_void_p, POINTER(c_int64), c_void_p, c_int, c_int, c_int,
                                c_int, c_int, ctypes.c_longlong, c_int, c_void_p, c_size_t, c_void_p]),
    "wn_forward_chunk_images": (c_int, [c_void_p, c_int, c_int, c_int]),
    "wn_set_chunk_pixels": (c_int, [c_void_p, ctypes.c_longlong]),
    "wn_set_train_mode": (c_int, [c_void_p, c_int]),
    "wn_f8_overflowed": (c_int, [c_void_p]),
    "wn_peer_alloc": (c_int, [c_size_t, POINTER(c_void_p), c_void_p]),
    "wn_peer_open": (c_int, [c_void_p, POINTER(c_void_p)]),
    "wn_peer_close": (c_int, [c_void_p]),
    "wn_peer_free": (c_int, [c_void_p]),
    "wn_memcpy_async": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "wn_stream_write_value32": (c_int, [c_void_p, c_void_p, ctypes.c_uint32]),
    "wn_stream_wait_value32": (c_int, [c_void_p, c_void_p, ctypes.c_uint32]),
    "wn_train_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "wn_forward_train": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_void_p,
                                 c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "wn_backward": (c_int, [c_void_p, c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_int, c_int, c_int, c_void_p,
                            c_size_t, c_void_p]),
    "wn_submodule_train_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "wn_confidence_maps_train": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_void_p,
                                         c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "wn_confidence_maps_backward": (c_int, [c_void_p, c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_int, c_int,
                                            c_int, c_void_p, c_size_t, c_void_p]),
    "wn_refine_train": (c_int, [c_void_p, c_int, c_void_p, c_void_p, POINTER(c_int64), c_void_p, c_int, c_int, c_int,
                                c_void_p, c_size_t, c_void_p]),
    "wn_refine_backward": (c_int, [c_void_p, c_int, c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_int, c_int,
                                   c_int, c_void_p, c_size_t, c_void_p]),
    "wn_backward_tiled_workspace_bytes":(c_size_t, [c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong]),
    "wn_backward_tiled": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_void_p,
                                  POINTER(c_void_p), POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int,
                                  ctypes.c_longlong, c_void_p, c_size_t, c_void_p]),
    "wn_submodule_backward_tiled_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong,
                                                               c_int]),
    "wn_confidence_maps_backward_tiled": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64),
                                                  c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_int, c_int, c_int,
                                                  c_int, c_int, ctypes.c_longlong, c_void_p, c_size_t, c_void_p]),
    "wn_refine_backward_tiled": (c_int, [c_void_p, c_int, c_void_p, c_void_p, POINTER(c_int64), c_void_p,
                                         POINTER(c_void_p), POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int,
                                         ctypes.c_longlong, c_void_p, c_size_t, c_void_p]),
    "wn_forward_ragged_workspace_bytes": (c_size_t, [POINTER(c_int), POINTER(c_int), c_int, c_int, c_int,
                                                     ctypes.c_longlong, c_int]),
    "wn_forward_ragged": (c_int, [c_void_p, POINTER(RaggedTensors), c_int, c_int, c_int, ctypes.c_longlong, c_int,
                                  c_void_p, c_size_t, c_void_p]),
    "wn_train_ragged_workspace_bytes": (c_size_t, [POINTER(c_int), POINTER(c_int), c_int]),
    "wn_forward_train_ragged": (c_int, [c_void_p, POINTER(RaggedTensors), c_int, c_void_p, c_size_t, c_void_p]),
    "wn_backward_ragged": (c_int, [c_void_p, POINTER(c_int), POINTER(c_int), POINTER(c_void_p), POINTER(c_void_p),
                                   POINTER(c_void_p), c_int, c_void_p, c_size_t, c_void_p]),
    "wn_backward_ragged_tiled_workspace_bytes": (c_size_t, [POINTER(c_int), POINTER(c_int), c_int, c_int, c_int,
                                                            ctypes.c_longlong]),
    "wn_backward_ragged_tiled": (c_int, [c_void_p, POINTER(RaggedTensors), POINTER(c_void_p), POINTER(c_void_p),
                                         POINTER(c_void_p), c_int, c_int, c_int, ctypes.c_longlong, c_void_p, c_size_t,
                                         c_void_p]),
    "wn_debug_forward_layer": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int64), c_int,
                                       c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "wn_debug_backward_layer": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, POINTER(c_void_p), c_int, c_int,
                                        c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "wn_vgg_pack_weights": (c_int, [c_void_p, POINTER(c_void_p), c_void_p]),
    "wn_perceptual_loss_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, ctypes.c_longlong]),
    "wn_perceptual_loss": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_void_p, POINTER(c_int64), c_int, c_int,
                                   c_int, c_int, c_int, ctypes.c_longlong, c_void_p, c_void_p, c_void_p, c_size_t,
                                   c_void_p]),
    "wn_debug_vgg_layer": (c_int, [c_void_p, c_void_p, POINTER(c_int64), c_void_p, POINTER(c_int64), c_int, c_int,
                                   c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "wn_enable_timing": (c_int, [c_void_p, c_int]),
    "wn_read_timings": (c_int, [c_void_p, POINTER(c_float), POINTER(c_int)]),
}

# ... and include/waternet_b200_metrics.h, the SSIM / PSNR statistics (csrc/metrics.cu)
_METRICS_SIGNATURES = {
    "wn_quality_workspace_bytes": (c_size_t, [POINTER(c_int), POINTER(c_int), c_int]),
    "wn_quality": (c_int, [c_void_p, POINTER(QualityImage), c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
}

# ... and include/waternet_b200_ssim.h, SSIM's gradient (csrc/metrics.cu)
_SSIM_SIGNATURES = {
    "wn_ssim_grad_workspace_bytes": (c_size_t, [POINTER(c_int), POINTER(c_int), c_int]),
    "wn_ssim_grad": (c_int, [c_void_p, POINTER(SSIMGradImage), c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)                # the entry points of include/waternet_b200.h
METRICS_SYMBOLS = tuple(_METRICS_SIGNATURES)         # ... of include/waternet_b200_metrics.h
SSIM_SYMBOLS = tuple(_SSIM_SIGNATURES)               # ... of include/waternet_b200_ssim.h

_lib = None


class WaterNetLibraryError(RuntimeError):
    pass


def load() -> ctypes.CDLL:
    """dlopen the library and attach the prototypes.  Fails loudly when absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("WATERNET_B200_LIB", LIB_PATH)  # experiment variants (see build.py); default in-tree
    if not os.path.exists(path):
        raise WaterNetLibraryError(
            f"{path} is missing: the CUDA library has not been built. "
            "Run `python -m waternet_b200.build` (needs nvcc 12.9); there is no CPU fallback."
        )
    lib = ctypes.CDLL(path)
    for name, (res, args) in {**_SIGNATURES, **_METRICS_SIGNATURES, **_SSIM_SIGNATURES}.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.wn_abi_version() != ABI_VERSION:
        raise WaterNetLibraryError(
            f"libwaternet_b200.so ABI {lib.wn_abi_version()} != binding ABI {ABI_VERSION}; rebuild it")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().wn_last_error()
        raise WaterNetLibraryError(f"{what} failed (code {rc}): {msg.decode() if msg else ''}")
