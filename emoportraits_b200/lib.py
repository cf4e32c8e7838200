"""ctypes binding of libemoport.so (the C-ABI declared in include/emoportraits_b200.h).

There is NO fallback: if the shared library is missing or fails to load, importing the ops raises.
"""
from __future__ import annotations

import ctypes as C
import os
import pathlib

_HERE = pathlib.Path(__file__).resolve().parent
# EMO_LIB=<path>: load another build of the same sources instead (tools/conv_bound_probe.py uses the instrumented
# libemoport_dbg.so that `python -m emoportraits_b200.csrc.build --debug` writes next to the product library)
LIB_PATH = pathlib.Path(os.environ["EMO_LIB"]).resolve() if os.environ.get("EMO_LIB") else _HERE / "csrc" / "libemoport.so"

ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3

c_void_p, c_int, c_ll, c_float, c_double = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_double


class GridSample3dDesc(C.Structure):
    _fields_ = [("in_", c_void_p), ("in_layout", c_int), ("N", c_int), ("C", c_int), ("Din", c_int), ("Hin", c_int),
                ("Win", c_int), ("grid", c_void_p), ("theta", c_void_p), ("Dout", c_int), ("Hout", c_int),
                ("Wout", c_int), ("out", c_void_p), ("out_hi", c_void_p), ("out_lo", c_void_p), ("os_n", c_ll),
                ("os_c", c_ll), ("os_d", c_ll), ("os_h", c_ll), ("os_w", c_ll), ("out_lo2", c_void_p),
                ("plane_fp16", c_int), ("plane_scale", c_float)]


class GridSample2dAffineDesc(C.Structure):
    _fields_ = [("in_", c_void_p), ("N", c_int), ("C", c_int), ("Hin", c_int), ("Win", c_int), ("theta", c_void_p),
                ("Hout", c_int), ("Wout", c_int), ("mean", c_void_p), ("std", c_void_p), ("out", c_void_p),
                ("C_pad", c_int), ("out_nchw", c_void_p)]


class ResizeBilinearDesc(C.Structure):
    _fields_ = [("in_", c_void_p), ("N", c_int), ("C", c_int), ("Hin", c_int), ("Win", c_int), ("Hout", c_int),
                ("Wout", c_int), ("mean", c_void_p), ("std", c_void_p), ("out", c_void_p), ("C_pad", c_int)]


class GnFinalizeDesc(C.Structure):
    _fields_ = [("stats", c_void_p), ("N", c_int), ("C", c_int), ("G", c_int), ("count", c_double), ("eps", c_float),
                ("gamma", c_void_p), ("beta", c_void_p), ("ada_w", c_void_p), ("ada_b", c_void_p), ("A", c_void_p),
                ("B", c_void_p)]


class ApplyDesc(C.Structure):
    _fields_ = [("x", c_void_p), ("N", c_int), ("C", c_int), ("D", c_int), ("H", c_int), ("W", c_int),
                ("A", c_void_p), ("B", c_void_p), ("ab_per_sample", c_int), ("res", c_void_p), ("A2", c_void_p),
                ("B2", c_void_p), ("act", c_int), ("up", c_int), ("out", c_void_p), ("out_hi", c_void_p),
                ("out_lo", c_void_p), ("out_lo2", c_void_p), ("stats", c_void_p), ("G", c_int), ("count", c_double),
                ("eps", c_float), ("gamma", c_void_p), ("beta", c_void_p), ("ada_w", c_void_p), ("ada_b", c_void_p),
                ("plane_fp16", c_int), ("plane_scale", c_float)]


class GnHeadDesc(C.Structure):
    _fields_ = [("x", c_void_p), ("N", c_int), ("C", c_int), ("S", c_ll), ("stats", c_void_p), ("G", c_int),
                ("count", c_double), ("eps", c_float), ("gamma", c_void_p), ("beta", c_void_p), ("w", c_void_p),
                ("bias", c_void_p), ("Cout", c_int), ("act_out", c_int), ("out", c_void_p)]


class ConvDesc(C.Structure):
    _fields_ = [("a_hi", c_void_p), ("a_lo", c_void_p), ("N", c_int), ("Din", c_int), ("Hin", c_int), ("Win", c_int),
                ("Cin", c_int), ("w_hi", c_void_p), ("w_lo", c_void_p), ("Cout", c_int), ("Cout_pad", c_int),
                ("kd", c_int), ("kh", c_int), ("kw", c_int), ("sd", c_int), ("sh", c_int), ("sw", c_int),
                ("pd", c_int), ("ph", c_int), ("pw", c_int), ("Dout", c_int), ("Hout", c_int), ("Wout", c_int),
                ("bias", c_void_p), ("residual", c_void_p), ("res_shift", c_int), ("act", c_int),
                ("post_add", c_void_p), ("out", c_void_p), ("out_nchw", c_int), ("stats", c_void_p), ("G", c_int),
                ("a_lo2", c_void_p), ("w_lo2", c_void_p), ("acc_chunk_mmas", c_int),
                ("splitk_ws", c_void_p), ("splitk_ws_elems", c_ll), ("upconv", c_int),
                ("operand_fp16", c_int), ("out_scale", c_float), ("post", c_void_p)]


class ConvPlanInfo(C.Structure):
    _fields_ = [("kernel", c_int), ("KC", c_int), ("NP", c_int), ("fp16", c_int), ("BN", c_int), ("ksplit", c_int),
                ("yreuse", c_int), ("sa", c_int), ("sb", c_int), ("stages", c_int), ("flush", c_int), ("tw", c_int),
                ("th", c_int), ("td", c_int), ("m_tiles", c_int), ("n_tiles", c_int), ("grid", c_int), ("finish", c_int)]


# emo_conv_plan_info.kernel and .finish (EMO_CONV_KERNEL_* / EMO_CONV_FINISH_*)
CONV_KERNELS = ("conv<64,2>", "conv<32,2>", "conv<64,3>", "conv<32,3>", "f16<64,2>", "f16<32,2>", "ps<64,2>")
CONV_FINISH = ("none", "finalize", "post", "finalize+apply", "apply")
# the one-plane fp16 kernels (operand mode ops.H1) follow as ids 7, 8, 9 (EMO_CONV_KERNEL_H1_*)
CONV_KERNELS_H1 = ("h1<64,1>", "h1<32,1>", "h1ps<64,1>")


def conv_kernel_name(kernel: int) -> str:
    """name of an emo_conv_plan_info.kernel id"""
    return (CONV_KERNELS + CONV_KERNELS_H1)[kernel]


class ConvDirectDesc(C.Structure):
    _fields_ = [("x", c_void_p), ("N", c_int), ("Hin", c_int), ("Win", c_int), ("Cin_pad", c_int), ("w", c_void_p),
                ("Cout", c_int), ("kh", c_int), ("kw", c_int), ("stride", c_int), ("pad", c_int), ("Hout", c_int),
                ("Wout", c_int), ("bias", c_void_p), ("out", c_void_p), ("stats", c_void_p), ("G", c_int)]


class LinearDesc(C.Structure):
    _fields_ = [("x", c_void_p), ("xs_m", c_ll), ("xs_k", c_ll), ("w", c_void_p), ("bias", c_void_p),
                ("add", c_void_p), ("scale", c_float), ("act", c_int), ("M", c_int), ("N", c_int), ("K", c_int),
                ("out", c_void_p), ("os_m", c_ll), ("os_n", c_ll)]


class ResampleDesc(C.Structure):
    _fields_ = [("x", c_void_p), ("N", c_int), ("D", c_int), ("H", c_int), ("W", c_int), ("C", c_int), ("fd", c_int),
                ("fh", c_int), ("fw", c_int), ("add", c_void_p), ("out", c_void_p), ("stats", c_void_p), ("G", c_int)]


class PoseDesc(C.Structure):
    _fields_ = [("srt", c_void_p), ("source_theta", c_void_p), ("N", c_int), ("mix", c_int), ("invert_warp", c_int),
                ("theta_out", c_void_p), ("theta_warp", c_void_p), ("align2d", c_void_p),
                ("theta_in", c_void_p), ("mix_old", c_int), ("smooth_init", c_int), ("smooth_state", c_void_p),
                ("smooth_momentum", C.c_float), ("smooth_one_minus", C.c_float)]


# every symbol include/emoportraits_b200.h declares, with its prototype
SYMBOLS = {
    "emo_last_error": (C.c_char_p, []),
    "emo_version": (c_int, []),
    "emo_device_info": (c_int, [C.POINTER(c_int), C.POINTER(c_int)]),
    "emo_grid_sample3d": (c_int, [C.POINTER(GridSample3dDesc), c_void_p]),
    "emo_grid_sample2d_affine": (c_int, [C.POINTER(GridSample2dAffineDesc), c_void_p]),
    "emo_resize_bilinear": (c_int, [C.POINTER(ResizeBilinearDesc), c_void_p]),
    "emo_gn_stats": (c_int, [c_void_p, c_int, c_ll, c_int, c_int, c_void_p, c_void_p]),
    "emo_gn_finalize": (c_int, [C.POINTER(GnFinalizeDesc), c_void_p]),
    "emo_apply": (c_int, [C.POINTER(ApplyDesc), c_void_p]),
    "emo_gn_head": (c_int, [C.POINTER(GnHeadDesc), c_void_p]),
    "emo_conv_igemm": (c_int, [C.POINTER(ConvDesc), c_void_p]),
    "emo_conv_plan": (c_int, [C.POINTER(ConvDesc), c_int, C.POINTER(ConvPlanInfo)]),
    "emo_conv_direct": (c_int, [C.POINTER(ConvDirectDesc), c_void_p]),
    "emo_stem_pack": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    "emo_linear": (c_int, [C.POINTER(LinearDesc), c_void_p]),
    "emo_upsample_trilinear": (c_int, [C.POINTER(ResampleDesc), c_void_p]),
    "emo_avgpool": (c_int, [C.POINTER(ResampleDesc), c_void_p]),
    "emo_maxpool2d_3x3s2": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "emo_global_avgpool": (c_int, [c_void_p, c_int, c_ll, c_int, c_void_p, c_void_p]),
    "emo_pose_theta": (c_int, [C.POINTER(PoseDesc), c_void_p]),
    "emo_split_bf16": (c_int, [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p]),
    "emo_split_f16": (c_int, [c_void_p, c_ll, c_float, c_void_p, c_void_p, c_void_p]),
    "emo_u8_to_image": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "emo_image_to_u8": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "emo_resize_bicubic": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "emo_s2_prepare": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_float, c_void_p]),
    "emo_s2_finish": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "emo_s2_prepare_composite": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                         c_void_p, c_float, c_void_p]),
    "emo_s2_masked_stem": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p]),
    "emo_s2_finish_masked": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "emo_composite": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    "emo_l2_flush": (c_int, [c_void_p, c_ll, c_void_p]),
    "emo_l2_flush_clean": (c_int, [c_void_p, c_ll, c_void_p]),
    "emo_parsing_prepare": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "emo_parsing_masks": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "emo_resize_area": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "emo_resample_u8": (c_int, [c_void_p, c_int, c_int, c_ll, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_ll, c_int,
                                c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "emo_mask_dilate": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p]),
}

# EMO_DRY_RUN=1: host-logic test mode for the GPU-less CI box — every C-ABI call is validated for presence in the
# library and then SKIPPED (outputs stay uninitialised).  It computes nothing and is not a fallback: results are garbage
# by construction; it only lets `pytest -m "not gpu"` walk the network-assembly code paths (shapes, layouts, launch order).
DRY_RUN = os.environ.get("EMO_DRY_RUN") == "1"

_lib = None
launch_count = 0  # number of kernel-launching C-ABI calls made through call() (bench.py's gpu_launches)


class EmoError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load the native library.  Fails loudly: there is no CPU or torch fallback for the hot path."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise EmoError(f"{LIB_PATH} is missing: build it with `python -m emoportraits_b200.csrc.build` "
                       "(or __graft_entry__.build()). The hot path has no fallback.")
    import torch  # noqa: F401  (makes libcudart.so.12 resident before our library is resolved)

    try:
        lib = C.CDLL(str(LIB_PATH), mode=C.RTLD_GLOBAL)
    except OSError:
        # CPU-only box without a resident cudart: preload the toolkit's runtime, then retry
        for cand in ("libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
            try:
                C.CDLL(cand, mode=C.RTLD_GLOBAL)
                break
            except OSError:
                continue
        lib = C.CDLL(str(LIB_PATH), mode=C.RTLD_GLOBAL)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def call(name: str, *args) -> None:
    global launch_count
    lib = load()
    if DRY_RUN:
        assert hasattr(lib, name)
        launch_count += 1
        return
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise EmoError(f"{name} failed ({rc}): {lib.emo_last_error().decode()}")
    launch_count += 1
