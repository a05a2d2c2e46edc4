"""ctypes binding of csrc/libggufb200.so (the C ABI in include/ggufb200.h).

There is deliberately no fallback: if the shared library is missing or a call fails the
caller gets an exception.  Nothing in this package computes a dequant on the CPU.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libggufb200.so")
_lib = None

F16, BF16, F32 = 0, 1, 2
ALGO_AUTO, ALGO_GEMV, ALGO_FUSED_MMA, ALGO_DEQUANT_MMA, ALGO_FUSED_TMEM, ALGO_GEMV_FAST = 0, 1, 2, 3, 4, 5
ALGO_FUSED_SYNC = 6             # ggufb200_linear_fallback only
ALGO_MASK = 0xFF
# per-call switches OR-ed into `algo` (include/ggufb200.h)
FLAG_EXACT_W, FLAG_GENERIC, FLAG_TILE384, FLAG_NOSPLIT, FLAG_UNSTAGED, FLAG_TILE192 = 0x100, 0x200, 0x400, 0x800, 0x1000, 0x2000
FLAG_W_STABLE = 0x4000          # ggufb200_linear: no kernel still in flight writes the packed weight (prefetch under the previous kernel's tail)
DEQUANT_SRC_STABLE = 0x100      # same promise for ggufb200_dequant, OR-ed into math_dtype
OP_DEQUANT, OP_LINEAR, OP_ROWS, OP_LINEAR_MMA, OP_DEQUANT_FALLBACK, OP_QUANTIZE, OP_LINEAR_GRAD = 0, 1, 2, 3, 4, 5, 6
OP_LINEAR_FALLBACK, OP_ROWS_FALLBACK, OP_QUANTIZE_K = 7, 8, 9
LOWRANK_MAX_PATCHES, LOWRANK_MAX_RANK = 8, 1024   # ggufb200_dequant_lowrank: descriptors per call, rank of one factor pair
PATCH_LOWRANK, PATCH_KRON = 0, 1                   # ggufb200_weight_patch.kind
DORA_AXIS_OUT, DORA_AXIS_IN = 0, 1                 # ggufb200_dora_patch.axis


class GGUFB200Error(RuntimeError):
    pass


class KronPatch(ctypes.Structure):
    """ggufb200_kron_patch (include/ggufb200.h): one LoKr patch of ggufb200_dequant_kron."""
    _fields_ = [("A", ctypes.c_void_p), ("B", ctypes.c_void_p), ("a1", ctypes.c_int64), ("a2", ctypes.c_int64), ("b1", ctypes.c_int64),
                ("b2", ctypes.c_int64), ("band_dim", ctypes.c_int32), ("scale", ctypes.c_float), ("band_start", ctypes.c_int64),
                ("band_size", ctypes.c_int64)]


class LowrankPatch(ctypes.Structure):
    """ggufb200_lowrank_patch (include/ggufb200.h): one LoRA (a2 = None) or LoHa patch of ggufb200_dequant_lowrank."""
    _fields_ = [("a1", ctypes.c_void_p), ("b1", ctypes.c_void_p), ("a2", ctypes.c_void_p), ("b2", ctypes.c_void_p), ("r1", ctypes.c_int64),
                ("r2", ctypes.c_int64), ("scale", ctypes.c_float)]


class WeightPatch(ctypes.Structure):
    """ggufb200_weight_patch (include/ggufb200.h): one patch of ggufb200_dequant_patched, `lowrank` or `kron` as `kind` says."""
    _fields_ = [("kind", ctypes.c_int32), ("lowrank", LowrankPatch), ("kron", KronPatch)]


class DoraPatch(ctypes.Structure):
    """ggufb200_dora_patch (include/ggufb200.h): the DoRA step of one patch of ggufb200_dequant_patched_dora (factor None: plain)."""
    _fields_ = [("factor", ctypes.c_void_p), ("axis", ctypes.c_int32), ("group", ctypes.c_int32), ("strength", ctypes.c_float)]


def build(verbose: bool = False) -> str:
    """Compile the CUDA sources in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    out = subprocess.run(["bash", os.path.join(_HERE, "csrc", "build.sh")], capture_output=True, text=True)
    if verbose or out.returncode != 0:
        print(out.stdout, out.stderr)
    if out.returncode != 0:
        raise GGUFB200Error("nvcc build of libggufb200.so failed")
    return LIB_PATH


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise GGUFB200Error(
            f"{LIB_PATH} is missing: build it with comfyui-gguf_b200/csrc/build.sh (or __graft_entry__.build()). "
            "This package has no CPU / torch fallback for the dequant + Linear hot path."
        )
    L = ctypes.CDLL(LIB_PATH)
    c_int, c_i64, c_vp, c_sz = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_size_t
    L.ggufb200_version.restype = c_int
    L.ggufb200_strerror.restype = ctypes.c_char_p
    L.ggufb200_strerror.argtypes = [c_int]
    L.ggufb200_type_info.argtypes = [c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]
    L.ggufb200_supported.argtypes = [c_int, c_int]
    L.ggufb200_set_tuning.argtypes = [c_int, c_int]
    L.ggufb200_dequant.argtypes = [c_int, c_vp, c_i64, c_vp, c_int, c_int, c_vp]
    L.ggufb200_dequant_fallback.argtypes = [c_int, c_vp, c_i64, c_vp, c_int, c_int, c_vp]
    L.ggufb200_dequant_kron.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_int, c_int, ctypes.POINTER(KronPatch), c_int, c_vp]
    L.ggufb200_dequant_lowrank.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_int, c_int, ctypes.POINTER(LowrankPatch), c_int, c_vp]
    L.ggufb200_dequant_patched.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_int, c_int, ctypes.POINTER(WeightPatch), c_int, c_vp]
    L.ggufb200_dequant_patched_dora.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_int, c_int, ctypes.POINTER(WeightPatch),
                                                ctypes.POINTER(DoraPatch), c_int, c_vp]
    L.ggufb200_quantize.argtypes = [c_int, c_vp, c_int, c_i64, c_vp, c_int, c_vp]
    L.ggufb200_quantize_k.argtypes = [c_int, c_vp, c_int, c_i64, c_vp, c_int, c_vp]
    L.ggufb200_unpack_int.argtypes = [c_int, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp]
    L.ggufb200_dequant_rows.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_i64, c_vp, c_int, c_int, c_vp]
    L.ggufb200_dequant_rows_fallback.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_i64, c_vp, c_int, c_vp]
    L.ggufb200_linear_fallback_workspace.restype = c_sz
    L.ggufb200_linear_fallback_workspace.argtypes = [c_int, c_i64, c_i64, c_i64, c_int, c_int]
    L.ggufb200_linear_fallback_route.argtypes = [c_int, c_i64, c_i64, c_i64, c_int, c_int]
    L.ggufb200_linear_fallback.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_int, c_vp, c_int, c_vp, c_i64, c_vp, c_sz, c_int, c_vp]
    L.ggufb200_linear_plan.restype = c_int
    L.ggufb200_linear_plan.argtypes = [c_int, c_i64, c_i64, c_i64, c_sz, c_int] + [ctypes.POINTER(c_int)] * 4
    L.ggufb200_linear_workspace.restype = c_sz
    L.ggufb200_linear_workspace.argtypes = [c_int, c_i64, c_i64, c_i64, c_int, c_int]
    L.ggufb200_linear_workspace_ex.restype = c_sz
    L.ggufb200_linear_workspace_ex.argtypes = [c_int, c_i64, c_i64, c_i64, c_int, c_int, c_int]
    L.ggufb200_linear.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_int, c_int, c_vp, c_int, c_vp, c_i64,
                                  c_vp, c_sz, c_int, c_vp]
    L.ggufb200_linear_spans.argtypes = [c_int, c_vp, c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_int, c_int, c_vp, c_int, c_vp, c_i64,
                                        c_vp, c_sz, c_int, c_vp]
    L.ggufb200_repack_bytes.restype = c_sz
    L.ggufb200_repack_bytes.argtypes = [c_int, c_i64, c_i64]
    L.ggufb200_repack.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_vp]
    if hasattr(L, "ggufb200_linear_lora"):
        L.ggufb200_linear_lora.argtypes = [c_int, c_vp, c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_int, c_vp, c_int, c_vp, c_i64, c_vp, c_vp, c_i64,
                                           c_vp, c_sz, c_int, c_vp]
    L.ggufb200_linear_lora_ex.argtypes = [c_int, c_vp, c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_int, c_vp, c_int, c_vp, c_i64, c_vp, c_i64, c_int,
                                          c_vp, c_vp, c_i64, c_vp, c_sz, c_int, c_vp]
    L.ggufb200_gemm.argtypes = [c_vp, c_i64, c_i64, c_i64, c_vp, c_i64, c_i64, c_int, c_vp, c_int, c_vp, c_i64, c_vp]
    L.ggufb200_linear_lora_scaled.argtypes = [c_int, c_vp, c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_int, c_vp, c_int, c_vp, c_i64, c_vp, c_i64,
                                              c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_sz, c_int, c_vp]
    L.ggufb200_gemm_scaled.argtypes = [c_vp, c_i64, c_i64, c_i64, c_vp, c_i64, c_i64, c_int, c_vp, c_int, c_vp, c_vp, c_i64, c_vp]
    L.ggufb200_scale_columns.argtypes = [c_vp, c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_i64, c_vp]
    L.ggufb200_linear_grad_input_workspace.restype = c_sz
    L.ggufb200_linear_grad_input_workspace.argtypes = [c_int, c_i64, c_i64, c_int]
    L.ggufb200_linear_grad_input.argtypes = [c_int, c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_int, c_int, c_vp, c_i64, c_vp, c_sz, c_int, c_vp]
    _lib = L
    return L


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise GGUFB200Error(f"{what}: {lib().ggufb200_strerror(rc).decode()} (rc={rc})")


EXPORTS = (
    "ggufb200_version", "ggufb200_strerror", "ggufb200_type_info", "ggufb200_supported", "ggufb200_dequant",
    "ggufb200_unpack_int", "ggufb200_dequant_rows", "ggufb200_linear_workspace", "ggufb200_linear", "ggufb200_gemm",
    "ggufb200_set_tuning", "ggufb200_linear_plan", "ggufb200_linear_workspace_ex",
    "ggufb200_repack_bytes", "ggufb200_repack", "ggufb200_linear_spans", "ggufb200_linear_lora",
    "ggufb200_linear_lora_ex", "ggufb200_dequant_kron", "ggufb200_dequant_fallback", "ggufb200_linear_lora_scaled",
    "ggufb200_gemm_scaled", "ggufb200_scale_columns", "ggufb200_dequant_lowrank", "ggufb200_dequant_patched",
    "ggufb200_dequant_patched_dora", "ggufb200_quantize", "ggufb200_linear_grad_input_workspace", "ggufb200_linear_grad_input",
    "ggufb200_dequant_rows_fallback", "ggufb200_linear_fallback_workspace", "ggufb200_linear_fallback", "ggufb200_linear_fallback_route",
    "ggufb200_quantize_k",
)
