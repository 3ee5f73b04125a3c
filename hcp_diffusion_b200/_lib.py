"""ctypes binding of libhcpb200.so (the C-ABI CUDA library, include/hcp_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, an exception is raised.
PyTorch is used for device memory, streams and autograd plumbing only; every kernel on the hot path lives in the
library this module loads.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("HCP_LIB", os.path.join(_HERE, "lib", "libhcpb200.so"))     # HCP_LIB: an alternative build (A/B experiments)
CSRC = os.path.join(_HERE, "csrc")
SOURCES = ["gemm.cu", "host_util.cu", "attention.cu", "norms.cu", "misc.cu", "step.cu", "wgrad.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--shared", "-Xcompiler", "-fPIC"]

MAX_SEG = 3


class HcpError(RuntimeError):
    pass


def build(verbose: bool = False) -> str:
    """Compile the CUDA sources for sm_90a into lib/libhcpb200.so (nvcc cross-compiles without a GPU)."""
    os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    newest = max(os.path.getmtime(p) for p in srcs + [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "wgmma.cuh"),
                                                      os.path.join(CSRC, "host_util.h"), os.path.join(_HERE, "..", "include", "hcp_b200.h")])
    if os.path.exists(LIB_PATH) and os.path.getmtime(LIB_PATH) >= newest:
        return LIB_PATH
    cmd = ["nvcc", *NVCC_FLAGS, *os.environ.get("HCP_EXTRA_NVCC_FLAGS", "").split(), "-o", LIB_PATH, *srcs, "-lcudart"]
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    return LIB_PATH


class GemmArgs(C.Structure):
    _fields_ = [
        ("nseg", C.c_int32),
        ("a", C.c_void_p * MAX_SEG), ("b", C.c_void_p * MAX_SEG),
        ("lda", C.c_int64 * MAX_SEG), ("ldb", C.c_int64 * MAX_SEG),
        ("k", C.c_int64 * MAX_SEG), ("n_rows_b", C.c_int64 * MAX_SEG),
        ("M", C.c_int64), ("N", C.c_int64),
        ("bias", C.c_void_p), ("rowbias", C.c_void_p), ("rows_per_group", C.c_int64), ("rowbias_ld", C.c_int64),
        ("residual", C.c_void_p), ("ldr", C.c_int64),
        ("out", C.c_void_p), ("ldo", C.c_int64),
        ("flags", C.c_int32),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
        ("out2", C.c_void_p), ("ldo2", C.c_int64), ("n_main", C.c_int64),
    ]


class ConvArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("w", C.c_void_p),
        ("B", C.c_int64), ("Hin", C.c_int64), ("Win", C.c_int64), ("Cin", C.c_int64), ("Cout", C.c_int64),
        ("stride", C.c_int32), ("mode", C.c_int32),
        ("bias", C.c_void_p), ("rowbias", C.c_void_p), ("rowbias_ld", C.c_int64), ("residual", C.c_void_p), ("out", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
        ("lora_t", C.c_void_p), ("lora_b", C.c_void_p), ("lora_r", C.c_int64), ("lora_ld", C.c_int64), ("w_tiled", C.c_int32),
    ]


class AttnArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("ldq", C.c_int64), ("k", C.c_void_p), ("ldk", C.c_int64), ("v", C.c_void_p), ("ldv", C.c_int64),
        ("B", C.c_int64), ("H", C.c_int64), ("Lq", C.c_int64), ("Lkv", C.c_int64), ("d", C.c_int64),
        ("scale", C.c_float), ("kv_bias", C.c_void_p),
        ("o", C.c_void_p), ("ldo", C.c_int64), ("lse", C.c_void_p),
    ]


class AttnBwdArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("ldq", C.c_int64), ("k", C.c_void_p), ("ldk", C.c_int64), ("v", C.c_void_p), ("ldv", C.c_int64),
        ("o", C.c_void_p), ("ldo", C.c_int64), ("dout", C.c_void_p), ("lddo", C.c_int64),
        ("B", C.c_int64), ("H", C.c_int64), ("Lq", C.c_int64), ("Lkv", C.c_int64), ("d", C.c_int64),
        ("scale", C.c_float), ("kv_bias", C.c_void_p), ("lse", C.c_void_p),
        ("dq", C.c_void_p), ("lddq", C.c_int64), ("dk", C.c_void_p), ("lddk", C.c_int64), ("dv", C.c_void_p), ("lddv", C.c_int64),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
    ]


class GroupNormArgs(C.Structure):
    _fields_ = [
        ("x1", C.c_void_p), ("x2", C.c_void_p),
        ("B", C.c_int64), ("HW", C.c_int64), ("C1", C.c_int64), ("C2", C.c_int64), ("G", C.c_int64),
        ("gamma", C.c_void_p), ("beta", C.c_void_p), ("eps", C.c_float), ("silu", C.c_int32),
        ("stats", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
        ("y", C.c_void_p), ("dy", C.c_void_p), ("add1", C.c_void_p), ("add2", C.c_void_p), ("dx1", C.c_void_p), ("dx2", C.c_void_p),
    ]


class LoraJob(C.Structure):
    _fields_ = [
        ("w_down", C.c_void_p), ("w_up", C.c_void_p), ("alpha", C.c_float),
        ("rank", C.c_int32), ("in_dim", C.c_int32), ("out_dim", C.c_int32),
        ("c0", C.c_int32), ("o0", C.c_int32), ("out_tot", C.c_int32), ("ld_r", C.c_int32),
        ("A", C.c_void_p), ("AT", C.c_void_p), ("Bl", C.c_void_p), ("BlT", C.c_void_p),
    ]


class LoraMergeJob(C.Structure):
    _fields_ = [
        ("w_host", C.c_void_p), ("w_down", C.c_void_p * 4), ("w_up", C.c_void_p * 4), ("alpha", C.c_float * 4), ("rank", C.c_int32 * 4),
        ("nblocks", C.c_int32), ("in_dim", C.c_int32), ("out_dim", C.c_int32), ("o0", C.c_int32), ("out_tot", C.c_int32), ("tile0", C.c_int32),
        ("tiled", C.c_int32), ("pad_", C.c_int32), ("W", C.c_void_p), ("WT", C.c_void_p),
    ]


class LoraConvJob(C.Structure):
    _fields_ = [
        ("w_down", C.c_void_p), ("rank", C.c_int32), ("cin", C.c_int32), ("c0", C.c_int32), ("ld_r", C.c_int32), ("flip", C.c_int32),
        ("pad_", C.c_int32), ("wt", C.c_void_p), ("wd", C.c_void_p),
    ]


class RepackJob(C.Structure):
    _fields_ = [
        ("src", C.c_void_p), ("dst0", C.c_void_p), ("dst1", C.c_void_p),
        ("kind", C.c_int32), ("rows", C.c_int32), ("K", C.c_int32), ("o0", C.c_int32), ("n_tot", C.c_int32), ("flip", C.c_int32),
    ]


class LoraGradBlock(C.Structure):
    _fields_ = [
        ("n_lo", C.c_int64), ("n_hi", C.c_int64), ("c0", C.c_int32), ("rank", C.c_int32), ("scale", C.c_float),
        ("transpose_out", C.c_int32), ("dst", C.c_void_p), ("dst_ld", C.c_int64),
    ]


_lib = None
_lock = threading.Lock()

# every exported symbol of include/hcp_b200.h (checked by tests/test_abi.py)
EXPORTS = [
    "hcp_version", "hcp_last_error_string", "hcp_device_check", "hcp_launch_count", "hcp_gemm_bf16", "hcp_splitk_workspace_bytes", "hcp_conv3x3_bf16",
    "hcp_attn_fwd_bf16", "hcp_attn_bwd_workspace_bytes", "hcp_attn_bwd_bf16",
    "hcp_groupnorm_workspace_bytes", "hcp_groupnorm_fwd_bf16", "hcp_groupnorm_bwd_bf16",
    "hcp_layernorm_fwd_bf16", "hcp_layernorm_bwd_bf16", "hcp_geglu_fwd_bf16", "hcp_geglu_bwd_bf16",
    "hcp_upsample2x_fwd_bf16", "hcp_upsample2x_bwd_bf16", "hcp_add_bf16",
    "hcp_sinusoid_f32", "hcp_conv_in_f32", "hcp_conv_out_f32", "hcp_conv_out_dgrad_f32", "hcp_skinny_linear", "hcp_cast_f32_to_bf16",
    "hcp_lora_pack", "hcp_lora_merge", "hcp_lora_pack_conv", "hcp_lora_grad", "hcp_lora_grad_pair", "hcp_lora_grad_conv3x3", "hcp_add_noise", "hcp_mse_loss", "hcp_sumsq", "hcp_adamw_flat",
    "hcp_adamw_flat_dev", "hcp_snr_mse_loss", "hcp_ema_flat", "hcp_dropout_bf16", "hcp_counter_add_u64", "hcp_cfg_mix_f32",
    "hcp_wgrad_bf16", "hcp_wgrad_conv3x3_bf16", "hcp_colsum_bf16", "hcp_norm_affine_grad_bf16", "hcp_small_linear_bwd_f32", "hcp_silu_f32",
    "hcp_conv_in_wgrad_f32", "hcp_conv_out_wgrad_f32", "hcp_repack_weights",
]


def lib() -> C.CDLL:
    """Load libhcpb200.so (fails loudly when it has not been built -- there is no CPU / eager fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise HcpError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(hcp_diffusion_b200 has no fallback path)")
            l = C.CDLL(LIB_PATH)
            l.hcp_last_error_string.restype = C.c_char_p
            l.hcp_launch_count.restype = C.c_ulonglong
            l.hcp_launch_count.argtypes = []
            l.hcp_attn_bwd_workspace_bytes.restype = C.c_size_t
            l.hcp_attn_bwd_workspace_bytes.argtypes = [C.c_int64] * 5
            l.hcp_splitk_workspace_bytes.restype = C.c_size_t
            l.hcp_splitk_workspace_bytes.argtypes = [C.c_int64] * 3
            l.hcp_groupnorm_workspace_bytes.restype = C.c_size_t
            l.hcp_groupnorm_workspace_bytes.argtypes = [C.c_int64] * 3
            vp, i64, f32, i32 = C.c_void_p, C.c_int64, C.c_float, C.c_int
            l.hcp_gemm_bf16.argtypes = [C.POINTER(GemmArgs), vp]
            l.hcp_conv3x3_bf16.argtypes = [C.POINTER(ConvArgs), vp]
            l.hcp_attn_fwd_bf16.argtypes = [C.POINTER(AttnArgs), vp]
            l.hcp_attn_bwd_bf16.argtypes = [C.POINTER(AttnBwdArgs), vp]
            l.hcp_groupnorm_fwd_bf16.argtypes = [C.POINTER(GroupNormArgs), vp]
            l.hcp_groupnorm_bwd_bf16.argtypes = [C.POINTER(GroupNormArgs), vp]
            l.hcp_layernorm_fwd_bf16.argtypes = [vp, vp, vp, f32, i64, i64, vp, vp, vp]
            l.hcp_layernorm_bwd_bf16.argtypes = [vp, vp, vp, vp, vp, i64, i64, vp, vp]
            l.hcp_geglu_fwd_bf16.argtypes = [vp, i64, i64, vp, vp]
            l.hcp_geglu_bwd_bf16.argtypes = [vp, vp, i64, i64, vp, vp]
            l.hcp_upsample2x_fwd_bf16.argtypes = [vp, i64, i64, i64, i64, vp, vp]
            l.hcp_upsample2x_bwd_bf16.argtypes = [vp, i64, i64, i64, i64, vp, vp]
            l.hcp_add_bf16.argtypes = [vp, vp, i64, vp, vp]
            l.hcp_conv_in_f32.argtypes = [vp, vp, vp, i64, i64, i64, i64, i64, vp, vp]
            l.hcp_conv_out_f32.argtypes = [vp, vp, vp, i64, i64, i64, i64, i64, vp, vp]
            l.hcp_conv_out_dgrad_f32.argtypes = [vp, vp, i64, i64, i64, i64, i64, vp, vp]
            l.hcp_skinny_linear.argtypes = [vp, vp, vp, i64, i64, i64, i32, i32, vp, vp]
            l.hcp_cast_f32_to_bf16.argtypes = [vp, i64, vp, vp]
            l.hcp_sinusoid_f32.argtypes = [vp, i64, i64, i64, vp, i64, vp]
            l.hcp_lora_pack.argtypes = [vp, i64, vp]
            l.hcp_lora_pack_conv.argtypes = [vp, i64, vp]
            l.hcp_lora_merge.argtypes = [vp, i64, i64, vp, C.c_int32, vp]
            l.hcp_lora_grad_conv3x3.argtypes = [vp, i64, vp, i64, i64, i64, i64, C.c_int32, C.POINTER(LoraGradBlock), C.c_int32, vp]
            l.hcp_lora_grad.argtypes = [vp, i64, vp, i64, i64, i64, i64, C.POINTER(LoraGradBlock), C.c_int32, vp]
            l.hcp_lora_grad_pair.argtypes = [vp, vp, i64, i64, C.POINTER(LoraGradBlock), vp, vp, i64, i64, C.POINTER(LoraGradBlock),
                                             C.c_int32, i64, i64, vp]
            l.hcp_add_noise.argtypes = [vp, vp, vp, vp, i64, i64, vp, vp]
            l.hcp_mse_loss.argtypes = [vp, vp, i64, f32, vp, vp, vp]
            l.hcp_sumsq.argtypes = [vp, i64, vp, vp]
            l.hcp_adamw_flat.argtypes = [vp, vp, vp, vp, i64, vp, f32, f32, f32, f32, f32, vp, f32, vp, vp]
            l.hcp_adamw_flat_dev.argtypes = [vp, vp, vp, vp, i64, vp, f32, vp, f32, vp, vp]
            l.hcp_snr_mse_loss.argtypes = [vp, vp, vp, vp, f32, C.c_int32, i64, i64, f32, vp, vp, vp]
            l.hcp_ema_flat.argtypes = [vp, vp, i64, vp, f32, f32, f32, vp]
            l.hcp_dropout_bf16.argtypes = [vp, i64, vp, i64, vp, i64, i64, i64, i64, f32, vp, C.c_uint32, vp, i64, vp]
            l.hcp_counter_add_u64.argtypes = [vp, C.c_uint64, vp]
            l.hcp_wgrad_bf16.argtypes = [vp, i64, i64, vp, i64, i64, i64, f32, vp, i64, i64, vp]
            l.hcp_wgrad_conv3x3_bf16.argtypes = [vp, i64, vp, i64, i64, i64, i64, C.c_int32, f32, vp, vp]
            l.hcp_colsum_bf16.argtypes = [vp, i64, i64, i64, i64, f32, vp, i64, vp]
            l.hcp_norm_affine_grad_bf16.argtypes = [vp, vp, i64, i64, vp, vp, vp, vp, i64, i64, i64, C.c_int32, vp, vp, vp]
            l.hcp_small_linear_bwd_f32.argtypes = [vp, i64, vp, vp, i64, i64, i64, vp, vp, vp, vp]
            l.hcp_silu_f32.argtypes = [vp, vp, i64, vp, vp]
            l.hcp_conv_in_wgrad_f32.argtypes = [vp, vp, i64, i64, i64, i64, i64, vp, vp, vp]
            l.hcp_conv_out_wgrad_f32.argtypes = [vp, vp, i64, i64, i64, i64, i64, vp, vp, vp]
            l.hcp_repack_weights.argtypes = [vp, i64, vp]
            l.hcp_cfg_mix_f32.argtypes = [vp, vp, vp, i64, i64, f32, f32, C.c_int32, C.c_int32, vp, vp]
            _lib = l
    return _lib


def __getattr__(name: str):
    # `_lib.launch_count`: kernels launched by the library so far, counted inside libhcpb200 itself (bench.py `gpu_launches`)
    if name == "launch_count":
        return int(lib().hcp_launch_count())
    raise AttributeError(name)


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise HcpError(f"{what} failed (rc={rc}): {lib().hcp_last_error_string().decode()}")


def call(name: str, *args) -> None:
    rc = getattr(lib(), name)(*args)
    if rc != 0:
        raise HcpError(f"{name} failed (rc={rc}): {lib().hcp_last_error_string().decode()}")


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()
