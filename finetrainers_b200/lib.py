"""ctypes binding of libb2d.so (the C ABI declared in include/b2d.h).

The product path has NO fallback: if the library is missing or the device is not sm_90 every op raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2d.so")
_lib = None
_lock = threading.Lock()


class B2DError(RuntimeError):
    pass


class GemmDesc(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("lda", C.c_int64),
        ("B", C.c_void_p), ("ldb", C.c_int64),
        ("A2", C.c_void_p), ("lda2", C.c_int64),
        ("B2", C.c_void_p), ("ldb2", C.c_int64),
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("K2", C.c_int32),
        ("a_mn_major", C.c_int32), ("b_mn_major", C.c_int32),
        ("a2_group_n", C.c_int32),
        ("splits", C.c_int32), ("batch", C.c_int32),
        ("a_boff_row", C.c_int64), ("a_boff_col", C.c_int64), ("b_boff_row", C.c_int64), ("b_boff_col", C.c_int64),
        ("c_boff", C.c_int64),
        ("epi", C.c_int32),
        ("alpha", C.c_float),
        ("out", C.c_void_p), ("ldc", C.c_int64),
        ("out2", C.c_void_p), ("ldc2", C.c_int64),
        ("bias", C.c_void_p),
        ("res", C.c_void_p), ("ldres", C.c_int64),
        ("aux", C.c_void_p), ("ldaux", C.c_int64),
        ("gate_table", C.c_void_p), ("gate_temb", C.c_void_p),
        ("gate2_table", C.c_void_p), ("gate2_temb", C.c_void_p),
        ("temb_stride", C.c_int64),
        ("rows_per_sample", C.c_int32),
        ("block_n", C.c_int32),
        ("max_ctas", C.c_int32),
        ("a2_boff_row", C.c_int64), ("b2_boff_row", C.c_int64), ("bias_boff", C.c_int64),
        ("cta_pair", C.c_int32),
    ]


def build(verbose: bool = False) -> str:
    """Compile libb2d.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).  Serialised across processes
    with a file lock: N torchrun ranks on a source-only checkout must not link the same output concurrently."""
    import fcntl
    cmd = ["make", "-C", os.path.join(_HERE, "csrc"), "-j", str(min(8, os.cpu_count() or 1))]
    with open(os.path.join(_HERE, "csrc", ".build.lock"), "w") as lk:
        fcntl.flock(lk, fcntl.LOCK_EX)
        try:
            r = subprocess.run(cmd, capture_output=True, text=True)
        finally:
            fcntl.flock(lk, fcntl.LOCK_UN)
    if r.returncode != 0:
        raise B2DError("building libb2d.so failed:\n" + r.stdout[-4000:] + r.stderr[-4000:])
    if verbose:
        print(r.stdout[-2000:])
    return LIB_PATH


def load():
    """Load libb2d.so or raise — never falls back to another implementation."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            try:  # source-only checkout: compile once with nvcc (no other implementation exists to fall back to)
                build()
            except Exception as e:  # noqa: BLE001
                raise B2DError(f"{LIB_PATH} not found and building it failed ({e}); there is no CPU or PyTorch "
                               "fallback for the b200 hot path") from e
        lib = C.CDLL(LIB_PATH)
        lib.b2d_last_error.restype = C.c_char_p
        lib.b2d_version.restype = C.c_int
        lib.b2d_launch_count.restype = C.c_int64
        _lib = lib
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().b2d_last_error().decode()
        raise B2DError(f"libb2d {what} failed (code {rc}): {msg}")


EXPORTS = [
    "b2d_version", "b2d_last_error", "b2d_device_check", "b2d_launch_count", "b2d_gemm",
    "b2d_norm_modulate_fwd", "b2d_norm_modulate_bwd", "b2d_colscale", "b2d_rope_table",
    "b2d_qkv_norm_rope_hd_fwd", "b2d_qkv_norm_rope_hd_bwd",
    "b2d_attn_fwd_hd", "b2d_attn_bwd_hd",
    "b2d_prep_noise_pack", "b2d_prep_posterior_noise_pack", "b2d_loss_mse", "b2d_timestep_sinusoid", "b2d_cast_f32_bf16",
    "b2d_sumsq", "b2d_adamw_clip", "b2d_upcast_fp8_bf16", "b2d_splitk_reduce_bf16", "b2d_cfg_euler_step",
    "b2d_cfg_euler_step_cond", "b2d_rope_table_wan", "b2d_wan_prep", "b2d_patch_permute", "b2d_layer_norm_affine_fwd",
    "b2d_layer_norm_affine_bwd", "b2d_qkv_norm_rope_ph_fwd", "b2d_qkv_norm_rope_ph_bwd", "b2d_attn_dual_fwd_hd",
    "b2d_attn_dual_bwd_hd", "b2d_wan_i2v_prep", "b2d_gelu_erf",
]
