"""ctypes binding of include/lanpaint_b200.h.

There is deliberately no fallback: if the library is missing or a call fails
the caller gets an exception.  (The product never routes through `oracle/`.)
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_LIB_PATH = os.environ.get("LANPAINT_B200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "_lib",
                                                               "liblanpaint_b200.so")

ABI_VERSION = 5
TABLE_STRIDE = 32

RNG_TAPE, RNG_PHILOX, RNG_TORCH = 0, 1, 2
DTYPE_F32, DTYPE_BF16, DTYPE_F16 = 0, 1, 2
HEADS_DEAD = 0x100  # LP_HEADS_DEAD: or-ed into Heads.dtype when nothing reads the heads after the launch
T_INVS = 2  # LP_T_INVS
SUBSTEP_FIRST, SUBSTEP_FUSE_NEXT, SUBSTEP_STORE_C, SUBSTEP_MERGE_NOISE = 1, 2, 4, 8

# every symbol include/lanpaint_b200.h declares (checked by tests/test_abi.py)
SYMBOLS = (
    "lp_abi_version", "lp_status_string", "lp_last_cuda_error", "lp_set_option", "lp_selftest_index_math", "lp_selftest_box_muller", "lp_selftest_normal_fast", "lp_build_coef_table", "lp_build_coef_table_dt",
    "lp_torch_randn_geometry", "lp_pack_mask_f32", "lp_prologue_f32", "lp_substep", "lp_substep_f32", "lp_substep_cfg_f32", "lp_advance_f32",
    "lp_boundary", "lp_boundary_ancestral", "lp_boundary_multistep", "lp_boundary_midpoint", "lp_boundary_deis", "lp_boundary_gradient_estimation",
    "lp_boundary_heun", "lp_boundary_known_rows", "lp_boundary_ancestral_rows", "lp_boundary_midpoint_rows",
    "lp_boundary_deis_rows", "lp_boundary_gradient_estimation_rows", "lp_synth_denoiser", "lp_known_words", "lp_pack_known", "lp_substep_known", "lp_boundary_known",
    "lp_epilogue_f32", "lp_epilogue_euler_f32", "lp_step_boundary_f32", "lp_epilogue_cfg_f32", "lp_stop_stats_f32", "lp_fill_normal_f32", "lp_synth_denoiser_f32", "lp_l2_persist_capacity", "lp_l2_persist_set", "lp_l2_persist_clear", "lp_l2_flush", "lp_torch_cpu_randn_f32",
)


class NativeError(RuntimeError):
    pass


class Hyper(C.Structure):
    _fields_ = [("step_size", C.c_double), ("lam", C.c_double), ("beta", C.c_double),
                ("min_step_frac", C.c_double), ("flow", C.c_int32), ("reserved", C.c_int32)]


class Heads(C.Structure):
    """lp_heads: the model's prediction(s) of one call (x0 / x0_BIG, or raw cond / uncond with combine=1)."""
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("dtype", C.c_int32), ("combine", C.c_int32),
                ("cfg", C.c_float), ("cfg_big", C.c_float)]


class Dims(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("per_row", C.c_int64), ("spatial", C.c_int64),
                ("mask_row_stride", C.c_int64), ("mask_channel_stride", C.c_int64), ("row_split", C.c_int64)]


class Rng(C.Structure):
    _fields_ = [("mode", C.c_int32), ("reserved", C.c_int32), ("tape0", C.c_void_p), ("tape1", C.c_void_p),
                ("seed", C.c_uint64), ("draw0", C.c_uint64), ("draw1", C.c_uint64), ("state", C.c_void_p)]


class Known(C.Structure):
    """lp_known: the known-operand layout (known bits + packed y / noise) of one job's y, noise and mask."""
    _fields_ = [("words", C.c_void_p), ("y", C.c_void_p), ("noise", C.c_void_p)]


class Ancestral(C.Structure):
    """lp_ancestral: one outer step of sample_euler_ancestral (sigma_from, sigma_down - sigma_from, s_noise, sigma_up)."""
    _fields_ = [("sigma", C.c_float), ("down", C.c_float), ("s_noise", C.c_float), ("sigma_up", C.c_float)]


class Multistep(C.Structure):
    """lp_multistep: one outer step of sample_dpmpp_2m (ratio, expm1(-h), c_cur, c_old)."""
    _fields_ = [("ratio", C.c_float), ("em1", C.c_float), ("c_cur", C.c_float), ("c_old", C.c_float)]


class Midpoint(C.Structure):
    """lp_midpoint: one update of sample_dpm_2, x_out = x_base + ((x_in - out) / sigma) * dt."""
    _fields_ = [("sigma", C.c_float), ("dt", C.c_float)]


class Deis(C.Structure):
    """lp_deis: one step of sample_deis, x = x + c_cur*d [+ c_prev1*d_prev1 [+ c_prev2*d_prev2]], d = (x - out)/sigma."""
    _fields_ = [("sigma", C.c_float), ("c_cur", C.c_float), ("c_prev1", C.c_float), ("c_prev2", C.c_float)]


class GradientEstimation(C.Structure):
    """lp_gradient_estimation: one step of sample_gradient_estimation, x = x + d*dt [+ (gm1*(d - d_prev))*dt], or
    x = out when final; d = (x - out)/sigma."""
    _fields_ = [("sigma", C.c_float), ("dt", C.c_float), ("gm1", C.c_float), ("final", C.c_int)]


class Heun(C.Structure):
    """lp_heun: the corrector of sample_heun, x = x + ((((x - out_prev)/sigma) + ((x2 - out)/sigma_next)) / 2) * dt."""
    _fields_ = [("sigma", C.c_float), ("sigma_next", C.c_float), ("dt", C.c_float)]


_lib: Optional[C.CDLL] = None


def lib_path() -> str:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load (once) and type the library.  Raises NativeError when it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise NativeError(
            f"{_LIB_PATH} is missing: build it with `python -m lanpaint_b200.build` "
            "(nvcc, sm_90a).  lanpaint_b200 has no CPU or eager-PyTorch fallback.")
    lib = C.CDLL(_LIB_PATH)
    p, i64, u64, i32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_int
    lib.lp_abi_version.restype = i32
    lib.lp_abi_version.argtypes = []
    lib.lp_status_string.restype = C.c_char_p
    lib.lp_status_string.argtypes = [i32]
    lib.lp_last_cuda_error.restype = i32
    lib.lp_last_cuda_error.argtypes = []
    lib.lp_set_option.restype = i32
    lib.lp_set_option.argtypes = [C.c_char_p, i32]
    lib.lp_selftest_index_math.restype = i64
    lib.lp_selftest_index_math.argtypes = [i64]
    lib.lp_selftest_box_muller.restype = i32
    lib.lp_selftest_box_muller.argtypes = [i64, u64, p, p]
    lib.lp_selftest_normal_fast.restype = i32
    lib.lp_selftest_normal_fast.argtypes = [C.c_uint32, i32, p, p, p]
    lib.lp_build_coef_table.restype = i32
    lib.lp_build_coef_table.argtypes = [p, p, p, p, p, i64, C.POINTER(Hyper), p]
    lib.lp_build_coef_table_dt.restype = i32
    lib.lp_build_coef_table_dt.argtypes = [p, p, p, p, C.c_double, C.c_int32, i64, p]
    lib.lp_torch_randn_geometry.restype = i32
    lib.lp_torch_randn_geometry.argtypes = [i64, i32, C.POINTER(i64), C.POINTER(u64)]
    lib.lp_pack_mask_f32.restype = i32
    lib.lp_pack_mask_f32.argtypes = [p, p, i64, i32, p]
    lib.lp_prologue_f32.restype = i32
    lib.lp_prologue_f32.argtypes = [p, p, p, p, p, p, p, C.POINTER(Dims), p]
    lib.lp_substep.restype = i32
    lib.lp_substep.argtypes = [p, C.POINTER(Heads), p, p, p, p, p, p, C.POINTER(Dims), C.POINTER(Rng), i32, p]
    lib.lp_boundary.restype = i32
    lib.lp_boundary.argtypes = [C.POINTER(Heads), p, p, p, p, p, C.c_float, p, C.POINTER(Dims), p]
    lib.lp_known_words.restype = i64
    lib.lp_known_words.argtypes = [i64]
    lib.lp_pack_known.restype = i32
    lib.lp_pack_known.argtypes = [p, C.POINTER(Dims), p, p, p, p, p, p]
    lib.lp_substep_known.restype = i32
    lib.lp_substep_known.argtypes = [p, C.POINTER(Heads), p, p, C.POINTER(Known), p, p, p, p, C.POINTER(Dims),
                                     C.POINTER(Rng), i32, p]
    lib.lp_boundary_known.restype = i32
    lib.lp_boundary_known.argtypes = [C.POINTER(Heads), p, p, p, C.POINTER(Known), p, p, C.c_float, p, C.POINTER(Dims), p]
    lib.lp_boundary_ancestral.restype = i32
    lib.lp_boundary_ancestral.argtypes = [C.POINTER(Heads), p, p, p, C.POINTER(Known), p, p, C.POINTER(Ancestral),
                                          C.POINTER(Rng), p, C.POINTER(Dims), p]
    lib.lp_boundary_multistep.restype = i32
    lib.lp_boundary_multistep.argtypes = [C.POINTER(Heads), p, p, p, C.POINTER(Known), p, p, p, C.POINTER(Multistep), p,
                                          C.POINTER(Dims), p]
    lib.lp_boundary_midpoint.restype = i32
    lib.lp_boundary_midpoint.argtypes = [C.POINTER(Heads), p, p, p, C.POINTER(Known), p, p, p, p, C.POINTER(Midpoint), p,
                                         C.POINTER(Dims), p]
    lib.lp_boundary_deis.restype = i32
    lib.lp_boundary_deis.argtypes = [C.POINTER(Heads), p, p, p, C.POINTER(Known), p, p, p, p, p, C.POINTER(Deis), p,
                                     C.POINTER(Dims), p]
    lib.lp_boundary_gradient_estimation.restype = i32
    lib.lp_boundary_gradient_estimation.argtypes = [C.POINTER(Heads), p, p, p, C.POINTER(Known), p, p, p, p,
                                                    C.POINTER(GradientEstimation), p, C.POINTER(Dims), p]
    lib.lp_boundary_heun.restype = i32
    lib.lp_boundary_heun.argtypes = [C.POINTER(Heads), p, p, p, C.POINTER(Known), p, p, p, p, C.POINTER(Heun), p,
                                     C.POINTER(Dims), p]
    # the row-bounded forms: `out_rows` (int64) right after `out`
    for name in ("lp_boundary_known", "lp_boundary_ancestral", "lp_boundary_midpoint", "lp_boundary_deis",
                 "lp_boundary_gradient_estimation"):
        f, g = getattr(lib, name), getattr(lib, name + "_rows")
        out = {"lp_boundary_midpoint": 8}.get(name, 6)   # position of `out`
        g.restype = i32
        g.argtypes = f.argtypes[:out + 1] + [i64] + f.argtypes[out + 1:]
    lib.lp_synth_denoiser.restype = i32
    lib.lp_synth_denoiser.argtypes = [p, p, p, i32, i64, p, p]
    lib.lp_substep_f32.restype = i32
    lib.lp_substep_f32.argtypes = [p, p, p, p, p, p, p, p, p, C.POINTER(Dims), C.POINTER(Rng), i32, p]
    lib.lp_substep_cfg_f32.restype = i32
    lib.lp_substep_cfg_f32.argtypes = [p, p, p, C.c_float, C.c_float, p, p, p, p, p, p, C.POINTER(Dims), C.POINTER(Rng),
                                       i32, p]
    lib.lp_epilogue_cfg_f32.restype = i32
    lib.lp_epilogue_cfg_f32.argtypes = [p, p, C.c_float, p, p, p, p, C.c_float, C.POINTER(Dims), p]
    lib.lp_advance_f32.restype = i32
    lib.lp_advance_f32.argtypes = [p, p, p, p, C.POINTER(Dims), C.POINTER(Rng), i32, p]
    lib.lp_epilogue_f32.restype = i32
    lib.lp_epilogue_f32.argtypes = [p, p, p, p, C.POINTER(Dims), p]
    lib.lp_epilogue_euler_f32.restype = i32
    lib.lp_epilogue_euler_f32.argtypes = [p, p, p, p, p, C.c_float, C.POINTER(Dims), p]
    lib.lp_step_boundary_f32.restype = i32
    lib.lp_step_boundary_f32.argtypes = [p, p, p, p, p, p, C.c_float, p, C.POINTER(Dims), p]
    lib.lp_stop_stats_f32.restype = i32
    lib.lp_stop_stats_f32.argtypes = [p, p, p, p, p, C.POINTER(Dims), p, p]
    lib.lp_fill_normal_f32.restype = i32
    lib.lp_fill_normal_f32.argtypes = [p, i64, C.POINTER(Rng), p]
    lib.lp_synth_denoiser_f32.restype = i32
    lib.lp_synth_denoiser_f32.argtypes = [p, p, p, i64, p, p]
    lib.lp_l2_persist_capacity.restype = i32
    lib.lp_l2_persist_capacity.argtypes = [i32, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.lp_l2_persist_set.restype = i32
    lib.lp_l2_persist_set.argtypes = [p, C.c_size_t, p]
    lib.lp_l2_persist_clear.restype = i32
    lib.lp_l2_persist_clear.argtypes = [p]
    lib.lp_l2_flush.restype = i32
    lib.lp_l2_flush.argtypes = [p, C.c_size_t, p]
    lib.lp_torch_cpu_randn_f32.restype = i32
    lib.lp_torch_cpu_randn_f32.argtypes = [p, i64, u64, p, C.POINTER(i64), p]
    v = lib.lp_abi_version()
    if v != ABI_VERSION:
        raise NativeError(f"ABI mismatch: library {v}, binding {ABI_VERSION}")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        lib = load()
        msg = lib.lp_status_string(rc).decode()
        raise NativeError(f"{what}: {msg} (status {rc}, cudaError {lib.lp_last_cuda_error()})")
