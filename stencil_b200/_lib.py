"""ctypes binding of the C ABI (include/stencil_b200.h -> stencil_b200/libstencil_b200.so).

There is no CPU fallback: if the shared library is missing or a CUDA call fails, the call raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Sequence

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SB_LIB_PATH") or os.path.join(_HERE, "libstencil_b200.so")


class StencilError(RuntimeError):
    pass


class Pitched(C.Structure):
    """sb_pitched: the cudaPitchedPtr the reference passes around (ptr, pitch bytes, rows per plane)."""

    _fields_ = [("ptr", C.c_void_p), ("pitch", C.c_int64), ("ysize", C.c_int64)]


class BoxCopy(C.Structure):
    """sb_box_copy"""

    _fields_ = [
        ("dst", Pitched),
        ("dst_pos", C.c_int64 * 3),
        ("src", Pitched),
        ("src_pos", C.c_int64 * 3),
        ("extent", C.c_int64 * 3),
        ("elem_size", C.c_int64),
    ]


I3 = C.c_int64 * 3
I27 = C.c_int64 * 27

class AstarothParams(C.Structure):
    """sb_astaroth_params: the uniforms solve<> reads through DCONST (astaroth/user_kernels.h:389-427)."""

    _fields_ = [(n, C.c_double) for n in ("inv_dsx", "inv_dsy", "inv_dsz", "dt", "cs2_sound", "gamma", "cp_sound", "lnrho0", "lnT0", "mu0", "nu_visc", "zeta", "eta")]


class HaloPush(C.Structure):
    """sb_halo_push: the six face neighbours' output allocations (-x, +x, -y, +y, -z, +z)."""

    _fields_ = [("nbr", Pitched * 6), ("nbr_zsize", C.c_int64 * 6), ("x_dense", C.c_int64 * 2), ("x_recv", C.c_void_p * 2)]


class BcRegion(C.Structure):
    """sb_bc_region: one ghost box a boundary condition writes, with its source map."""

    _fields_ = [
        ("dir", C.c_int64 * 3),
        ("pos", C.c_int64 * 3),
        ("extent", C.c_int64 * 3),
        ("mirror", C.c_int64 * 3),
        ("faces", C.c_int32),
        ("reserved", C.c_int32),
    ]


class Message(C.Structure):
    """sb_message: one halo message of the exchange plan."""

    _fields_ = [
        ("dir", C.c_int64 * 3),
        ("dst_idx", C.c_int64 * 3),
        ("src_pos", C.c_int64 * 3),
        ("dst_pos", C.c_int64 * 3),
        ("extent", C.c_int64 * 3),
    ]


class Staged(C.Structure):
    """sb_staged: quantity q of message msg at byte offset of a staging buffer."""

    _fields_ = [("msg", C.c_int64), ("q", C.c_int64), ("offset", C.c_int64)]


class BcQuantity(C.Structure):
    """sb_bc_quantity: one quantity of a boundary-condition plan."""

    _fields_ = [
        ("data", Pitched),
        ("elem_size", C.c_int64),
        ("value", C.c_double * 6),
        ("dtype", C.c_int32),
        ("kind", C.c_int32 * 6),
    ]


class ReduceItem(C.Structure):
    """sb_reduce_item: one reduction over a box [lo, hi) of compute cells (global coordinates)."""

    _fields_ = [
        ("kind", C.c_int32),
        ("dtype", C.c_int32),
        ("src", Pitched * 3),
        ("acc_origin", C.c_int64 * 3),
        ("lo", C.c_int64 * 3),
        ("hi", C.c_int64 * 3),
    ]


class ReduceResult(C.Structure):
    """sb_reduce_result"""

    _fields_ = [("min", C.c_double), ("max", C.c_double), ("sum", C.c_double), ("sumsq", C.c_double), ("count", C.c_int64)]


REDUCE_SCALAR, REDUCE_DIFF, REDUCE_NORM3 = 0, 1, 2  # sb_reduce_kind

EXACT_WORDS = 34  # SB_EXACT_WORDS
EXACT_NAN, EXACT_POS_INF, EXACT_NEG_INF = 1, 2, 4  # SB_EXACT_NAN, SB_EXACT_POS_INF, SB_EXACT_NEG_INF


class ExactSum(C.Structure):
    """sb_exact_sum: the exact sum of the finite terms, 2176-bit two's complement in units of 2^-1074 (word[0] least
    significant), and the flags of the non-finite terms."""

    _fields_ = [("word", C.c_uint64 * EXACT_WORDS), ("flags", C.c_uint64)]


class ReduceExactPart(C.Structure):
    """sb_reduce_exact_part"""

    _fields_ = [("min", C.c_double), ("max", C.c_double), ("count", C.c_int64), ("sum", ExactSum), ("sumsq", ExactSum)]


class StencilTerm(C.Structure):
    """sb_stencil_term: one term of a linear stencil operator (source 0 = src, 1 = aux; offset; weight)."""

    _fields_ = [("source", C.c_int32), ("offset", C.c_int32 * 3), ("weight", C.c_double)]


STENCIL_MAX_TERMS, STENCIL_MAX_REACH = 64, 4  # SB_STENCIL_MAX_TERMS, SB_STENCIL_MAX_REACH


class StencilVTerm(C.Structure):
    """sb_stencil_vterm: a term that may also read coefficient field `coef` (-1: none) at `coef_offset`."""

    _fields_ = [("source", C.c_int32), ("offset", C.c_int32 * 3), ("coef", C.c_int32), ("coef_offset", C.c_int32 * 3), ("weight", C.c_double)]


STENCIL_MAX_COEFS, STENCIL_COEF_REACH = 4, 1  # SB_STENCIL_MAX_COEFS, SB_STENCIL_COEF_REACH


class StencilSysTerm(C.Structure):
    """sb_stencil_sys_term: a term of a system: output, input read at offset, coefficient input (-1: none) at coef_offset."""

    _fields_ = [("output", C.c_int32), ("input", C.c_int32), ("offset", C.c_int32 * 3), ("coef", C.c_int32), ("coef_offset", C.c_int32 * 3),
                ("weight", C.c_double)]


# SB_STENCIL_SYS_MAX_INPUTS, SB_STENCIL_SYS_MAX_OUTPUTS, SB_STENCIL_SYS_MAX_TERMS
STENCIL_SYS_MAX_INPUTS, STENCIL_SYS_MAX_OUTPUTS, STENCIL_SYS_MAX_TERMS = 8, 4, 128

I6 = C.c_int32 * 6

TRANSFER_RESTRICT, TRANSFER_PROLONG = 0, 1  # sb_transfer_kind

KRYLOV_DOT, KRYLOV_XPBY, KRYLOV_UPDATE, KRYLOV_BICG_P = 0, 1, 2, 4  # sb_krylov_mode (3 is not a mode)

FUSED_MAX_GROUPS = 4096  # SB_FUSED_MAX_GROUPS


class StepSync(C.Structure):
    """sb_step_sync: per-face mailbox rows of the in-kernel handshake of sb_jacobi3d_fused_sync."""

    _fields_ = [("wait_rows", C.c_void_p * 6), ("signal_rows", C.c_void_p * 6), ("wait_value", C.c_uint32), ("signal_value", C.c_uint32)]


# every symbol include/stencil_b200.h declares: (restype, argtypes)
_SIGS = {
    "sb_last_error": (C.c_char_p, []),
    "sb_version": (C.c_int, []),
    "sb_launch_count": (C.c_uint64, []),
    "sb_halo_pos": (C.c_int, [I3, I3, I27, C.c_int, I3]),
    "sb_halo_extent": (C.c_int, [I3, I3, I27, I3]),
    "sb_raw_size": (C.c_int, [I3, I27, I3]),
    "sb_prime_factors": (C.c_int, [C.c_int64, C.POINTER(C.c_int64), C.c_int]),
    "sb_rank_partition": (C.c_int, [I3, C.c_int64, I3, I3, I3]),
    "sb_node_partition": (C.c_int, [I3, I27, C.c_int64, C.c_int64, I3, I3, I3, I3]),
    "sb_subdomain_size": (C.c_int, [I3, I3, I3, I3]),
    "sb_subdomain_origin": (C.c_int, [I3, I3, I3, I3]),
    "sb_interior": (C.c_int, [I3, I3, I27, I3, I3]),
    "sb_exterior": (C.c_int, [I3, I3, I27, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "sb_pack": (C.c_int, [C.c_void_p, Pitched, I3, I3, C.c_int64, C.c_void_p]),
    "sb_unpack": (C.c_int, [Pitched, C.c_void_p, I3, I3, C.c_int64, C.c_void_p]),
    "sb_translate": (C.c_int, [Pitched, I3, Pitched, I3, I3, C.c_int64, C.c_void_p]),
    "sb_copy_plan_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.POINTER(BoxCopy), C.c_int64]),
    "sb_copy_plan_launch": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sb_copy_plan_bytes": (C.c_int64, [C.c_void_p]),
    "sb_copy_plan_num_tiles": (C.c_int64, [C.c_void_p]),
    "sb_copy_plan_destroy": (C.c_int, [C.c_void_p]),
    "sb_bc_regions": (C.c_int, [I3, I27, I6, C.POINTER(BcRegion), C.c_int]),
    "sb_exchange_messages": (C.c_int, [I3, I3, I3, C.c_int32 * 3, I27, I3, C.POINTER(Message), C.c_int]),
    "sb_staging_layout": (C.c_int, [I3, I3, I3, C.c_int32 * 3, I27, I3, I3, C.POINTER(C.c_int64), C.c_int, C.POINTER(Staged), C.c_int, C.POINTER(C.c_int64)]),
    "sb_staging_layout_subset": (C.c_int, [I3, I3, I3, C.c_int32 * 3, I27, I3, I3, C.POINTER(C.c_int64), C.c_int, C.c_uint64, C.POINTER(Staged), C.c_int,
                                           C.POINTER(C.c_int64)]),
    "sb_bc_plan_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.POINTER(BcQuantity), C.c_int64, I3, I27]),
    "sb_bc_plan_launch": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sb_bc_plan_bytes": (C.c_int64, [C.c_void_p]),
    "sb_bc_plan_destroy": (C.c_int, [C.c_void_p]),
    "sb_reduce_plan_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.POINTER(ReduceItem), C.c_int64]),
    "sb_reduce_plan_launch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_reduce_plan_bytes": (C.c_int64, [C.c_void_p]),
    "sb_reduce_plan_destroy": (C.c_int, [C.c_void_p]),
    "sb_reduce_combine": (C.c_int, [C.POINTER(ReduceResult), C.c_int64, C.POINTER(ReduceResult)]),
    "sb_reduce_exact_plan_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.POINTER(ReduceItem), C.c_int64]),
    "sb_reduce_exact_plan_launch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_reduce_exact_plan_bytes": (C.c_int64, [C.c_void_p]),
    "sb_reduce_exact_plan_destroy": (C.c_int, [C.c_void_p]),
    "sb_reduce_exact_combine": (C.c_int, [C.POINTER(ReduceExactPart), C.c_int64, C.POINTER(ReduceExactPart)]),
    "sb_reduce_exact_round": (C.c_int, [C.POINTER(ReduceExactPart), C.POINTER(ReduceResult)]),
    "sb_krylov_plan_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.POINTER(Pitched), C.c_int, I3, I3, I3]),
    "sb_krylov_plan_launch": (C.c_int, [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]),
    "sb_krylov_plan_launch2": (C.c_int, [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_void_p]),
    "sb_krylov_plan_bytes": (C.c_int64, [C.c_void_p]),
    "sb_krylov_plan_destroy": (C.c_int, [C.c_void_p]),
    "sb_stencil_check": (C.c_int, [C.POINTER(StencilTerm), C.c_int, I27]),
    "sb_stencil_laplacian": (C.c_int, [C.c_int, C.c_double * 3, C.POINTER(StencilTerm), C.c_int]),
    "sb_stencil_plan_create": (
        C.c_int,
        [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(StencilTerm), C.c_int, Pitched, Pitched, Pitched, I3, C.c_int64, C.c_int,
         C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
    ),
    "sb_stencil_vcheck": (C.c_int, [C.POINTER(StencilVTerm), C.c_int, I27]),
    "sb_stencil_div_grad": (C.c_int, [C.c_double * 3, C.POINTER(StencilVTerm), C.c_int]),
    "sb_stencil_vplan_create": (
        C.c_int,
        [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(StencilVTerm), C.c_int, Pitched, Pitched, Pitched, C.POINTER(Pitched), C.c_int,
         I3, C.c_int64, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
    ),
    "sb_stencil_ccheck": (C.c_int, [C.POINTER(StencilVTerm), C.c_int, I27, C.c_int]),
    "sb_stencil_relax": (C.c_int, [C.POINTER(StencilTerm), C.c_int, C.c_double, C.POINTER(StencilTerm), C.c_int]),
    "sb_stencil_cplan_create": (
        C.c_int,
        [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(StencilVTerm), C.c_int, Pitched, Pitched, Pitched, C.POINTER(Pitched), C.c_int,
         C.c_int, C.c_int, I3, C.c_int64, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
    ),
    "sb_stencil_dplan_create": (
        C.c_int,
        [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(StencilVTerm), C.c_int, Pitched, Pitched, Pitched, C.POINTER(Pitched), C.c_int,
         C.c_double, C.c_int, C.c_int, I3, C.c_int64, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
    ),
    "sb_stencil_sys_check": (C.c_int, [C.POINTER(StencilSysTerm), C.c_int, C.c_int, C.c_int, I27]),
    "sb_stencil_grad": (C.c_int, [C.c_int, C.c_double * 3, C.POINTER(StencilSysTerm), C.c_int]),
    "sb_stencil_div": (C.c_int, [C.c_int, C.c_double * 3, C.POINTER(StencilSysTerm), C.c_int]),
    "sb_stencil_curl": (C.c_int, [C.c_int, C.c_double * 3, C.POINTER(StencilSysTerm), C.c_int]),
    "sb_stencil_sys_plan_create": (
        C.c_int,
        [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(StencilSysTerm), C.c_int, C.POINTER(Pitched), C.c_int, C.POINTER(Pitched), C.c_int,
         I3, C.c_int64, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
    ),
    "sb_stencil_plan_launch": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sb_stencil_plan_bytes": (C.c_int64, [C.c_void_p]),
    "sb_stencil_plan_destroy": (C.c_int, [C.c_void_p]),
    "sb_transfer_check": (C.c_int, [I3, I3, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "sb_transfer_plan_create": (
        C.c_int,
        [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, Pitched, I3, C.c_int64, Pitched, I3, C.c_int64, Pitched, I3, I3],
    ),
    "sb_transfer_oplan_create": (
        C.c_int,
        [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(StencilTerm), C.c_int, Pitched, I3, C.c_int64, Pitched, I3, C.c_int64, Pitched,
         C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
    ),
    "sb_transfer_voplan_create": (
        C.c_int,
        [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(StencilVTerm), C.c_int, Pitched, I3, C.c_int64, Pitched, I3, C.c_int64, Pitched,
         C.POINTER(Pitched), C.c_int, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
    ),
    "sb_transfer_fplan_create": (
        C.c_int,
        [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, Pitched, I3, C.c_int64, Pitched, I3, C.c_int64, I3, I3],
    ),
    "sb_transfer_plan_launch": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sb_transfer_plan_bytes": (C.c_int64, [C.c_void_p]),
    "sb_transfer_plan_destroy": (C.c_int, [C.c_void_p]),
    "sb_signal": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_uint32, C.c_int, C.c_void_p]),
    "sb_wait": (C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_int, C.c_void_p]),
    "sb_jacobi3d": (C.c_int, [Pitched, Pitched, C.c_int, I3, I3, I3, I3, I3, C.c_void_p]),
    "sb_jacobi3d_regions": (C.c_int, [Pitched, Pitched, C.c_int, I3, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64), I3, I3, C.c_void_p]),
    "sb_astaroth_substep": (C.c_int, [C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int, I3, I3, I3, C.POINTER(AstarothParams), C.c_int, C.c_void_p]),
    "sb_jacobi3d_fused": (C.c_int, [Pitched, Pitched, C.c_int, I3, I3, I3, I3, I3, C.POINTER(HaloPush), C.c_void_p]),
    "sb_jacobi3d_fused_sync": (C.c_int, [Pitched, Pitched, C.c_int, I3, I3, I3, I3, I3, C.POINTER(HaloPush), C.POINTER(StepSync), C.c_void_p]),
    "sb_fill": (C.c_int, [Pitched, C.c_int, I3, I3, I3, C.c_double, C.c_void_p]),
    "sb_sqdiff": (C.c_int, [Pitched, Pitched, C.c_int, I3, I3, I3, C.c_void_p, C.c_void_p]),
    "sb_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "sb_malloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_size_t, C.c_int]),
    "sb_free": (C.c_int, [C.c_void_p, C.c_int]),
    "sb_memset": (C.c_int, [C.c_void_p, C.c_int, C.c_size_t, C.c_int, C.c_void_p]),
    "sb_memcpy": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "sb_stream_sync": (C.c_int, [C.c_int, C.c_void_p]),
    "sb_device_sync": (C.c_int, [C.c_int]),
    "sb_enable_peer": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "sb_ipc_export": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sb_ipc_import": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]),
    "sb_ipc_close": (C.c_int, [C.c_void_p, C.c_int]),
}

_lib = None


def lib() -> C.CDLL:
    """Load the shared library (once).  Raises StencilError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise StencilError(
                f"{LIB_PATH} not found: build it with `make` (or `python -c 'import __graft_entry__ as g; g.build()'`); "
                "stencil_b200 has no CPU fallback"
            )
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)  # AttributeError if the header and the library drifted apart
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc: int) -> int:
    if rc < 0:
        raise StencilError(f"stencil_b200 error {rc}: {lib().sb_last_error().decode()}")
    return rc


def i3(v: Sequence[int]) -> I3:
    return I3(int(v[0]), int(v[1]), int(v[2]))


def o3():
    return I3(0, 0, 0)


def t3(a) -> tuple:
    return (int(a[0]), int(a[1]), int(a[2]))


def stream_ptr(stream) -> C.c_void_p:
    """Accept None (default stream), an int handle, or a torch.cuda.Stream."""
    if stream is None:
        return C.c_void_p(0)
    if isinstance(stream, int):
        return C.c_void_p(stream)
    return C.c_void_p(stream.cuda_stream)
