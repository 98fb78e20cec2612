"""ctypes binding of ``libfugue_b200.so`` (the C ABI declared in ``include/fugue_b200.h``).

There is no CPU fallback: if the shared library is missing, loading raises
``FugueB200LibraryError`` and every engine entry point fails with it.
"""
import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfugue_b200.so")


class FugueB200LibraryError(RuntimeError):
    pass


class FugueB200KernelError(RuntimeError):
    pass


_lib: Optional[C.CDLL] = None


class ExprIns(C.Structure):
    """``fb_expr_ins`` of include/fugue_b200.h."""
    _fields_ = [("op", C.c_int32), ("kind", C.c_int32), ("b", C.c_int32), ("flags", C.c_int32),
                ("imm", C.c_int64)]


class MapUnit(C.Structure):
    """``fb_map_unit`` of include/fugue_b200.h (K4 fused map epilogue)."""
    _fields_ = [("src2", C.c_void_p), ("mode", C.c_int32), ("reserved", C.c_int32), ("a", C.c_uint64),
                ("b", C.c_uint64), ("c", C.c_uint64)]


REGEX_MAX_STATES, REGEX_MAX_RANGES, REGEX_MAX_SLOTS, REGEX_MAX_REWRITE = 64, 512, 8, 512
REGEX_MAX_CLOSURES = 2 * (REGEX_MAX_STATES + 2)
REGEX_MAX_ENTRIES = REGEX_MAX_CLOSURES * (REGEX_MAX_STATES + 1)


class RegexProgram(C.Structure):
    """``fb_regex_program`` of include/fugue_b200.h (K15)."""
    _fields_ = [("npos", C.c_int32), ("nranges", C.c_int32), ("nslots", C.c_int32), ("op", C.c_int32),
                ("group_pair", C.c_int32), ("nrewrite", C.c_int32), ("restart", C.c_int32), ("reserved", C.c_int32),
                ("ascii", C.c_uint64 * 128), ("range_mask", C.c_uint64 * REGEX_MAX_RANGES),
                ("range_lo", C.c_uint32 * REGEX_MAX_RANGES), ("cl_mask", C.c_uint64 * REGEX_MAX_CLOSURES),
                ("cl_accept", C.c_uint8 * REGEX_MAX_CLOSURES), ("cl_off", C.c_uint16 * (REGEX_MAX_CLOSURES + 1)),
                ("ent_target", C.c_uint8 * REGEX_MAX_ENTRIES), ("ent_save", C.c_uint8 * REGEX_MAX_ENTRIES),
                ("rewrite", C.c_int16 * REGEX_MAX_REWRITE)]


_vp = C.c_void_p
_i32p = C.POINTER(C.c_int32)
_vpp = C.POINTER(C.c_void_p)

# name -> (restype, argtypes); mirrors include/fugue_b200.h one to one
SIGNATURES = {
    "fb_abi_version": (C.c_int, []),
    "fb_last_error": (C.c_char_p, []),
    "fb_device_info": (C.c_int, [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_size_t),
                                 C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "fb_partition_ids": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _vpp, _i32p, _vpp,
                                   C.c_uint32, _vp]),
    "fb_row_hash64": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _vpp, _i32p, _vpp, _vp]),
    "fb_debug_fastmod_host": (C.c_uint32, [C.c_uint64, C.c_uint32]),
    "fb_partition_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_uint32]),
    "fb_partition_plan": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _vpp, _i32p, _vpp,
                                    C.c_uint32, _vp, C.c_size_t, _vp]),
    "fb_partition_apply": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _vpp, _i32p, _vpp,
                                     C.c_uint32, _vp, C.c_size_t, _vp, C.c_int, _vpp, _i32p,
                                     _vpp]),
    "fb_partition_apply_ex": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _vpp, _i32p, _vpp,
                                        C.c_uint32, _vp, C.c_size_t, _vp, C.c_int, _vpp, _i32p,
                                        _vpp, C.c_int, C.c_int]),
    "fb_partition_map_tail_bytes": (C.c_size_t, [C.c_int]),
    "fb_partition_apply_map": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _vpp, _i32p, _vpp,
                                         C.c_uint32, _vp, C.c_size_t, _vp, C.c_int, _vpp, _vpp, _vp, _vp, C.c_int]),
    "fb_partition_cols": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _vpp, _i32p, _i32p,
                                    C.c_int, _vpp, C.c_uint32, _vpp, _vp, _vp, C.c_size_t]),
    "fb_radix_pass": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, C.c_int, C.c_int, _vpp, _i32p, _vpp, _vp, C.c_size_t,
                                _vp]),
    "fb_bits_to_bytes": (C.c_int, [C.c_int, _vp, _vp, C.c_int64, C.c_int64, _vp]),
    "fb_bytes_to_bits": (C.c_int, [C.c_int, _vp, _vp, C.c_int64, _vp, _vp]),
    "fb_groupby_table_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "fb_groupby_u64": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int, _vpp, _vpp, _i32p, C.c_int64,
                                 C.c_uint32, _vp, _vp, _vp]),
    "fb_groupby_extract": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _i32p, _vp, _vp, _vp, _vp, _vp]),
    "fb_join_table_bytes": (C.c_size_t, [C.c_int64]),
    "fb_join_build_u64": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_uint32, _vp, _vp, _vp]),
    "fb_join_probe_count_u64": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_uint32, _vp,
                                          C.c_int, _vp, _vp]),
    "fb_join_probe_write_u64": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_uint32, _vp,
                                          C.c_int, _vp, _vp, _vp, _vp, _vp]),
    "fb_join_mark_matched": (C.c_int, [C.c_int, _vp, _vp, C.c_int64, _vp]),
    "fb_join2_table_bytes": (C.c_size_t, [C.c_int64]),
    "fb_join2_build": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_uint32, _vp, _vp, _vp]),
    "fb_join2_tiles_bytes": (C.c_size_t, [C.c_int64]),
    "fb_join2_probe": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, C.c_int64, C.c_uint32, _vp, C.c_int,
                                 _vp, _vp, _vp, _vp, _vp]),
    "fb_join2_build_probe": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, C.c_int64, _vp, _vp, _vp, C.c_int64,
                                       C.c_uint32, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp]),
    "fb_join2_emit": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int64, C.c_uint32, _vp, _vp, _vp, _vp,
                                C.c_int, _vpp, _vpp, _i32p, C.c_int, _vpp, _vpp, _i32p, _vpp, _vpp]),
    "fb_exclusive_scan_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "fb_exclusive_scan_i64": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, _vp, C.c_size_t]),
    "fb_compact_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "fb_compact_indices": (C.c_int, [C.c_int, _vp, _vp, C.c_int64, _vp, _vp, _vp, C.c_size_t]),
    "fb_gather_rows": (C.c_int, [C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int64]),
    "fb_scatter_rows": (C.c_int, [C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int64]),
    "fb_asof_search": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int, C.c_int, C.c_int,
                                 C.c_int, C.c_uint64, _vp]),
    "fb_range_join_count": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp, _vp,
                                      C.c_size_t, C.c_int, C.c_int, _vp]),
    "fb_range_join_emit": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp, _vp,
                                     C.c_size_t, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp]),
    "fb_copy_runs_dma": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp]),
    "fb_copy_runs_dma_streams": (C.c_int, [C.c_int, C.c_int64, _vp, _vp, _vp, _vp, C.c_int]),
    "fb_pull_runs_tma": (C.c_int, [C.c_int, _vp, C.c_int, _vp, _vp, _vp, C.c_int]),
    "fb_eval_expr": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _vpp, _i32p, _vpp, C.c_int, _vp, C.c_int,
                               _i32p, _vpp, _vpp]),
    "fb_copy_segments": (C.c_int, [C.c_int, _vp, C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, _vp,
                                   C.c_int64]),
    "fb_segmented_scan_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "fb_segmented_scan": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int, _i32p, _vpp, _vpp, _vpp,
                                    _vpp, _vp, C.c_size_t]),
    "fb_segmented_moments_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "fb_segmented_moments": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int, _vpp, _vpp, _vpp, _vpp,
                                       _vp, C.c_size_t]),
    "fb_segmented_comoments_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "fb_segmented_comoments": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int, _vpp, _vpp, _vpp, _vpp,
                                         _vpp, _vpp, _vpp, _vpp, _vpp, _vpp, _vp, C.c_size_t]),
    "fb_segmented_shape_moments_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "fb_segmented_shape_moments": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int, _vpp, _vpp, _vpp,
                                             _vpp, _vpp, _vpp, _vp, C.c_size_t]),
    "fb_segmented_ewm_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "fb_segmented_ewm": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int, _vpp, _vpp, C.POINTER(C.c_double),
                                   _i32p, _i32p, _vpp, C.POINTER(C.c_double), _vpp, _vpp, _vpp, _vpp, _vpp, _vp,
                                   C.c_size_t]),
    "fb_window_frame_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int]),
    "fb_window_frame": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                  _i32p, _vpp, _vpp, _vpp, _vpp, _vp, C.c_size_t]),
    "fb_window_range_bounds_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "fb_window_range_bounds": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, _vp, C.c_int, C.c_int,
                                         C.c_uint64, C.c_uint64, C.c_int, _vp, _vp, _vp, C.c_size_t]),
    "fb_window_bounded_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "fb_window_bounded": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int, _i32p, _vpp, _vpp, _vpp, _vpp, _vp,
                                    C.c_size_t]),
    "fb_window_tree": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int, _i32p, _vpp, _vpp, _vp, C.c_size_t]),
    "fb_window_value": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int64, C.c_int64, C.c_int, _vp, _vp,
                                  C.c_int, C.POINTER(C.c_int64), _i32p, _vpp, _vpp, _vpp, _vpp]),
    "fb_window_distribution_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "fb_window_distribution": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, _vp, _vp, C.c_int,
                                         C.POINTER(C.c_int64), _vpp, _vp, C.c_size_t]),
    "fb_quantile_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64]),
    "fb_segmented_quantile": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, _vp, C.c_int, C.c_int,
                                        C.POINTER(C.c_double), _i32p, _vp, _vpp, _vp, C.c_size_t]),
    "fb_string_length": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, _vp]),
    "fb_string_like": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, C.c_int, C.POINTER(C.c_int16), _vp, _vp]),
    "fb_string_transform": (C.c_int, [C.c_int, _vp, C.c_int, C.c_int64, _vp, _vp, _vp, _vp, C.c_int64, C.c_int64,
                                      C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.c_int,
                                      C.POINTER(C.c_int16), C.c_int, _vp, _vp, _vp, _vp]),
    "fb_string_hash": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, C.c_int, _vp]),
    "fb_string_first_equal": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "fb_string_parse": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, _vp]),
    "fb_debug_string_parse_host": (C.c_int, [C.c_int64, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp]),
    "fb_value_format": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, C.c_int, _vp, _vp, _vp]),
    "fb_debug_value_format_host": (C.c_int, [C.c_int64, _vp, _vp, C.c_int, _vp, _vp, _vp]),
    "fb_regex_match": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "fb_regex_transform": (C.c_int, [C.c_int, _vp, C.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "fb_debug_regex_host": (C.c_int, [C.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
}


def build_hint() -> str:
    return ("build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C fugue_b200/csrc`")


def load() -> C.CDLL:
    """Load the CUDA library once; raise loudly when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FugueB200LibraryError(
            f"{LIB_PATH} not found - the B200 engine has no CPU fallback; {build_hint()}")
    try:
        lib = C.CDLL(LIB_PATH)
    except OSError as e:  # pragma: no cover
        raise FugueB200LibraryError(f"cannot load {LIB_PATH}: {e}") from e
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise FugueB200LibraryError(
                f"{LIB_PATH} does not export {name}; rebuild ({build_hint()})") from e
        fn.restype = res
        fn.argtypes = args
    if lib.fb_abi_version() != 1:
        raise FugueB200LibraryError("libfugue_b200.so ABI version mismatch; rebuild")
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().fb_last_error()
        raise FugueB200KernelError(msg.decode() if msg else f"fugue_b200 error {rc}")


def ptr_array(ptrs) -> "C.Array":
    arr = (C.c_void_p * max(len(ptrs), 1))()
    for i, p in enumerate(ptrs):
        arr[i] = p
    return arr


def f64_array(vals) -> "C.Array":
    arr = (C.c_double * max(len(vals), 1))()
    for i, v in enumerate(vals):
        arr[i] = float(v)
    return arr


def i32_array(vals) -> "C.Array":
    arr = (C.c_int32 * max(len(vals), 1))()
    for i, v in enumerate(vals):
        arr[i] = int(v)
    return arr
