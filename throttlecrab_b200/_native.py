"""Build and load libgcra_b200.so (the C ABI in include/gcra_b200.h) with ctypes.

There is no CPU fallback: importing works anywhere (so the symbol table can be checked on a
box without a GPU), but creating an engine fails loudly when the library or a CUDA device
is missing.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_PKG)
_SRC = os.path.join(_PKG, "csrc")
SO_PATH = os.environ.get("GCRA_SO") or os.path.join(_PKG, "libgcra_b200.so")   # GCRA_SO: tuning variants

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "--shared", "-Xcompiler", "-fPIC", "-Xcompiler", "-pthread", "-ldl"]

REQ_DTYPE = np.dtype([("key_hash", "<u8"), ("max_burst", "<i8"), ("count_per_period", "<i8"),
                      ("period", "<i8"), ("quantity", "<i8"), ("now_ns", "<i8")])
RES_DTYPE = np.dtype([("remaining", "<i8"), ("reset_after_ns", "<i8"), ("retry_after_ns", "<i8"),
                      ("status", "<i4"), ("allowed", "u1"), ("pad", "u1", (3,))])
REQ16_DTYPE = np.dtype([("key_hash", "<u8"), ("quantity", "<i4"), ("policy", "<u4")])
POLICY_DTYPE = np.dtype([("max_burst", "<i8"), ("count_per_period", "<i8"), ("period", "<i8")])
assert REQ_DTYPE.itemsize == 48 and RES_DTYPE.itemsize == 32 and REQ16_DTYPE.itemsize == 16

OK, NEGATIVE_QUANTITY, INVALID_RATE_LIMIT, INTERNAL = 0, 1, 2, 3
STORE_PERIODIC, STORE_PROBABILISTIC, STORE_ADAPTIVE, STORE_MANUAL = 0, 1, 2, 3
FLAG_TIGHT_TABLE, FLAG_INDEX_PATH, FLAG_SORT_PATH, FLAG_RANDOM_SEED = 1, 2, 4, 8


class Config(C.Structure):
    _fields_ = [("capacity", C.c_uint64), ("device", C.c_int32), ("store_kind", C.c_int32),
                ("p0", C.c_uint64), ("p1", C.c_uint64), ("p2", C.c_uint64),
                ("created_ns", C.c_int64), ("max_batch", C.c_uint32), ("flags", C.c_uint32),
                ("hash_seed", C.c_uint64 * 2)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in
                ("len", "occupied_slots", "table_slots", "stash_entries", "allowed", "denied",
                 "errors", "expired_hits", "sweeps", "swept", "grows", "purges",
                 "index_batches", "residue_rows", "residue_batches", "drains", "path_switches")]


def sources():
    return [os.path.join(_SRC, f) for f in sorted(os.listdir(_SRC))] + \
        [os.path.join(_ROOT, "include", "gcra_b200.h")]


def build(force=False, verbose=False):
    """nvcc cross-compiles for sm_90a (H100) without a GPU; the .so is kept in-tree."""
    srcs = sources()
    if os.environ.get("GCRA_SO"):
        return SO_PATH                      # a prebuilt tuning variant
    if not force and os.path.exists(SO_PATH) and all(
            os.path.getmtime(s) <= os.path.getmtime(SO_PATH) for s in srcs):
        return SO_PATH
    cmd = ["nvcc"] + NVCC_FLAGS + ["-o", SO_PATH, os.path.join(_SRC, "gcra_b200.cu")]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd)
    return SO_PATH


# name -> (restype, argtypes); every symbol include/gcra_b200.h declares
_vp, _u64, _i64, _u32, _i32 = C.c_void_p, C.c_uint64, C.c_int64, C.c_uint32, C.c_int32
_pi64, _pu8, _pu64 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)
SYMBOLS = {
    "gcra_create": (_i32, [C.POINTER(Config), C.POINTER(_vp)]),
    "gcra_destroy": (None, [_vp]),
    "gcra_last_error": (C.c_char_p, [_vp]),
    "gcra_hash_key": (_u64, [C.c_char_p, _u64]),
    "gcra_hash_key_seeded": (_u64, [C.c_char_p, _u64, _u64, _u64]),
    "gcra_engine_hash_key": (_u64, [_vp, C.c_char_p, _u64]),
    "gcra_get_hash_seed": (None, [_vp, C.POINTER(_u64 * 2)]),
    "gcra_hash_key_ids": (None, [C.c_char_p, _u64, _vp, _u64, _vp]),
    "gcra_derive_params": (_i32, [_i64, _i64, _i64, _pi64, _pi64]),
    "gcra_store_get": (_i32, [_vp, C.c_char_p, _u64, _i64, _pi64, _pu8]),
    "gcra_store_cas": (_i32, [_vp, C.c_char_p, _u64, _i64, _i64, _u64, _i64, _pu8]),
    "gcra_store_set_nx": (_i32, [_vp, C.c_char_p, _u64, _i64, _u64, _i64, _pu8]),
    "gcra_rate_limit": (_i32, [_vp, C.c_char_p, _u64, _i64, _i64, _i64, _i64, _i64, _vp]),
    "gcra_rate_limit_batch": (_i32, [_vp, _u64, _vp, _vp]),
    "gcra_rate_limit_batch_device": (_i32, [_vp, _u64, _vp, _vp, _vp]),
    "gcra_rate_limit_batch_device_pipelined": (_i32, [_vp, _u64, _vp, _vp, _vp]),
    "gcra_pipeline_join": (_i32, [_vp, _vp]),
    "gcra_set_policies": (_i32, [_vp, _u32, _vp]),
    "gcra_rate_limit_batch16": (_i32, [_vp, _u64, _vp, _i64, _vp]),
    "gcra_rate_limit_batch16_device": (_i32, [_vp, _u64, _vp, _i64, _vp, _vp]),
    "gcra_ring_create": (_i32, [_vp, _u32, _u32, _i32]),
    "gcra_ring_requests": (_vp, [_vp, _u32]),
    "gcra_ring_results": (_vp, [_vp, _u32]),
    "gcra_ring_submit": (_i32, [_vp, _u32, _u32, _i64]),
    "gcra_ring_wait": (_i32, [_vp, _u32]),
    "gcra_ring_poll": (_i32, [_vp, _u32, C.POINTER(_i32)]),
    "gcra_sweep": (_i32, [_vp, _i64, _pu64]),
    "gcra_policy_tick": (_i32, [_vp, _i64, _pu64]),
    "gcra_len": (_u64, [_vp]),
    "gcra_get_stats": (_i32, [_vp, C.POINTER(Stats)]),
    "gcra_track_denied": (_i32, [_vp, _u32]),
    "gcra_top_denied": (_i32, [_vp, _u32, _vp, _vp, C.POINTER(_u32), _pu64]),
    "gcra_peek": (_i32, [_vp, _u64, _pi64, _pi64, _pu8]),
    "gcra_snapshot_save": (_i32, [_vp, C.c_char_p]),
    "gcra_snapshot_load": (_i32, [_vp, C.c_char_p]),
    "gcra_sync": (_i32, [_vp]),
    "gcra_last_kernel_ms": (_i32, [_vp, C.POINTER(C.c_float * 4)]),
    "gcra_last_kernel_ms_detail": (_i32, [_vp, C.POINTER(C.c_float * 7)]),
    "gcra_debug_set": (None, [_vp, _u32]),
    "gcra_last_sweep_ms": (_i32, [_vp, C.POINTER(C.c_float)]),
    "gcra_launch_count": (_u64, [_vp]),
    "gcra_shard_unique_ids": (_i32, [_vp]),
    "gcra_shard_init": (_i32, [_vp, _i32, _i32, _vp, _u32]),
    "gcra_shard_submit": (_i32, [_vp, _u64, _vp, _vp, _vp]),
    "gcra_shard_join": (_i32, [_vp, _vp]),
    "gcra_shard_wait_tick": (_i32, [_vp, _u32, _vp]),
    "gcra_p2p_prepare": (_i32, [_vp, _i32, _i32, _u32, _vp, C.POINTER(_vp)]),
    "gcra_p2p_connect": (_i32, [_vp, _vp, _vp]),
    "gcra_p2p_submit": (_i32, [_vp, _u64, _vp, _vp, _vp]),
    "gcra_p2p_submit_route": (_i32, [_vp, _u64, _vp, _vp]),
    "gcra_p2p_submit_finish": (_i32, [_vp, _vp]),
    "gcra_p2p_wait_tick": (_i32, [_vp, _u32, _vp]),
    "gcra_p2p_join": (_i32, [_vp, _vp]),
    "gcra_p2p_error": (_i32, [_vp, C.POINTER(_u32)]),
    "gcra_p2p_set_timing": (_i32, [_vp, _i32]),
    "gcra_p2p_last_tick_ms": (_i32, [_vp, C.POINTER(C.c_float * 5)]),
    "gcra_actor_create": (_i32, [_vp, _u32, _u32, C.POINTER(_vp)]),
    "gcra_actor_throttle": (_i32, [_vp, C.c_char_p, _u64, _i64, _i64, _i64, _i64, _i64, _vp]),
    "gcra_actor_stats": (_i32, [_vp, C.POINTER(_u64 * 3)]),
    "gcra_actor_destroy": (None, [_vp]),
    "gcra_resp_parse_throttle": (_i32, [_vp, C.c_char_p, _u64, _i64, _u32, _vp, _pu64, C.POINTER(_u32), C.POINTER(_i32)]),
    "gcra_resp_format_replies": (_u64, [_vp, _vp, _u32, _vp, _u64]),
    "gcra_owner_of": (_u32, [_u64, _u32]),
    "gcra_route_partition": (_i32, [_vp, _u64, _vp, _u32, _vp, _vp, _vp, _vp]),
    "gcra_route_unpermute": (_i32, [_vp, _u64, _vp, _vp, _vp, _vp]),
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            build()
        L = C.CDLL(SO_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)      # AttributeError if the header and the library disagree
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib
