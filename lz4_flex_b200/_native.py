"""Loader/builder of liblz4b200.so (the CUDA C-ABI library, include/lz4b200.h).

The library is built in-tree with nvcc for sm_90a and loaded with ctypes.  There is no Python or
CPU implementation behind these bindings: if the library is missing it is rebuilt, and if it cannot be
loaded or no CUDA device exists, every call fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

_PKG = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_PKG, "csrc")
SO_PATH = os.environ.get("LZ4B200_SO_OVERRIDE") or os.path.join(_PKG, "liblz4b200.so")   # override: tuning builds only
HEADER = os.path.join(os.path.dirname(_PKG), "include", "lz4b200.h")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC",
]


def _sources():
    return [os.path.join(_CSRC, f) for f in sorted(os.listdir(_CSRC)) if f.endswith(".cu")]


def _stale() -> bool:
    if not os.path.exists(SO_PATH):
        return True
    t = os.path.getmtime(SO_PATH)
    deps = [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)] + [HEADER]
    return any(os.path.getmtime(d) > t for d in deps)


AB_SO_PATH = os.path.join(_PKG, "liblz4b200_ab.so")


def build_ab(force: bool = False) -> str:
    """The A/B library: the same sources with -DLZ4B200_AB_VARIANTS, i.e. the product kernels PLUS every variant that
    lost its measurement (thread-per-block, single-thread solo, tagged tables, v1 encoder, converged / batched decoders)
    and the environment switches that select them.  Only tests/test_gpu_kernel_variants.py and tests/dev/* load it (through
    LZ4B200_SO_OVERRIDE in a child process); the product library carries none of it."""
    if not force and os.path.exists(AB_SO_PATH):
        t = os.path.getmtime(AB_SO_PATH)
        deps = [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)] + [HEADER]
        if all(os.path.getmtime(d) <= t for d in deps):
            return AB_SO_PATH
    return _compile(AB_SO_PATH, ["-DLZ4B200_AB_VARIANTS"], force=True)


def build(force: bool = False, verbose: bool = False) -> str:
    """nvcc -gencode arch=compute_90a,code=sm_90a ... -> lz4_flex_b200/liblz4b200.so"""
    if os.environ.get("LZ4B200_SO_OVERRIDE"):
        return SO_PATH
    if not force and not _stale():
        return SO_PATH
    return _compile(SO_PATH, [], force, verbose)


def _compile(out_path: str, extra: list, force: bool = False, verbose: bool = False) -> str:
    SO_PATH = out_path
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found and liblz4b200.so is missing or stale")
    # several ranks of one torchrun job may get here at once: one builds (under a file lock, into a temporary that
    # is renamed into place), the others wait and find a fresh library
    import fcntl
    with open(SO_PATH + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and out_path == globals()["SO_PATH"] and not _stale():
                return SO_PATH
            tmp = f"{SO_PATH}.tmp{os.getpid()}"
            cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + _sources()
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                if os.path.exists(tmp):
                    os.remove(tmp)
                raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
            os.replace(tmp, SO_PATH)
            if verbose:
                print(r.stderr)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return SO_PATH


class FrameInfoC(C.Structure):
    _fields_ = [
        ("block_size_id", C.c_int32), ("block_checksums", C.c_int32), ("content_checksum", C.c_int32),
        ("has_content_size", C.c_int32), ("content_size", C.c_uint64), ("linked", C.c_int32),
        ("reserved", C.c_int32),
    ]


class FrameResultC(C.Structure):
    _fields_ = [("consumed", C.c_uint64), ("written", C.c_uint64), ("err_expected", C.c_uint64),
                ("err_actual", C.c_uint64), ("status", C.c_int32), ("block_status", C.c_int32)]


class FrameDecoderStepC(C.Structure):
    _fields_ = [("consumed", C.c_uint64), ("written", C.c_uint64), ("need", C.c_uint64), ("frame_done", C.c_int32),
                ("pad", C.c_int32), ("result", FrameResultC)]


class FrameIndexInfoC(C.Structure):
    _fields_ = [("block_size", C.c_uint64), ("nblocks", C.c_uint64), ("content_len", C.c_uint64), ("linked", C.c_int32),
                ("pad", C.c_int32), ("result", FrameResultC)]


_lib = None

_vp, _sz, _u32, _i32 = C.c_void_p, C.c_size_t, C.c_uint32, C.c_int
_psz = C.POINTER(C.c_size_t)

# name -> (restype, argtypes).  Kept in one table so tests can check every symbol the header declares.
SIGNATURES = {
    "lz4b200_abi_version": (_i32, []),
    "lz4b200_host_pointer_kind": (_i32, [_vp]),
    "lz4b200_status_string": (C.c_char_p, [_i32]),
    "lz4b200_last_cuda_error": (C.c_char_p, [_vp]),
    "lz4b200_ctx_create": (_i32, [_i32, C.POINTER(_vp)]),
    "lz4b200_ctx_destroy": (None, [_vp]),
    "lz4b200_ctx_set_priority": (None, [_vp, _i32]),
    "lz4b200_ctx_stream": (_vp, [_vp]),
    "lz4b200_ctx_last_kernel": (C.c_char_p, [_vp, _i32]),
    "lz4b200_max_output_size": (_sz, [_sz]),
    "lz4b200_compress_into": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz]),
    "lz4b200_compress_prepend_size": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz]),
    "lz4b200_decompress_into": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz, _psz, _psz]),
    "lz4b200_uncompressed_size": (_i32, [_vp, _sz, _psz]),
    "lz4b200_decompress_size_prepended": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz, _psz, _psz]),
    "lz4b200_compress_batch_device": (_i32, [_vp] * 10 + [_sz, _u32, _vp]),
    "lz4b200_decompress_batch_device": (_i32, [_vp] * 10 + [_sz, _vp]),
    "lz4b200_compress_batch_host": (_i32, [_vp] * 6 + [_sz] + [_vp] * 3 + [_sz]),
    "lz4b200_decompress_batch_host": (_i32, [_vp] * 10 + [_sz]),
    "lz4b200_compress_into_with_table": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz, C.POINTER(C.c_int)]),
    "lz4b200_compress_into_with_dict": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _psz]),
    "lz4b200_compress_prepend_size_with_dict": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _psz]),
    "lz4b200_decompress_into_with_dict": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _psz, _psz, _psz]),
    "lz4b200_decompress_size_prepended_with_dict": (_i32, [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _psz, _psz, _psz]),
    "lz4b200_compress_batch_device_with_dict": (_i32, [_vp] * 5 + [_sz] + [_vp] * 5 + [_sz, _u32, _vp]),
    "lz4b200_decompress_batch_device_with_dict": (_i32, [_vp] * 5 + [_sz] + [_vp] * 6 + [_sz, _vp]),
    "lz4b200_compress_batch_host_with_dict": (_i32, [_vp] * 5 + [_sz, _vp, _sz] + [_vp] * 3 + [_sz]),
    "lz4b200_decompress_batch_host_with_dict": (_i32, [_vp] * 5 + [_sz] + [_vp] * 6 + [_sz]),
    "lz4b200_compress_prepend_size_batch_device": (_i32, [_vp] * 4 + [_sz, _u32, _vp, _sz] + [_vp] * 3),
    "lz4b200_compress_prepend_size_batch_device_with_dict": (_i32, [_vp] * 4 + [_sz, _u32, _vp, _sz, _vp, _sz] + [_vp] * 3),
    "lz4b200_decompress_size_prepended_batch_device": (_i32, [_vp] * 4 + [_sz, _vp, _sz] + [_vp] * 5),
    "lz4b200_decompress_size_prepended_batch_device_with_dict": (_i32, [_vp] * 4 + [_sz, _vp, _sz, _vp, _sz] + [_vp] * 5),
    "lz4b200_frame_bound": (_sz, [_sz, C.POINTER(FrameInfoC)]),
    "lz4b200_frame_compress": (_i32, [_vp, _vp, _sz, C.POINTER(FrameInfoC), _sz, _vp, _sz, _psz]),
    "lz4b200_frame_compress_device": (_i32, [_vp, _vp, _sz, C.POINTER(FrameInfoC), _sz, _vp, _sz, _vp, _vp]),
    "lz4b200_frame_compress_batch_device": (_i32, [_vp, _vp, _vp, _vp, C.POINTER(FrameInfoC), _vp, _sz, _vp, _sz, _vp]),
    "lz4b200_frame_compress_linked_batch_device": (_i32, [_vp, _vp, _vp, _vp, C.POINTER(FrameInfoC), _vp, _sz, _vp, _sz,
                                                           _vp]),
    "lz4b200_frame_compress_batch_device_async_scratch": (_sz, [_vp, _sz, _sz, _sz]),
    "lz4b200_frame_compress_batch_device_async": (_i32, [_vp, _vp, _vp, _vp, C.POINTER(FrameInfoC), _vp, _sz, _vp, _vp,
                                                         _sz, _sz, _sz, _vp, _sz, _vp]),
    "lz4b200_frame_compress_linked_batch_device_async": (_i32, [_vp, _vp, _vp, _vp, C.POINTER(FrameInfoC), _vp, _sz, _vp,
                                                                _vp, _sz, _sz, _sz, _vp, _sz, _vp]),
    "lz4b200_frame_compress_blocks_device": (_i32, [_vp, _vp, _sz, _sz, C.c_uint64, _vp, _sz, _vp, _vp, _vp]),
    "lz4b200_frame_blocks_bound": (_sz, [_sz, _sz]),
    "lz4b200_frame_range_compress": (_i32, [_vp, _vp, _sz, _sz, C.c_uint64, _vp, _vp, _vp]),
    "lz4b200_frame_range_pack": (_i32, [_vp, _vp, _vp, _vp]),
    "lz4b200_peer_alloc": (_i32, [_vp, _sz, C.POINTER(_vp), _vp]),
    "lz4b200_peer_open": (_i32, [_vp, _vp, C.POINTER(_vp)]),
    "lz4b200_peer_close": (_i32, [_vp, _vp]),
    "lz4b200_peer_free": (_i32, [_vp, _vp]),
    "lz4b200_frame_write_header": (_sz, [C.POINTER(FrameInfoC), _vp, _sz]),
    "lz4b200_frame_decompress": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz, C.POINTER(C.c_int)]),
    "lz4b200_frame_decoded_bound": (_i32, [_vp, _sz, _psz]),
    "lz4b200_frame_decompress_next": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz, _psz, C.POINTER(C.c_int),
                                             C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "lz4b200_frame_decompress_next_device": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz, _psz, C.POINTER(C.c_int),
                                                    C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), _vp]),
    "lz4b200_frame_decoded_bound_device": (_i32, [_vp, _vp, _sz, _psz, _vp]),
    "lz4b200_frame_decompress_batch_device": (_i32, [_vp] * 8 + [_sz, _vp]),
    "lz4b200_frame_decompress_batch_device_async_scratch": (_sz, [_sz, _sz]),
    "lz4b200_frame_decompress_batch_device_async": (_i32, [_vp] * 8 + [_sz, _sz, _vp, _sz, _vp]),
    "lz4b200_frame_decoded_bound_batch_device": (_i32, [_vp] * 5 + [_sz, _vp]),
    "lz4b200_frame_split_device_scratch": (_sz, [_sz, _sz]),
    "lz4b200_frame_split_device": (_i32, [_vp, _vp, _sz, _vp, _vp, _sz, _vp, _sz, _vp, _sz, _vp]),
    "lz4b200_frame_decompress_device": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz, C.POINTER(C.c_int),
                                               C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), _vp]),
    "lz4b200_frame_index_device": (_i32, [_vp, _vp, _sz, _vp, _sz, _psz, C.POINTER(FrameIndexInfoC), _vp]),
    "lz4b200_frame_decompress_ranges_device": (_i32, [_vp, _vp, _sz, C.POINTER(FrameIndexInfoC)] + [_vp] * 6 + [_sz, _vp]),
    "lz4b200_frame_index_batch_device": (_i32, [_vp] * 4 + [_sz, _vp, _sz, _psz, _vp, _vp, _vp]),
    "lz4b200_frame_decompress_ranges_batch_device": (_i32, [_vp] * 4 + [_sz] + [_vp] * 3 + [_sz] + [_vp] * 6 + [_sz, _vp]),
    "lz4b200_ctx_last_range_blocks": (C.c_uint64, [_vp]),
    "lz4b200_ctx_set_frame_budget": (None, [_vp, _sz]),
    "lz4b200_ctx_device_bytes": (_sz, [_vp]),
    "lz4b200_frame_decoder_create": (_i32, [_vp, C.POINTER(_vp)]),
    "lz4b200_frame_decoder_destroy": (None, [_vp]),
    "lz4b200_frame_decoder_decode_device": (_i32, [_vp, _vp, _sz, _i32, _vp, _sz, C.POINTER(FrameDecoderStepC), _vp]),
    "lz4b200_frame_encoder_create": (_i32, [_vp, C.POINTER(FrameInfoC), C.POINTER(_vp)]),
    "lz4b200_frame_encoder_destroy": (None, [_vp]),
    "lz4b200_frame_encoder_bound": (_sz, [_vp, _sz, _i32]),
    "lz4b200_frame_encoder_content_len": (C.c_uint64, [_vp]),
    "lz4b200_frame_encoder_encode_device": (_i32, [_vp, _vp, _sz, _i32, _vp, _sz, _vp, _vp]),
    "lz4b200_xxh32": (_u32, [_vp, _sz, _u32]),
    "lz4b200_xxh32_reset": (None, [_vp, _u32]),
    "lz4b200_xxh32_update": (None, [_vp, _vp, _sz]),
    "lz4b200_xxh32_digest": (_u32, [_vp]),
}


def lib():
    """The loaded C-ABI library (built on demand)."""
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(SO_PATH)
        for name, (res, args) in SIGNATURES.items():
            f = getattr(L, name)
            f.restype = res
            f.argtypes = args
        _lib = L
    return _lib


def status_string(code: int) -> str:
    return lib().lz4b200_status_string(code).decode()
