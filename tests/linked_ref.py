"""The linked-frame parity reference (tests/cpp/linked_frame_ref.c): lz4_flex's FrameEncoder with BlockMode::Linked,
restated in C, built with gcc on first use into tests/cpp/_build and called through ctypes.  Test infrastructure only."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "linked_frame_ref.c")
SO = os.path.join(HERE, "cpp", "_build", "liblinked_frame_ref.so")

BLOCK_CHECKSUMS, CONTENT_CHECKSUM, CONTENT_SIZE = 1, 2, 4          # the C oracle's frame flag bits

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO) or os.path.getmtime(SO) < os.path.getmtime(SRC):
            if shutil.which("gcc") is None:
                raise RuntimeError("gcc is required to build the linked-frame reference")
            os.makedirs(os.path.dirname(SO), exist_ok=True)
            tmp = f"{SO}.tmp{os.getpid()}"
            subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-Wall", "-Wextra", "-Werror", "-o", tmp, SRC],
                           check=True)
            os.replace(tmp, SO)
        L = C.CDLL(SO)
        L.lfr_frame_bound.restype = C.c_size_t
        L.lfr_frame_bound.argtypes = [C.c_size_t, C.c_int, C.c_size_t]
        L.lfr_frame_compress.restype = C.c_int64
        L.lfr_frame_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_uint, C.c_size_t, C.c_void_p, C.c_size_t]
        _lib = L
    return _lib


def frame_compress(data, block_size_id: int = 0, flags: int = 0, flush_every: int = 0) -> bytes:
    """FrameEncoder::with_frame_info(info, Vec::new()), write_all(data) (in chunks of flush_every bytes, each followed
    by flush(), when flush_every > 0) and finish() with linked blocks.  flags: the C oracle's frame flag bits (the
    linked bit, 8, is implied and ignored)."""
    src = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    cap = lib().lfr_frame_bound(src.size, block_size_id, flush_every)
    out = np.empty(cap, dtype=np.uint8)
    r = lib().lfr_frame_compress(src.ctypes.data if src.size else None, src.size, block_size_id, flags & 7, flush_every,
                                 out.ctypes.data, cap)
    assert r >= 0, r
    return out[:r].tobytes()
