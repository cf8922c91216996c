"""lz4_flex_b200 — an H100-native (sm_90a) LZ4 block codec behind lz4_flex's API surface.

Layout mirrors the crate: `block` (compress*/decompress* free functions, error enums), `frame`
(FrameEncoder/FrameDecoder/FrameInfo), and the crate-root re-exports of lib.rs:96-105.  Everything
computes on the GPU through the C ABI in include/lz4b200.h (lz4_flex_b200/liblz4b200.so); there is no
CPU codec in this package.
"""
from . import block, frame, errors  # noqa: F401
from .block import (compress, compress_into, compress_prepend_size, decompress, decompress_into,  # noqa: F401
                    decompress_size_prepended, get_maximum_output_size, uncompressed_size)

__all__ = ["block", "frame", "errors", "compress", "compress_into", "compress_prepend_size", "decompress",
           "decompress_into", "decompress_size_prepended", "get_maximum_output_size", "uncompressed_size"]
