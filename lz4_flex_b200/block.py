"""lz4_flex::block, H100 edition.

Same names, argument meaning and error behaviour as the crate's block API (reference
src/block/compress.rs:588-692, src/block/decompress.rs:454-517, src/block/mod.rs:151-157); every call
goes through the C ABI in include/lz4b200.h into the sm_90a kernels.  The single-block functions are
1:1 replacements and PCIe-bound by construction; `compress_batch` / `decompress_batch` (many independent
blocks per launch) are the throughput path, and `DeviceBatch` is the device-pointer form bench.py times.
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import Iterable, Sequence

import numpy as np

from . import _native
from .errors import CudaError, block_error, error_from_status

BLOCK_FRESH = 0
BLOCK_CONT = 1
BLOCK_HASH5_ALWAYS = 2

WINDOW_SIZE = 64 * 1024          # block/mod.rs:35
MINMATCH = 4                     # block/mod.rs:70
MFLIMIT = 12                     # block/mod.rs:46
LZ4_MIN_LENGTH = MFLIMIT + 1     # block/mod.rs:61
MAX_DISTANCE = (1 << 16) - 1     # block/mod.rs:64


class Context:
    """One lz4b200_ctx: a stream plus scratch on one GPU.  Not shareable between threads at the same time."""

    def __init__(self, device: int = 0, high_priority: bool = False):
        L = _native.lib()
        h = C.c_void_p()
        st = L.lz4b200_ctx_create(device, C.byref(h))
        if st != 0:
            raise CudaError(f"lz4b200_ctx_create(device={device}) failed: no usable CUDA device "
                            f"(status {st}); there is no CPU fallback")
        self._h = h
        self.device = device
        if high_priority:                                   # decode side of a two-context streaming pipeline
            L.lz4b200_ctx_set_priority(h, 1)

    @property
    def handle(self):
        return self._h

    @property
    def stream(self) -> int:
        return _native.lib().lz4b200_ctx_stream(self._h)

    def last_cuda_error(self) -> str:
        return _native.lib().lz4b200_last_cuda_error(self._h).decode()

    def close(self):
        if self._h:
            _native.lib().lz4b200_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_tls = threading.local()


def default_context(device: int | None = None) -> Context:
    """Thread-local context on the current torch device (or device 0)."""
    if device is None:
        device = 0
        try:
            import torch
            if torch.cuda.is_available():
                device = torch.cuda.current_device()
        except Exception:
            pass
    ctxs = getattr(_tls, "ctxs", None)
    if ctxs is None:
        ctxs = _tls.ctxs = {}
    if device not in ctxs:
        ctxs[device] = Context(device)
    return ctxs[device]


def _raise(ctx: Context, status: int, expected: int = 0, actual: int = 0):
    if status in (200, 201):
        raise error_from_status(status, detail=ctx.last_cuda_error())
    raise block_error(status, expected, actual)


def _as_u8(data) -> np.ndarray:
    if isinstance(data, np.ndarray):
        a = data
        if a.dtype != np.uint8:
            a = a.view(np.uint8)
        return np.ascontiguousarray(a).reshape(-1)
    return np.frombuffer(data, dtype=np.uint8)


def _ptr(a: np.ndarray) -> int:
    return a.ctypes.data if a.size else 0


# ---- sizes ----------------------------------------------------------------------------------------

def get_maximum_output_size(input_len: int) -> int:
    """block::get_maximum_output_size (compress.rs:588-590): 16 + 4 + floor(1.1 * n)."""
    return 16 + 4 + (input_len * 110 // 100)


def uncompressed_size(input) -> tuple[int, bytes]:
    """block::uncompressed_size (block/mod.rs:151-157): (size, rest)."""
    b = bytes(input[:4]) if not isinstance(input, np.ndarray) else input[:4].tobytes()
    if len(b) < 4:
        from .errors import ExpectedAnotherByte
        raise ExpectedAnotherByte()
    return int.from_bytes(b, "little"), input[4:]


# ---- single block ----------------------------------------------------------------------------------

def compress_into(input, output, ctx: Context | None = None) -> int:
    """block::compress_into (compress.rs:599): compress `input` into the writable buffer `output`
    (bytearray / numpy uint8); returns bytes written.  Raises CompressOutputTooSmall up-front when
    len(output) < get_maximum_output_size(len(input)), like the reference (compress.rs:338-340)."""
    ctx = ctx or default_context()
    src = _as_u8(input)
    dst = _as_u8(output) if isinstance(output, np.ndarray) else np.frombuffer(output, dtype=np.uint8)
    w = C.c_size_t(0)
    st = _native.lib().lz4b200_compress_into(ctx.handle, _ptr(src), src.size, _ptr(dst), dst.size, C.byref(w))
    if st != 0:
        _raise(ctx, st)
    return w.value


def compress(input, ctx: Context | None = None) -> bytes:
    """block::compress (compress.rs:679)."""
    src = _as_u8(input)
    out = np.empty(get_maximum_output_size(src.size), dtype=np.uint8)
    n = compress_into(src, out, ctx)
    return out[:n].tobytes()


def compress_prepend_size(input, ctx: Context | None = None) -> bytes:
    """block::compress_prepend_size (compress.rs:673): u32 LE uncompressed length + block."""
    ctx = ctx or default_context()
    src = _as_u8(input)
    out = np.empty(get_maximum_output_size(src.size) + 4, dtype=np.uint8)
    w = C.c_size_t(0)
    st = _native.lib().lz4b200_compress_prepend_size(ctx.handle, _ptr(src), src.size, _ptr(out), out.size,
                                                     C.byref(w))
    if st != 0:
        _raise(ctx, st)
    return out[: w.value].tobytes()


def decompress_into(input, output, ctx: Context | None = None) -> int:
    """block::decompress_into (decompress.rs:454): returns bytes written; raises the reference's
    DecompressError variants."""
    ctx = ctx or default_context()
    src = _as_u8(input)
    dst = _as_u8(output) if isinstance(output, np.ndarray) else np.frombuffer(output, dtype=np.uint8)
    w, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    st = _native.lib().lz4b200_decompress_into(ctx.handle, _ptr(src), src.size, _ptr(dst), dst.size,
                                               C.byref(w), C.byref(e1), C.byref(e2))
    if st != 0:
        _raise(ctx, st, e1.value, e2.value)
    return w.value


def decompress(input, min_uncompressed_size: int, ctx: Context | None = None) -> bytes:
    """block::decompress (decompress.rs:508): output may be shorter than `min_uncompressed_size`."""
    out = np.empty(max(min_uncompressed_size, 0), dtype=np.uint8)
    n = decompress_into(input, out, ctx)
    return out[:n].tobytes()


def decompress_size_prepended(input, ctx: Context | None = None) -> bytes:
    """block::decompress_size_prepended (decompress.rs:496)."""
    size, rest = uncompressed_size(input)
    return decompress(rest, size, ctx)


# ---- reusable table ---------------------------------------------------------------------------------------

class CompressTable:
    """block::CompressTable (compress.rs:709-735): Small (u16 entries, 4-byte hash, inputs < 65 535 bytes) or Large
    (u32 entries, 5-byte hash, any size).  The table's memory lives on the GPU; this object carries the variant, which
    is what decides the bytes produced."""
    SMALL, LARGE = 0, 1

    def __init__(self, kind: int = 0):
        self.kind = kind

    @classmethod
    def small(cls) -> "CompressTable":
        return cls(cls.SMALL)

    @classmethod
    def large(cls) -> "CompressTable":
        return cls(cls.LARGE)


def compress_into_with_table(input, output, table: CompressTable, ctx: Context | None = None) -> int:
    """block::compress_into_with_table (compress.rs:744-766).  A Small table handed an input of >= 65 535 bytes is
    upgraded to Large and stays Large."""
    ctx = ctx or default_context()
    src = _as_u8(input)
    dst = _as_u8(output) if isinstance(output, np.ndarray) else np.frombuffer(output, dtype=np.uint8)
    w, k = C.c_size_t(0), C.c_int(table.kind)
    st = _native.lib().lz4b200_compress_into_with_table(ctx.handle, _ptr(src), src.size, _ptr(dst), dst.size,
                                                        C.byref(w), C.byref(k))
    table.kind = k.value
    if st != 0:
        _raise(ctx, st)
    return w.value


# ---- external dictionary ------------------------------------------------------------------------------

def compress_into_with_dict(input, output, dict_data, ctx: Context | None = None) -> int:
    """block::compress_into_with_dict (compress.rs:610-616)."""
    ctx = ctx or default_context()
    src, d = _as_u8(input), _as_u8(dict_data)
    dst = _as_u8(output) if isinstance(output, np.ndarray) else np.frombuffer(output, dtype=np.uint8)
    w = C.c_size_t(0)
    st = _native.lib().lz4b200_compress_into_with_dict(ctx.handle, _ptr(src), src.size, _ptr(d), d.size, _ptr(dst),
                                                       dst.size, C.byref(w))
    if st != 0:
        _raise(ctx, st)
    return w.value


def compress_with_dict(input, ext_dict, ctx: Context | None = None) -> bytes:
    """block::compress_with_dict (compress.rs:685-687)."""
    src = _as_u8(input)
    out = np.empty(get_maximum_output_size(src.size), dtype=np.uint8)
    n = compress_into_with_dict(src, out, ext_dict, ctx)
    return out[:n].tobytes()


def compress_prepend_size_with_dict(input, ext_dict, ctx: Context | None = None) -> bytes:
    """block::compress_prepend_size_with_dict (compress.rs:692-694)."""
    ctx = ctx or default_context()
    src, d = _as_u8(input), _as_u8(ext_dict)
    out = np.empty(get_maximum_output_size(src.size) + 4, dtype=np.uint8)
    w = C.c_size_t(0)
    st = _native.lib().lz4b200_compress_prepend_size_with_dict(ctx.handle, _ptr(src), src.size, _ptr(d), d.size,
                                                               _ptr(out), out.size, C.byref(w))
    if st != 0:
        _raise(ctx, st)
    return out[: w.value].tobytes()


def decompress_into_with_dict(input, output, ext_dict, ctx: Context | None = None) -> int:
    """block::decompress_into_with_dict (decompress.rs:462-468)."""
    ctx = ctx or default_context()
    src, d = _as_u8(input), _as_u8(ext_dict)
    dst = _as_u8(output) if isinstance(output, np.ndarray) else np.frombuffer(output, dtype=np.uint8)
    w, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    st = _native.lib().lz4b200_decompress_into_with_dict(ctx.handle, _ptr(src), src.size, _ptr(d), d.size, _ptr(dst),
                                                         dst.size, C.byref(w), C.byref(e1), C.byref(e2))
    if st != 0:
        _raise(ctx, st, e1.value, e2.value)
    return w.value


def decompress_with_dict(input, min_uncompressed_size: int, ext_dict, ctx: Context | None = None) -> bytes:
    """block::decompress_with_dict (decompress.rs:478-490)."""
    out = np.empty(max(min_uncompressed_size, 0), dtype=np.uint8)
    n = decompress_into_with_dict(input, out, ext_dict, ctx)
    return out[:n].tobytes()


def decompress_size_prepended_with_dict(input, ext_dict, ctx: Context | None = None) -> bytes:
    """block::decompress_size_prepended_with_dict (decompress.rs:522-528)."""
    size, rest = uncompressed_size(input)
    return decompress_with_dict(rest, size, ext_dict, ctx)


def compress_blocks_with_dict(blocks: Iterable[bytes], ext_dict, ctx: Context | None = None) -> list[bytes]:
    """Many independent blocks sharing one dictionary, one launch (lz4b200_compress_batch_host_with_dict)."""
    ctx = ctx or default_context()
    blocks = [bytes(b) for b in blocks]
    d = _as_u8(ext_dict)
    lens = np.array([len(b) for b in blocks], dtype=np.uint32)
    offs = np.zeros(len(blocks), dtype=np.uint64)
    if len(blocks) > 1:
        offs[1:] = np.cumsum(lens[:-1].astype(np.uint64))
    src = np.frombuffer(b"".join(blocks) or b"\0", dtype=np.uint8)
    cap = int(sum(get_maximum_output_size(int(x)) for x in lens))
    out = np.empty(max(cap, 1), dtype=np.uint8)
    out_off = np.zeros(len(blocks), dtype=np.uint64)
    out_len = np.zeros(len(blocks), dtype=np.uint32)
    status = np.zeros(len(blocks), dtype=np.int32)
    st = _native.lib().lz4b200_compress_batch_host_with_dict(
        ctx.handle, _ptr(src), _ptr(offs), _ptr(lens), _ptr(d), d.size, _ptr(out), out.size, _ptr(out_off),
        _ptr(out_len), _ptr(status), len(blocks))
    if st != 0:
        _raise(ctx, st)
    bad = np.nonzero(status)[0]
    if bad.size:
        _raise(ctx, int(status[bad[0]]))
    return [out[int(o): int(o) + int(l)].tobytes() for o, l in zip(out_off, out_len)]


def decompress_blocks_with_dict(blocks: Iterable[bytes], caps: Sequence[int], ext_dict, ctx: Context | None = None):
    """Many independent blocks sharing one dictionary; returns (outputs, status[], expected[])."""
    ctx = ctx or default_context()
    blocks = [bytes(b) for b in blocks]
    d = _as_u8(ext_dict)
    lens = np.array([len(b) for b in blocks], dtype=np.uint32)
    offs = np.zeros(len(blocks), dtype=np.uint64)
    if len(blocks) > 1:
        offs[1:] = np.cumsum(lens[:-1].astype(np.uint64))
    src = np.frombuffer(b"".join(blocks) or b"\0", dtype=np.uint8)
    caps = np.asarray(caps, dtype=np.uint32)
    ooff = np.zeros(len(blocks), dtype=np.uint64)
    if len(blocks) > 1:
        ooff[1:] = np.cumsum(caps[:-1].astype(np.uint64))
    out = np.zeros(max(int(caps.astype(np.uint64).sum()), 1), dtype=np.uint8)
    out_len = np.zeros(len(blocks), dtype=np.uint32)
    status = np.zeros(len(blocks), dtype=np.int32)
    expected = np.zeros(len(blocks), dtype=np.uint64)
    st = _native.lib().lz4b200_decompress_batch_host_with_dict(
        ctx.handle, _ptr(src), _ptr(offs), _ptr(lens), _ptr(d), d.size, _ptr(out), _ptr(ooff), _ptr(caps),
        _ptr(out_len), _ptr(status), _ptr(expected), len(blocks))
    if st != 0:
        _raise(ctx, st)
    outs = [out[int(o): int(o) + int(l)].tobytes() for o, l in zip(ooff, out_len)]
    return outs, status, expected


# ---- many blocks, host memory ----------------------------------------------------------------------

def compress_batch(src, in_off: Sequence[int], in_len: Sequence[int], flags: Sequence[int] | None = None,
                   out: np.ndarray | None = None, ctx: Context | None = None):
    """Compress many independent blocks of the host buffer `src` in one launch.

    Returns (out, out_off, out_len): compressed blocks packed back to back in `out`.
    `flags[b]` is BLOCK_FRESH (block API), or BLOCK_CONT / BLOCK_HASH5_ALWAYS for frame blocks."""
    ctx = ctx or default_context()
    src = _as_u8(src)
    nb = len(in_len)
    in_off = np.ascontiguousarray(in_off, dtype=np.uint64)
    in_len = np.ascontiguousarray(in_len, dtype=np.uint32)
    fl = None if flags is None else np.ascontiguousarray(flags, dtype=np.uint8)
    if out is None:
        cap = int(sum(get_maximum_output_size(int(x)) for x in in_len)) if nb < 4096 else \
            int(in_len.astype(np.uint64).sum() * 110 // 100 + 20 * nb)
        out = np.empty(cap, dtype=np.uint8)
    out_off = np.zeros(nb, dtype=np.uint64)
    out_len = np.zeros(nb, dtype=np.uint32)
    status = np.zeros(nb, dtype=np.int32)
    st = _native.lib().lz4b200_compress_batch_host(
        ctx.handle, _ptr(src), _ptr(in_off), _ptr(in_len), _ptr(fl) if fl is not None else None,
        _ptr(out), out.size, _ptr(out_off), _ptr(out_len), _ptr(status), nb)
    if st != 0:
        _raise(ctx, st)
    bad = np.nonzero(status)[0]
    if bad.size:
        _raise(ctx, int(status[bad[0]]))
    return out, out_off, out_len


def decompress_batch(src, in_off: Sequence[int], in_len: Sequence[int], out: np.ndarray,
                     out_off: Sequence[int], out_cap: Sequence[int], ctx: Context | None = None,
                     raise_on_error: bool = True):
    """Decompress many independent blocks in one launch.  Returns (out_len, status, err_expected)."""
    ctx = ctx or default_context()
    src = _as_u8(src)
    nb = len(in_len)
    in_off = np.ascontiguousarray(in_off, dtype=np.uint64)
    in_len = np.ascontiguousarray(in_len, dtype=np.uint32)
    out_off = np.ascontiguousarray(out_off, dtype=np.uint64)
    out_cap = np.ascontiguousarray(out_cap, dtype=np.uint32)
    out_len = np.zeros(nb, dtype=np.uint32)
    status = np.zeros(nb, dtype=np.int32)
    expected = np.zeros(nb, dtype=np.uint64)
    st = _native.lib().lz4b200_decompress_batch_host(
        ctx.handle, _ptr(src), _ptr(in_off), _ptr(in_len), _ptr(out), _ptr(out_off), _ptr(out_cap),
        _ptr(out_len), _ptr(status), _ptr(expected), nb)
    if st != 0:
        _raise(ctx, st)
    if raise_on_error:
        bad = np.nonzero(status)[0]
        if bad.size:
            b = int(bad[0])
            _raise(ctx, int(status[b]), int(expected[b]), int(out_cap[b]))
    return out_len, status, expected


def compress_blocks(blocks: Iterable[bytes], flags: Sequence[int] | None = None,
                    ctx: Context | None = None) -> list[bytes]:
    """Convenience: list of inputs -> list of compressed blocks (one launch)."""
    blocks = [bytes(b) for b in blocks]
    if not blocks:
        return []
    lens = np.array([len(b) for b in blocks], dtype=np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens[:-1], dtype=np.uint64)]).astype(np.uint64)
    src = np.frombuffer(b"".join(blocks) or b"\0", dtype=np.uint8)
    out, out_off, out_len = compress_batch(src, offs, lens, flags, ctx=ctx)
    return [out[int(o): int(o) + int(n)].tobytes() for o, n in zip(out_off, out_len)]


def decompress_blocks(blocks: Iterable[bytes], caps: Sequence[int], ctx: Context | None = None,
                      raise_on_error: bool = True):
    """Convenience: list of compressed blocks + capacities -> (list of outputs, status, expected)."""
    blocks = [bytes(b) for b in blocks]
    if not blocks:
        return [], np.zeros(0, np.int32), np.zeros(0, np.uint64)
    lens = np.array([len(b) for b in blocks], dtype=np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens[:-1], dtype=np.uint64)]).astype(np.uint64)
    caps = np.asarray(caps, dtype=np.uint32)
    ooff = np.concatenate([[0], np.cumsum(caps[:-1], dtype=np.uint64)]).astype(np.uint64)
    src = np.frombuffer(b"".join(blocks) or b"\0", dtype=np.uint8)
    out = np.zeros(max(int(caps.astype(np.uint64).sum()), 1), dtype=np.uint8)
    out_len, status, expected = decompress_batch(src, offs, lens, out, ooff, caps, ctx, raise_on_error)
    outs = [out[int(o): int(o) + int(n)].tobytes() for o, n in zip(ooff, out_len)]
    return outs, status, expected


# ---- many blocks, device memory (torch tensors as the allocator; the measured path) ----------------

class DeviceBatch:
    """Descriptor arrays of a batch of blocks resident in HBM.  All tensors are torch CUDA tensors;
    torch is only the allocator/stream provider here — the work is the C-ABI call."""

    def __init__(self, in_off, in_len, out_off, out_cap, flags=None, device=None):
        import torch
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.nblocks = len(in_len)
        self.max_in_len = int(np.max(in_len)) if self.nblocks else 0
        t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt).view(np.int64 if dt == np.uint64 else (np.int32 if dt == np.uint32 else np.uint8))).to(dev)
        self.in_off = t(in_off, np.uint64)
        self.in_len = t(in_len, np.uint32)
        self.out_off = t(out_off, np.uint64)
        self.out_cap = t(out_cap, np.uint32)
        self.flags = None if flags is None else t(flags, np.uint8)
        self.out_len = torch.zeros(self.nblocks, dtype=torch.int32, device=dev)
        self.status = torch.zeros(self.nblocks, dtype=torch.int32, device=dev)
        self.expected = torch.zeros(self.nblocks, dtype=torch.int64, device=dev)

    def compress(self, d_in, d_out, ctx: Context, stream: int | None = None):
        """lz4b200_compress_batch_device on torch's current stream (or `stream`)."""
        import torch
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        st = _native.lib().lz4b200_compress_batch_device(
            ctx.handle, d_in.data_ptr(), self.in_off.data_ptr(), self.in_len.data_ptr(),
            self.flags.data_ptr() if self.flags is not None else None, d_out.data_ptr(),
            self.out_off.data_ptr(), self.out_cap.data_ptr(), self.out_len.data_ptr(),
            self.status.data_ptr(), self.nblocks, self.max_in_len, s)
        if st != 0:
            _raise(ctx, st)

    def decompress(self, d_in, d_out, ctx: Context, stream: int | None = None):
        """lz4b200_decompress_batch_device on torch's current stream (or `stream`)."""
        import torch
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        st = _native.lib().lz4b200_decompress_batch_device(
            ctx.handle, d_in.data_ptr(), self.in_off.data_ptr(), self.in_len.data_ptr(), d_out.data_ptr(),
            self.out_off.data_ptr(), self.out_cap.data_ptr(), self.out_len.data_ptr(),
            self.status.data_ptr(), self.expected.data_ptr(), self.nblocks, s)
        if st != 0:
            _raise(ctx, st)
