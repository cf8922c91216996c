"""lz4_flex::frame, H100 edition (encoder: independent-block mode; decoder: independent and linked blocks).

FrameInfo / BlockSize / BlockMode / FrameEncoder / FrameDecoder with the reference's names and behaviour
(src/frame/header.rs:39-192, src/frame/compress.rs:62-438, src/frame/decompress.rs:48-422).  The container
(header, BlockInfo words, checksums, end mark) is host bookkeeping; the blocks themselves are compressed
and decompressed in GPU batches through the C ABI.  Block boundaries, the stored-raw rule and — crucially —
each block's parse mode (FRESH for the first block of a table epoch, CONT afterwards, SURVEY.md §8a) follow
FrameEncoder::write/write_block exactly, so the produced frame is byte-identical to lz4_flex's.

BlockMode::Linked chains every block to its frame's earlier output.  The DECODER handles it on the device
(lz4_decompress_blocks_linked: a block waits for the predecessors an offset reaches into), so frames written by
`lz4` / LZ4F / pyarrow with their default linked blocks decode; the ENCODER refuses it (LinkedBlocksUnsupported):
a linked encode is one serial chain per frame, which is not what a GPU batch path is for.
"""
from __future__ import annotations

import ctypes as C
import enum
import io
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _native, block as _block
from .errors import (ContentChecksumError, ContentLengthError, IoError, LinkedBlocksUnsupported, error_from_status)

WINDOW_SIZE = 64 * 1024
_REPOSITION_LIMIT = 0xFFFFFFFF // 2          # u32::MAX as usize / 2  (frame/compress.rs:266)


class BlockSize(enum.IntEnum):
    """frame::BlockSize (header.rs:39-53)."""
    Auto = 0
    Max64KB = 4
    Max256KB = 5
    Max1MB = 6
    Max4MB = 7
    Max8MB = 8

    @staticmethod
    def from_buf_length(buf_len: int) -> "BlockSize":
        """header.rs:57-67"""
        if buf_len > 256 * 1024:
            return BlockSize.Max4MB
        if buf_len > 64 * 1024:
            return BlockSize.Max256KB
        return BlockSize.Max64KB

    def get_size(self) -> int:
        return {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20, 8: 8 << 20}[int(self)]


class BlockMode(enum.Enum):
    """frame::BlockMode (header.rs:83-91)."""
    Independent = 0
    Linked = 1


@dataclass
class FrameInfo:
    """frame::FrameInfo (header.rs:130-192)."""
    content_size: Optional[int] = None
    dict_id: Optional[int] = None
    block_size: BlockSize = BlockSize.Auto
    block_mode: BlockMode = BlockMode.Independent
    block_checksums: bool = False
    content_checksum: bool = False
    legacy_frame: bool = False

    def to_c(self) -> _native.FrameInfoC:
        return _native.FrameInfoC(int(self.block_size), int(self.block_checksums), int(self.content_checksum),
                                  int(self.content_size is not None), int(self.content_size or 0),
                                  int(self.block_mode == BlockMode.Linked), 0)

    def header_bytes(self) -> bytes:
        """FrameInfo::write (header.rs:232-275)."""
        buf = (C.c_uint8 * 19)()
        ci = self.to_c()
        n = _native.lib().lz4b200_frame_write_header(C.byref(ci), buf, 19)
        return bytes(buf[:n])


class _Xxh32:
    def __init__(self, seed: int = 0):
        self._st = (C.c_uint8 * 48)()
        _native.lib().lz4b200_xxh32_reset(self._st, seed)

    def update(self, data: bytes):
        a = np.frombuffer(data, dtype=np.uint8)
        _native.lib().lz4b200_xxh32_update(self._st, a.ctypes.data if a.size else None, a.size)

    def digest(self) -> int:
        return _native.lib().lz4b200_xxh32_digest(self._st)


def xxh32(data, seed: int = 0) -> int:
    a = np.frombuffer(data, dtype=np.uint8)
    return _native.lib().lz4b200_xxh32(a.ctypes.data if a.size else None, a.size, seed)


# -----------------------------------------------------------------------------------------------------
# one-shot helpers over the C ABI
# -----------------------------------------------------------------------------------------------------

def compress_frame(data, frame_info: FrameInfo | None = None, ctx: _block.Context | None = None) -> bytes:
    """FrameEncoder::with_frame_info(info, Vec::new()); write_all(data); finish() — one C-ABI call."""
    ctx = ctx or _block.default_context()
    info = frame_info or FrameInfo()
    if info.block_mode == BlockMode.Linked:
        raise LinkedBlocksUnsupported()
    src = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    ci = info.to_c()
    cap = _native.lib().lz4b200_frame_bound(src.size, C.byref(ci))
    out = np.empty(cap, dtype=np.uint8)
    w = C.c_size_t(0)
    st = _native.lib().lz4b200_frame_compress(ctx.handle, src.ctypes.data if src.size else None, src.size,
                                              C.byref(ci), src.size, out.ctypes.data, cap, C.byref(w))
    if st != 0:
        raise error_from_status(st, detail=ctx.last_cuda_error())
    return out[: w.value].tobytes()


def decompress_next_frame(data, ctx: _block.Context | None = None):
    """The frame that starts at data[0], through lz4b200_frame_decompress_next: returns
    (decoded bytes, consumed input bytes, exception or None).  Bytes decoded before an error are returned with it.
    consumed == 0 with no bytes and no error means the input is exhausted (decompress.rs:113-128)."""
    ctx = ctx or _block.default_context()
    src = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    L = _native.lib()
    bound = C.c_size_t(0)
    L.lz4b200_frame_decoded_bound(src.ctypes.data if src.size else None, src.size, C.byref(bound))
    out = np.empty(max(bound.value, 1), dtype=np.uint8)
    used, w, bs = C.c_size_t(0), C.c_size_t(0), C.c_int(0)
    e1, e2 = C.c_uint64(0), C.c_uint64(0)
    st = L.lz4b200_frame_decompress_next(ctx.handle, src.ctypes.data if src.size else None, src.size, out.ctypes.data,
                                         bound.value, C.byref(used), C.byref(w), C.byref(bs), C.byref(e1), C.byref(e2))
    err = None if st == 0 else error_from_status(st, bs.value, ctx.last_cuda_error(), e1.value, e2.value)
    return out[: w.value].tobytes(), used.value, err


def decompress_frame(data, ctx: _block.Context | None = None, partial: bool = False):
    """Every concatenated frame of `data`, outputs joined (a convenience; the reference's reader stops at each
    EndMark — FrameDecoder below does too, and decompress_next_frame() exposes the boundaries).
    With partial=True returns (bytes_before_error, exception_or_None) instead of raising."""
    src = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    parts, pos, err = [], 0, None
    while pos < src.size:
        out, used, err = decompress_next_frame(src[pos:], ctx)
        parts.append(out)
        if err is not None or used == 0:
            break
        pos += used
    joined = b"".join(parts)
    if partial:
        return joined, err
    if err is not None:
        raise err
    return joined


# -----------------------------------------------------------------------------------------------------
# FrameEncoder
# -----------------------------------------------------------------------------------------------------

class FrameEncoder:
    """frame::FrameEncoder<W> (compress.rs:62-404): a writer that LZ4-frame-compresses into `w`.

    Blocks are cut exactly where the reference cuts them; they are queued and compressed on the GPU in
    batches of up to `batch_bytes` of input (and at flush()/finish()), so the bytes arriving in `w` are
    identical to lz4_flex's, only later."""

    def __init__(self, w, frame_info: FrameInfo | None = None, ctx: _block.Context | None = None,
                 batch_bytes: int = 256 << 20):
        self.w = w
        self._info = frame_info or FrameInfo()
        if self._info.block_mode == BlockMode.Linked:
            raise LinkedBlocksUnsupported()
        self._ctx = ctx
        self._batch_bytes = batch_bytes
        self._src = bytearray()            # the reference's `src` buffer (one block being filled)
        self._queue: list[tuple[bytes, int]] = []   # (block, flags) not yet compressed
        self._queued_bytes = 0
        self._stream_offset = 0            # src_stream_offset (compress.rs:80)
        self._content_len = 0
        self._hasher = _Xxh32(0)
        self._is_frame_open = False
        self._data_to_frame_written = False

    # -- constructors with the reference's names -----------------------------------------------------
    @classmethod
    def new(cls, w, **kw) -> "FrameEncoder":
        return cls(w, FrameInfo(), **kw)

    @classmethod
    def with_frame_info(cls, frame_info: FrameInfo, w, **kw) -> "FrameEncoder":
        return cls(w, frame_info, **kw)

    def frame_info(self) -> FrameInfo:
        return self._info

    def get_ref(self):
        return self.w

    def get_mut(self):
        return self.w

    def into_inner(self):
        return self.w

    # -- io::Write -------------------------------------------------------------------------------------
    def write(self, buf) -> int:
        buf = bytes(buf)
        if not self._is_frame_open and buf:
            self._begin_frame(len(buf))
        bs = self._info.block_size.get_size() if self._info.block_size != BlockSize.Auto else 0
        view = memoryview(buf)
        while len(view):
            room = bs - len(self._src)
            if room == 0:
                self._write_block()
                continue
            take = min(room, len(view))
            self._src += view[:take]
            view = view[take:]
        return len(buf)

    def write_all(self, buf):
        self.write(buf)

    def flush(self):
        if self._src:
            self._write_block()
        self._drain()
        if hasattr(self.w, "flush"):
            try:
                self.w.flush()
            except Exception:
                pass

    def try_finish(self):
        """compress.rs:166-181"""
        if self._src:
            self._write_block()
        self._drain()
        if not self._is_frame_open and not self._data_to_frame_written:
            self._begin_frame(0)
        self._end_frame()
        self._data_to_frame_written = True

    def finish(self):
        self.try_finish()
        return self.w

    def auto_finish(self) -> "AutoFinishEncoder":
        return AutoFinishEncoder(self)

    # -- internals -----------------------------------------------------------------------------------
    def _begin_frame(self, buf_len: int):
        """compress.rs:234-258"""
        self._is_frame_open = True
        if self._info.block_size == BlockSize.Auto:
            self._info.block_size = BlockSize.from_buf_length(buf_len)
        self.w.write(self._info.header_bytes())
        if self._content_len != 0:
            self._content_len = 0
            self._stream_offset = 0
            self._src.clear()
            self._hasher = _Xxh32(0)

    def _end_frame(self):
        """compress.rs:209-230"""
        self._is_frame_open = False
        if self._info.content_size is not None and self._info.content_size != self._content_len:
            raise ContentLengthError(self._info.content_size, self._content_len)
        self.w.write(b"\0\0\0\0")
        if self._info.content_checksum:
            self.w.write(self._hasher.digest().to_bytes(4, "little"))

    def _write_block(self):
        """compress.rs:261-371, minus the compression itself (queued)."""
        bs = self._info.block_size.get_size()
        if self._stream_offset + bs + WINDOW_SIZE >= _REPOSITION_LIMIT:       # compress.rs:266-271
            self._stream_offset = 0
        flags = _block.BLOCK_HASH5_ALWAYS | (_block.BLOCK_CONT if self._stream_offset else _block.BLOCK_FRESH)
        blk = bytes(self._src)
        self._src.clear()
        self._queue.append((blk, flags))
        self._queued_bytes += len(blk)
        if self._info.content_checksum:
            self._hasher.update(blk)
        self._content_len += len(blk)
        self._stream_offset += len(blk)
        if self._queued_bytes >= self._batch_bytes:
            self._drain()

    def _drain(self):
        if not self._queue:
            return
        ctx = self._ctx or _block.default_context()
        blocks = [b for b, _ in self._queue]
        flags = [f for _, f in self._queue]
        comp = _block.compress_blocks(blocks, flags, ctx)
        out = bytearray()
        for raw, c in zip(blocks, comp):
            if len(c) < len(raw):                                            # compress.rs:301-306
                out += len(c).to_bytes(4, "little"); payload = c
            else:
                out += (len(raw) | 0x80000000).to_bytes(4, "little"); payload = raw
            out += payload
            if self._info.block_checksums:
                out += xxh32(payload).to_bytes(4, "little")
        self.w.write(bytes(out))
        self._queue.clear()
        self._queued_bytes = 0


class AutoFinishEncoder:
    """frame::AutoFinishEncoder (compress.rs:417-438): finishes the stream when the scope ends."""

    def __init__(self, enc: FrameEncoder):
        self.encoder = enc

    def write(self, buf) -> int:
        return self.encoder.write(buf)

    def flush(self):
        self.encoder.flush()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        if self.encoder is not None:
            try:
                self.encoder.try_finish()
            except Exception:
                if exc[0] is None:
                    raise
            self.encoder = None
        return False


# -----------------------------------------------------------------------------------------------------
# FrameDecoder
# -----------------------------------------------------------------------------------------------------

class FrameDecoder(io.RawIOBase):
    """frame::FrameDecoder<R> (decompress.rs:48-422): a reader that decompresses LZ4 frames from `r`.

    Streaming with bounded memory, like the reference's block-at-a-time reader, but a GROUP of blocks at a time so the
    GPU gets a batch: the header and the BlockInfo chain are read from `r` incrementally; blocks are collected until
    their decoded bound reaches `group_bytes` (default 64 MiB) and then decoded in one C-ABI call.  Only one group of
    compressed and decoded bytes is ever held.  (A frame with linked blocks is one dependency chain and is collected
    whole.)  As in the reference, read() returns b"" at every EndMark (decompress.rs:310-331): read_to_end() returns the
    rest of the CURRENT frame and the next call continues with the next frame (tests/tests.rs:633-647).  Bytes decoded
    before a corrupt block are delivered first; the error surfaces on the read that reaches it."""

    def __init__(self, r, ctx: _block.Context | None = None, group_bytes: int = 64 << 20):
        super().__init__()
        self.r = r
        self._ctx = ctx
        self._group_bytes = max(int(group_bytes), 1)
        self._ready = bytearray()          # decoded, not yet handed out
        self._err: Exception | None = None
        self._hdr: bytes | None = None     # header bytes of the frame being read (None: between frames)
        self._bs = 0
        self._flg = 0
        self._content = None               # streaming XXH32 of the frame's content (if the header asks for it)
        self._content_len = 0
        self._content_size = None
        self._eof = False                  # the underlying reader is exhausted
        self._frame_done = False           # an EndMark was consumed: the next read() returns b"" once

    @classmethod
    def new(cls, r, **kw) -> "FrameDecoder":
        return cls(r, **kw)

    def get_ref(self):
        return self.r

    def get_mut(self):
        return self.r

    def into_inner(self):
        return self.r

    def readable(self) -> bool:
        return True

    # ---- underlying reader ----------------------------------------------------------------------------
    def _read_upto(self, n: int) -> bytes:
        """read_exact that tolerates short reads; returns fewer bytes only at the end of the reader."""
        chunks, got = [], 0
        while got < n:
            c = self.r.read(n - got)
            if not c:
                break
            chunks.append(bytes(c))
            got += len(c)
        return b"".join(chunks)

    # ---- frame header: read_frame_info, decompress.rs:109-176 -------------------------------------------
    def _read_header(self) -> bool:
        """False = end of data where a frame would start."""
        magic = self._read_upto(4)
        if len(magic) == 0:
            return False
        if len(magic) < 4:
            raise IoError("unexpected end of input in the magic number")
        if magic == b"\x02\x21\x4c\x18":                                      # legacy frame, header.rs:285-291
            self._hdr, self._bs, self._flg = magic, 8 << 20, 0x20
        else:
            rest = self._read_upto(3)
            if len(rest) == 0:
                return False                                                   # decompress.rs:124-128
            if len(rest) < 3:
                raise IoError("unexpected end of input in the frame header")
            m = int.from_bytes(magic, "little")
            if 0x184D2A50 <= m <= 0x184D2A5F:
                raise error_from_status(111)
            if m != 0x184D2204:
                raise error_from_status(102)
            flg = rest[0]
            extra = (8 if flg & 0x08 else 0) + (4 if flg & 0x01 else 0)
            more = self._read_upto(extra)
            if len(more) < extra:
                raise IoError("unexpected end of input in the frame header")
            hdr = magic + rest + more
            # validate exactly like the C walk does: decode the header as an empty frame
            _, _, err = decompress_next_frame(hdr + b"\0\0\0\0" + (b"\0\0\0\0" if flg & 0x04 else b""), self._ctx)
            if err is not None and not isinstance(err, (ContentLengthError, ContentChecksumError)):
                raise err
            self._hdr, self._flg = hdr, flg
            self._bs = {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20}[(rest[1] >> 4) & 7]
            self._content_size = int.from_bytes(hdr[6:14], "little") if flg & 0x08 else None
        self._content = _Xxh32(0) if self._flg & 0x04 else None
        self._content_len = 0
        return True

    # ---- one group of blocks: read_block, decompress.rs:189-342 ------------------------------------------
    def _fill(self):
        """Decode the next group of blocks of the current frame into self._ready (may set self._err / _frame_done)."""
        if self._hdr is None:
            if self._eof or not self._read_header():
                self._eof = True
                return
        linked = not (self._flg & 0x20)
        has_bc = bool(self._flg & 0x10)
        body, bound, closed, end_err = [], 0, False, None
        while linked or bound < self._group_bytes or not body:
            w = self._read_upto(4)
            if len(w) < 4:                                                      # EOF where a BlockInfo is due: Ok(0)
                self._eof = True
                break
            word = int.from_bytes(w, "little")
            if word == 0:
                closed = True
                break
            ln = word & 0x7FFFFFFF
            if ln > self._bs:
                end_err = error_from_status(110)
                break
            payload = self._read_upto(ln + (4 if has_bc else 0))
            if len(payload) < ln + (4 if has_bc else 0):
                end_err = IoError("unexpected end of input inside a block")
                self._eof = True
                break
            body.append(w + payload)
            bound += ln if word & 0x80000000 else min(self._bs, 255 * ln + 16)
        if body:
            # the group as a frame of its own: same block size / block-checksum / linkage flags, no content size or checksum
            if len(self._hdr) == 4:                                             # legacy frame: magic + blocks, no EndMark
                group = self._hdr + b"".join(body)
            else:
                mini_hdr = bytes([(self._flg & 0x30) | 0x40, self._hdr[5]])
                group = (b"\x04\x22\x4d\x18" + mini_hdr + bytes([(xxh32(mini_hdr) >> 8) & 0xFF]) + b"".join(body)
                         + b"\0\0\0\0")
            out, _, err = decompress_next_frame(group, self._ctx)
            self._ready += out
            self._content_len += len(out)
            if self._content is not None:
                self._content.update(out)
            if err is not None:
                self._err = err
                self._hdr = None
                return
        if end_err is not None:
            self._err = end_err
            self._hdr = None
            return
        if closed:
            err = None
            if self._content_size is not None and self._content_len != self._content_size:
                err = ContentLengthError(self._content_size, self._content_len)                 # decompress.rs:312-321
            if self._flg & 0x04:
                c = self._read_upto(4)
                if len(c) < 4:
                    err = err or IoError("unexpected end of input in the content checksum")
                elif err is None and int.from_bytes(c, "little") != self._content.digest():
                    err = ContentChecksumError()
            self._hdr = None
            self._frame_done = True
            self._err = err
        elif self._eof:
            self._hdr = None

    def read(self, size: int = -1) -> bytes:
        want_all = size is None or size < 0
        while (want_all or len(self._ready) < size) and self._err is None and not self._frame_done:
            if self._eof and self._hdr is None:
                break
            self._fill()
        if self._ready:
            n = len(self._ready) if want_all else min(size, len(self._ready))
            out = bytes(self._ready[:n])
            del self._ready[:n]
            if want_all and self._err is not None:
                e, self._err = self._err, None
                self._frame_done = False
                raise _with_partial(e, out)
            if want_all:
                self._frame_done = False
            return out
        if self._err is not None:
            e, self._err = self._err, None
            self._frame_done = False
            raise e
        self._frame_done = False                                                # the b"" of this EndMark
        return b""

    def readinto(self, b) -> int:
        data = self.read(len(b))
        b[: len(data)] = data
        return len(data)

    def read_to_end(self) -> bytes:
        """Read::read_to_end: the rest of the current frame (empty at the end of the data)."""
        return self.read(-1)


def _with_partial(e: Exception, partial: bytes) -> Exception:
    """read(-1) that hits an error after delivering bytes: the bytes travel on the exception (`.partial`), like the
    Vec a failed read_to_end leaves filled in the reference."""
    try:
        e.partial = partial
    except Exception:
        pass
    return e
