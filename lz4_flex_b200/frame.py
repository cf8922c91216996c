"""lz4_flex::frame, H100 edition (encoder: independent-block mode; decoder: independent and linked blocks).

FrameInfo / BlockSize / BlockMode / FrameEncoder / FrameDecoder with the reference's names and behaviour
(src/frame/header.rs:39-192, src/frame/compress.rs:62-438, src/frame/decompress.rs:48-422).  The container
(header, BlockInfo words, checksums, end mark) is host bookkeeping; the blocks themselves are compressed
and decompressed in GPU batches through the C ABI.  Block boundaries, the stored-raw rule and — crucially —
each block's parse mode (FRESH for the first block of a table epoch, CONT afterwards, SURVEY.md §8a) follow
FrameEncoder::write/write_block exactly, so the produced frame is byte-identical to lz4_flex's.
For data already in GPU memory, compress_frame_device() and decompress_frame_device() keep the whole container on the
device: header, EndMark and both checksums are written or verified by kernels, and no payload crosses PCIe.

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
from .errors import (ContentChecksumError, ContentLengthError, DecompressionError, IoError, LinkedBlocksUnsupported,
                     error_from_status)

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


def compress_frame_device(d_in, frame_info: FrameInfo | None = None, out=None, ctx: _block.Context | None = None,
                          stream: int | None = None):
    """compress_frame() for input in device memory, through lz4b200_frame_compress_device: the frame is written to
    `out` (a contiguous 1-D torch CUDA uint8 tensor; None: one of lz4b200_frame_bound bytes is allocated) and the view
    of `out` that holds it is returned, byte-identical to what compress_frame() gives for the same bytes.  The work,
    checksums included, runs on torch's current stream (or `stream`); the call returns once the frame length has been
    read back.  Raises what compress_frame() raises for the same arguments."""
    import torch
    _device_u8(d_in, "d_in")
    ctx = ctx or _block.default_context()
    info = frame_info or FrameInfo()
    if info.block_mode == BlockMode.Linked:
        raise LinkedBlocksUnsupported()
    ci = info.to_c()
    n = d_in.numel()
    if out is None:
        out = torch.empty(_native.lib().lz4b200_frame_bound(n, C.byref(ci)), dtype=torch.uint8, device=d_in.device)
    _device_u8(out, "out")
    s = stream if stream is not None else torch.cuda.current_stream(d_in.device).cuda_stream
    written = torch.empty(1, dtype=torch.int64, device=out.device)
    st = _native.lib().lz4b200_frame_compress_device(ctx.handle, d_in.data_ptr() if n else None, n, C.byref(ci), n,
                                                     out.data_ptr(), out.numel(), written.data_ptr(), s)
    if st != 0:
        raise error_from_status(st, detail=ctx.last_cuda_error())
    if stream is None:
        w = int(written.item())
    else:
        with torch.cuda.stream(torch.cuda.ExternalStream(stream, device=out.device)):
            w = int(written.item())                                           # copied and synchronised on `stream`
    return out[:w]


def _host_i64(v, what: str) -> np.ndarray:
    if hasattr(v, "is_cuda"):
        v = v.cpu().numpy()
    a = np.ascontiguousarray(v, dtype=np.int64)
    if a.ndim != 1:
        raise TypeError(f"{what} must be 1-D")
    if a.size and a.min() < 0:
        raise ValueError(f"{what} must not be negative")
    return a


def compress_frames_device(d_in, offsets, lengths, frame_info: FrameInfo | None = None, out=None,
                           ctx: _block.Context | None = None, stream: int | None = None):
    """compress_frame() for each of many inputs in device memory, in one call (lz4b200_frame_compress_batch_device):
    input i is d_in[offsets[i]:offsets[i] + lengths[i]], and its frame is byte-identical to what compress_frame() gives
    for those bytes.  The frames are written back to back into `out` (a contiguous 1-D torch CUDA uint8 tensor; None:
    one of the summed lz4b200_frame_bound bytes is allocated).  offsets and lengths are int64 sequences or arrays (a
    CUDA tensor is copied to the host first).  frame_info is shared by every frame; BlockSize.Auto picks each frame's
    block size from its own length, and a non-None content_size means "each frame records its own length" (the value
    itself is ignored).  The work runs on torch's current stream (or `stream`); the call returns once the total length
    has been read back.  Returns (view of `out` that holds the frames, CUDA int64 tensor of len(offsets) + 1 frame
    offsets: frame i is out[frame_offsets[i]:frame_offsets[i + 1]]).  Raises what compress_frame() raises."""
    import torch
    _device_u8(d_in, "d_in")
    ctx = ctx or _block.default_context()
    info = frame_info or FrameInfo()
    if info.block_mode == BlockMode.Linked:
        raise LinkedBlocksUnsupported()
    offs, lens = _host_i64(offsets, "offsets"), _host_i64(lengths, "lengths")
    n = offs.size
    if lens.size != n:
        raise ValueError("offsets and lengths differ in length")
    if n and int((offs + lens).max()) > d_in.numel():
        raise ValueError("an input runs past the end of d_in")
    ci = info.to_c()
    if out is None:
        # the sum of lz4b200_frame_bound over the frames, each with its resolved block size
        if info.block_size == BlockSize.Auto:
            bs = np.where(lens > 256 << 10, 4 << 20, np.where(lens > 64 << 10, 256 << 10, 64 << 10))
        else:
            bs = np.full(n, info.block_size.get_size(), dtype=np.int64)
        total = int((27 + lens + 8 * ((lens + bs - 1) // bs)).sum()) if n else 0
        out = torch.empty(total, dtype=torch.uint8, device=d_in.device)
    _device_u8(out, "out")
    s = stream if stream is not None else torch.cuda.current_stream(d_in.device).cuda_stream
    frame_offsets = torch.empty(n + 1, dtype=torch.int64, device=out.device)
    st = _native.lib().lz4b200_frame_compress_batch_device(
        ctx.handle, d_in.data_ptr() if d_in.numel() else None, offs.ctypes.data, lens.ctypes.data, C.byref(ci),
        out.data_ptr() if out.numel() else None, out.numel(), frame_offsets.data_ptr(), n, s)
    if st != 0:
        raise error_from_status(st, detail=ctx.last_cuda_error())
    if stream is None:
        total = int(frame_offsets[n].item())
    else:
        with torch.cuda.stream(torch.cuda.ExternalStream(stream, device=out.device)):
            total = int(frame_offsets[n].item())                              # copied and synchronised on `stream`
    return out[:total], frame_offsets


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


def _device_u8(t, what: str):
    if not (t.is_cuda and t.dtype.itemsize == 1 and t.dim() == 1 and t.is_contiguous()):
        raise TypeError(f"{what} must be a contiguous 1-D torch CUDA uint8 tensor")


def decompress_next_frame_device(d_in, d_out, ctx: _block.Context | None = None, stream: int | None = None):
    """The frame that starts at d_in[0], decoded from device memory into d_out through
    lz4b200_frame_decompress_next_device: returns (consumed, written, exception or None), the same values
    decompress_next_frame() gives for the same bytes in host memory.  d_in and d_out are torch CUDA uint8 tensors;
    the work runs on torch's current stream (or `stream`) and the call returns once d_out holds the result.  Bytes
    of d_out past `written` are left untouched."""
    import torch
    _device_u8(d_in, "d_in")
    _device_u8(d_out, "d_out")
    ctx = ctx or _block.default_context()
    s = stream if stream is not None else torch.cuda.current_stream(d_in.device).cuda_stream
    n, cap = d_in.numel(), d_out.numel()
    used, w, bs = C.c_size_t(0), C.c_size_t(0), C.c_int(0)
    e1, e2 = C.c_uint64(0), C.c_uint64(0)
    st = _native.lib().lz4b200_frame_decompress_next_device(
        ctx.handle, d_in.data_ptr() if n else None, n, d_out.data_ptr() if cap else None, cap, C.byref(used),
        C.byref(w), C.byref(bs), C.byref(e1), C.byref(e2), s)
    err = None if st == 0 else error_from_status(st, bs.value, ctx.last_cuda_error(), e1.value, e2.value)
    return used.value, w.value, err


def decoded_bound_device(d_in, ctx: _block.Context | None = None, stream: int | None = None) -> int:
    """Upper bound of the decoded size of every concatenated frame in the device tensor d_in."""
    import torch
    _device_u8(d_in, "d_in")
    ctx = ctx or _block.default_context()
    s = stream if stream is not None else torch.cuda.current_stream(d_in.device).cuda_stream
    bound = C.c_size_t(0)
    st = _native.lib().lz4b200_frame_decoded_bound_device(ctx.handle, d_in.data_ptr() if d_in.numel() else None,
                                                          d_in.numel(), C.byref(bound), s)
    if st != 0:
        raise error_from_status(st, detail=ctx.last_cuda_error())
    return bound.value


def decompress_frame_device(d_in, out=None, ctx: _block.Context | None = None):
    """Every concatenated frame of the device tensor d_in, decoded on the GPU into `out` (a torch CUDA uint8 tensor;
    None: one of lz4b200_frame_decoded_bound_device bytes is allocated).  Returns the view of `out` that holds the
    decoded bytes.  Raises what decompress_frame() raises for the same bytes."""
    import torch
    _device_u8(d_in, "d_in")
    ctx = ctx or _block.default_context()
    if out is None:
        out = torch.empty(max(decoded_bound_device(d_in, ctx), 1), dtype=torch.uint8, device=d_in.device)
    _device_u8(out, "out")
    pos, total = 0, 0
    while pos < d_in.numel():
        used, w, err = decompress_next_frame_device(d_in[pos:], out[total:], ctx)
        total += w
        if err is not None:
            raise err
        if used == 0:
            break
        pos += used
    return out[:total]


def _device_i64(v, device, what: str):
    import torch
    t = v if isinstance(v, torch.Tensor) else torch.as_tensor(np.asarray(v, dtype=np.int64))
    t = t.to(device=device, dtype=torch.int64).contiguous()
    if t.dim() != 1:
        raise TypeError(f"{what} must be 1-D")
    return t


@dataclass
class DecodedFrames:
    """What decompress_frames_device() returns: the output buffer, each frame's output offset, and one row per frame
    of lz4b200_frame_result as int64 (consumed, written, err_expected, err_actual, status | block_status << 32)."""
    out: "object"
    out_offsets: "object"
    results: "object"
    _host: Optional[np.ndarray] = None

    def __len__(self) -> int:
        return self.results.shape[0]

    def frame(self, i: int):
        """(view of frame i's decoded bytes in `out`, consumed, exception or None): the values
        decompress_next_frame_device() gives for the same frame."""
        if self._host is None:
            self._host = self.results.cpu().numpy()
            self._offs = self.out_offsets.cpu().numpy()
        consumed, written, e1, e2, packed = (int(x) for x in self._host[i])
        st = int(np.int32(packed & 0xFFFFFFFF))
        bs = int(np.int32((packed >> 32) & 0xFFFFFFFF))
        err = None if st == 0 else error_from_status(st, bs, "", e1, e2)
        o = int(self._offs[i])
        return self.out[o:o + written], consumed, err

    def __iter__(self):
        return (self.frame(i) for i in range(len(self)))


def decompress_frames_device(d_in, offsets, lengths, out=None, out_offsets=None, out_caps=None,
                             ctx: _block.Context | None = None, stream: int | None = None) -> DecodedFrames:
    """Many independent frames in the device tensor d_in, decoded on the GPU in one call
    (lz4b200_frame_decompress_batch_device): frame i is the one that starts at d_in[offsets[i]] in a region of
    lengths[i] bytes, and is decoded into out[out_offsets[i]:] with room for out_caps[i] bytes.  With out=None each
    region gets lz4b200_frame_decoded_bound_batch_device bytes, laid out back to back.  d_in and out are contiguous
    1-D torch CUDA uint8 tensors; offsets, lengths and caps are int64 tensors or sequences.  The work runs on torch's
    current stream (or `stream`); the call returns once `out` holds the result.  Frame i's result is exactly what
    decompress_next_frame_device() returns for it: see DecodedFrames.frame()."""
    import torch
    _device_u8(d_in, "d_in")
    ctx = ctx or _block.default_context()
    dev = d_in.device
    s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
    offs, lens = _device_i64(offsets, dev, "offsets"), _device_i64(lengths, dev, "lengths")
    n = offs.numel()
    if lens.numel() != n:
        raise ValueError("offsets and lengths differ in length")
    if (out is None) != (out_offsets is None) or (out is None) != (out_caps is None):
        raise ValueError("out, out_offsets and out_caps go together")
    if out is not None:
        _device_u8(out, "out")
        oo, caps = _device_i64(out_offsets, dev, "out_offsets"), _device_i64(out_caps, dev, "out_caps")
        if oo.numel() != n or caps.numel() != n:
            raise ValueError("out_offsets and out_caps need one entry per frame")
    else:
        caps = torch.zeros(n, dtype=torch.int64, device=dev)
    results = torch.zeros((n, 5), dtype=torch.int64, device=dev)
    if stream is not None:
        torch.cuda.current_stream(dev).synchronize()                       # the tensors above were filled on torch's stream
    L = _native.lib()
    in_ptr = d_in.data_ptr() if d_in.numel() else None
    if out is None:
        st = L.lz4b200_frame_decoded_bound_batch_device(ctx.handle, in_ptr, offs.data_ptr(), lens.data_ptr(),
                                                        caps.data_ptr(), n, s)
        if st != 0:
            raise error_from_status(st, detail=ctx.last_cuda_error())
        with torch.cuda.stream(torch.cuda.ExternalStream(s, device=dev)):
            ends = torch.cumsum(caps, 0)
            oo = ends - caps
            total = int(ends[-1].item()) if n else 0
        out = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
    st = L.lz4b200_frame_decompress_batch_device(ctx.handle, in_ptr, offs.data_ptr(), lens.data_ptr(), out.data_ptr(),
                                                 oo.data_ptr(), caps.data_ptr(), results.data_ptr(), n, s)
    if st != 0:
        raise error_from_status(st, detail=ctx.last_cuda_error())
    return DecodedFrames(out, oo, results)


_CONTENT_CHECKSUM = 108


@dataclass
class FrameIndex:
    """What index_frame_device() returns for one frame: its result, and one row per block it covers as an int64 CUDA
    tensor of shape (nblocks, 3) holding lz4b200_frame_index_entry: payload offset, decoded offset, and the BlockInfo
    word | decoded length << 32.  Blocks are those before the first failing block; `error` is the exception
    decompress_next_frame_device() would raise for the frame, except that the content checksum is not verified."""
    consumed: int
    content_len: int
    nblocks: int
    block_size: int
    linked: bool
    error: Optional[Exception]
    entries: "object"
    _info: "object" = None

    def decoded_lengths(self):
        return self.entries[:, 2] >> 32 if self.nblocks else self.entries[:, 2]


def index_frame_device(d_in, ctx: _block.Context | None = None, stream: int | None = None) -> FrameIndex:
    """Indexes the frame that starts at the device tensor d_in[0] (lz4b200_frame_index_device): the decoded offset and
    length of every block, found on the GPU without decoding, for decompress_ranges_device()."""
    import torch
    _device_u8(d_in, "d_in")
    ctx = ctx or _block.default_context()
    s = stream if stream is not None else torch.cuda.current_stream(d_in.device).cuda_stream
    L = _native.lib()
    n = d_in.numel()
    ptr = d_in.data_ptr() if n else None
    count, info = C.c_size_t(0), _native.FrameIndexInfoC()
    st = L.lz4b200_frame_index_device(ctx.handle, ptr, n, None, 0, C.byref(count), None, s)
    if st != 0:
        raise error_from_status(st, detail=ctx.last_cuda_error())
    entries = torch.empty((max(count.value, 1), 3), dtype=torch.int64, device=d_in.device)
    st = L.lz4b200_frame_index_device(ctx.handle, ptr, n, entries.data_ptr(), count.value, C.byref(count),
                                      C.byref(info), s)
    if st != 0:
        raise error_from_status(st, detail=ctx.last_cuda_error())
    r = info.result
    err = None if r.status in (0, _CONTENT_CHECKSUM) else error_from_status(r.status, r.block_status, "", r.err_expected,
                                                                            r.err_actual)
    return FrameIndex(r.consumed, info.content_len, info.nblocks, info.block_size, bool(info.linked), err,
                      entries[:info.nblocks], info)


def decompress_ranges_device(d_in, index: FrameIndex, starts, lengths, out=None, out_offsets=None,
                             ctx: _block.Context | None = None, stream: int | None = None):
    """Content bytes [starts[i], starts[i] + lengths[i]) of the frame `index` describes, for every i, decoded from the
    device tensor d_in in one call (lz4b200_frame_decompress_ranges_device).  Ranges are clipped to index.content_len
    like Python slices.  Range i goes to out[out_offsets[i]:]; with out=None the ranges are laid back to back (lengths
    are read on the host to size `out`).  Only the blocks a range touches are decoded; a linked frame's ranges decode
    from a look-back of earlier blocks, doubled while a requested byte still copies content before it.  Returns (out,
    out_offsets, written): CUDA int64 tensors, written[i] the clipped length of range i.
    Raises InvalidArgument for an index that does not fit the bytes, and DecompressionError when a block does not decode
    to its indexed length."""
    import torch
    _device_u8(d_in, "d_in")
    ctx = ctx or _block.default_context()
    dev = d_in.device
    s = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
    st_t, ln_t = _device_i64(starts, dev, "starts"), _device_i64(lengths, dev, "lengths")
    nr = st_t.numel()
    if ln_t.numel() != nr:
        raise ValueError("starts and lengths differ in length")
    if (out is None) != (out_offsets is None):
        raise ValueError("out and out_offsets go together")
    if out is None:
        a, b = _host_i64(starts, "starts"), _host_i64(lengths, "lengths")
        c = index.content_len
        s0 = np.minimum(a, c)
        clipped = np.minimum(b, c - s0)
        ends = np.cumsum(clipped)
        oo = torch.as_tensor(ends - clipped, dtype=torch.int64).to(dev)
        out = torch.empty(max(int(ends[-1]) if nr else 0, 1), dtype=torch.uint8, device=dev)
    else:
        _device_u8(out, "out")
        oo = _device_i64(out_offsets, dev, "out_offsets")
        if oo.numel() != nr:
            raise ValueError("out_offsets needs one entry per range")
    written = torch.zeros(nr, dtype=torch.int64, device=dev)
    if stream is not None:
        torch.cuda.current_stream(dev).synchronize()                       # the tensors above were filled on torch's stream
    st = _native.lib().lz4b200_frame_decompress_ranges_device(
        ctx.handle, d_in.data_ptr() if d_in.numel() else None, d_in.numel(), C.byref(index._info),
        index.entries.data_ptr() if index.nblocks else None, st_t.data_ptr(), ln_t.data_ptr(), out.data_ptr(),
        oo.data_ptr(), written.data_ptr(), nr, s)
    if st == 101:
        raise DecompressionError(ValueError("a block does not decode to its indexed length"))
    if st != 0:
        raise error_from_status(st, detail=ctx.last_cuda_error())
    return out, oo, written


class DeviceFrameDecoder:
    """FrameDecoder over device memory (lz4b200_frame_decoder): decodes frames whose compressed bytes arrive in device
    memory chunk by chunk, into caller-sized output pieces, in device memory that does not grow with the frame (the
    context's frame budget and a 64 KiB window).  Linked frames included."""

    def __init__(self, ctx: _block.Context | None = None):
        self.ctx = ctx or _block.default_context()
        h = C.c_void_p()
        st = _native.lib().lz4b200_frame_decoder_create(self.ctx.handle, C.byref(h))
        if st != 0:
            raise error_from_status(st, detail=self.ctx.last_cuda_error())
        self._h = h

    def close(self):
        if self._h:
            _native.lib().lz4b200_frame_decoder_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def decode(self, d_in, d_out, end_of_input: bool = False, stream: int | None = None):
        """Continues the frame in progress with d_in (or starts one at d_in[0]) and decodes into d_out; both are
        contiguous 1-D torch CUDA uint8 tensors.  Returns (consumed, written, need, done, err): the whole units of d_in
        used, the bytes of d_out written, the bytes from d_in[consumed] the next unit needs when the call stopped for
        input (else 0), whether the frame ended, and then the exception decompress_next_frame_device() would raise for
        it (or None).  Present the unconsumed rest of d_in again with more bytes after it; set end_of_input when d_in
        runs to the end of the input.  Raises IoError when d_out cannot hold the next block (nothing is consumed).
        The work runs on torch's current stream (or `stream`) and the call returns once d_out holds the result."""
        import torch
        _device_u8(d_in, "d_in")
        _device_u8(d_out, "d_out")
        s = stream if stream is not None else torch.cuda.current_stream(d_in.device).cuda_stream
        n, cap = d_in.numel(), d_out.numel()
        step = _native.FrameDecoderStepC()
        st = _native.lib().lz4b200_frame_decoder_decode_device(self._h, d_in.data_ptr() if n else None, n,
                                                                1 if end_of_input else 0,
                                                                d_out.data_ptr() if cap else None, cap, C.byref(step), s)
        if st != 0:
            raise error_from_status(st, detail=self.ctx.last_cuda_error())
        r = step.result
        err = None
        if step.frame_done and r.status != 0:
            err = error_from_status(r.status, r.block_status, self.ctx.last_cuda_error(), r.err_expected, r.err_actual)
        return step.consumed, step.written, step.need, bool(step.frame_done), err


_ENCODE_WRITE, _ENCODE_FLUSH, _ENCODE_FINISH = 0, 1, 2
_CONTENT_LENGTH = 109


class DeviceFrameEncoder:
    """FrameEncoder over device memory (lz4b200_frame_encoder): compresses a stream that arrives in device memory in
    pieces into LZ4 frames in device memory, in device memory that does not grow with the stream (one group of blocks
    that fits the context's frame budget).  For any sequence of write / flush / finish calls, the concatenated bytes
    the calls return are what FrameEncoder writes for the same sequence of write_all / flush / try_finish."""

    def __init__(self, frame_info: FrameInfo | None = None, ctx: _block.Context | None = None):
        self.ctx = ctx or _block.default_context()
        self._h = None
        info = frame_info or FrameInfo()
        if info.block_mode == BlockMode.Linked:
            raise LinkedBlocksUnsupported()
        self._info = info
        ci = info.to_c()
        h = C.c_void_p()
        st = _native.lib().lz4b200_frame_encoder_create(self.ctx.handle, C.byref(ci), C.byref(h))
        if st != 0:
            raise error_from_status(st, detail=self.ctx.last_cuda_error())
        self._h = h

    def close(self):
        if self._h:
            _native.lib().lz4b200_frame_encoder_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    @staticmethod
    def _op(flush: bool, finish: bool) -> int:
        return _ENCODE_FINISH if finish else _ENCODE_FLUSH if flush else _ENCODE_WRITE

    def bound(self, n: int, flush: bool = False, finish: bool = False) -> int:
        """The most bytes write(n bytes, flush=, finish=) can return in the encoder's current state."""
        return _native.lib().lz4b200_frame_encoder_bound(self._h, n, self._op(flush, finish))

    def write(self, d_in, out=None, flush: bool = False, finish: bool = False, stream: int | None = None):
        """write_all(d_in), then flush() or try_finish(); d_in and out are contiguous 1-D torch CUDA uint8 tensors
        (out None: one of bound() bytes is allocated).  Returns the view of `out` that holds the bytes the call wrote.
        The work runs on torch's current stream (or `stream`); the call returns once that length has been read back, and
        d_in may be reused once the stream has passed the call.  A finish that finds a content length other than the
        FrameInfo's raises ContentLengthError(expected, actual) with the flushed bytes as `.partial`, and closes the
        frame without an EndMark, as FrameEncoder.try_finish() does."""
        import torch
        _device_u8(d_in, "d_in")
        op = self._op(flush, finish)
        n = d_in.numel()
        if out is None:
            out = torch.empty(self.bound(n, flush, finish), dtype=torch.uint8, device=d_in.device)
        _device_u8(out, "out")
        s = stream if stream is not None else torch.cuda.current_stream(d_in.device).cuda_stream
        written = torch.empty(1, dtype=torch.int64, device=out.device)
        cap = out.numel()
        st = _native.lib().lz4b200_frame_encoder_encode_device(self._h, d_in.data_ptr() if n else None, n, op,
                                                               out.data_ptr() if cap else None, cap, written.data_ptr(), s)
        if st != 0 and st != _CONTENT_LENGTH:
            raise error_from_status(st, detail=self.ctx.last_cuda_error())
        if stream is None:
            w = int(written.item())
        else:
            with torch.cuda.stream(torch.cuda.ExternalStream(stream, device=out.device)):
                w = int(written.item())                                       # copied and synchronised on `stream`
        if st == _CONTENT_LENGTH:
            actual = int(_native.lib().lz4b200_frame_encoder_content_len(self._h))
            raise _with_partial(ContentLengthError(self._info.content_size, actual), out[:w])
        return out[:w]

    def flush(self, out=None, stream: int | None = None):
        """flush(): compresses what is buffered; returns the bytes written."""
        return self.write(self._empty(), out=out, flush=True, stream=stream)

    def finish(self, out=None, stream: int | None = None):
        """try_finish(): flushes and closes the frame (an empty frame when nothing was written); a later write opens the
        next frame.  Returns the bytes written."""
        return self.write(self._empty(), out=out, finish=True, stream=stream)

    def _empty(self):
        import torch
        return torch.empty(0, dtype=torch.uint8, device=torch.device("cuda", self.ctx.device))


def iter_decompress_device(read_into, out_bytes: int = 8 << 20, in_bytes: int = 16 << 20, ctx: _block.Context | None = None,
                           device=None):
    """Every concatenated frame of a compressed stream that arrives in device memory, decoded in bounded device memory.
    read_into(buf) writes the next compressed bytes to the start of the device tensor `buf` and returns how many (0 at
    the end of the input).  Yields (view, frame_done): views of an output buffer of out_bytes (at least the frames'
    block size: 8 MiB covers every frame), each valid until the next item is taken; frame_done marks a frame's last
    piece.  Raises what decompress_frame_device() raises, after yielding the bytes decoded before the error.  Compressed
    units must fit in_bytes (a 4 MiB block takes 4 MiB + 8 bytes)."""
    import torch
    dec = DeviceFrameDecoder(ctx)
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    buf = torch.empty(in_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(out_bytes, dtype=torch.uint8, device=dev)
    pos, have, eof = 0, 0, False
    try:
        while True:
            if not eof and (pos or have < in_bytes):
                if pos:
                    buf[:have - pos] = buf[pos:have].clone()
                    have, pos = have - pos, 0
                got = int(read_into(buf[have:]))
                eof = got == 0
                have += got
            consumed, written, need, done, err = dec.decode(buf[pos:have], out, end_of_input=eof)
            if done and consumed == 0 and written == 0 and err is None:
                return                                                     # end of data: nothing left to decode
            if written or done:
                yield out[:written], done
            if err is not None:
                raise err
            pos += consumed
            if need and pos == 0 and have == in_bytes:
                raise ValueError(f"a compressed unit of {need} bytes does not fit in_bytes={in_bytes}")
    finally:
        dec.close()


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
