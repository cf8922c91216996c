"""Random access into frames in device memory: the block index (lz4b200_frame_index_device) and the range decoder
(lz4b200_frame_decompress_ranges_device), against the one-frame device decoder and the oracle.

The index's result must be the device decoder's for the same bytes in every field (its content checksum aside, which
the index never verifies), its per-block decoded lengths the oracle's, and its sizing walk must fail exactly where the
block decoder fails: hand-built frames from test_gpu_linked_adversarial.py (offsets that reach frame byte 0 and one
byte further, OffsetOutOfBounds before OutputTooSmall, ...) and the reference's decoder known answers.  Ranges are
checked against slices of the oracle's whole-frame decode, with sentinel bytes around every output region."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import vectors
from lz4_flex_b200 import _native, block, corpus, errors, frame
from stream_frames import broken_frames, valid_frames
from test_gpu_launch_shapes import seq
from test_gpu_linked_adversarial import all_cases

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
CONTENT_CHECKSUM = 108


def device_next(ctx, f: bytes):
    """lz4b200_frame_decompress_next_device with a sufficient cap: (status, consumed, written, block_status,
    err_expected, err_actual, bytes)."""
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda") if f else torch.empty(0, dtype=torch.uint8,
                                                                                                 device="cuda")
    cap = max(frame.decoded_bound_device(d_in, ctx), 1)
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    used, w, bs, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_uint64(0), C.c_uint64(0)
    s = torch.cuda.current_stream().cuda_stream
    st = _native.lib().lz4b200_frame_decompress_next_device(
        ctx.handle, d_in.data_ptr() if f else None, len(f), out.data_ptr(), cap, C.byref(used), C.byref(w),
        C.byref(bs), C.byref(e1), C.byref(e2), s)
    return st, used.value, w.value, bs.value, e1.value, e2.value, out[:w.value].cpu().numpy().tobytes()


def check_index(ctx, f: bytes, name: str):
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda") if f else torch.empty(0, dtype=torch.uint8,
                                                                                                 device="cuda")
    idx = frame.index_frame_device(d_in, ctx)
    st, used, w, bst, e1, e2, data = device_next(ctx, f)
    r = idx._info.result
    want = 0 if st == CONTENT_CHECKSUM else st
    assert (r.status, r.consumed, r.written, r.block_status, r.err_expected, r.err_actual) == \
        (want, used, w, bst, e1, e2), name
    assert idx.content_len == w, name
    ent = idx.entries.cpu().numpy()
    lens = (ent[:, 2] >> 32).astype(np.int64) if idx.nblocks else np.zeros(0, np.int64)
    assert int(lens.sum()) == w, name
    assert (ent[:, 1] == np.concatenate([[0], np.cumsum(lens)[:-1]])).all() if idx.nblocks else True, name
    return idx, d_in, data


def oracle_block_lengths(f: bytes, idx, content: bytes):
    """Each indexed block's decoded length by the oracle: stored blocks their payload, compressed blocks decoded alone
    (independent) or with the last 64 KiB of content before them as dictionary (linked)."""
    out, pos = [], 0
    for off, _, word in idx.entries.cpu().numpy():
        word = int(word) & 0xFFFFFFFF
        payload = f[int(off):int(off) + (word & 0x7FFFFFFF)]
        if word & 0x80000000:
            n = len(payload)
        elif idx.linked:
            st, b, _, _ = oracle.decompress_with_dict(payload, idx.block_size, content[max(0, pos - 65536):pos])
            assert st == 0
            n = len(b)
        else:
            st, b, _, _ = oracle.decompress_block(payload, idx.block_size)
            assert st == 0
            n = len(b)
        out.append(n)
        pos += n
    return out


@pytest.fixture(scope="module")
def valid():
    return valid_frames()


def test_index_matches_device_decoder_on_valid_frames(ctx, valid):
    for name, f in valid:
        idx, _, data = check_index(ctx, f, name)
        assert idx.error is None, name
        got = [int(x) for x in idx.decoded_lengths().cpu()]
        assert got == oracle_block_lengths(f, idx, data), name


def test_index_matches_device_decoder_on_broken_frames(ctx):
    for name, f in broken_frames():
        check_index(ctx, f, name)


def test_sizing_walk_fails_where_the_decoder_fails(ctx):
    """Linked frames built from explicit sequences (every DecompressError, offsets that reach frame byte 0 exactly and
    one byte further, OffsetOutOfBounds before OutputTooSmall) and the reference's decoder known answers as the one
    block of an independent frame, plus a block that decodes to the block size + 1."""
    hand, rnd = all_cases()
    for c in hand + rnd[:400]:
        check_index(ctx, c.frame, c.name)
    hdr = bytes([0x60, 0x40])
    head = b"\x04\x22\x4d\x18" + hdr + bytes([(frame.xxh32(hdr) >> 8) & 0xFF])
    streams = [bytes(s) for _, s, *_ in vectors.DECODE_KATS] + [seq(b"x" * 65537), seq(b"ab", 1, 65535),
                                                               seq(b"ab", 1, 65534), seq(b"ab", 3, 4)]
    for s in streams:
        f = head + len(s).to_bytes(4, "little") + s + bytes(4)
        check_index(ctx, f, repr(s[:8]))


def _edges(idx):
    """(start, length) pairs on the edges: the whole content, inside one block, on block boundaries, across stored,
    short and empty blocks, empty ranges, and ranges that start at or past the end or run past it."""
    c = idx.content_len
    ent = idx.entries.cpu().numpy()
    offs = [int(x) for x in ent[:, 1]]
    lens = [int(x) for x in ent[:, 2] >> 32]
    r = [(0, c), (0, c + 10), (c, 5), (c + 7, 3), (0, 0), (c // 2, 0), (max(c - 1, 0), 100)]
    for k in range(len(offs)):
        d, L = offs[k], lens[k]
        r += [(d, L), (d, 1), (d + L // 3, L // 3), (max(d - 1, 0), 2), (d + L, 0)]
        if k + 2 < len(offs):
            r.append((d + L // 2, lens[k + 1] + L))
        if len(r) > 600:
            break
    return r


def run_ranges(ctx, d_in, idx, ranges, content: bytes, gap: int = 3):
    """Decode `ranges` into one buffer with `gap` sentinel bytes around every region and check each region against
    content[s:s + l] and every sentinel against SENTINEL."""
    st = np.array([a for a, _ in ranges], dtype=np.int64)
    ln = np.array([b for _, b in ranges], dtype=np.int64)
    c = idx.content_len
    clip = np.minimum(ln, c - np.minimum(st, c))
    oo = np.cumsum(clip + gap) - clip
    out = torch.full((int(oo[-1] + clip[-1] + gap),), SENTINEL, dtype=torch.uint8, device="cuda")
    _, _, written = frame.decompress_ranges_device(d_in, idx, st, ln, out=out, out_offsets=oo, ctx=ctx)
    assert (written.cpu().numpy() == clip).all()
    h = out.cpu().numpy()
    mask = np.ones(h.size, dtype=bool)
    for i, (a, _) in enumerate(ranges):
        o, n = int(oo[i]), int(clip[i])
        assert h[o:o + n].tobytes() == content[a:a + n], (i, a, n)
        mask[o:o + n] = False
    assert (h[mask] == SENTINEL).all()


def test_ranges_on_every_valid_frame(ctx, valid):
    rng = np.random.default_rng(7)
    for name, f in valid:
        idx, d_in, data = check_index(ctx, f, name)
        c = idx.content_len
        assert data == oracle.frame_decompress(f, c + 1)[1], name
        ranges = _edges(idx) + [(int(rng.integers(0, c + 1)), int(rng.integers(0, 300000))) for _ in range(200)]
        run_ranges(ctx, d_in, idx, ranges, data)


def test_default_layout(ctx):
    data = corpus.tiled("compression_66k_JSON.txt", 500000).tobytes()
    f = oracle.frame_compress(data, 4, 7, 3000)
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    idx = frame.index_frame_device(d_in, ctx)
    starts, lens = [0, 70000, 499990, 600000, 10], [10, 200000, 100, 5, 0]
    out, oo, written = frame.decompress_ranges_device(d_in, idx, starts, lens, ctx=ctx)
    h, oo = out.cpu().numpy(), oo.cpu().numpy()
    for i, (a, n) in enumerate(zip(starts, lens)):
        w = int(written[i])
        assert w == len(data[a:a + n])
        assert h[oo[i]:oo[i] + w].tobytes() == data[a:a + n]


def test_frames_with_a_failing_block(ctx):
    """Ranges are served up to content_len, the output before the first failing block, and clipped there."""
    served = 0
    for name, f in broken_frames():
        idx, d_in, data = check_index(ctx, f, name)
        if idx.error is None or idx.content_len == 0:
            continue
        c = idx.content_len
        run_ranges(ctx, d_in, idx, [(0, c + 100), (c // 3, c), (c, 10), (max(c - 5, 0), 5)], data)
        served += 1
    assert served >= 5


def test_budget(ctx):
    """At a 1 MiB frame budget, 4 MiB blocks and 1 000 ranges decode the same, and the range call's scratch stays
    within one block's slot (a window holds at least one block) and a small fixed part."""
    data = corpus.tiled("hdfs.json", (12 << 20) + 12345).tobytes()
    f = oracle.frame_compress(data, 7, 0)
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    small = block.Context()
    try:
        _native.lib().lz4b200_ctx_set_frame_budget(small.handle, 1 << 20)
        idx = frame.index_frame_device(d_in, small)
        before = _native.lib().lz4b200_ctx_device_bytes(small.handle)
        rng = np.random.default_rng(3)
        ranges = [(int(rng.integers(0, len(data))), int(rng.integers(0, 1 << 16))) for _ in range(1000)]
        run_ranges(small, d_in, idx, ranges, data)
        grown = _native.lib().lz4b200_ctx_device_bytes(small.handle) - before
        assert grown <= (4 << 20) * 9 // 8 + (2 << 20), grown
    finally:
        small.close()


@pytest.mark.parametrize("which", ["json 64k", "hdfs 4m"])
def test_scale(ctx, which):
    """10 000 random ranges in one call against slices of the source: a 1 GiB frame of 64 KiB JSON blocks, and a frame
    of 4 MiB hdfs blocks."""
    if which == "json 64k":
        src = torch.tensor(corpus.tiled("compression_66k_JSON.txt", 1 << 30), device="cuda")
        info = frame.FrameInfo(block_size=frame.BlockSize.Max64KB)
    else:
        src = torch.tensor(corpus.tiled("hdfs.json", 256 << 20), device="cuda")
        info = frame.FrameInfo(block_size=frame.BlockSize.Max4MB)
    f = frame.compress_frame_device(src, info, ctx=ctx)
    idx = frame.index_frame_device(f, ctx)
    assert idx.error is None and idx.content_len == src.numel()
    rng = np.random.default_rng(11)
    n = src.numel()
    st = rng.integers(0, n, 10000)
    ln = np.where(rng.random(10000) < 0.5, rng.integers(0, 4096, 10000), rng.integers(0, 1 << 20, 10000))
    out, oo, written = frame.decompress_ranges_device(f, idx, st, ln, ctx=ctx)
    clip = np.minimum(ln, n - st)
    assert (written.cpu().numpy() == clip).all()
    # each range against the source, compared on the device in one gather
    total = int(clip.sum())
    within = np.arange(total) - np.repeat(np.cumsum(clip) - clip, clip)
    pos_out = torch.as_tensor(np.repeat(oo.cpu().numpy(), clip) + within, device="cuda")
    pos_src = torch.as_tensor(np.repeat(st, clip) + within, device="cuda")
    assert torch.equal(out[pos_out], src[pos_src])


def test_bad_index_and_changed_bytes(ctx):
    """A truncated, edited or foreign index, and bytes changed after indexing: a status, never a fault.  Each case runs
    once."""
    data = corpus.tiled("compression_66k_JSON.txt", 400000).tobytes()
    f = oracle.frame_compress(data, 4, 0)
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    idx = frame.index_frame_device(d_in, ctx)
    ranges = ([0, 1000, 390000], [400000, 5000, 100])

    def call(d, ix):
        return frame.decompress_ranges_device(d, ix, *ranges, ctx=ctx)

    call(d_in, idx)
    # truncated: fewer entries than the info says cover the content
    t = frame.FrameIndex(**{**idx.__dict__, "entries": idx.entries[:-1].clone()})
    t._info = _native.FrameIndexInfoC.from_buffer_copy(idx._info)
    t._info.nblocks = idx.nblocks - 1
    with pytest.raises(ValueError):
        call(d_in, t)
    # edited: a decoded length, a payload offset past the input, a block size
    for col, delta in ((2, 1 << 32), (0, len(f)), (1, 7)):
        e = frame.FrameIndex(**{**idx.__dict__, "entries": idx.entries.clone()})
        e._info = idx._info
        e.entries[3, col] += delta
        with pytest.raises(ValueError):
            call(d_in, e)
    b = frame.FrameIndex(**idx.__dict__)
    b._info = _native.FrameIndexInfoC.from_buffer_copy(idx._info)
    b._info.block_size = 12345
    with pytest.raises(ValueError):
        call(d_in, b)
    # foreign: the index of another frame with the same block size
    g = oracle.frame_compress(corpus.load("dickens.txt")[:400000], 4, 0)
    other = frame.index_frame_device(torch.tensor(np.frombuffer(g, dtype=np.uint8), device="cuda"), ctx)
    with pytest.raises((ValueError, errors.DecompressionError)):
        call(d_in, other)
    # changed bytes: a compressed block's payload zeroed after indexing
    ent = idx.entries.cpu().numpy()
    k = next(i for i in range(idx.nblocks) if not int(ent[i, 2]) & 0x80000000)
    off, ln = int(ent[k, 0]), int(ent[k, 2]) & 0x7FFFFFFF
    z = d_in.clone()
    z[off:off + ln] = 0
    with pytest.raises(errors.DecompressionError):
        frame.decompress_ranges_device(z, idx, [int(ent[k, 1])], [10], ctx=ctx)
