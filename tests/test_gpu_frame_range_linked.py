"""Random access into linked frames in device memory: lz4b200_frame_decompress_ranges_device marker-decodes the
blocks a range needs from a bounded look-back instead of decoding from the frame's first block.

Every range is checked against slices of the oracle's whole-frame decode with sentinel bytes around every output
region, and lz4b200_ctx_last_range_blocks against the block decodes of the CPU model in test_linked_marker_model.py."""

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, block, corpus, errors, frame
from stream_frames import linked_frame
from test_gpu_frame_range_device import SENTINEL, _edges, check_index, run_ranges
from test_gpu_linked_adversarial import all_cases
from test_linked_marker_model import decode_ranges, golden_frames, model_frames

pytestmark = pytest.mark.gpu

MiB = 1 << 20


def last_blocks(ctx):
    return _native.lib().lz4b200_ctx_last_range_blocks(ctx.handle)


def entries_of(idx):
    """The index as the model takes it: (payload_off, decoded_off, word, decoded_len) per block."""
    e = idx.entries.cpu().numpy()
    return [(int(a), int(b), int(w) & 0xFFFFFFFF, int(w) >> 32) for a, b, w in e]


def counts_match(ctx, f, d_in, idx, ranges, content):
    _, decodes, _ = decode_ranges(f, entries_of(idx), ranges, idx.content_len)
    run_ranges(ctx, d_in, idx, ranges, content)
    if idx.linked:                                     # one golden frame of one block is flagged independent
        assert last_blocks(ctx) == decodes
    return decodes


@pytest.fixture(scope="module")
def frames():
    return golden_frames() + model_frames()


def test_ranges_against_the_oracle(ctx, frames):
    rng = np.random.default_rng(17)
    for name, f in frames:
        idx, d_in, data = check_index(ctx, f, name)
        assert idx.error is None, name
        c = idx.content_len
        assert data == oracle.frame_decompress(f, c + 1)[1], name
        ranges = _edges(idx) + [(int(rng.integers(0, c + 1)), int(rng.integers(0, 300000))) for _ in range(100)]
        counts_match(ctx, f, d_in, idx, ranges, data)


def test_block_counts_match_the_model(ctx, frames):
    """One 4 KiB range at the start, the middle and the end of every frame, one call each."""
    for name, f in frames:
        idx, d_in, data = check_index(ctx, f, name)
        c = idx.content_len
        for where in (0, c // 2, max(c - 4096, 0)):
            counts_match(ctx, f, d_in, idx, [(where, 4096)], data)


def test_separated_ranges_count_as_the_model(ctx):
    """Two 4 KiB ranges in blocks far apart need different look-backs: the one that resolves first stops, and the
    other's doubled look-back, which then covers the first one's blocks, is not sent further back by the first one's
    bytes.  2 MiB of dickens in 64 KiB blocks, one call per pair of blocks."""
    src = corpus.load("dickens.txt")[:2 * MiB]
    f = linked_frame(src, [65536])
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    idx = frame.index_frame_device(d_in, ctx)
    assert idx.error is None
    for b1, b2 in ((2, 9), (1, 12), (4, 7), (5, 20), (3, 30), (10, 25), (0, 31)):
        ranges = [(b1 * 65536 + 30000, 4096), (b2 * 65536 + 30000, 4096)]
        counts_match(ctx, f, d_in, idx, ranges, src)


@pytest.mark.parametrize("which", ["dickens", "json"])
def test_64_mib_frames(ctx, which):
    """A 4 KiB range in the last block of a 64 MiB linked frame of 64 KiB blocks.  On dickens the look-back stays a few
    blocks, as the model counts; the hdfs JSON log copies itself from block to block and its look-back reaches block 0.
    Either way the bytes are exact."""
    src = corpus.tiled("dickens.txt" if which == "dickens" else "hdfs.json", 64 * MiB).tobytes()
    f = linked_frame(src, [65536])
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    idx = frame.index_frame_device(d_in, ctx)
    assert idx.error is None and idx.content_len == len(src)
    if which == "dickens":
        assert counts_match(ctx, f, d_in, idx, [(len(src) - 5000, 4096)], src) <= 16
    else:                                              # the model would decode ~2 000 blocks in Python: no model here
        run_ranges(ctx, d_in, idx, [(len(src) - 5000, 4096)], src)
        assert last_blocks(ctx) >= idx.nblocks


def test_frames_with_a_failing_block(ctx):
    """Linked frames with a failing block (every DecompressError, OffsetOutOfBounds at content byte 0, a bad
    checksum): ranges are clipped to the indexed content and equal the oracle's bytes before the first failing
    block."""
    hand, rnd = all_cases()
    served = 0
    for c in hand + rnd[:300]:
        idx, d_in, _ = check_index(ctx, c.frame, c.name)
        if not idx.linked or idx.content_len == 0:
            continue
        n = idx.content_len
        assert len(c.data) >= n, c.name
        run_ranges(ctx, d_in, idx, [(0, n + 100), (n // 3, n), (n, 10), (max(n - 5, 0), 5)], c.data)
        served += 1
    assert served >= 20


def _frame(blocks, flg=0x40, bsid=4):
    """A linked frame of the given (word, payload) blocks."""
    hdr = bytes([flg, bsid << 4])
    parts = [b"\x04\x22\x4d\x18", hdr, bytes([(frame.xxh32(hdr) >> 8) & 0xFF])]
    for word, payload in blocks:
        parts.append(word.to_bytes(4, "little") + payload)
    parts.append(bytes(4))
    return b"".join(parts)


def _forged(idx, entries, content_len):
    e = frame.FrameIndex(**{**idx.__dict__, "entries": torch.tensor(entries, dtype=torch.int64, device="cuda")})
    e._info = _native.FrameIndexInfoC.from_buffer_copy(idx._info)
    e._info.nblocks = len(entries)
    e._info.content_len = content_len
    return e


def _call_with_sentinels(ctx, d_in, ix, starts, lens):
    """The call into sentinel-filled output; returns the error raised (or None) and whether only the range regions
    were written."""
    total = sum(lens) + 8 * len(lens) + 8
    out = torch.full((total,), SENTINEL, dtype=torch.uint8, device="cuda")
    oo = np.cumsum([8] + [ln + 8 for ln in lens[:-1]])
    err = None
    try:
        frame.decompress_ranges_device(d_in, ix, starts, lens, out=out, out_offsets=oo, ctx=ctx)
    except (ValueError, errors.DecompressionError) as e:
        err = e
    h = out.cpu().numpy()
    mask = np.ones(total, dtype=bool)
    for o, ln in zip(oo, lens):
        mask[o:o + ln] = False
    return err, bool((h[mask] == SENTINEL).all())


def test_untrusted_index(ctx):
    """Edited decoded offsets and lengths, a foreign index, bytes changed after indexing, and a forged entry whose
    block copies from before content byte 0: a status, and nothing outside the range regions written."""
    data = corpus.load("dickens.txt")[:400000]
    f = linked_frame(data, [65536])
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    idx = frame.index_frame_device(d_in, ctx)
    starts, lens = [0, 140000, 390000], [5000, 4096, 10000]
    assert _call_with_sentinels(ctx, d_in, idx, starts, lens) == (None, True)
    ent = idx.entries.cpu().numpy()
    for row, col, delta in ((3, 2, 1 << 32), (3, 1, 7), (2, 2, -(1 << 32)), (5, 1, -1)):
        e = ent.copy()
        e[row, col] += delta
        err, clean = _call_with_sentinels(ctx, d_in, _forged(idx, e.tolist(), idx.content_len), starts, lens)
        assert isinstance(err, ValueError) and clean, (row, col)
    # lengths moved between two blocks, offsets kept consistent: the blocks decode to other lengths
    e = ent.copy()
    e[2, 2] -= 1000 << 32
    e[6, 2] += 1000 << 32
    e[3:, 1] -= 1000
    err, clean = _call_with_sentinels(ctx, d_in, _forged(idx, e.tolist(), idx.content_len), starts, lens)
    assert isinstance(err, errors.DecompressionError) and clean
    g = linked_frame(corpus.load("compression_66k_JSON.txt") * 6, [65536])
    other = frame.index_frame_device(torch.tensor(np.frombuffer(g, dtype=np.uint8), device="cuda"), ctx)
    err, clean = _call_with_sentinels(ctx, d_in, other, starts, lens)
    assert err is not None and clean
    k = next(i for i in range(idx.nblocks) if i > 2 and not int(ent[i, 2]) & 0x80000000)
    z = d_in.clone()
    z[int(ent[k, 0]) + 10:int(ent[k, 0]) + 400] = 0
    err, clean = _call_with_sentinels(ctx, z, idx, [int(ent[k, 1])], [100])
    assert isinstance(err, errors.DecompressionError) and clean
    # block 1 copies 4 bytes from 11 back, one byte before content byte 0: the index stops before it; a forged
    # entry for it must fail in the range decoder, not read before its entries
    h = _frame([(10 | 0x80000000, b"0123456789"), (5, bytes([0x00, 11, 0, 0x10]) + b"Z")])
    d_h = torch.tensor(np.frombuffer(h, dtype=np.uint8), device="cuda")
    hidx = frame.index_frame_device(d_h, ctx)
    assert hidx.nblocks == 1 and hidx.content_len == 10 and hidx.error is not None
    forged = _forged(hidx, [[11, 0, 10 | 0x80000000 | (10 << 32)], [25, 10, 5 | (5 << 32)]], 15)
    forged._info.result.status = 0
    for starts, lens in (([10], [5]), ([12], [3]), ([0], [15])):
        err, clean = _call_with_sentinels(ctx, d_h, forged, starts, lens)
        assert isinstance(err, errors.DecompressionError) and clean, starts


def test_budget(ctx):
    """At a 1 MiB frame budget, a 64 MiB linked frame of 4 MiB blocks decodes the same, each window one block (segments
    carry their last 64 KiB from window to window), and the call's scratch stays within test_budget's bound for the
    independent path with four bytes of entry per content byte: one block's entries, its 64 KiB of carry, and a small
    fixed part."""
    data = corpus.tiled("hdfs.json", 64 * MiB - 12345).tobytes()
    f = linked_frame(data, [4 * MiB], bsid=7)
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    small = block.Context()
    try:
        _native.lib().lz4b200_ctx_set_frame_budget(small.handle, 1 << 20)
        idx = frame.index_frame_device(d_in, small)
        before = _native.lib().lz4b200_ctx_device_bytes(small.handle)
        rng = np.random.default_rng(3)
        ranges = [(int(rng.integers(0, len(data))), int(rng.integers(0, 1 << 16))) for _ in range(300)]
        ranges += [(10 * MiB - 100, 9 * MiB), (len(data) - 4096, 4096)]
        _, decodes, _ = decode_ranges(f, entries_of(idx), ranges, idx.content_len)
        run_ranges(small, d_in, idx, ranges, data)
        assert last_blocks(small) == decodes
        grown = _native.lib().lz4b200_ctx_device_bytes(small.handle) - before
        assert grown <= 4 * ((4 << 20) * 9 // 8) + (2 << 20), grown
    finally:
        small.close()


def test_scale(ctx):
    """10 000 random 4 KiB ranges over a 256 MiB linked frame of 64 KiB JSON blocks, against the source."""
    src = corpus.tiled("compression_66k_JSON.txt", 256 * MiB)
    f = linked_frame(src.tobytes(), [65536])
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    idx = frame.index_frame_device(d_in, ctx)
    assert idx.error is None and idx.content_len == src.size
    rng = np.random.default_rng(11)
    n = src.size
    st = rng.integers(0, n, 10000)
    ln = rng.integers(0, 4097, 10000)
    out, oo, written = frame.decompress_ranges_device(d_in, idx, st, ln, ctx=ctx)
    clip = np.minimum(ln, n - st)
    assert (written.cpu().numpy() == clip).all()
    total = int(clip.sum())
    within = np.arange(total) - np.repeat(np.cumsum(clip) - clip, clip)
    d_src = torch.tensor(src, device="cuda")
    pos_out = torch.as_tensor(np.repeat(oo.cpu().numpy(), clip) + within, device="cuda")
    pos_src = torch.as_tensor(np.repeat(st, clip) + within, device="cuda")
    assert torch.equal(out[pos_out], d_src[pos_src])
    assert last_blocks(ctx) >= idx.nblocks             # tiled JSON copies itself: look-backs reach block 0


def test_teardown_frees_the_entries(ctx):
    """The entry window is context scratch: counted by lz4b200_ctx_device_bytes while the context lives, and returned to
    the device when it is destroyed."""
    data = corpus.tiled("dickens.txt", 96 * MiB).tobytes()
    f = linked_frame(data, [4 * MiB], bsid=7)
    d_in = torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    c = block.Context()
    idx = frame.index_frame_device(d_in, c)
    before = _native.lib().lz4b200_ctx_device_bytes(c.handle)
    out = torch.empty(64 * MiB, dtype=torch.uint8, device="cuda")
    frame.decompress_ranges_device(d_in, idx, [0], [64 * MiB], out=out, out_offsets=[0], ctx=c)
    assert torch.equal(out.cpu(), torch.frombuffer(bytearray(data[:64 * MiB]), dtype=torch.uint8))
    grown = _native.lib().lz4b200_ctx_device_bytes(c.handle) - before
    assert grown >= 4 * 48 * MiB, grown                 # the entries of a window of the 64 MiB the range spans
    del idx, out
    c.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert torch.cuda.mem_get_info()[0] >= free0 - 64 * MiB
