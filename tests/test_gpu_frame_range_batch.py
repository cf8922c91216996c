"""Random access into many frames in device memory per call: the batch index (lz4b200_frame_index_batch_device) against
the one-frame index of every region, and the batch range decoder (lz4b200_frame_decompress_ranges_batch_device)
against the oracle and the one-frame range call on every frame, with sentinel bytes around every output region."""

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, block, corpus, errors, frame
from stream_frames import broken_frames, linked_frame, valid_frames
from test_gpu_frame_range_device import SENTINEL, _edges
from test_gpu_linked_adversarial import all_cases

pytestmark = pytest.mark.gpu

MiB = 1 << 20


def last_blocks(ctx):
    return _native.lib().lz4b200_ctx_last_range_blocks(ctx.handle)


def pack(frames, rng, junk=True):
    """The frames' bytes back to back with junk between them: (device tensor, offsets, lengths)."""
    parts, offs, lens, pos = [], [], [], 0
    for f in frames:
        gap = bytes(rng.integers(0, 256, int(rng.integers(0, 40))).astype(np.uint8)) if junk else b""
        parts.append(gap)
        pos += len(gap)
        offs.append(pos)
        lens.append(len(f))
        parts.append(f)
        pos += len(f)
    buf = b"".join(parts) + b"\0"
    return torch.tensor(np.frombuffer(buf, dtype=np.uint8), device="cuda"), offs, lens


def assert_same_index(ix, i, one, name):
    got = ix.frame(i)
    assert bytes(got._info) == bytes(one._info), name
    assert torch.equal(got.entries, one.entries), name


def test_index_parity(ctx):
    """Every valid and broken fixture frame and a few hundred hand-built linked cases, shuffled, with junk between the
    regions, trailing bytes inside some and empty regions: each frame's info and entries are the one-frame index's."""
    rng = np.random.default_rng(21)
    hand, rnd = all_cases()
    items = valid_frames() + broken_frames(mutations=120) + [(c.name, c.frame) for c in hand + rnd[:300]]
    items += [(f"empty {k}", b"") for k in range(5)]
    for k in range(0, 40, 4):                                   # trailing bytes inside the region
        name, f = items[k]
        items.append((name + " + trailing", f + bytes(rng.integers(0, 256, 1 + k).astype(np.uint8))))
    rng.shuffle(items)
    d_in, offs, lens = pack([f for _, f in items], rng)
    ix = frame.index_frames_device(d_in, offs, lens, ctx)
    assert len(ix) == len(items)
    eo = ix.entry_offsets.cpu().numpy()
    assert (eo[1:] >= eo[:-1]).all()
    for i, (name, _) in enumerate(items):
        one = frame.index_frame_device(d_in[offs[i]:offs[i] + lens[i]], ctx)
        assert_same_index(ix, i, one, name)


def mixed_frames():
    """(frame, content) of independent and linked frames with 64 KiB and 4 MiB blocks."""
    j = corpus.tiled("compression_66k_JSON.txt", 900000).tobytes()
    d = corpus.load("dickens.txt")
    h = corpus.tiled("hdfs.json", 9 * MiB + 777).tobytes()
    return [(oracle.frame_compress(j, 4, 7), j), (oracle.frame_compress(h, 7, 0), h),
            (linked_frame(d[:800000], [65536, 20000, 7000], 4, True, True), d[:800000]),
            (linked_frame(h, [4 * MiB], 7), h),
            (oracle.frame_compress(j[:300000], 4, 2, 1000), j[:300000]),
            (linked_frame(j[:400000], [65536], 4), j[:400000]),
            (oracle.frame_compress(b"", 4, 7), b"")]


def run_batch(ctx, d_in, ix, calls, contents, gap=3):
    """The (frame, start, length) calls in one batch call, into one buffer with `gap` sentinel bytes around every region;
    each region is checked against its frame's content and every sentinel against SENTINEL.  Returns the host buffer and
    the offsets."""
    fr = np.array([c[0] for c in calls], dtype=np.int64)
    st = np.array([c[1] for c in calls], dtype=np.int64)
    ln = np.array([c[2] for c in calls], dtype=np.int64)
    cl = np.array([len(contents[f]) for f in fr], dtype=np.int64)
    clip = np.minimum(ln, cl - np.minimum(st, cl))
    oo = np.cumsum(clip + gap) - clip
    out = torch.full((int(oo[-1] + clip[-1] + gap),), SENTINEL, dtype=torch.uint8, device="cuda")
    _, _, written = frame.decompress_frames_ranges_device(d_in, ix, fr, st, ln, out=out, out_offsets=oo, ctx=ctx)
    assert (written.cpu().numpy() == clip).all()
    h = out.cpu().numpy()
    mask = np.ones(h.size, dtype=bool)
    for i, (f, a, _) in enumerate(calls):
        o, n = int(oo[i]), int(clip[i])
        assert h[o:o + n].tobytes() == contents[f][a:a + n], (i, f, a, n)
        mask[o:o + n] = False
    assert (h[mask] == SENTINEL).all()
    return h, oo, clip


def test_mixed_ranges_match_oracle_and_one_frame_calls(ctx):
    """Independent and linked frames with 64 KiB and 4 MiB blocks in one call: every frame's edge ranges plus random
    ranges over random frames, in random order.  Each range equals the oracle's slice and the one-frame call's bytes,
    and the call's block decodes are the sum of the one-frame calls' (segments never merge across frames)."""
    rng = np.random.default_rng(5)
    fs = mixed_frames()
    d_in, offs, lens = pack([f for f, _ in fs], rng)
    ix = frame.index_frames_device(d_in, offs, lens, ctx)
    contents = [c for _, c in fs]
    for k, (f, c) in enumerate(fs):
        assert oracle.frame_decompress(f, len(c) + 1)[1] == c
        assert ix.frame(k).content_len == len(c) and ix.frame(k).error is None
    per = [[(a, b) for a, b in _edges(ix.frame(k))] for k in range(len(fs))]
    for _ in range(2000):
        k = int(rng.integers(0, len(fs)))
        c = len(contents[k])
        per[k].append((int(rng.integers(0, c + 1)), int(rng.integers(0, 70000))))
    calls = [(k, a, b) for k in range(len(fs)) for a, b in per[k]]
    order = rng.permutation(len(calls))
    calls = [calls[i] for i in order]
    h, oo, clip = run_batch(ctx, d_in, ix, calls, contents)
    batch_blocks = last_blocks(ctx)
    # the one-frame call on each frame with that frame's ranges
    want_blocks = 0
    for k in range(len(fs)):
        mine = [i for i, c in enumerate(calls) if c[0] == k]
        region = d_in[offs[k]:offs[k] + lens[k]]
        out, o1, w1 = frame.decompress_ranges_device(region, ix.frame(k), [calls[i][1] for i in mine],
                                                     [calls[i][2] for i in mine], ctx=ctx)
        want_blocks += last_blocks(ctx)
        o1, w1, out = o1.cpu().numpy(), w1.cpu().numpy(), out.cpu().numpy()
        for q, i in enumerate(mine):
            assert w1[q] == clip[i]
            assert out[o1[q]:o1[q] + w1[q]].tobytes() == h[oo[i]:oo[i] + clip[i]].tobytes(), (k, calls[i])
    assert batch_blocks == want_blocks


def test_default_layout(ctx):
    fs = mixed_frames()[:3]
    d_in, offs, lens = pack([f for f, _ in fs], np.random.default_rng(1), junk=False)
    ix = frame.index_frames_device(d_in, offs, lens, ctx)
    calls = [(2, 5000, 100), (0, 0, 10), (1, 10 ** 12, 5), (0, 899990, 100)]
    out, oo, written = frame.decompress_frames_ranges_device(d_in, ix, *zip(*calls), ctx=ctx)
    h, oo = out.cpu().numpy(), oo.cpu().numpy()
    for i, (k, a, n) in enumerate(calls):
        want = fs[k][1][a:a + n]
        assert int(written[i]) == len(want)
        assert h[oo[i]:oo[i] + len(want)].tobytes() == want
    with pytest.raises(ValueError):
        frame.decompress_frames_ranges_device(d_in, ix, [3], [0], [1], ctx=ctx)


def test_untrusted_input(ctx):
    """A frame id out of range, a forged info, an entry span past the entries and a forged entry in one frame of many are
    each InvalidArgument with the output untouched; a changed payload byte is a decode error."""
    fs = mixed_frames()
    d_in, offs, lens = pack([f for f, _ in fs], np.random.default_rng(2))
    ix = frame.index_frames_device(d_in, offs, lens, ctx)
    calls = ([0, 1, 2, 3, 4], [1000, 5000, 70000, 4 * MiB - 10, 0], [3000, 100, 9000, 20, 50])
    out = torch.full((64 * 1024,), SENTINEL, dtype=torch.uint8, device="cuda")
    oo = [0, 4000, 8000, 20000, 30000]

    def call(x, frames=calls[0], d=d_in):
        return frame.decompress_frames_ranges_device(d, x, frames, *calls[1:], out=out, out_offsets=oo, ctx=ctx)

    call(ix)
    out.fill_(SENTINEL)
    bad = []
    for frames in ([0, 1, 2, 3, 7], [0, 1, 2, 3, -1]):
        bad.append((ix, frames))
    for col, delta in ((0, 12345), (1, 1), (2, 1)):                # block size, nblocks, content length
        t = {k: getattr(ix, k).clone() for k in ("infos", "entries", "entry_offsets", "offsets", "lengths")}
        t["infos"][2, col] += delta
        bad.append((frame.FrameIndexes(**t), calls[0]))
    t = {k: getattr(ix, k).clone() for k in ("infos", "entries", "entry_offsets", "offsets", "lengths")}
    t["entry_offsets"][len(fs) - 2] = ix.entries.shape[0] - int(ix.infos[len(fs) - 2, 1]) + 1
    bad.append((frame.FrameIndexes(**t), calls[0]))
    for col, delta in ((2, 1 << 32), (0, 10 ** 9), (1, 3)):        # decoded length, payload offset, decoded offset
        t = {k: getattr(ix, k).clone() for k in ("infos", "entries", "entry_offsets", "offsets", "lengths")}
        t["entries"][int(ix.entry_offsets[4]) + 7, col] += delta
        bad.append((frame.FrameIndexes(**t), calls[0]))
    for x, frames in bad:
        with pytest.raises(ValueError):
            call(x, frames)
        assert (out.cpu().numpy() == SENTINEL).all()
    # a compressed payload byte changed after indexing
    e = ix.frame(0).entries.cpu().numpy()
    k = next(i for i in range(e.shape[0]) if not int(e[i, 2]) & 0x80000000 and int(e[i, 1]) <= 1000 < int(e[i, 1]) +
             (int(e[i, 2]) >> 32))
    z = d_in.clone()
    z[offs[0] + int(e[k, 0]):offs[0] + int(e[k, 0]) + (int(e[k, 2]) & 0x7FFFFFFF)] = 0
    with pytest.raises(errors.DecompressionError):
        call(ix, d=z)


def test_one_mib_budget(ctx):
    """At a 1 MiB frame budget: the index goes in many passes, a frame of tens of thousands of tiny blocks takes the
    one-frame path, ranges go in many windows, and more than 65 536 ranges cross the planner's chunk; the results are the
    default budget's and the content's."""
    rng = np.random.default_rng(9)
    j = corpus.tiled("compression_66k_JSON.txt", 2 * MiB).tobytes()
    d = corpus.load("dickens.txt")
    fs = [(oracle.frame_compress(j[k * 9000:k * 9000 + 150000], 4, 7, 700), j[k * 9000:k * 9000 + 150000])
          for k in range(200)]
    fs.append((oracle.frame_compress(j[:1500000], 4, 0, 48), j[:1500000]))            # about 31 000 blocks
    fs.append((linked_frame(d[:3 * MiB], [4 * MiB], 7), d[:3 * MiB]))
    fs.append((linked_frame(d[:600000], [65536, 3000], 4), d[:600000]))
    fs.append((oracle.frame_compress(d[:5 * MiB], 7, 0), d[:5 * MiB]))
    order = rng.permutation(len(fs))
    fs = [fs[i] for i in order]
    d_in, offs, lens = pack([f for f, _ in fs], rng)
    ref = frame.index_frames_device(d_in, offs, lens, ctx)
    small = block.Context()
    try:
        _native.lib().lz4b200_ctx_set_frame_budget(small.handle, MiB)
        ix = frame.index_frames_device(d_in, offs, lens, small)
        assert torch.equal(ix.infos, ref.infos) and torch.equal(ix.entries, ref.entries)
        assert torch.equal(ix.entry_offsets, ref.entry_offsets)
        assert max(int(x) for x in ix.infos[:, 1].cpu()) > 30000
        contents = [c for _, c in fs]
        calls = []
        for _ in range(70000):
            k = int(rng.integers(0, len(fs)))
            calls.append((k, int(rng.integers(0, len(contents[k]) + 1)), int(rng.integers(0, 3000))))
        for k in range(len(fs)):
            calls.append((k, 0, len(contents[k])))
        run_batch(small, d_in, ix, calls, contents, gap=1)
    finally:
        small.close()


def test_scale_compressed_frames(ctx):
    """compress_frames_device packs 4 096 x 256 KiB of JSON; the frames are indexed in one call and 10 000 random
    ranges over them read in one call, every range checked against the source on the device."""
    n, size = 4096, 256 << 10
    src = torch.tensor(corpus.tiled("compression_66k_JSON.txt", n * size + 4099), device="cuda")
    starts = np.arange(n, dtype=np.int64) * size + np.arange(n) % 4
    frames_, foff = frame.compress_frames_device(src, starts, [size] * n,
                                                 frame.FrameInfo(block_size=frame.BlockSize.Max64KB), ctx=ctx)
    fo = foff.cpu().numpy()
    ix = frame.index_frames_device(frames_, fo[:-1], np.diff(fo), ctx)
    cl = ix.content_lens()
    assert (cl == size).all()
    rng = np.random.default_rng(4)
    fr = rng.integers(0, n, 10000)
    st = rng.integers(0, size, 10000)
    ln = rng.integers(0, 8192, 10000)
    out, oo, written = frame.decompress_frames_ranges_device(frames_, ix, fr, st, ln, ctx=ctx)
    clip = np.minimum(ln, size - st)
    assert (written.cpu().numpy() == clip).all()
    total = int(clip.sum())
    within = np.arange(total) - np.repeat(np.cumsum(clip) - clip, clip)
    pos_out = torch.as_tensor(np.repeat(oo.cpu().numpy(), clip) + within, device="cuda")
    pos_src = torch.as_tensor(np.repeat(starts[fr] + st, clip) + within, device="cuda")
    assert torch.equal(out[pos_out], src[pos_src])


def test_teardown_frees_the_batch_scratch(ctx):
    """The batch index and range scratch is context scratch: counted by lz4b200_ctx_device_bytes while the context lives,
    and returned to the device when it is destroyed."""
    fs = mixed_frames()
    d_in, offs, lens = pack([f for f, _ in fs], np.random.default_rng(3))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    c = block.Context()
    ix = frame.index_frames_device(d_in, offs, lens, c)
    grown = _native.lib().lz4b200_ctx_device_bytes(c.handle)
    assert grown > 0
    out, _, _ = frame.decompress_frames_ranges_device(d_in, ix, [3, 1], [0, 0], [16 * MiB, 16 * MiB], ctx=c)
    assert out[:len(fs[3][1])].cpu().numpy().tobytes() == fs[3][1]
    assert _native.lib().lz4b200_ctx_device_bytes(c.handle) > grown
    del ix, out
    c.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert torch.cuda.mem_get_info()[0] >= free0 - 64 * MiB
