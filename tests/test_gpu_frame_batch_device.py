"""GPU parity of the batch frame decoder: lz4b200_frame_decompress_batch_device gives every frame of a batch exactly
what lz4b200_frame_decompress_next returns for that frame's bytes in host memory on the same context — status,
consumed, written, block_status, err_expected, err_actual and the output bytes — and writes nothing else of d_out.
lz4b200_frame_decoded_bound_batch_device equals lz4b200_frame_decoded_bound per single-frame region."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, block, corpus, frame
from lz4_flex_b200.frame import BlockSize, FrameInfo

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
GAP = 64
ALL = oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM | oracle.F_CONTENT_SIZE
GDIR = os.path.join(os.path.dirname(__file__), "golden", "linked")


def _ptr(a):
    return a.ctypes.data if a.size else None


def host_bound(f: bytes) -> int:
    src = np.frombuffer(f, dtype=np.uint8)
    b = C.c_size_t(0)
    assert _native.lib().lz4b200_frame_decoded_bound(_ptr(src), src.size, C.byref(b)) == 0
    return b.value


def host_next(ctx, f: bytes, cap: int):
    src = np.frombuffer(f, dtype=np.uint8)
    out = np.zeros(max(cap, 1), dtype=np.uint8)
    used, w, bs, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_uint64(0), C.c_uint64(0)
    st = _native.lib().lz4b200_frame_decompress_next(ctx.handle, _ptr(src), src.size, out.ctypes.data if cap else None,
                                                     cap, C.byref(used), C.byref(w), C.byref(bs), C.byref(e1), C.byref(e2))
    return (st, used.value, w.value, bs.value, e1.value, e2.value), out[:w.value].tobytes()


def layout(sizes, rng, gap):
    """Offsets for regions of `sizes` bytes with `gap` + 0..15 bytes before each."""
    offs, pos = [], 0
    for n in sizes:
        pos += gap + int(rng.integers(0, 16))
        offs.append(pos)
        pos += n
    return offs, pos + gap


def run_batch(ctx, frames, caps, seed=0, stream=None):
    """Decodes `frames` (with output caps `caps`) in one batch call; returns per frame ((six fields), bytes) and checks
    that every byte of d_out outside the frames' written bytes still holds the sentinel."""
    rng = np.random.default_rng(seed)
    n = len(frames)
    in_off, in_total = layout([len(f) for f in frames], rng, 0)
    h_in = np.full(max(in_total, 1), 0x5A, dtype=np.uint8)
    for f, o in zip(frames, in_off):
        h_in[o:o + len(f)] = np.frombuffer(f, dtype=np.uint8)
    out_off, out_total = layout(caps, rng, GAP)
    d_in = torch.from_numpy(h_in).cuda()
    d_out = torch.full((out_total,), SENTINEL, dtype=torch.uint8, device="cuda")
    t = lambda v: torch.tensor(v, dtype=torch.int64, device="cuda")
    d_foff, d_flen, d_ooff, d_ocap = t(in_off), t([len(f) for f in frames]), t(out_off), t(caps)
    res = torch.full((max(n, 1), 5), -1, dtype=torch.int64, device="cuda")
    s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    st = _native.lib().lz4b200_frame_decompress_batch_device(
        ctx.handle, d_in.data_ptr(), d_foff.data_ptr(), d_flen.data_ptr(), d_out.data_ptr(), d_ooff.data_ptr(),
        d_ocap.data_ptr(), res.data_ptr(), n, s)
    assert st == 0, ctx.last_cuda_error()
    r = res.cpu().numpy()
    o = d_out.cpu().numpy()
    mask = np.ones(out_total, dtype=bool)
    got = []
    for i in range(n):
        consumed, written, e1, e2, packed = (int(x) for x in r[i])
        fst, bst = int(np.int32(packed & 0xFFFFFFFF)), int(np.int32((packed >> 32) & 0xFFFFFFFF))
        got.append(((fst, consumed, written, bst, e1, e2), o[out_off[i]:out_off[i] + written].tobytes()))
        mask[out_off[i]:out_off[i] + written] = False
    assert (o[mask] == SENTINEL).all(), "bytes outside the frames' written output were modified"
    return got


def check_batch(ctx, frames, caps=None, seed=0):
    """The batch call against one host call per frame; returns the host results."""
    if caps is None:
        caps = [host_bound(f) for f in frames]
    want = [host_next(ctx, f, c) for f, c in zip(frames, caps)]
    got = run_batch(ctx, frames, caps, seed)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g[0] == w[0], (i, len(frames[i]), caps[i], g[0], w[0])
        assert g[1] == w[1], i
    return want


def _rehead(f: bytes, flg=None, bd=None, size=None, dict_id=None) -> bytes:
    old_flg = f[4]
    hlen = 7 + (8 if old_flg & 0x08 else 0) + (4 if old_flg & 0x01 else 0)
    flg = old_flg if flg is None else flg
    bd = f[5] if bd is None else bd
    h = bytes([flg, bd])
    if flg & 0x08:
        h += (int.from_bytes(f[6:14], "little") if size is None else size).to_bytes(8, "little")
    if flg & 0x01:
        h += (dict_id or 0).to_bytes(4, "little")
    return f[:4] + h + bytes([(frame.xxh32(h) >> 8) & 0xFF]) + f[hlen:]


def linked_fixtures():
    return [open(os.path.join(GDIR, m["file"]), "rb").read() for m in json.load(open(os.path.join(GDIR, "manifest.json")))]


def block_positions(f: bytes):
    blocks, pos = [], 15
    while True:
        w = int.from_bytes(f[pos:pos + 4], "little")
        if w == 0:
            return blocks
        blocks.append((pos, w & 0x7FFFFFFF))
        pos += 8 + (w & 0x7FFFFFFF)


def mixed_cases():
    """(frame, cap or None) over everything the one-frame device tests cover."""
    cases = []
    datas = (b"", b"a", corpus.load("compression_1k.txt"), corpus.load("compression_66k_JSON.txt"),
             corpus.tiled("compression_66k_JSON.txt", 5 * 65536 + 777).tobytes(),
             corpus.load("dickens.txt")[: (9 << 20) + 5], bytes(300000), corpus.adversarial_blocks(6, 0.5).tobytes())
    for bs in (0, 4, 5, 6, 7):
        for checks in (0, ALL):
            for d in datas:
                cases.append((oracle.frame_compress(d, bs, checks), None))
    for tiny in (b"", b"\x04", b"\x04\x22\x4d", b"\x04\x22\x4d\x18", b"\x04\x22\x4d\x18\x60", b"\x02\x21\x4c\x18"):
        cases.append((tiny, None))
    cases.append((corpus.load("dickens.lz4"), None))
    for f in linked_fixtures():
        cases += [(f, None)] * 3
    rnd = corpus.xorshift64star_bytes(3 * 65536 + 100).tobytes()
    cases.append((oracle.frame_compress(rnd, 4, ALL), None))                              # stored blocks
    j = corpus.tiled("compression_66k_JSON.txt", 700000).tobytes()
    f1, f2 = oracle.frame_compress(j[:200000], 4, ALL, 9000), oracle.frame_compress(j[200000:], 5, oracle.F_CONTENT_CHECKSUM)
    cases += [(f1, None), (f1 + f2, None)]                                                 # flushed; two frames in one region
    g = corpus.tiled("compression_66k_JSON.txt", 300000).tobytes()
    f = oracle.frame_compress(g, 4, ALL)
    for name, h in {"magic": bytes([f[0] ^ 1]) + f[1:], "version": _rehead(f, flg=(f[4] & 0x3F) | 0x80),
                    "reserved flg": _rehead(f, flg=f[4] | 0x02), "reserved bd": _rehead(f, bd=f[5] | 0x01),
                    "block size": _rehead(f, bd=(f[5] & 0x8F) | 0x30), "dictionary": _rehead(f, flg=f[4] | 0x01, dict_id=7),
                    "header checksum": f[:14] + bytes([f[14] ^ 1]) + f[15:],
                    "skippable": b"\x50\x2a\x4d\x18" + (4).to_bytes(4, "little") + b"abcd" + f}.items():
        cases.append((h, None))
    blocks = block_positions(f)
    w0 = blocks[0][1]
    cuts = list(range(0, 21)) + [15 + 4 + w0 // 2, 15 + 4 + w0, 15 + 4 + w0 + 2]
    cuts += [len(f) - 11, len(f) - 8, len(f) - 6, len(f) - 4, len(f) - 2, len(f) - 1]
    cases += [(f[:c], None) for c in cuts]                                                 # truncation in every region
    for k in (0, len(blocks) // 2, len(blocks) - 1):                                       # block checksum flipped
        p, ln = blocks[k]
        h = bytearray(f)
        h[p + 4 + ln] ^= 0x10
        cases.append((bytes(h), None))
    h = bytearray(f)
    h[-1] ^= 1
    cases.append((bytes(h), None))                                                         # content checksum flipped
    cases += [(_rehead(f, size=len(g) + d), None) for d in (-1, 1)]                        # content size both ways
    h = bytearray(f)
    h[15:19] = (65537).to_bytes(4, "little")
    cases.append((bytes(h), None))                                                         # BlockTooBig
    good = oracle.compress_block(g[:65536])
    bad = bytes([0x44]) + b"abcd" + b"\x00\x00" + bytes([0x50]) + b"hello"
    body = b"".join(len(b).to_bytes(4, "little") + b for b in (good, bad))
    cases.append((FrameInfo(block_size=BlockSize.Max64KB).header_bytes() + body + b"\0\0\0\0", None))   # zero offset
    for src in (oracle.frame_compress(g, 4, ALL), oracle.frame_compress(g, 5, 0, 30000)):  # caps 0, one short, exact
        cases += [(src, 0), (src, len(g) - 1), (src, len(g)), (src, 1)]
    return cases


def mutations(count, seed):
    j = corpus.tiled("compression_66k_JSON.txt", 500000).tobytes()
    bases = [oracle.frame_compress(j, 4, ALL), oracle.frame_compress(j, 5, 0)] + linked_fixtures()[:2]
    rng = np.random.default_rng(seed)
    out = []
    for t in range(count):
        g = bytearray(bases[t % len(bases)])
        for _ in range(int(rng.integers(1, 4))):
            p = int(rng.integers(0, 40)) if rng.random() < 0.3 else int(rng.integers(0, len(g)))
            g[p] = int(rng.integers(0, 256))
        if t % 4 == 3:
            g = g[:int(rng.integers(0, len(g) + 1))]
        out.append(bytes(g))
    return out


def _caps(cases):
    return [host_bound(f) if c is None else c for f, c in cases]


def test_mixed_batch_matches_host(ctx):
    cases = mixed_cases()
    frames, caps = [f for f, _ in cases], _caps(cases)
    want = check_batch(ctx, frames, caps, seed=1)
    statuses = {w[0][0] for w in want}
    assert {0, 101, 102, 107, 108, 109, 110, 111, 115}.issubset(statuses), statuses
    # the region with two concatenated frames decodes the first and says where it ended
    assert any(w[0][0] == 0 and 0 < w[0][1] < len(f) for f, w in zip(frames, want))


def test_mutations_and_isolation(ctx):
    frames = mutations(500, 77)
    good = oracle.frame_compress(corpus.tiled("compression_66k_JSON.txt", 200000).tobytes(), 4, ALL)
    mixed = [x for m in frames for x in (m, good)]                     # every mutated frame between good frames
    caps = [host_bound(f) for f in mixed]
    want = check_batch(ctx, mixed, caps, seed=2)
    assert len({w[0][0] for w in want}) >= 4
    assert all(w[0][0] == 0 for w in want[1::2])
    perm = np.random.default_rng(3).permutation(len(mixed))             # shuffled: every frame's result unchanged
    got = run_batch(ctx, [mixed[p] for p in perm], [caps[p] for p in perm], seed=4)
    for k, p in enumerate(perm):
        assert got[k] == (want[p][0], want[p][1]), k


def test_small_budget(ctx):
    """A context of this test's own with a 1 MiB frame budget: many groups, and frames larger than the budget."""
    c2 = block.Context(0)
    try:
        _native.lib().lz4b200_ctx_set_frame_budget(c2.handle, 1 << 20)
        j = corpus.tiled("compression_66k_JSON.txt", 3 << 20).tobytes()
        big = oracle.frame_compress(j, 4, ALL)                          # independent, 48 blocks: the one-frame path
        big_linked = _rehead(big, flg=big[4] & ~0x20)                   # the same blocks as one 3 MiB linked chain
        small = [oracle.frame_compress(j[i * 70000:(i + 1) * 70000], 4, ALL) for i in range(40)]
        frames = small[:20] + [big, big_linked] + small[20:] + [big, big]
        caps = _caps([(f, None) for f in frames])
        caps[-1] = (1 << 20) + 100000                                   # OUTPUT_FULL after the host's first 1 MiB group
        caps[-2] = len(j) - 1
        want = check_batch(ctx=c2, frames=frames, caps=caps, seed=5)
        assert want[20][0][0] == want[21][0][0] == 0 and want[-1][0][0] == 115 and want[-1][0][2] > 0
        check_batch(c2, mutations(100, 9), seed=6)
        check_batch(c2, linked_fixtures() * 8, seed=7)
    finally:
        c2.close()


def test_scale_single_block_json_frames(ctx):
    data = corpus.tiled("compression_66k_JSON.txt", 16384 * 65536)
    frames = [oracle.frame_compress(data[i * 65536:(i + 1) * 65536].tobytes(), 4,
                                    oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM) for i in range(16384)]
    lens = np.array([len(f) for f in frames], dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    d_in = torch.from_numpy(np.frombuffer(b"".join(frames), dtype=np.uint8).copy()).cuda()
    r = frame.decompress_frames_device(d_in, offs, lens, ctx=ctx)
    res = r.results.cpu().numpy()
    assert (res[:, 4] == 0).all() and (res[:, 1] == 65536).all() and (res[:, 0] == lens).all()
    oo = r.out_offsets.cpu().numpy()
    assert (oo == np.arange(16384) * 65536).all()
    assert torch.equal(r.out[:16384 * 65536], torch.from_numpy(data[:16384 * 65536]).cuda())


def test_scale_linked_interleaved(ctx):
    fixtures = linked_fixtures()
    j = corpus.tiled("compression_66k_JSON.txt", 300000).tobytes()
    ind = [oracle.frame_compress(j[:100000 + 17 * i], 4, ALL) for i in range(8)]
    frames = [x for i in range(2000) for x in (fixtures[i % len(fixtures)], ind[i % len(ind)])]
    got = run_batch(ctx, frames, [host_bound(f) for f in frames], seed=8)
    want = {id(f): host_next(ctx, f, host_bound(f)) for f in fixtures + ind}
    for f, g in zip(frames, got):
        assert g == want[id(f)]


def test_bounds_and_arguments(ctx):
    L = _native.lib()
    cases = mixed_cases()[::3] + [(f, None) for f in mutations(60, 11)]
    frames = [f for f, _ in cases]
    offs, total = layout([len(f) for f in frames], np.random.default_rng(12), 0)
    h = np.zeros(max(total, 1), dtype=np.uint8)
    for f, o in zip(frames, offs):
        h[o:o + len(f)] = np.frombuffer(f, dtype=np.uint8)
    d_in = torch.from_numpy(h).cuda()
    t = lambda v: torch.tensor(v, dtype=torch.int64, device="cuda")
    d_off, d_len = t(offs), t([len(f) for f in frames])
    d_b = torch.zeros(len(frames), dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    assert L.lz4b200_frame_decoded_bound_batch_device(ctx.handle, d_in.data_ptr(), d_off.data_ptr(), d_len.data_ptr(),
                                                      d_b.data_ptr(), len(frames), s) == 0
    got = d_b.cpu().numpy().tolist()
    several = 0
    for f, b in zip(frames, got):
        if b != host_bound(f):                                          # a region of several frames: the first one's
            (st, consumed, *_), _ = host_next(ctx, f, host_bound(f))
            assert 0 < consumed < len(f) and b == host_bound(f[:consumed]), (len(f), b, host_bound(f))
            several += 1
    assert several <= 1 + len(frames) // 20
    p = d_in.data_ptr()
    res = torch.zeros((1, 5), dtype=torch.int64, device="cuda")
    args = [ctx.handle, p, d_off.data_ptr(), d_len.data_ptr(), p, d_off.data_ptr(), d_len.data_ptr(), res.data_ptr()]
    assert L.lz4b200_frame_decompress_batch_device(*args, 0, s) == 0
    assert L.lz4b200_frame_decompress_batch_device(None, *args[1:], 0, s) == 200
    for k in range(1, 8):
        a = list(args)
        a[k] = None
        assert L.lz4b200_frame_decompress_batch_device(*a, 1, s) == 200, k
        assert L.lz4b200_frame_decompress_batch_device(*a, 0, s) == 0, k
    assert L.lz4b200_frame_decompress_batch_device(*args, 1 << 32, s) == 200
    bargs = [ctx.handle, p, d_off.data_ptr(), d_len.data_ptr(), d_b.data_ptr()]
    assert L.lz4b200_frame_decoded_bound_batch_device(None, *bargs[1:], 0, s) == 200
    for k in range(1, 5):
        a = list(bargs)
        a[k] = None
        assert L.lz4b200_frame_decoded_bound_batch_device(*a, 1, s) == 200, k
    assert L.lz4b200_frame_decoded_bound_batch_device(*bargs, 1 << 32, s) == 200
    assert (res == 0).all()


def test_python_matches_next_frame_device(ctx):
    frames = [f for f, _ in mixed_cases()[::4]] + mutations(40, 13)
    lens = [len(f) for f in frames]
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    d_in = torch.from_numpy(np.frombuffer(b"".join(frames), dtype=np.uint8).copy()).cuda()
    want = []
    for f in frames:
        d_out = torch.empty(max(host_bound(f), 1), dtype=torch.uint8, device="cuda")
        used, w, err = frame.decompress_next_frame_device(torch.from_numpy(np.frombuffer(f, np.uint8).copy()).cuda()
                                                          if f else torch.empty(0, dtype=torch.uint8, device="cuda"),
                                                          d_out[:host_bound(f)], ctx)
        want.append((d_out[:w].cpu().numpy().tobytes(), used, type(err), repr(err)))

    def same(r):
        for i, (view, used, err) in enumerate(r):
            assert (view.cpu().numpy().tobytes(), used, type(err), repr(err)) == want[i], i

    same(frame.decompress_frames_device(d_in, offs, lens, ctx=ctx))                      # default allocation
    side = torch.cuda.Stream()
    same(frame.decompress_frames_device(d_in, torch.from_numpy(offs).cuda(), lens, ctx=ctx, stream=side.cuda_stream))
    a = frame.decompress_frames_device(d_in, offs, lens, ctx=ctx)                         # two calls back to back
    caps = [host_bound(f) for f in frames]
    oo = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
    out = torch.full((sum(caps) + 1,), SENTINEL, dtype=torch.uint8, device="cuda")
    b = frame.decompress_frames_device(d_in, offs, lens, out, oo, caps, ctx=ctx)
    same(a)
    same(b)
    assert b.out is out
