"""GPU parity of the device-resident frame decoder: lz4b200_frame_decompress_next_device on bytes in HBM returns
exactly what lz4b200_frame_decompress_next returns for the same bytes in host memory — status, consumed, written,
block_status, err_expected, err_actual and the output bytes — and writes nothing past `written`.
lz4b200_frame_decoded_bound_device equals lz4b200_frame_decoded_bound on every input."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, corpus, errors, frame
from lz4_flex_b200.frame import BlockSize, FrameInfo

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
ALL = oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM | oracle.F_CONTENT_SIZE


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
    return st, used.value, w.value, bs.value, e1.value, e2.value, out[:w.value].tobytes()


def to_device(f: bytes, mis: int = 0):
    """f in a device buffer at byte offset `mis` from a 256-byte aligned allocation."""
    buf = torch.zeros(len(f) + mis + 16, dtype=torch.uint8, device="cuda")
    if f:
        buf[mis:mis + len(f)] = torch.from_numpy(np.frombuffer(f, dtype=np.uint8).copy()).cuda()
    return buf[mis:mis + len(f)]


def device_next(ctx, f: bytes, cap: int, mis: int = 0, stream=None):
    d_in = to_device(f, mis)
    out = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    used, w, bs, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_uint64(0), C.c_uint64(0)
    s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
    st = _native.lib().lz4b200_frame_decompress_next_device(
        ctx.handle, d_in.data_ptr() if len(f) else None, len(f), out.data_ptr() if cap else None, cap, C.byref(used),
        C.byref(w), C.byref(bs), C.byref(e1), C.byref(e2), s)
    o = out.cpu().numpy()
    assert (o[w.value:] == SENTINEL).all(), "bytes past `written` were modified"
    return st, used.value, w.value, bs.value, e1.value, e2.value, o[:w.value].tobytes()


def device_bound(ctx, f: bytes) -> int:
    d_in = to_device(f, 3)
    b = C.c_size_t(0)
    st = _native.lib().lz4b200_frame_decoded_bound_device(ctx.handle, d_in.data_ptr() if len(f) else None, len(f),
                                                          C.byref(b), torch.cuda.current_stream().cuda_stream)
    assert st == 0
    return b.value


def check(ctx, f: bytes, cap=None, mis: int = 0, bound=True):
    """Device and host calls agree on every field; returns the host result."""
    if cap is None:
        cap = host_bound(f)
    h = host_next(ctx, f, cap)
    d = device_next(ctx, f, cap, mis)
    assert d[:6] == h[:6], (d[:6], h[:6])
    assert d[6] == h[6]
    if bound:
        assert device_bound(ctx, f) == host_bound(f)
    return h


def _flags(checks: bool) -> int:
    return ALL if checks else 0


@pytest.mark.parametrize("bs", [BlockSize.Auto, BlockSize.Max64KB, BlockSize.Max256KB, BlockSize.Max1MB, BlockSize.Max4MB])
@pytest.mark.parametrize("checks", [False, True])
def test_one_shot_matrix(ctx, bs, checks):
    for data in (b"", b"a", corpus.load("compression_1k.txt"), corpus.load("compression_66k_JSON.txt"),
                 corpus.tiled("compression_66k_JSON.txt", 5 * 65536 + 777).tobytes(),
                 corpus.load("dickens.txt")[: (9 << 20) + 5], bytes(300000),
                 corpus.adversarial_blocks(6, 0.5).tobytes()):
        f = oracle.frame_compress(data, int(bs), _flags(checks))
        h = check(ctx, f)
        assert h[0] == 0 and h[6] == data and h[1] == len(f)


def test_concatenated_and_flushed_frames(ctx):
    j = corpus.tiled("compression_66k_JSON.txt", 700000).tobytes()
    f1 = oracle.frame_compress(j[:200000], 4, ALL, 9000)                     # flushed short blocks
    f2 = oracle.frame_compress(j[200000:], 5, oracle.F_CONTENT_CHECKSUM)
    cat = f1 + f2
    h = check(ctx, cat)
    assert h[0] == 0 and h[1] == len(f1) and h[6] == j[:200000]
    check(ctx, cat[h[1]:])
    got = frame.decompress_frame_device(to_device(cat, 5), ctx=ctx)
    assert got.cpu().numpy().tobytes() == frame.decompress_frame(cat, ctx) == j


def test_legacy_linked_stored_and_empty(ctx):
    import json
    import os
    d = corpus.load("dickens.lz4")
    assert check(ctx, d)[6] == corpus.load("dickens.txt")
    gdir = os.path.join(os.path.dirname(__file__), "golden", "linked")
    for m in json.load(open(os.path.join(gdir, "manifest.json"))):
        f = open(os.path.join(gdir, m["file"]), "rb").read()
        assert check(ctx, f)[0] == 0, m["file"]
    rnd = corpus.xorshift64star_bytes(3 * 65536 + 100).tobytes()
    f = oracle.frame_compress(rnd, 4, ALL)
    assert int.from_bytes(f[15:19], "little") == (65536 | 0x80000000)
    assert check(ctx, f)[6] == rnd
    for tiny in (b"", b"\x04", b"\x04\x22\x4d", b"\x04\x22\x4d\x18", b"\x04\x22\x4d\x18\x60", b"\x02\x21\x4c\x18"):
        check(ctx, tiny)
    assert check(ctx, b"\x04\x22\x4d\x18")[:3] == (0, 4, 0)                     # magic only: end of data


def _frame_regions():
    j = corpus.tiled("compression_66k_JSON.txt", 300000).tobytes()
    f = oracle.frame_compress(j, 4, ALL)
    return j, f


def _rehead(f: bytes, flg=None, bd=None, size=None, dict_id=None) -> bytes:
    """The frame with a rewritten header (valid header checksum)."""
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


def test_truncation_in_every_region(ctx):
    j, f = _frame_regions()
    hlen = 15
    w0 = int.from_bytes(f[hlen:hlen + 4], "little") & 0x7FFFFFFF
    last_end = len(f) - 8                                                      # EndMark at [len-8, len-4)
    cuts = list(range(0, hlen + 6))                                            # header, first BlockInfo
    cuts += [hlen + 4 + w0 // 2, hlen + 4 + w0, hlen + 4 + w0 + 2]             # payload, block checksum
    cuts += [last_end - 3, last_end, last_end + 2, last_end + 4, len(f) - 2, len(f) - 1, len(f)]   # EndMark, content checksum
    for c in cuts:
        check(ctx, f[:c])


def test_corrupted_headers(ctx):
    _, f = _frame_regions()
    cases = {
        "magic": bytes([f[0] ^ 1]) + f[1:],
        "version": _rehead(f, flg=(f[4] & 0x3F) | 0x80),
        "reserved flg": _rehead(f, flg=f[4] | 0x02),
        "reserved bd": _rehead(f, bd=f[5] | 0x01),
        "block size": _rehead(f, bd=(f[5] & 0x8F) | 0x30),
        "dictionary": _rehead(f, flg=f[4] | 0x01, dict_id=7),
        "header checksum": f[:14] + bytes([f[14] ^ 1]) + f[15:],
        "skippable": b"\x50\x2a\x4d\x18" + (4).to_bytes(4, "little") + b"abcd" + f,
    }
    want = {"magic": 102, "version": 104, "reserved flg": 103, "reserved bd": 103, "block size": 105, "dictionary": 112,
            "header checksum": 106, "skippable": 111}
    for name, g in cases.items():
        h = check(ctx, g)
        assert h[0] == want[name], name


def test_checksums_sizes_offsets_and_too_big(ctx):
    j, f = _frame_regions()
    blocks = []
    pos = 15
    while True:
        w = int.from_bytes(f[pos:pos + 4], "little")
        if w == 0:
            break
        blocks.append((pos, w & 0x7FFFFFFF))
        pos += 8 + (w & 0x7FFFFFFF)
    assert len(blocks) >= 4
    for k in (0, len(blocks) // 2, len(blocks) - 1):                           # block checksum flipped
        p, ln = blocks[k]
        g = bytearray(f)
        g[p + 4 + ln] ^= 0x10
        h = check(ctx, bytes(g))
        assert h[0] == 107 and h[1] == p + 4 + ln and h[6] == j[:65536 * k]
    g = bytearray(f)
    g[-1] ^= 1                                                                 # content checksum flipped
    assert check(ctx, bytes(g))[0] == 108
    for size in (len(j) - 1, len(j) + 1):                                      # content size too small / too large
        h = check(ctx, _rehead(f, size=size))
        assert h[0] == 109 and (h[4], h[5]) == (size, len(j))
    g = bytearray(f)
    g[15:19] = (65537).to_bytes(4, "little")                                   # BlockTooBig
    assert check(ctx, bytes(g))[0] == 110
    # a zeroed match offset in the second block, after a good first block
    good = oracle.compress_block(j[:65536])
    bad = bytes([0x44]) + b"abcd" + b"\x00\x00" + bytes([0x50]) + b"hello"
    body = b"".join(len(b).to_bytes(4, "little") + b for b in (good, bad))
    g = FrameInfo(block_size=BlockSize.Max64KB).header_bytes() + body + b"\0\0\0\0"
    h = check(ctx, g)
    assert h[0] == 101 and h[6] == j[:65536]


def test_random_mutations(ctx):
    j = corpus.tiled("compression_66k_JSON.txt", 500000).tobytes()
    f = oracle.frame_compress(j, 4, ALL)
    rng = np.random.default_rng(77)
    seen = set()
    for t in range(520):
        g = bytearray(f)
        for _ in range(int(rng.integers(1, 4))):
            p = int(rng.integers(0, 40)) if rng.random() < 0.3 else int(rng.integers(0, len(g)))
            g[p] = int(rng.integers(0, 256))
        if t % 4 == 3:
            g = g[:int(rng.integers(0, len(g) + 1))]
        h = check(ctx, bytes(g), bound=(t % 10 == 0))
        seen.add(h[0])
    assert len(seen) >= 4, seen


def test_caps_and_alignment(ctx):
    j = corpus.tiled("compression_66k_JSON.txt", 400000).tobytes()
    for f in (oracle.frame_compress(j, 4, ALL), oracle.frame_compress(j, 5, 0, 30000)):
        for cap in (0, 1, len(j) - 1, len(j), len(j) + 1):
            check(ctx, f, cap, bound=False)
        for mis in range(1, 16):
            check(ctx, f, None, mis, bound=(mis == 1))


def test_many_blocks_small_budget(ctx):
    data = corpus.tiled("compression_66k_JSON.txt", 20000 * 150).tobytes()
    f = oracle.frame_compress(data, 7, oracle.F_CONTENT_CHECKSUM | oracle.F_BLOCK_CHECKSUMS, 150)
    _native.lib().lz4b200_ctx_set_frame_budget(ctx.handle, 1 << 20)
    try:
        h = check(ctx, f)
        assert h[0] == 0 and h[6] == data
        g = bytearray(f)
        g[-1] ^= 1
        assert check(ctx, bytes(g), bound=False)[0] == 108
        check(ctx, f, len(data) // 2, bound=False)                           # OUTPUT_FULL at a group boundary
    finally:
        _native.lib().lz4b200_ctx_set_frame_budget(ctx.handle, 256 << 20)


def test_device_round_trip_without_host_data(ctx):
    """Header, device-compressed blocks and EndMark assembled in one device buffer, decoded in place on the GPU."""
    L = _native.lib()
    bs = 64 << 10
    src = torch.from_numpy(corpus.tiled("hdfs.json", 3 << 20)).cuda()
    info = FrameInfo(block_size=BlockSize.Max64KB).to_c()
    hdr = (C.c_uint8 * 19)()
    hlen = L.lz4b200_frame_write_header(C.byref(info), hdr, 19)
    bound = L.lz4b200_frame_blocks_bound(src.numel(), bs)
    buf = torch.zeros(hlen + bound + 4, dtype=torch.uint8, device="cuda")
    buf[:hlen] = torch.tensor(list(hdr[:hlen]), dtype=torch.uint8)
    d_total = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    assert L.lz4b200_frame_compress_blocks_device(ctx.handle, src.data_ptr(), src.numel(), bs, 0, buf[hlen:].data_ptr(),
                                                  bound, d_total.data_ptr(), None, s) == 0
    total = int(d_total.item())
    buf[hlen + total:hlen + total + 4] = 0                                    # EndMark
    f = buf[:hlen + total + 4]
    out = frame.decompress_frame_device(f, ctx=ctx)
    assert out.numel() == src.numel() and torch.equal(out, src)
    used, w, err = frame.decompress_next_frame_device(f, torch.empty(src.numel(), dtype=torch.uint8, device="cuda"), ctx)
    assert (used, w, err) == (f.numel(), src.numel(), None)


def test_python_errors_match_host(ctx):
    _, f = _frame_regions()
    for g in (f[:100], bytes([f[0] ^ 1]) + f[1:], f[:-1] + bytes([f[-1] ^ 1])):
        with pytest.raises(errors.FrameError) as want:
            frame.decompress_frame(g, ctx)
        with pytest.raises(errors.FrameError) as got:
            frame.decompress_frame_device(to_device(g), ctx=ctx)
        assert type(got.value) is type(want.value)
    # the context's own stream
    j = corpus.load("compression_66k_JSON.txt")
    g = oracle.frame_compress(j, 4, ALL)
    out = torch.empty(len(j), dtype=torch.uint8, device="cuda")
    used, w, err = frame.decompress_next_frame_device(to_device(g), out, ctx, stream=ctx.stream)
    assert (used, w, err) == (len(g), len(j), None) and out.cpu().numpy().tobytes() == j
