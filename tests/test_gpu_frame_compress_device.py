"""GPU parity of the device-resident frame encoder: lz4b200_frame_compress_device on input in HBM returns the status
lz4b200_frame_compress returns for the same input in host memory, and on success writes the same bytes, which are
the bytes the C oracle (lz4_flex's FrameEncoder) writes.  *d_written equals the host call's `written`, nothing past
the frame is written, and after an argument error neither the output nor *d_written is touched."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, corpus, errors, frame
from lz4_flex_b200.frame import BlockMode, BlockSize, FrameInfo

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
UNSET = -7                                            # *d_written before the call
ALL = oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM | oracle.F_CONTENT_SIZE
CHECKS = {"none": 0, "block": oracle.F_BLOCK_CHECKSUMS, "content": oracle.F_CONTENT_CHECKSUM,
          "content_size": oracle.F_CONTENT_SIZE, "all": ALL}
BLOCK_SIZES = [BlockSize.Auto, BlockSize.Max64KB, BlockSize.Max256KB, BlockSize.Max1MB, BlockSize.Max4MB]


def _ptr(a):
    return a.ctypes.data if a.size else None


def _json(n: int) -> bytes:
    return corpus.tiled("compression_66k_JSON.txt", n).tobytes() if n else b""


def matrix_inputs():
    lens = [0, 1, 15, 16, 17, 4096, 65535, 65536, 65537, 262143, 262144, 262145, (1 << 20) + 7]
    ins = [(f"json{n}", _json(n)) for n in lens]
    ins += [("random300k", corpus.xorshift64star_bytes(300000).tobytes()), ("zeros1m", bytes(1 << 20)),
            ("json3m", _json(3 << 20)), ("dickens2m", corpus.load("dickens.txt")[:2 << 20])]
    return ins


@pytest.fixture(scope="module")
def inputs():
    return matrix_inputs()


def info_of(bs, flags: int, n: int, **kw) -> FrameInfo:
    return FrameInfo(block_size=BlockSize(int(bs)), block_checksums=bool(flags & oracle.F_BLOCK_CHECKSUMS),
                     content_checksum=bool(flags & oracle.F_CONTENT_CHECKSUM),
                     content_size=n if flags & oracle.F_CONTENT_SIZE else None, **kw)


def bound(ci, n: int) -> int:
    return _native.lib().lz4b200_frame_bound(n, C.byref(ci))


def host_compress(ctx, data: bytes, ci, first_write_len=None, cap=None):
    src = np.frombuffer(data, dtype=np.uint8)
    cap = bound(ci, src.size) if cap is None else cap
    out = np.empty(max(cap, 1), dtype=np.uint8)
    w = C.c_size_t(0)
    st = _native.lib().lz4b200_frame_compress(ctx.handle, _ptr(src), src.size, C.byref(ci),
                                              src.size if first_write_len is None else first_write_len,
                                              out.ctypes.data, cap, C.byref(w))
    return st, w.value, out[:w.value].tobytes()


def to_device(data: bytes, mis: int = 0):
    """data in a device buffer at byte offset `mis` from an aligned allocation."""
    buf = torch.zeros(len(data) + mis + 16, dtype=torch.uint8, device="cuda")
    if data:
        buf[mis:mis + len(data)] = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    return buf[mis:mis + len(data)]


def device_compress(ctx, data: bytes, ci, first_write_len=None, cap=None, mis_in=0, mis_out=0):
    """The device call on `data` at d_in offset mis_in into a sentinel-filled buffer at offset mis_out; checks that
    nothing outside the frame (and, after an error, nothing at all) was written.  Returns (status, written, frame)."""
    n = len(data)
    cap = bound(ci, n) if cap is None else cap
    d_in = to_device(data, mis_in)
    buf = torch.full((mis_out + cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_w = torch.full((1,), UNSET, dtype=torch.int64, device="cuda")
    st = _native.lib().lz4b200_frame_compress_device(
        ctx.handle, d_in.data_ptr() if n else None, n, C.byref(ci), n if first_write_len is None else first_write_len,
        buf[mis_out:].data_ptr(), cap, d_w.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    o = buf.cpu().numpy()
    w = int(d_w.item())
    if st != 0:
        assert w == UNSET and (o == SENTINEL).all(), "an argument error touched the output"
        return st, None, None
    assert (o[:mis_out] == SENTINEL).all() and (o[mis_out + w:] == SENTINEL).all(), "bytes outside the frame written"
    return st, w, o[mis_out:mis_out + w].tobytes()


def check(ctx, data: bytes, bs, flags: int, **kw) -> bytes:
    """Device call == host call == oracle; returns the frame."""
    ci = info_of(bs, flags, len(data)).to_c()
    hs, hw, hf = host_compress(ctx, data, ci)
    ds, dw, df = device_compress(ctx, data, ci, **kw)
    assert hs == ds == 0, (hs, ds)
    assert dw == hw
    assert df == hf
    assert df == oracle.frame_compress(data, int(bs), flags)
    return df


@pytest.mark.parametrize("checks", list(CHECKS))
@pytest.mark.parametrize("bs", BLOCK_SIZES)
def test_option_matrix(ctx, inputs, bs, checks):
    for name, data in inputs:
        try:
            check(ctx, data, bs, CHECKS[checks])
        except AssertionError as e:
            raise AssertionError(f"{name}: {e}") from e


def test_empty_frame_content_checksum(ctx):
    f = check(ctx, b"", BlockSize.Max64KB, oracle.F_CONTENT_CHECKSUM)
    assert f[-8:] == b"\0\0\0\0" + (0x02CC5D05).to_bytes(4, "little")


def test_auto_block_size_from_first_write_len(ctx):
    data = _json(50000)
    for first in (70000, 300000, 1, 50000):
        for flags in (0, ALL):
            ci = info_of(BlockSize.Auto, flags, len(data)).to_c()
            h = host_compress(ctx, data, ci, first)
            d = device_compress(ctx, data, ci, first)
            assert h[0] == 0 and d == h, first


def test_alignment(ctx):
    ins = [_json(17), _json(65537), corpus.xorshift64star_bytes(300000).tobytes(), _json((1 << 20) + 7)]
    for k in range(1, 16):
        for data in ins:
            for bs, flags in ((BlockSize.Max64KB, ALL), (BlockSize.Auto, oracle.F_CONTENT_CHECKSUM)):
                check(ctx, data, bs, flags, mis_in=k, mis_out=(5 * k) % 16)
        check(ctx, ins[1], BlockSize.Max256KB, ALL, mis_in=k, mis_out=k)


def test_errors_match_host(ctx):
    data = _json(100000)
    n = len(data)
    cases = {
        "linked": (FrameInfo(block_size=BlockSize.Max64KB, block_mode=BlockMode.Linked).to_c(), None),
        "content size": (FrameInfo(block_size=BlockSize.Max64KB, content_size=n + 1).to_c(), None),
        "cap": (info_of(BlockSize.Max64KB, ALL, n).to_c(), bound(info_of(BlockSize.Max64KB, ALL, n).to_c(), n) - 1),
    }
    for bad in (1, 8):
        ci = FrameInfo().to_c()
        ci.block_size_id = bad
        cases[f"block size id {bad}"] = (ci, 1 << 20)
    want = {"linked": 114, "content size": 109, "cap": 1, "block size id 1": 200, "block size id 8": 200}
    for name, (ci, cap) in cases.items():
        hs = host_compress(ctx, data, ci, cap=cap)[0]
        ds = device_compress(ctx, data, ci, cap=cap)[0]
        assert hs == ds == want[name], (name, hs, ds)
    # the Python wrapper raises what compress_frame raises
    d_in = to_device(data)
    for info in (FrameInfo(block_mode=BlockMode.Linked), FrameInfo(content_size=n - 1),
                 FrameInfo(block_size=BlockSize.Max8MB)):
        with pytest.raises(Exception) as want_e:
            frame.compress_frame(data, info, ctx)
        with pytest.raises(Exception) as got_e:
            frame.compress_frame_device(d_in, info, ctx=ctx)
        assert type(got_e.value) is type(want_e.value)
    with pytest.raises(errors.LinkedBlocksUnsupported):
        frame.compress_frame_device(d_in, FrameInfo(block_mode=BlockMode.Linked), ctx=ctx)
    info = FrameInfo(block_size=BlockSize.Max64KB)
    small = torch.empty(bound(info.to_c(), n) - 1, dtype=torch.uint8, device="cuda")
    with pytest.raises(errors.CompressOutputTooSmall):
        frame.compress_frame_device(d_in, info, out=small, ctx=ctx)


def test_streams_and_ordering(ctx):
    data = _json(3 << 20)
    info = FrameInfo(block_size=BlockSize.Max64KB, block_checksums=True, content_checksum=True, content_size=len(data))
    want = frame.compress_frame(data, info, ctx)
    d_in = to_device(data, 3)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    f = frame.compress_frame_device(d_in, info, ctx=ctx, stream=side.cuda_stream)
    assert f.cpu().numpy().tobytes() == want
    f = frame.compress_frame_device(d_in, info, ctx=ctx, stream=ctx.stream)
    assert f.cpu().numpy().tobytes() == want

    # two calls back to back on one context and stream, no synchronisation between them
    other = corpus.load("dickens.txt")[:(1 << 20) + 3]
    info2 = FrameInfo(block_size=BlockSize.Max256KB, block_checksums=True)
    d_other = to_device(other, 1)
    outs = [torch.full((bound(i.to_c(), len(x)) + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
            for i, x in ((info, data), (info2, other))]
    d_w = torch.zeros(2, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    L = _native.lib()
    for k, (x, d, i) in enumerate(((data, d_in, info), (other, d_other, info2))):
        ci = i.to_c()
        assert L.lz4b200_frame_compress_device(ctx.handle, d.data_ptr(), len(x), C.byref(ci), len(x),
                                               outs[k].data_ptr(), outs[k].numel() - 64,
                                               d_w[k:].data_ptr(), s) == 0
    torch.cuda.synchronize()
    w = d_w.tolist()
    assert outs[0][:w[0]].cpu().numpy().tobytes() == want
    assert outs[1][:w[1]].cpu().numpy().tobytes() == frame.compress_frame(other, info2, ctx)
    assert (outs[1][w[1]:] == SENTINEL).all()


def test_round_trip(ctx):
    for data in (_json(5 * 65536 + 777), corpus.load("dickens.txt")[:3 << 20], bytes(1 << 20),
                 corpus.adversarial_blocks(6, 0.5).tobytes()):
        for bs in (BlockSize.Max64KB, BlockSize.Max1MB):
            info = FrameInfo(block_size=bs, block_checksums=True, content_checksum=True, content_size=len(data))
            x = to_device(data, 7)
            f = frame.compress_frame_device(x, info, ctx=ctx)
            back = frame.decompress_frame_device(f, ctx=ctx)
            assert torch.equal(back, x)
            assert frame.decompress_frame(f.cpu().numpy().tobytes(), ctx) == data


def test_content_hash_lengths_and_offsets(ctx):
    rnd = corpus.xorshift64star_bytes((1 << 20) + 64).tobytes()
    buf = to_device(rnd)
    info = FrameInfo(block_size=BlockSize.Max64KB, content_checksum=True)
    for n in list(range(0, 301)) + [(1 << 20) + k for k in range(16)]:
        for off in range(16):
            f = frame.compress_frame_device(buf[off:off + n], info, ctx=ctx)
            got = int.from_bytes(f[-4:].cpu().numpy().tobytes(), "little")
            assert got == frame.xxh32(rnd[off:off + n]), (n, off)


def test_decoder_content_hash_carry(ctx):
    """Group outputs that end mid-stripe: the decoder carries the content hash state over them."""
    data = _json(3000000)
    _native.lib().lz4b200_ctx_set_frame_budget(ctx.handle, 1 << 20)
    try:
        for f in (oracle.frame_compress(data, 5, oracle.F_CONTENT_CHECKSUM, 9001),
                  oracle.frame_compress(data, 7, ALL, 150)):
            for g in (f, f[:-1] + bytes([f[-1] ^ 1])):
                d_out = torch.full((len(data) + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
                used, w, err = frame.decompress_next_frame_device(to_device(g, 5), d_out, ctx)
                hout, hused, herr = frame.decompress_next_frame(g, ctx)
                assert (used, w) == (hused, len(hout))
                assert type(err) is type(herr)
                assert d_out[:w].cpu().numpy().tobytes() == hout == data
    finally:
        _native.lib().lz4b200_ctx_set_frame_budget(ctx.handle, 256 << 20)


def test_full_size_json_1gib(ctx):
    data = corpus.tiled("compression_66k_JSON.txt", 1 << 30)
    info = FrameInfo(block_size=BlockSize.Max64KB, block_checksums=True, content_checksum=True, content_size=data.size)
    want = frame.compress_frame(data, info, ctx)
    x = torch.from_numpy(data).cuda()
    f = frame.compress_frame_device(x, info, ctx=ctx)
    assert f.numel() == len(want)
    assert torch.equal(f, torch.from_numpy(np.frombuffer(want, dtype=np.uint8).copy()).cuda())


def test_full_size_513_blocks_of_4mib(ctx):
    """The only whole frame that crosses the FRESH block at index 511 of a 4 MiB-block frame."""
    data = corpus.tiled("hdfs.json", 513 << 22)
    want = oracle.frame_compress(data, 7, ALL)
    info = FrameInfo(block_size=BlockSize.Max4MB, block_checksums=True, content_checksum=True, content_size=data.size)
    x = torch.from_numpy(data).cuda()
    f = frame.compress_frame_device(x, info, ctx=ctx)
    assert f.numel() == len(want)
    assert torch.equal(f, torch.from_numpy(np.frombuffer(want, dtype=np.uint8).copy()).cuda())
