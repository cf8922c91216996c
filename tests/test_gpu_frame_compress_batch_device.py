"""GPU parity of the batch frame encoder: lz4b200_frame_compress_batch_device writes, for every input of a batch, the
frame lz4b200_frame_compress writes for the same bytes (block size Auto resolved from the input's length, the content
size recorded per frame), which is the frame the C oracle (lz4_flex's FrameEncoder) writes.  The frames lie back to back
from d_out[0], d_frame_off holds their offsets and the total, nothing past the total is written, and after an argument
error neither d_out nor d_frame_off is touched."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, corpus, errors, frame
from lz4_flex_b200.frame import BlockMode, BlockSize, FrameInfo

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
UNSET = -7
ALL = oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM | oracle.F_CONTENT_SIZE
CHECKS = {"none": 0, "block": oracle.F_BLOCK_CHECKSUMS, "content": oracle.F_CONTENT_CHECKSUM,
          "content_size": oracle.F_CONTENT_SIZE, "all": ALL}
BLOCK_SIZES = [BlockSize.Auto, BlockSize.Max64KB, BlockSize.Max256KB, BlockSize.Max1MB, BlockSize.Max4MB]
INVALID, LINKED, TOO_SMALL = 200, 114, 1


def _json(n: int) -> bytes:
    return corpus.tiled("compression_66k_JSON.txt", n).tobytes() if n else b""


@pytest.fixture(scope="module")
def inputs():
    lens = [0, 1, 15, 16, 17, 4096, 65535, 65536, 65537, 262143, 262144, 262145, (1 << 20) + 7]
    ins = [_json(n) for n in lens]
    ins += [corpus.xorshift64star_bytes(300000).tobytes(), bytes(1 << 20), _json(3 << 20),
            corpus.load("dickens.txt")[:2 << 20]]
    return ins


def info_of(bs, flags: int) -> FrameInfo:
    """The shared FrameInfo; a content size of 0 only says 'record each frame's length'."""
    return FrameInfo(block_size=BlockSize(int(bs)), block_checksums=bool(flags & oracle.F_BLOCK_CHECKSUMS),
                     content_checksum=bool(flags & oracle.F_CONTENT_CHECKSUM),
                     content_size=0 if flags & oracle.F_CONTENT_SIZE else None)


def resolved(info: FrameInfo, n: int) -> FrameInfo:
    """info_f: Auto resolved from n, the content size set to n when the batch records sizes."""
    bs = BlockSize.from_buf_length(n) if info.block_size == BlockSize.Auto else info.block_size
    return FrameInfo(block_size=bs, block_checksums=info.block_checksums, content_checksum=info.content_checksum,
                     content_size=n if info.content_size is not None else None)


def bound(info: FrameInfo, n: int) -> int:
    ci = resolved(info, n).to_c()
    return _native.lib().lz4b200_frame_bound(n, C.byref(ci))


def host_frame(ctx, data: bytes, info: FrameInfo) -> bytes:
    ci = resolved(info, len(data)).to_c()
    src = np.frombuffer(data, dtype=np.uint8)
    cap = _native.lib().lz4b200_frame_bound(src.size, C.byref(ci))
    out = np.empty(cap, dtype=np.uint8)
    w = C.c_size_t(0)
    st = _native.lib().lz4b200_frame_compress(ctx.handle, src.ctypes.data if src.size else None, src.size,
                                              C.byref(ci), src.size, out.ctypes.data, cap, C.byref(w))
    assert st == 0, st
    return out[:w.value].tobytes()


class Batch:
    """The inputs in one device buffer, input i at an odd gap after input i - 1 (so most start unaligned), and a
    sentinel-filled output buffer whose base is `mis_out` bytes past an aligned allocation."""

    def __init__(self, datas, info: FrameInfo, mis_out: int = 0, cap=None, seed: int = 0):
        rng = np.random.default_rng(seed)
        self.datas, self.info = datas, info
        gaps = rng.integers(0, 16, size=len(datas))
        offs, pos = [], 0
        for d, g in zip(datas, gaps):
            pos += int(g)
            offs.append(pos)
            pos += len(d)
        self.off = np.array(offs, dtype=np.int64)
        self.len = np.array([len(d) for d in datas], dtype=np.int64)
        host = np.zeros(pos + 16, dtype=np.uint8)
        for d, o in zip(datas, offs):
            host[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
        self.d_in = torch.from_numpy(host).cuda()
        self.need = sum(bound(info, len(d)) for d in datas)
        self.cap = self.need if cap is None else cap
        self.mis_out = mis_out
        self.buf = torch.full((mis_out + self.cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.d_off = torch.full((len(datas) + 1,), UNSET, dtype=torch.int64, device="cuda")

    def enqueue(self, context, stream=None, **override):
        """The C call; `override` replaces any of its arguments by name."""
        ci = self.info.to_c()
        a = dict(ctx=context.handle, d_in=self.d_in.data_ptr(), in_off=self.off.ctypes.data, in_len=self.len.ctypes.data,
                 info=C.byref(ci), d_out=self.buf[self.mis_out:].data_ptr(), out_cap=self.cap,
                 d_frame_off=self.d_off.data_ptr(), nframes=len(self.datas),
                 stream=torch.cuda.current_stream().cuda_stream if stream is None else stream)
        a.update(override)
        return _native.lib().lz4b200_frame_compress_batch_device(*a.values())

    def result(self):
        """(frames, offsets) after a successful call; checks the packing and the sentinel."""
        torch.cuda.synchronize()
        offs = self.d_off.cpu().numpy()
        o = self.buf.cpu().numpy()
        total = int(offs[-1])
        assert offs[0] == 0 and (np.diff(offs) > 0).all() and total <= self.cap
        assert (o[:self.mis_out] == SENTINEL).all() and (o[self.mis_out + total:] == SENTINEL).all(), "past the total"
        body = o[self.mis_out:self.mis_out + total].tobytes()
        return [body[offs[i]:offs[i + 1]] for i in range(len(self.datas))], offs

    def untouched(self):
        torch.cuda.synchronize()
        assert (self.buf.cpu().numpy() == SENTINEL).all() and (self.d_off.cpu().numpy() == UNSET).all()


def check_batch(ctx, b: Batch, flags=None, bs=None, host=True):
    frames, offs = b.result()
    lens = []
    for i, (d, f) in enumerate(zip(b.datas, frames)):
        if host:
            assert f == host_frame(ctx, d, b.info), f"frame {i} ({len(d)} bytes) differs from the host call"
        if flags is not None:
            assert f == oracle.frame_compress(d, int(bs), flags), f"frame {i} ({len(d)} bytes) differs from the oracle"
        lens.append(len(f))
    assert offs.tolist() == [0] + np.cumsum(lens).tolist()
    return frames


def last_kernel(ctx) -> str:
    return _native.lib().lz4b200_ctx_last_kernel(ctx.handle, 0).decode()


@pytest.mark.parametrize("checks", list(CHECKS))
@pytest.mark.parametrize("bs", BLOCK_SIZES)
def test_option_matrix(ctx, inputs, bs, checks):
    b = Batch(inputs, info_of(bs, CHECKS[checks]), mis_out=int(bs) + len(checks))
    assert b.enqueue(ctx) == 0
    k = last_kernel(ctx)                           # before the host calls below launch their own
    if bs == BlockSize.Auto:                       # 64 KiB and 4 MiB blocks in one launch: both encoders run
        assert "split<unsigned short" in k and "split<unsigned int" in k, k
    check_batch(ctx, b, CHECKS[checks], bs)


def test_tiny_frames_shuffled(ctx):
    rng = np.random.default_rng(5)
    src = _json(1 << 20) + corpus.xorshift64star_bytes(1 << 20).tobytes()
    recs = []
    for _ in range(100000):
        n = int(rng.integers(0, 2049))
        o = int(rng.integers(0, len(src) - n))
        recs.append(src[o:o + n])
    info = info_of(BlockSize.Auto, oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM)
    b = Batch(recs, info, mis_out=3)
    assert b.enqueue(ctx) == 0
    assert last_kernel(ctx).startswith("lz4_compress_blocks_gtab<")    # > 24 blocks per SM: the global-table encoder
    first = check_batch(ctx, b, oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM, BlockSize.Auto, host=False)
    perm = rng.permutation(len(recs))
    b2 = Batch([recs[i] for i in perm], info, seed=1)
    assert b2.enqueue(ctx) == 0
    again, _ = b2.result()
    assert all(again[j] == first[i] for j, i in enumerate(perm))


def test_volume_16384_frames(ctx):
    n, bs = 16384, 65536
    data = _json(n * bs)
    datas = [data[i * bs:(i + 1) * bs] for i in range(n)]
    b = Batch(datas, info_of(BlockSize.Max64KB, ALL), mis_out=1)
    assert b.enqueue(ctx) == 0
    check_batch(ctx, b, ALL, BlockSize.Max64KB, host=False)


def test_table_epoch_is_frame_local(ctx):
    """A 513-block frame of 4 MiB blocks after frames with blocks: its block 511 is FRESH by its frame-local index (the
    batch index is 514)."""
    big = corpus.tiled("hdfs.json", 513 << 22)
    info = FrameInfo(block_size=BlockSize.Max4MB, block_checksums=True, content_checksum=True, content_size=0)
    small = [_json(5 << 20), b"", _json(3)]
    ci = resolved(info, big.size).to_c()
    want = np.empty(_native.lib().lz4b200_frame_bound(big.size, C.byref(ci)), dtype=np.uint8)
    w = C.c_size_t(0)
    assert _native.lib().lz4b200_frame_compress(ctx.handle, big.ctypes.data, big.size, C.byref(ci), big.size,
                                                want.ctypes.data, want.size, C.byref(w)) == 0
    d_big = torch.from_numpy(big).cuda()
    d_in = torch.cat([torch.from_numpy(np.frombuffer(b"".join(small), dtype=np.uint8).copy()).cuda(), d_big])
    lens = [len(s) for s in small] + [big.size]
    out, offs = frame.compress_frames_device(d_in, np.cumsum([0] + lens[:-1]), lens, info, ctx=ctx)
    offs = offs.tolist()
    for i, s in enumerate(small):
        assert out[offs[i]:offs[i + 1]].cpu().numpy().tobytes() == host_frame(ctx, s, info)
    assert offs[4] - offs[3] == w.value
    assert torch.equal(out[offs[3]:offs[4]], torch.from_numpy(want[:w.value]).cuda())


def test_back_to_back_and_side_stream(ctx, inputs):
    a = Batch(inputs, info_of(BlockSize.Max64KB, ALL), mis_out=5)
    b = Batch([_json(100000), b"", corpus.load("dickens.txt")[:(1 << 20) + 3]] * 3,
              info_of(BlockSize.Auto, oracle.F_CONTENT_CHECKSUM), mis_out=2, seed=9)
    torch.cuda.synchronize()
    assert a.enqueue(ctx) == 0 and b.enqueue(ctx) == 0          # no synchronisation between the two calls
    check_batch(ctx, a)
    check_batch(ctx, b)
    side = torch.cuda.Stream()
    c = Batch(inputs[::-1], info_of(BlockSize.Max256KB, oracle.F_BLOCK_CHECKSUMS), mis_out=7)
    torch.cuda.synchronize()
    assert c.enqueue(ctx, stream=side.cuda_stream) == 0
    side.synchronize()
    check_batch(ctx, c)


def test_device_round_trip(ctx, inputs):
    info = info_of(BlockSize.Auto, ALL)
    b = Batch(inputs, info, seed=3)
    assert b.enqueue(ctx) == 0
    torch.cuda.synchronize()
    total = int(b.d_off[-1].item())
    out = b.buf[:total]
    dec = frame.decompress_frames_device(out, b.d_off[:-1], b.d_off[1:] - b.d_off[:-1], ctx=ctx)
    for i, (view, used, err) in enumerate(dec):
        assert err is None and used == int(b.d_off[i + 1] - b.d_off[i])
        assert torch.equal(view, b.d_in[int(b.off[i]):int(b.off[i] + b.len[i])])


def test_argument_errors_in_order(ctx):
    datas = [_json(100000), b"", _json(70000)]
    info = info_of(BlockSize.Max64KB, ALL)
    lib = _native.lib()

    def status(finfo=info, cap=None, **override):
        b = Batch(datas, finfo, cap=cap)
        st = b.enqueue(ctx, **override)
        if st != 0:
            b.untouched()
        return st, b

    linked = FrameInfo(block_mode=BlockMode.Linked)
    bad_id = FrameInfo()
    bad_id.block_size = BlockSize.Max8MB
    assert status(ctx=None)[0] == INVALID
    assert status(info=None)[0] == INVALID
    assert status(d_frame_off=None)[0] == INVALID
    for k in ("in_off", "in_len", "d_out"):
        assert status(**{k: None})[0] == INVALID, k
    assert status(d_in=None)[0] == INVALID
    assert status(linked, d_in=None)[0] == INVALID                 # the null input is reported first
    assert status(linked)[0] == LINKED
    ci = linked.to_c()
    ci.block_size_id = 3
    assert status(linked, info=C.byref(ci))[0] == LINKED          # linked before the block size
    for bad in (1, 3, 8):
        ci = FrameInfo().to_c()
        ci.block_size_id = bad
        assert status(info=C.byref(ci), out_cap=0)[0] == INVALID, bad   # the block size before the capacity
    assert status(nframes=1 << 32, out_cap=0)[0] == INVALID
    huge = np.array([1 << 47, 1 << 47], dtype=np.int64)           # 2^32 blocks of 64 KiB
    zeros = np.zeros(3, dtype=np.int64)
    assert status(in_len=huge.ctypes.data, in_off=zeros.ctypes.data, nframes=2,
                  out_cap=0)[0] == INVALID
    need = Batch(datas, info).need
    assert status(cap=need - 1)[0] == TOO_SMALL
    st, b = status(cap=need)
    assert st == 0
    check_batch(ctx, b)

    # empty inputs need no d_in; nframes == 0 writes only the total
    st, b = status(d_in=None, in_len=zeros.ctypes.data)
    assert st == 0
    frames, _ = b.result()
    assert frames == [host_frame(ctx, b"", info)] * 3
    d_off = torch.full((1,), UNSET, dtype=torch.int64, device="cuda")
    ci = info.to_c()
    assert lib.lz4b200_frame_compress_batch_device(ctx.handle, None, None, None, C.byref(ci), None, 0,
                                                   d_off.data_ptr(), 0, torch.cuda.current_stream().cuda_stream) == 0
    assert d_off.item() == 0


def test_python_wrapper(ctx, inputs):
    datas = inputs[:9] + [inputs[-1]]
    lens = [len(d) for d in datas]
    offs = np.cumsum([0] + lens[:-1])
    d_in = torch.from_numpy(np.frombuffer(b"".join(datas), dtype=np.uint8).copy()).cuda()
    info = FrameInfo(block_checksums=True, content_checksum=True, content_size=12345)   # the value is ignored
    want = [frame.compress_frame(d, FrameInfo(block_checksums=True, content_checksum=True, content_size=len(d)), ctx)
            for d in datas]
    want_offs = np.cumsum([0] + [len(w) for w in want]).tolist()

    out, fo = frame.compress_frames_device(d_in, offs, lens, info, ctx=ctx)
    assert fo.is_cuda and fo.dtype == torch.int64 and fo.tolist() == want_offs
    assert out.cpu().numpy().tobytes() == b"".join(want)

    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):                                    # torch's current stream is the default
        out, fo = frame.compress_frames_device(d_in, torch.tensor(offs).cuda(), lens, info, ctx=ctx)
    side.synchronize()
    assert out.cpu().numpy().tobytes() == b"".join(want) and fo.tolist() == want_offs
    big = torch.full((sum(bound(info, n) for n in lens) + 100,), SENTINEL, dtype=torch.uint8, device="cuda")
    out, fo = frame.compress_frames_device(d_in, offs, lens, info, out=big, ctx=ctx, stream=side.cuda_stream)
    assert out.data_ptr() == big.data_ptr() and out.cpu().numpy().tobytes() == b"".join(want)
    assert (big[out.numel():] == SENTINEL).all()
    out, fo = frame.compress_frames_device(d_in, [], [], info, ctx=ctx)
    assert out.numel() == 0 and fo.tolist() == [0]

    for bad in (FrameInfo(block_mode=BlockMode.Linked), FrameInfo(block_size=BlockSize.Max8MB)):
        with pytest.raises(Exception) as want_e:
            frame.compress_frame(datas[1], bad, ctx)
        with pytest.raises(Exception) as got_e:
            frame.compress_frames_device(d_in, offs, lens, bad, ctx=ctx)
        assert type(got_e.value) is type(want_e.value)
    with pytest.raises(errors.LinkedBlocksUnsupported):
        frame.compress_frames_device(d_in, offs, lens, FrameInfo(block_mode=BlockMode.Linked), ctx=ctx)
    small = torch.empty(want_offs[-1], dtype=torch.uint8, device="cuda")
    with pytest.raises(errors.CompressOutputTooSmall):
        frame.compress_frames_device(d_in, offs, lens, info, out=small, ctx=ctx)
    with pytest.raises(ValueError):
        frame.compress_frames_device(d_in, [0], [d_in.numel() + 1], info, ctx=ctx)
