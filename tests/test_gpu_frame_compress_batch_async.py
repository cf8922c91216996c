"""GPU tests of the sync-free batch frame encoder (lz4b200_frame_compress_batch_device_async and its linked form;
Python: frame.compress_frames_device_async, compress_linked_frames_device_async): every frame inside capacity is
byte-identical to the synchronous call's at the same place, the call returns while the stream still sleeps, it
replays in a CUDA graph on new inputs, it applies its three limits as a prefix rule, and it refuses bad arguments with
its outputs untouched."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, block, corpus, frame
from lz4_flex_b200.frame import BlockMode, BlockSize, FrameInfo
from test_gpu_enc_window import env_context
from test_gpu_frame_compress_batch_device import ALL, BLOCK_SIZES, CHECKS, bound, info_of, inputs  # noqa: F401

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
UNSET = -7
OK, TOO_SMALL, INVALID, LINKED = 0, 1, 200, 114
SIZE_MAX = (1 << 64) - 1
BS = {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20}


@pytest.fixture(scope="module")
def sync_ctx():
    c = block.Context(0)
    yield c
    c.close()


def linked_info(info: FrameInfo) -> FrameInfo:
    return FrameInfo(block_size=info.block_size, block_checksums=info.block_checksums,
                     content_checksum=info.content_checksum, content_size=info.content_size,
                     block_mode=BlockMode.Linked)


def frame_cost(info: FrameInfo, n: int):
    bsid = int(info.block_size) or (7 if n > 256 << 10 else 5 if n > 64 << 10 else 4)
    return -(-n // BS[bsid]), n, bound(info, n)


class Batch:
    """The inputs in one device buffer whose base is 3 bytes past an allocation, input i at an odd gap after input
    i - 1; device offsets and lengths; a sentinel-filled output whose base is `mis_out` bytes past an allocation."""

    def __init__(self, datas, info: FrameInfo, mis_out: int = 5, seed: int = 0, cap=None):
        rng = np.random.default_rng(seed)
        self.datas, self.info, self.n = datas, info, len(datas)
        offs, pos = [], 0
        for d, g in zip(datas, rng.integers(0, 16, size=len(datas))):
            pos += int(g)
            offs.append(pos)
            pos += len(d)
        self.off = np.array(offs, dtype=np.int64)
        self.len = np.array([len(d) for d in datas], dtype=np.int64)
        host = np.zeros(pos + 3 + 16, dtype=np.uint8)
        for d, o in zip(datas, offs):
            host[3 + o:3 + o + len(d)] = np.frombuffer(d, dtype=np.uint8)
        self.alloc = torch.from_numpy(host).cuda()
        self.d_in = self.alloc[3:3 + pos]
        self.d_off = torch.from_numpy(self.off).cuda()
        self.d_len = torch.from_numpy(self.len).cuda()
        self.need = sum(bound(info, len(d)) for d in datas)
        self.cap = self.need if cap is None else cap
        self.mis_out = mis_out

    def out(self):
        buf = torch.full((self.mis_out + self.cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        return buf, buf[self.mis_out:self.mis_out + self.cap]

    def sync(self, ctx, linked=False):
        """(bytes up to the total, frame offsets) of the synchronous call."""
        info = linked_info(self.info) if linked else self.info
        ci = info.to_c()
        buf = torch.empty(max(self.need, 1), dtype=torch.uint8, device="cuda")
        offs = torch.empty(self.n + 1, dtype=torch.int64, device="cuda")
        fn = (_native.lib().lz4b200_frame_compress_linked_batch_device if linked
              else _native.lib().lz4b200_frame_compress_batch_device)
        st = fn(ctx.handle, self.d_in.data_ptr(), self.off.ctypes.data, self.len.ctypes.data, C.byref(ci),
                buf.data_ptr(), self.need, offs.data_ptr(), self.n, ctx.stream)
        assert st == 0, st
        torch.cuda.synchronize()
        o = offs.cpu().numpy()
        return buf[:int(o[-1])].cpu().numpy().tobytes(), o

    def run(self, ctx, linked=False, **kw):
        buf, out = self.out()
        fn = frame.compress_linked_frames_device_async if linked else frame.compress_frames_device_async
        info = linked_info(self.info) if linked else self.info
        r = fn(self.d_in, self.d_off, self.d_len, out, frame_info=info, ctx=ctx, **kw)
        torch.cuda.synchronize()
        return buf, r


def check_full(b: Batch, buf, r, want):
    """Every frame compressed, the bytes and offsets of the synchronous call, nothing else written."""
    body, offs = want
    got_offs = r.frame_offsets.cpu().numpy()
    assert got_offs.tolist() == offs.tolist()
    assert (r.statuses.cpu().numpy() == OK).all()
    h = buf.cpu().numpy()
    assert (h[:b.mis_out] == SENTINEL).all() and (h[b.mis_out + len(body):] == SENTINEL).all(), "past the total"
    assert h[b.mis_out:b.mis_out + len(body)].tobytes() == body


@pytest.mark.parametrize("checks", list(CHECKS))
@pytest.mark.parametrize("bs", BLOCK_SIZES)
def test_matches_sync(ctx, sync_ctx, inputs, bs, checks):   # noqa: F811
    flags = CHECKS[checks]
    b = Batch(inputs, info_of(bs, flags), mis_out=1 + int(bs) % 7, seed=int(bs) * 11 + flags)
    want = b.sync(sync_ctx)
    buf, r = b.run(ctx)
    check_full(b, buf, r, want)
    body, offs = want
    for i, d in enumerate(b.datas):                                  # the oracle on the short ones
        if len(d) <= 300000:
            assert body[offs[i]:offs[i + 1]] == oracle.frame_compress(d, int(bs), flags), i


@pytest.mark.parametrize("checks", ["none", "all"])
@pytest.mark.parametrize("bs", BLOCK_SIZES)
def test_linked_matches_sync(ctx, sync_ctx, inputs, bs, checks):   # noqa: F811
    b = Batch(inputs, info_of(bs, CHECKS[checks]), mis_out=3, seed=int(bs) * 13)
    check_full(b, *b.run(ctx, linked=True), b.sync(sync_ctx, linked=True))


def test_does_not_wait(ctx, sync_ctx, inputs):   # noqa: F811
    b = Batch(inputs, info_of(BlockSize.Auto, ALL), seed=3)
    want = b.sync(sync_ctx)
    b.run(ctx)                                                        # warm the allocator's cache
    s = torch.cuda.Stream()
    buf, out = b.out()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)
        r = frame.compress_frames_device_async(b.d_in, b.d_off, b.d_len, out, frame_info=b.info, ctx=ctx)
        assert not s.query(), "the call waited for the device"
    s.synchronize()
    check_full(b, buf, r, want)
    # the C call itself, linked, on a stream that is still sleeping
    L = _native.lib()
    want = b.sync(sync_ctx, linked=True)
    n, mb, mi = b.n, frame.default_compress_max_blocks(b.d_in.numel(), b.n), b.d_in.numel()
    nbytes = L.lz4b200_frame_compress_batch_device_async_scratch(ctx.handle, n, mb, mi)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    offs = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    sts = torch.empty(n, dtype=torch.int32, device="cuda")
    buf, out = b.out()
    ci = linked_info(b.info).to_c()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)
        assert L.lz4b200_frame_compress_linked_batch_device_async(
            ctx.handle, b.d_in.data_ptr(), b.d_off.data_ptr(), b.d_len.data_ptr(), C.byref(ci), out.data_ptr(),
            out.numel(), offs.data_ptr(), sts.data_ptr(), n, mb, mi, scratch.data_ptr(), nbytes, s.cuda_stream) == 0
        assert not s.query(), "the call waited for the device"
    s.synchronize()
    check_full(b, buf, frame.CompressedFrames(out, offs, sts), want)


def _graph_batches():
    """Three batches of different contents, lengths, offsets and kinds of data."""
    j = corpus.tiled("compression_66k_JSON.txt", 4 << 20).tobytes()
    d = corpus.load("dickens.txt")
    rnd = corpus.xorshift64star_bytes(1 << 20).tobytes()
    a = [j[1000 * i: 1000 * i + 3000 + 25000 * i] for i in range(20)]
    bb = [d[70000 * i: 70000 * i + 5 + 61000 * (i % 7)] for i in range(20)]
    c = [(rnd if i % 2 else bytes(1 << 20))[: 17 * i * i] for i in range(20)]
    c[4] = b""
    return [a, bb, c]


def test_cuda_graph_replays_new_inputs(ctx, sync_ctx):
    info = info_of(BlockSize.Auto, ALL)
    batches = [Batch(x, info, seed=50 + k) for k, x in enumerate(_graph_batches())]
    wants = [x.sync(sync_ctx) for x in batches]
    n = batches[0].n
    in_total = max(x.d_in.numel() for x in batches)
    out_cap = frame.compress_out_cap(n, in_total, info)
    d_in = torch.zeros(in_total + 1, dtype=torch.uint8, device="cuda")[1:]              # unaligned
    d_off, d_len = (torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(2))
    buf = torch.full((out_cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    out = buf[:out_cap]

    def call():
        return frame.compress_frames_device_async(d_in, d_off, d_len, out, frame_info=info, ctx=ctx)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()                                                        # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="global"):
        r = call()

    def load(x):
        d_in.zero_()
        d_in[:x.d_in.numel()].copy_(x.d_in)
        d_off.copy_(x.d_off)
        d_len.copy_(x.d_len)
        buf.fill_(SENTINEL)

    def check(want):
        body, offs = want
        assert r.frame_offsets.cpu().numpy().tolist() == offs.tolist()
        assert (r.statuses.cpu().numpy() == OK).all()
        h = buf.cpu().numpy()
        assert h[:len(body)].tobytes() == body and (h[len(body):] == SENTINEL).all()

    for x, want in zip(batches, wants):
        load(x)
        g.replay()
        torch.cuda.synchronize()
        check(want)
    # a replay on a side stream while the same context compresses other frames synchronously on its own stream
    load(batches[1])
    torch.cuda.synchronize()
    other = batches[0]
    with torch.cuda.stream(side):
        g.replay()
    o_out, o_offs = frame.compress_frames_device(other.d_in, other.off, other.len, frame_info=info, ctx=ctx,
                                                 stream=ctx.stream)
    torch.cuda.synchronize()
    check(wants[1])
    assert o_out.cpu().numpy().tobytes() == wants[0][0] and o_offs.cpu().numpy().tolist() == wants[0][1].tolist()


def _rule(b: Batch, limits):
    """The statuses the capacity rule gives, restated."""
    sums, sts = [0, 0, 0], []
    for d in b.datas:
        sums = [s + c for s, c in zip(sums, frame_cost(b.info, len(d)))]
        sts.append(INVALID if sums[0] > limits[0] or sums[1] > limits[1] else TOO_SMALL if sums[2] > limits[2] else OK)
    return sts


@pytest.mark.parametrize("linked", [False, True])
@pytest.mark.parametrize("limit", ["max_blocks", "max_in_bytes", "out_cap"])
def test_capacity_prefix_rule(ctx, sync_ctx, inputs, limit, linked):   # noqa: F811
    info = info_of(BlockSize.Auto, ALL)
    b0 = Batch(inputs, info, seed=9)
    body, offs = b0.sync(sync_ctx, linked=linked)
    totals = [sum(c) for c in zip(*(frame_cost(info, len(d)) for d in inputs))]
    i = ["max_blocks", "max_in_bytes", "out_cap"].index(limit)
    seen = set()
    for t in (0, totals[i] - 1, totals[i]):
        limits = [totals[0], totals[1], b0.need]
        limits[i] = t
        b = Batch(inputs, info, seed=9, cap=limits[2])
        buf, r = b.run(ctx, linked=linked, max_blocks=limits[0], max_in_bytes=limits[1])
        sts = r.statuses.cpu().numpy().tolist()
        want_sts = _rule(b, limits)
        assert sts == want_sts
        seen |= set(sts)
        k = next((f for f, s in enumerate(sts) if s != OK), b.n)      # the first frame past capacity
        got_offs = r.frame_offsets.cpu().numpy()
        assert got_offs[:k + 1].tolist() == offs[:k + 1].tolist()
        assert (got_offs[k:] == offs[k]).all(), "frames past capacity have no bytes"
        h = buf.cpu().numpy()
        end = int(offs[k])
        assert h[b.mis_out:b.mis_out + end].tobytes() == body[:end]
        assert (h[:b.mis_out] == SENTINEL).all() and (h[b.mis_out + end:] == SENTINEL).all(), "past the end"
    assert OK in seen and (INVALID in seen or TOO_SMALL in seen)


def test_arguments(ctx):
    L = _native.lib()
    datas = [b"abc" * 100, b"", b"xyz" * 5000]
    b = Batch(datas, FrameInfo(block_size=BlockSize.Max64KB))
    n, mb, mi = b.n, 16, b.d_in.numel()
    nbytes = L.lz4b200_frame_compress_batch_device_async_scratch(ctx.handle, n, mb, mi)
    assert nbytes > 0
    assert L.lz4b200_frame_compress_batch_device_async_scratch(ctx.handle, 0, mb, mi) == 0
    assert L.lz4b200_frame_compress_batch_device_async_scratch(ctx.handle, 1 << 32, 1, 1) == SIZE_MAX
    assert L.lz4b200_frame_compress_batch_device_async_scratch(ctx.handle, 1, 1 << 32, 1) == SIZE_MAX
    assert L.lz4b200_frame_compress_batch_device_async_scratch(None, 1, 1, 1) == SIZE_MAX
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    buf, out = b.out()
    offs = torch.full((n + 1,), UNSET, dtype=torch.int64, device="cuda")
    sts = torch.full((n,), UNSET, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def call(linked=False, **kw):
        ci = kw.pop("ci", b.info.to_c())
        a = dict(ctx=ctx.handle, d_in=b.d_in.data_ptr(), d_in_off=b.d_off.data_ptr(), d_in_len=b.d_len.data_ptr(),
                 info=C.byref(ci), d_out=out.data_ptr(), out_cap=out.numel(), d_frame_off=offs.data_ptr(),
                 d_status=sts.data_ptr(), nframes=n, max_blocks=mb, max_in_bytes=mi, d_scratch=scratch.data_ptr(),
                 scratch_bytes=nbytes, stream=s)
        a.update(kw)
        fn = (L.lz4b200_frame_compress_linked_batch_device_async if linked
              else L.lz4b200_frame_compress_batch_device_async)
        return fn(*a.values())

    def info_c(**kw):
        ci = b.info.to_c()
        for k, v in kw.items():
            setattr(ci, k, v)
        return ci

    cases = [dict(ctx=None), dict(info=None), dict(d_frame_off=None)]
    cases += [{k: None} for k in ("d_in", "d_in_off", "d_in_len", "d_out", "d_status", "d_scratch")]   # out_cap > 0
    cases += [dict(nframes=1 << 32), dict(max_blocks=1 << 32), dict(scratch_bytes=nbytes - 1)]
    cases += [dict(ci=info_c(block_size_id=bad)) for bad in (1, 2, 3, 8, -1)]
    for kw in cases:
        assert call(**kw) == INVALID, kw
    assert call(ci=info_c(linked=1)) == LINKED
    assert call(linked=True) == INVALID                               # the linked form wants linked blocks
    assert call(linked=True, ci=info_c(linked=1, block_size_id=9)) == INVALID
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == SENTINEL).all()
    assert (offs.cpu().numpy() == UNSET).all() and (sts.cpu().numpy() == UNSET).all()
    # no frames: d_frame_off[0] = 0, the rest of the arrays may be null
    assert call(nframes=0, d_in=None, d_in_off=None, d_in_len=None, d_out=None, d_status=None, d_scratch=None,
                scratch_bytes=0) == OK
    torch.cuda.synchronize()
    assert offs.cpu().numpy().tolist() == [0] + [UNSET] * n
    # Python: out is required, frame_info must match the form
    with pytest.raises(ValueError):
        frame.compress_linked_frames_device_async(b.d_in, b.d_off, b.d_len, out, frame_info=b.info, ctx=ctx)
    with pytest.raises(ValueError):
        frame.compress_frames_device_async(b.d_in, b.d_off, b.d_len[:2], out, ctx=ctx)


def test_global_table_shape_in_scratch(sync_ctx):
    """LZ4B200_ENC_G16=871 keeps its tables in global memory: the scratch holds the region, and a batch of more than
    24 blocks per SM (which takes that encoder) matches the synchronous call."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    j = corpus.tiled("compression_66k_JSON.txt", 64 << 20).tobytes()
    n = sm * 24 + 300
    datas = [j[(i * 7919) % (60 << 20):(i * 7919) % (60 << 20) + 20000 + (i * 37) % 40000] for i in range(n)]
    b = Batch(datas, info_of(BlockSize.Max64KB, ALL), seed=12)
    want = b.sync(sync_ctx)
    L = _native.lib()
    plain = L.lz4b200_frame_compress_batch_device_async_scratch(sync_ctx.handle, n, n, b.d_in.numel())
    with env_context({"LZ4B200_ENC_G16": "871"}) as c:
        wide = L.lz4b200_frame_compress_batch_device_async_scratch(c.handle, n, n, b.d_in.numel())
        assert wide > plain
        buf, r = b.run(c, max_blocks=n)
        assert "gtabg<8, 7, 1>" in L.lz4b200_ctx_last_kernel(c.handle, 0).decode()
        check_full(b, buf, r, want)


def _scale(ctx, sync_ctx, datas, info, seed, linked=False):
    b = Batch(datas, info, seed=seed)
    want = b.sync(sync_ctx, linked=linked)
    buf, r = b.run(ctx, linked=linked)
    got_offs = r.frame_offsets.cpu().numpy()
    assert got_offs.tolist() == want[1].tolist()
    assert (r.statuses.cpu().numpy() == OK).all()
    total = len(want[0])
    assert torch.equal(buf[b.mis_out:b.mis_out + total].cpu(), torch.frombuffer(bytearray(want[0]), dtype=torch.uint8))
    assert (buf[b.mis_out + total:] == SENTINEL).all() and (buf[:b.mis_out] == SENTINEL).all()


def test_scale_single_block_json_frames(ctx, sync_ctx):
    data = corpus.tiled("compression_66k_JSON.txt", 16384 * 65536)
    _scale(ctx, sync_ctx, [data[i * 65536:(i + 1) * 65536].tobytes() for i in range(16384)],
           info_of(BlockSize.Max64KB, ALL), 71)


def test_scale_one_gib_auto(ctx, sync_ctx):
    data = corpus.tiled("compression_66k_JSON.txt", 1 << 30).tobytes()
    _scale(ctx, sync_ctx, [data], info_of(BlockSize.Auto, oracle.F_CONTENT_CHECKSUM | oracle.F_CONTENT_SIZE), 72)


def test_scale_linked_dickens_frames(ctx, sync_ctx):
    data = corpus.tiled("dickens.txt", 256 << 20)
    _scale(ctx, sync_ctx, [data[i << 20:(i + 1) << 20].tobytes() for i in range(256)],
           info_of(BlockSize.Max64KB, oracle.F_CONTENT_CHECKSUM), 73, linked=True)
