"""GPU parity of the sync-free batch frame decoder: lz4b200_frame_decompress_batch_device_async gives every frame what
lz4b200_frame_decompress_batch_device gives it on a context whose frame budget holds the frame in one group (every
result field and every written byte), writes nothing else of d_out, returns before the device has run, replays from
a CUDA graph on new inputs, and applies its block capacity as a prefix rule."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, block, corpus, frame
from stream_frames import broken_frames, linked_frame, valid_frames
from test_gpu_frame_batch_device import ALL, SENTINEL, host_bound, layout, linked_fixtures, mixed_cases, mutations

pytestmark = pytest.mark.gpu

INVALID = 200
CANARY_GAP = 64


@pytest.fixture(scope="module")
def sync_ctx():
    """The synchronous call's context: a frame budget that holds every frame here in one group."""
    c = block.Context(0)
    _native.lib().lz4b200_ctx_set_frame_budget(c.handle, 8 << 30)
    yield c
    c.close()


class Batch:
    """Frames laid out in one device input with gaps, and output regions of the given caps with canary gaps."""

    def __init__(self, frames, caps, seed=0, in_total=None, out_total=None):
        rng = np.random.default_rng(seed)
        self.n = len(frames)
        self.in_off, total = layout([len(f) for f in frames], rng, 0)
        h = np.full(max(in_total or total, total, 1), 0x5A, dtype=np.uint8)
        for f, o in zip(frames, self.in_off):
            h[o:o + len(f)] = np.frombuffer(f, dtype=np.uint8)
        self.h_in = h
        self.lens = [len(f) for f in frames]
        self.caps = list(caps)
        self.out_off, ototal = layout(self.caps, rng, CANARY_GAP)
        self.out_total = max(out_total or ototal, ototal)
        t = lambda v: torch.tensor(v, dtype=torch.int64, device="cuda")
        self.d_in = torch.from_numpy(h).cuda()
        self.d_off, self.d_len, self.d_ooff, self.d_cap = t(self.in_off), t(self.lens), t(self.out_off), t(self.caps)

    def out(self):
        return torch.full((self.out_total,), SENTINEL, dtype=torch.uint8, device="cuda")

    def sync(self, ctx):
        """lz4b200_frame_decompress_batch_device: (results, out)."""
        out = self.out()
        res = torch.full((max(self.n, 1), 5), -1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        st = _native.lib().lz4b200_frame_decompress_batch_device(
            ctx.handle, self.d_in.data_ptr(), self.d_off.data_ptr(), self.d_len.data_ptr(), out.data_ptr(),
            self.d_ooff.data_ptr(), self.d_cap.data_ptr(), res.data_ptr(), self.n, torch.cuda.current_stream().cuda_stream)
        assert st == 0, ctx.last_cuda_error()
        return res[:self.n], out

    def run_async(self, ctx, max_blocks=None, stream=None):
        out = self.out()
        r = frame.decompress_frames_device_async(self.d_in, self.d_off, self.d_len, out, self.d_ooff, self.d_cap,
                                                 max_blocks=max_blocks, ctx=ctx, stream=stream)
        torch.cuda.synchronize()
        return r.results, out


def written_mask(res, out_off, total):
    mask = np.ones(total, dtype=bool)
    for i, w in enumerate(res[:, 1].tolist()):
        mask[out_off[i]:out_off[i] + w] = False
    return mask


def check_same(b: Batch, got, want, host_canaries=True):
    """Every result field and every byte of the output buffer equal the synchronous call's; nothing of d_out outside
    the written bytes changed."""
    (rg, og), (rw, ow) = got, want
    assert torch.equal(rg, rw), [(i, rg[i].tolist(), rw[i].tolist()) for i in range(b.n) if not torch.equal(rg[i], rw[i])][:5]
    assert torch.equal(og, ow), "decoded bytes differ from the synchronous call's"
    if host_canaries:
        o = og.cpu().numpy()
        assert (o[written_mask(rg.cpu().numpy(), b.out_off, b.out_total)] == SENTINEL).all(), "bytes outside written"


def walk_blocks(ctx, b: Batch, first=0, count=1):
    """The blocks the walks of frames [first, first + count) record together (the batch index's count)."""
    total = C.c_size_t(0)
    assert _native.lib().lz4b200_frame_index_batch_device(
        ctx.handle, b.d_in.data_ptr(), b.d_off[first:].data_ptr(), b.d_len[first:].data_ptr(), count, None, 0,
        C.byref(total), None, None, torch.cuda.current_stream().cuda_stream) == 0
    return total.value


def _caps(cases):
    return [host_bound(f) if c is None else c for f, c in cases]


def test_mixed_matches_sync(ctx, sync_ctx):
    cases = mixed_cases() + [(f, None) for _, f in valid_frames()] + [(f, None) for _, f in broken_frames()]
    frames, caps = [f for f, _ in cases], _caps(cases)
    b = Batch(frames, caps, seed=1)
    want = b.sync(sync_ctx)
    statuses = set((want[0][:, 4] & 0xFFFFFFFF).tolist())
    assert {0, 101, 102, 107, 108, 109, 110, 111, 115}.issubset(statuses), statuses
    check_same(b, b.run_async(ctx, max_blocks=walk_blocks(ctx, b, 0, b.n)), want)   # flushed frames pass the default
    # caps of 0, one short and exact for every frame of the stream matrix
    vf = [f for _, f in valid_frames()]
    bounds = [host_bound(f) for f in vf]
    for k, pick in enumerate((lambda x: 0, lambda x: max(x - 1, 0), lambda x: x)):
        b = Batch(vf, [pick(x) for x in bounds], seed=10 + k)
        check_same(b, b.run_async(ctx, max_blocks=walk_blocks(ctx, b, 0, b.n)), b.sync(sync_ctx))


def test_mutations_match_sync(ctx, sync_ctx):
    frames = mutations(500, 77)
    good = oracle.frame_compress(corpus.tiled("compression_66k_JSON.txt", 200000).tobytes(), 4, ALL)
    mixed = [x for m in frames for x in (m, good)]
    b = Batch(mixed, [host_bound(f) for f in mixed], seed=2)
    want = b.sync(sync_ctx)
    assert len(set((want[0][:, 4] & 0xFFFFFFFF).tolist())) >= 4
    check_same(b, b.run_async(ctx), want)


def test_does_not_wait(ctx, sync_ctx):
    frames = [f for f, _ in mixed_cases()[::3]] + linked_fixtures()
    b = Batch(frames, [host_bound(f) for f in frames], seed=3)
    want = b.sync(sync_ctx)
    out = b.out()
    frame.decompress_frames_device_async(b.d_in, b.d_off, b.d_len, out, b.d_ooff, b.d_cap, ctx=ctx)   # warm the cache
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = b.out()
        torch.cuda._sleep(1 << 30)
        r = frame.decompress_frames_device_async(b.d_in, b.d_off, b.d_len, out, b.d_ooff, b.d_cap, ctx=ctx)
        assert not s.query(), "the call waited for the device"
    s.synchronize()
    check_same(b, (r.results, out), want)
    # the C call itself, on a stream that is still sleeping
    L = _native.lib()
    nbytes = L.lz4b200_frame_decompress_batch_device_async_scratch(b.n, frame.default_max_blocks(b.d_in.numel(), b.n))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    res = torch.empty((b.n, 5), dtype=torch.int64, device="cuda")
    out = b.out()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)
        assert L.lz4b200_frame_decompress_batch_device_async(
            ctx.handle, b.d_in.data_ptr(), b.d_off.data_ptr(), b.d_len.data_ptr(), out.data_ptr(), b.d_ooff.data_ptr(),
            b.d_cap.data_ptr(), res.data_ptr(), b.n, frame.default_max_blocks(b.d_in.numel(), b.n), scratch.data_ptr(),
            nbytes, s.cuda_stream) == 0
        assert not s.query(), "the call waited for the device"
    s.synchronize()
    check_same(b, (res, out), want)


def _batches(n):
    """Three batches of n frames each, of different kinds and sizes."""
    j = corpus.tiled("compression_66k_JSON.txt", 3 << 20).tobytes()
    d = corpus.load("dickens.txt")
    rng = np.random.default_rng(21)
    a = [oracle.frame_compress(j[: 1000 + 9000 * i], 4 + i % 2, ALL if i % 3 == 0 else 0) for i in range(n)]
    bb = [linked_frame(d[50000 * i: 50000 * i + 300000], [65536, 9000 + 100 * i], 4, i % 2 == 1, True, i % 3 == 0)
          for i in range(n)]
    c = mutations(n, 22)
    c[int(rng.integers(0, n))] = b""
    return [a, bb, c]


def test_cuda_graph_replays_new_inputs(ctx, sync_ctx):
    n = 24
    sets = _batches(n)
    first = [Batch(fr, [host_bound(f) for f in fr], seed=30 + k) for k, fr in enumerate(sets)]
    in_total = max(x.h_in.size for x in first)
    out_total = max(x.out_total for x in first)
    batches = [Batch(fr, x.caps, seed=30 + k, in_total=in_total, out_total=out_total)
               for k, (x, fr) in enumerate(zip(first, sets))]
    wants = [x.sync(sync_ctx) for x in batches]
    d_in = torch.zeros(in_total, dtype=torch.uint8, device="cuda")
    d_off, d_len, d_ooff, d_cap = (torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(4))
    out = torch.full((out_total,), SENTINEL, dtype=torch.uint8, device="cuda")
    max_blocks = frame.default_max_blocks(in_total, n)

    def call():
        return frame.decompress_frames_device_async(d_in, d_off, d_len, out, d_ooff, d_cap, max_blocks=max_blocks,
                                                    ctx=ctx)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()                                                          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="global"):
        r = call()

    def load(x):
        d_in.copy_(x.d_in)
        d_off.copy_(x.d_off)
        d_len.copy_(x.d_len)
        d_ooff.copy_(x.d_ooff)
        d_cap.copy_(x.d_cap)
        out.fill_(SENTINEL)

    for x, want in zip(batches, wants):
        load(x)
        g.replay()
        torch.cuda.synchronize()
        check_same(x, (r.results.clone(), out.clone()), want)
    # a replay on a second stream while the same context decodes other frames synchronously on its own stream
    load(batches[1])
    torch.cuda.synchronize()
    other = Batch(sets[0] + linked_fixtures(), batches[0].caps + [host_bound(f) for f in linked_fixtures()], seed=40)
    other_out = other.out()
    other_res = torch.full((other.n, 5), -1, dtype=torch.int64, device="cuda")
    with torch.cuda.stream(side):
        g.replay()
    st = _native.lib().lz4b200_frame_decompress_batch_device(
        ctx.handle, other.d_in.data_ptr(), other.d_off.data_ptr(), other.d_len.data_ptr(), other_out.data_ptr(),
        other.d_ooff.data_ptr(), other.d_cap.data_ptr(), other_res.data_ptr(), other.n, ctx.stream)
    assert st == 0
    torch.cuda.synchronize()
    check_same(batches[1], (r.results.clone(), out.clone()), wants[1])
    check_same(other, (other_res, other_out), other.sync(sync_ctx))


def test_capacity_prefix_rule(ctx, sync_ctx):
    cases = mixed_cases()[::3] + [(f, None) for f in linked_fixtures()]
    frames, caps = [f for f, _ in cases], _caps(cases)
    b = Batch(frames, caps, seed=50)
    rw, ow = b.sync(sync_ctx)
    counts = [walk_blocks(ctx, b, i) for i in range(b.n)]
    total = sum(counts)
    assert total > 0 and counts[-1] > 0
    incl = np.cumsum(counts)
    for cap in (0, total - 1, total):
        rg, og = b.run_async(ctx, max_blocks=cap)
        inside = incl <= cap
        assert inside.any() and (cap == total) == inside.all()
        rgh, rwh = rg.cpu().numpy(), rw.cpu().numpy()
        o, w = og.cpu().numpy(), ow.cpu().numpy()
        for i in range(b.n):
            region = slice(b.out_off[i], b.out_off[i] + b.caps[i])
            if inside[i]:
                assert (rgh[i] == rwh[i]).all(), (cap, i)
                assert (o[region][:rwh[i, 1]] == w[region][:rwh[i, 1]]).all(), (cap, i)
            else:
                assert rgh[i].tolist() == [0, 0, 0, 0, INVALID], (cap, i, rgh[i])
        assert (o[written_mask(rgh, b.out_off, b.out_total)] == SENTINEL).all(), cap
        if cap == total:
            check_same(b, (rg, og), (rw, ow), host_canaries=False)


def test_arguments(ctx):
    L = _native.lib()
    j = corpus.load("compression_66k_JSON.txt")
    fr = [oracle.frame_compress(j, 4, ALL)] * 3
    b = Batch(fr, [host_bound(f) for f in fr], seed=60)
    nb = L.lz4b200_frame_decompress_batch_device_async_scratch(3, 10)
    assert nb > 0 and L.lz4b200_frame_decompress_batch_device_async_scratch(0, 10) == 0
    assert L.lz4b200_frame_decompress_batch_device_async_scratch(1 << 32, 1) == (1 << 64) - 1
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    out = b.out()
    res = torch.full((3, 5), 7, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    args = [ctx.handle, b.d_in.data_ptr(), b.d_off.data_ptr(), b.d_len.data_ptr(), out.data_ptr(), b.d_ooff.data_ptr(),
            b.d_cap.data_ptr(), res.data_ptr()]
    call = lambda a, n=3, mb=10, sp=scratch.data_ptr(), sb=nb: L.lz4b200_frame_decompress_batch_device_async(
        *a, n, mb, sp, sb, s)
    assert call(args, sb=nb - 1) == INVALID
    assert call([None] + args[1:]) == INVALID
    for k in range(1, 8):
        a = list(args)
        a[k] = None
        assert call(a) == INVALID, k
        assert call(a, n=0, sp=None, sb=0) == 0, k
    assert call(args, sp=None) == INVALID
    assert call(args, n=1 << 32) == INVALID
    assert call(args, mb=1 << 32) == INVALID
    torch.cuda.synchronize()
    assert (res == 7).all() and (out == SENTINEL).all()
    assert call(args) == 0
    torch.cuda.synchronize()
    assert (res[:, 4] == 0).all() and (res[:, 1] == len(j)).all()


def _scale(ctx, sync_ctx, frames, seed):
    b = Batch(frames, [host_bound(f) for f in frames], seed=seed)
    want = b.sync(sync_ctx)
    got = b.run_async(ctx)
    assert (want[0][:, 4] == 0).all()
    check_same(b, got, want, host_canaries=False)
    mask = torch.from_numpy(written_mask(got[0].cpu().numpy(), b.out_off, b.out_total)).cuda()
    assert (got[1][mask] == SENTINEL).all()


def test_scale_one_gib_frame(ctx, sync_ctx):
    data = corpus.tiled("compression_66k_JSON.txt", 1 << 30).tobytes()
    _scale(ctx, sync_ctx, [oracle.frame_compress(data, 4, oracle.F_CONTENT_CHECKSUM)], 70)


def test_scale_single_block_frames(ctx, sync_ctx):
    data = corpus.tiled("compression_66k_JSON.txt", 16384 * 65536)
    _scale(ctx, sync_ctx, [oracle.frame_compress(data[i * 65536:(i + 1) * 65536].tobytes(), 4, ALL)
                           for i in range(16384)], 71)


def test_scale_linked_dickens_frames(ctx, sync_ctx):
    data = corpus.tiled("dickens.txt", 256 << 20)
    _scale(ctx, sync_ctx, [linked_frame(data[i << 20:(i + 1) << 20].tobytes(), [65536], 4, False, True)
                           for i in range(256)], 72)
