"""GPU parity of the streaming device frame decoder (lz4b200_frame_decoder): presented in any chunks, with any out_cap
of at least the block size, it writes what lz4b200_frame_decompress_next writes for the same bytes and ends the frame
with the same result (consumed excepted after a block decode error: the end of the failing block and its checksum).
Also: nothing past `written` is touched, OUTPUT_FULL consumes nothing and changes nothing, the context's device memory
does not grow with the frame, other work on the context may come between two calls, and the Python wrappers raise
what the one-shot calls raise."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, block, corpus, errors, frame
from lz4_flex_b200.frame import BlockSize, FrameInfo
from stream_frames import broken_frames, linked_frame, random_splits, unit_ends, valid_frames

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
LEGACY = b"\x02\x21\x4c\x18"


def _ptr(a):
    return a.ctypes.data if a.size else None


def host_next(ctx, f: bytes):
    """lz4b200_frame_decompress_next with cap = the decoded bound: (status, consumed, written, block_status,
    err_expected, err_actual, bytes)."""
    L = _native.lib()
    src = np.frombuffer(f, dtype=np.uint8)
    b = C.c_size_t(0)
    assert L.lz4b200_frame_decoded_bound(_ptr(src), src.size, C.byref(b)) == 0
    out = np.zeros(max(b.value, 1), dtype=np.uint8)
    used, w, bs, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_uint64(0), C.c_uint64(0)
    st = L.lz4b200_frame_decompress_next(ctx.handle, _ptr(src), src.size, out.ctypes.data, b.value, C.byref(used),
                                         C.byref(w), C.byref(bs), C.byref(e1), C.byref(e2))
    return st, used.value, w.value, bs.value, e1.value, e2.value, out[:w.value].tobytes()


def block_size(f: bytes) -> int:
    if f[:4] == LEGACY:
        return 8 << 20
    if len(f) >= 6 and f[:4] == b"\x04\x22\x4d\x18" and (f[5] >> 4) & 7 >= 4:
        return 65536 << (2 * (((f[5] >> 4) & 7) - 4))
    return 4 << 20


class Decoder:
    def __init__(self, ctx):
        self.ctx = ctx
        self.h = C.c_void_p()
        assert _native.lib().lz4b200_frame_decoder_create(ctx.handle, C.byref(self.h)) == 0

    def close(self):
        _native.lib().lz4b200_frame_decoder_destroy(self.h)

    def call(self, d_in, eof, d_out, stream=None):
        s = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        step = _native.FrameDecoderStepC()
        n, cap = d_in.numel(), d_out.numel()
        st = _native.lib().lz4b200_frame_decoder_decode_device(self.h, d_in.data_ptr() if n else None, n, int(eof),
                                                                d_out.data_ptr() if cap else None, cap, C.byref(step), s)
        return st, step


def to_device(f: bytes, mis: int = 0):
    buf = torch.zeros(len(f) + mis + 16, dtype=torch.uint8, device="cuda")
    if f:
        buf[mis:mis + len(f)] = torch.from_numpy(np.frombuffer(f, dtype=np.uint8).copy()).cuda()
    return buf[mis:mis + len(f)]


def stream_decode(dec, f: bytes, splits, caps, mis_in=0, mis_out=0, stream=None, sentinel=True):
    """Presents f to the decoder in chunks ending at `splits` (end_of_input on the last), with out_cap from `caps`
    (a function of the call number).  Checks the bytes past `written` after every call.  Returns (bytes, result, sum
    of step.consumed, calls)."""
    d = to_device(f, mis_in)
    parts, pos, si, calls, consumed = [], 0, 0, 0, 0
    while True:
        cap = caps(calls)
        obuf = torch.full((cap + mis_out + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        end = splits[si]
        eof = si == len(splits) - 1
        st, step = dec.call(d[pos:end], eof, obuf[mis_out:mis_out + cap], stream)
        calls += 1
        assert st == 0, (st, calls)
        assert step.consumed <= end - pos and step.written <= cap
        if sentinel:
            assert bool((obuf[mis_out + step.written:] == SENTINEL).all()) and bool((obuf[:mis_out] == SENTINEL).all())
        if step.written:
            parts.append(obuf[mis_out:mis_out + step.written].cpu().numpy().tobytes())
        pos += step.consumed
        consumed += step.consumed
        if step.frame_done:
            r = step.result
            return b"".join(parts), (r.status, r.consumed, r.written, r.block_status, r.err_expected, r.err_actual), consumed, calls
        if step.need:
            assert not eof and step.need > end - pos
            si += 1
        else:
            assert step.consumed or step.written, "no progress"


def check(dec, ctx, f: bytes, splits, caps, **kw):
    h = host_next(ctx, f)
    got, r, consumed, calls = stream_decode(dec, f, splits, caps, **kw)
    assert got == h[6], (len(got), len(h[6]), r, h[:6])
    assert r[1] == consumed
    if h[0] == 101:
        assert r[0] == 101 and r[2:] == h[2:6]
        assert 0 < r[1] <= len(f)
    else:
        assert r == h[:6], (r, h[:6])
    return h, calls


@pytest.fixture(scope="module")
def dec(ctx):
    d = Decoder(ctx)
    yield d
    d.close()


def test_valid_frames_every_split(ctx, dec):
    rng = np.random.default_rng(1)
    for name, f in valid_frames():
        bs, n = block_size(f), len(f)
        ends = unit_ends(f)
        ends = ends if ends[-1] == n else ends + [n]
        h, _ = check(dec, ctx, f, [n], lambda i: bs)
        assert h[0] == 0, name
        check(dec, ctx, f, ends, lambda i: bs, mis_in=3, mis_out=5)
        caps = [bs + int(rng.integers(0, 3 * bs)) for _ in range(4096)]
        step = int(rng.choice([5000, 200000, 3 << 20])) if n > 100000 else int(rng.choice([7, 300]))
        check(dec, ctx, f, random_splits(n, rng, step), lambda i: caps[i % 4096],
              mis_in=int(rng.integers(0, 16)), mis_out=int(rng.integers(0, 16)))


def test_broken_and_mutated_frames(ctx, dec):
    rng = np.random.default_rng(2)
    seen = set()
    for name, f in broken_frames(seed=3, mutations=500):
        bs, n = block_size(f), len(f)
        step = int(rng.choice([1, 900, 70000])) if n < 20000 else int(rng.choice([900, 70000]))
        splits = [n] if rng.random() < 0.3 else random_splits(n, rng, step)
        h, _ = check(dec, ctx, f, splits, lambda i: bs + int(rng.integers(0, 2)) * bs)
        seen.add(h[0])
    assert {0, 101, 102, 106, 107, 108, 110, 111, 113} <= seen, seen
    check(dec, ctx, b"", [0], lambda i: 65536)                               # end of data: OK, 0, 0


def test_large_linked_frames_cross_block_matches(ctx, dec):
    dk = corpus.load("dickens.txt")
    data = dk[:5 << 20] + corpus.tiled("compression_66k_JSON.txt", 3 << 20).tobytes()
    rng = np.random.default_rng(4)
    for checks in (False, True):
        f = linked_frame(data, [65536, 20000, 7000, 1000, 40000, 65536, 300], 4, checks, checks, checks)
        h, calls = check(dec, ctx, f, random_splits(len(f), rng, 300000), lambda i: 65536)
        assert h[0] == 0 and h[6] == data and calls > 100
        check(dec, ctx, f, [len(f)], lambda i: int(rng.integers(65536, 3 << 20)), mis_out=7, sentinel=False)
    f = linked_frame(data[:3 << 20], [262144, 9000, 100000], 5, True, True, False)
    check(dec, ctx, f, random_splits(len(f), rng, 50000), lambda i: 262144 + int(rng.integers(0, 600000)))
    # many blocks per group and groups cut by a 1 MiB budget, the window carried between them
    _native.lib().lz4b200_ctx_set_frame_budget(ctx.handle, 1 << 20)
    try:
        f = linked_frame(data, [3000, 700, 20000], 4, True, True, True)
        check(dec, ctx, f, [len(f)], lambda i: 8 << 20, sentinel=False)
        g = bytearray(f)
        g[len(g) // 2] ^= 0x40                                                 # a corrupt block deep in the chain
        check(dec, ctx, bytes(g), random_splits(len(g), rng, 1 << 20), lambda i: 8 << 20, sentinel=False)
    finally:
        _native.lib().lz4b200_ctx_set_frame_budget(ctx.handle, 256 << 20)


def test_output_full_consumes_nothing(ctx, dec):
    j = corpus.tiled("compression_66k_JSON.txt", 900000).tobytes()
    for f in (oracle.frame_compress(j, 4, 7), linked_frame(j, [65536, 5000], 4, True, True, True)):
        want = host_next(ctx, f)
        d = to_device(f, 1)
        parts, pos, calls = [], 0, 0
        while True:
            calls += 1
            if calls % 3 == 0:                                                # too small for the next block
                small = torch.full((100,), SENTINEL, dtype=torch.uint8, device="cuda")
                st, step = dec.call(d[pos:], True, small)
                assert st == 115 and step.consumed == step.written == step.need == step.frame_done == 0
                assert bool((small == SENTINEL).all())
                continue
            out = torch.empty(65536 + 64 * calls, dtype=torch.uint8, device="cuda")
            st, step = dec.call(d[pos:], True, out)
            assert st == 0
            parts.append(out[:step.written].cpu().numpy().tobytes())
            pos += step.consumed
            if step.frame_done:
                break
        r = step.result
        assert b"".join(parts) == want[6] and (r.status, r.consumed, r.written) == want[:3]


def test_bounded_device_memory(ctx):
    budget = 4 << 20
    fresh = block.Context(0)                                                   # holds nothing but the decoder's scratch
    L = _native.lib()
    L.lz4b200_ctx_set_frame_budget(fresh.handle, budget)
    dec = Decoder(fresh)
    try:
        def run(f, src):
            d = to_device(f)
            out = torch.empty(4 << 20, dtype=torch.uint8, device="cuda")
            pos, off = 0, 0
            while True:
                end = min(len(f), pos + (1 << 20))
                st, step = dec.call(d[pos:end], end == len(f), out)
                assert st == 0
                if step.written:
                    assert torch.equal(out[:step.written], src[off:off + step.written])
                    off += step.written
                pos += step.consumed
                if step.frame_done:
                    assert step.result.status == 0 and off == src.numel()
                    return L.lz4b200_ctx_device_bytes(fresh.handle)

        big = corpus.tiled("hdfs.json", 512 << 20)
        src = torch.from_numpy(big).cuda()
        f_big = frame.compress_frame(big.tobytes(), FrameInfo(block_size=BlockSize.Max64KB), ctx=ctx)
        f_small = frame.compress_frame(big[:16 << 20].tobytes(), FrameInfo(block_size=BlockSize.Max64KB), ctx=ctx)
        small_bytes = run(f_small, src[:16 << 20])
        big_bytes = run(f_big, src)
        bound = 3 * (budget + (64 << 10)) + (4 << 20)                          # slots, staged input, descriptors
        assert big_bytes == small_bytes and big_bytes < bound, (small_bytes, big_bytes, bound)

        lin = corpus.load("dickens.txt")[:8 << 20] * 8
        lsrc = torch.from_numpy(np.frombuffer(lin, dtype=np.uint8).copy()).cuda()
        f_lin = linked_frame(lin, [65536, 30000], 4, True, True)
        f_lin16 = linked_frame(lin[:16 << 20], [65536, 30000], 4, True, True)
        l16 = run(f_lin16, lsrc[:16 << 20])
        l64 = run(f_lin, lsrc)
        assert l64 == l16 and l64 < bound, (l16, l64, bound)
    finally:
        dec.close()
        fresh.close()


def test_interleaved_decoders_and_other_work(ctx):
    j = corpus.tiled("compression_66k_JSON.txt", 2 << 20).tobytes()
    dk = corpus.load("dickens.txt")[:3 << 20]
    fa = linked_frame(dk, [65536, 9000, 30000], 4, True, True, True)
    fb = oracle.frame_compress(j, 5, 7)
    wa, wb = host_next(ctx, fa), host_next(ctx, fb)
    side = torch.cuda.Stream()
    for stream in (None, side.cuda_stream):
        da, db = Decoder(ctx), Decoder(ctx)
        ia, ib = to_device(fa, 3), to_device(fb)
        pa = pb = 0
        outs = {id(da): [], id(db): []}
        done = {id(da): None, id(db): None}
        blocks = [j[i:i + 65536] for i in range(0, 8 * 65536, 65536)]
        comp = [oracle.compress_block(b) for b in blocks]
        while done[id(da)] is None or done[id(db)] is None:
            for dec, d, key in ((da, ia, "a"), (db, ib, "b")):
                if done[id(dec)] is not None:
                    continue
                pos = pa if key == "a" else pb
                out = torch.empty(300000, dtype=torch.uint8, device="cuda")
                end = min(d.numel(), pos + 200000)
                st, step = dec.call(d[pos:end], end == d.numel(), out, stream)
                assert st == 0
                outs[id(dec)].append(out[:step.written].cpu().numpy().tobytes())
                if key == "a":
                    pa += step.consumed
                else:
                    pb += step.consumed
                if step.frame_done:
                    done[id(dec)] = step.result
                # other work on the same context between two calls: a frame batch and a block batch
                got = frame.decompress_frames_device(to_device(fb + fa), [0, len(fb)], [len(fb), len(fa)], ctx=ctx)
                assert got.frame(0)[2] is None
                o, status, _ = block.decompress_blocks(comp, [65536] * len(comp), ctx=ctx)
                assert not status.any() and o[3] == blocks[3]
        for dec, want, key in ((da, wa, id(da)), (db, wb, id(db))):
            r = done[key]
            assert b"".join(outs[key]) == want[6] and (r.status, r.consumed, r.written) == want[:3]
            dec.close()


def test_argument_errors_and_python_wrapper(ctx, dec):
    L = _native.lib()
    step = _native.FrameDecoderStepC()
    out = torch.empty(65536, dtype=torch.uint8, device="cuda")
    d = to_device(oracle.frame_compress(b"abc" * 1000, 4, 7))
    s = torch.cuda.current_stream().cuda_stream
    assert L.lz4b200_frame_decoder_decode_device(None, d.data_ptr(), d.numel(), 1, out.data_ptr(), 65536, C.byref(step), s) == 200
    assert L.lz4b200_frame_decoder_decode_device(dec.h, d.data_ptr(), d.numel(), 1, out.data_ptr(), 65536, None, s) == 200
    assert L.lz4b200_frame_decoder_decode_device(dec.h, None, 5, 1, out.data_ptr(), 65536, C.byref(step), s) == 200
    assert L.lz4b200_frame_decoder_decode_device(dec.h, d.data_ptr(), d.numel(), 1, None, 10, C.byref(step), s) == 200
    h = C.c_void_p()
    assert L.lz4b200_frame_decoder_create(None, C.byref(h)) == 200
    assert L.lz4b200_frame_decoder_create(ctx.handle, None) == 200
    assert L.lz4b200_ctx_device_bytes(None) == 0 and L.lz4b200_ctx_device_bytes(ctx.handle) > 0
    # the argument errors left the decoder untouched
    st, step = dec.call(d, True, out)
    assert st == 0 and step.frame_done and step.result.status == 0 and step.written == 3000

    # Python: DeviceFrameDecoder and iter_decompress_device against decompress_frame / decompress_next_frame_device
    j = corpus.tiled("compression_66k_JSON.txt", 1 << 20).tobytes()
    dk = corpus.load("dickens.txt")[:1 << 20]
    stream_bytes = (oracle.frame_compress(j, 4, 7) + linked_frame(dk, [65536, 4000], 4, True, True, True) +
                    corpus.load("dickens.lz4")[:300000] + oracle.frame_compress(b"", 4, 0))
    want = frame.decompress_frame(stream_bytes, ctx, partial=True)
    src = to_device(stream_bytes, 1)
    rng = np.random.default_rng(9)
    pos = [0]

    def read_into(buf):
        n = min(buf.numel(), src.numel() - pos[0], int(rng.integers(1, 3 << 20)))
        buf[:n] = src[pos[0]:pos[0] + n]
        pos[0] += n
        return n

    pieces, ends = [], 0
    with pytest.raises(errors.FrameError) as got:
        for view, done in frame.iter_decompress_device(read_into, ctx=ctx):
            pieces.append(view.cpu().numpy().tobytes())
            ends += done
    assert b"".join(pieces) == want[0] and ends >= 2 and type(got.value) is type(want[1])

    pdec = frame.DeviceFrameDecoder(ctx)
    fr = oracle.frame_compress(j, 4, 7)
    for g in (fr, fr[:100], bytes([fr[0] ^ 1]) + fr[1:], fr[:-1] + bytes([fr[-1] ^ 1]),
              linked_frame(dk, [5000], 4, False, True)[:-1] + b"\x01"):
        d_g = to_device(g, 2)
        out = torch.empty(max(len(j), 1 << 20), dtype=torch.uint8, device="cuda")
        used, w, err = frame.decompress_next_frame_device(d_g, out, ctx)
        want_bytes = out[:w].cpu().numpy().tobytes()
        pos_, parts = 0, []
        while True:
            o = torch.empty(65536, dtype=torch.uint8, device="cuda")
            c, wr, need, done, e = pdec.decode(d_g[pos_:], o, end_of_input=True)
            parts.append(o[:wr].cpu().numpy().tobytes())
            pos_ += c
            if done:
                break
        assert b"".join(parts) == want_bytes and pos_ == used
        assert type(e) is type(err) and str(e) == str(err)
    with pytest.raises(errors.IoError):
        pdec.decode(to_device(fr), torch.empty(10, dtype=torch.uint8, device="cuda"), end_of_input=True)
    pdec.close()
