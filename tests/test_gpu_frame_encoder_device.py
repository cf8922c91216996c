"""GPU tests of the streaming frame encoder over device memory (lz4b200_frame_encoder, frame.DeviceFrameEncoder).

For random sequences of writes, flushes and finishes, the concatenated bytes of the calls must equal both what
frame.FrameEncoder writes for the same sequence and what a CPU restatement of FrameEncoder (frame/compress.rs:173-404)
built on the C oracle's persistent table (oracle.FrameTable) and oracle.xxh32 writes.  Every call must stay within its
bound and leave the bytes past *d_written alone.  The file also covers a single write with FINISH against the one-shot
device call, the argument errors, misaligned buffers, asynchronous use (input overwritten after each call, a whole
sequence without a sync, a side stream, other work on the context in between), content-length errors, a round trip
through DeviceFrameDecoder, a frame that crosses the 2 GiB table reposition, and device memory that does not grow with
the stream."""
import ctypes as C
import io
import struct

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, block, corpus, frame
from lz4_flex_b200.errors import ContentLengthError, LinkedBlocksUnsupported
from lz4_flex_b200.frame import BlockMode, BlockSize, FrameInfo

pytestmark = pytest.mark.gpu

WRITE, FLUSH, FINISH = 0, 1, 2
OK, TOO_SMALL, CONTENT_LENGTH, LINKED, INVALID = 0, 1, 109, 114, 200
SENTINEL = 0xA5
UNSET = -7
SIZES = {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20}
MiB = 1 << 20


# ---- fixtures --------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def sources():
    n = 6 * MiB
    return {
        "json": corpus.tiled("compression_66k_JSON.txt", n).tobytes(),
        "dickens": corpus.load("dickens.txt")[:n],
        "random": corpus.xorshift64star_bytes(2 * MiB).tobytes() * 3,
        "zeros": bytes(n),
    }


def to_device(data: bytes, mis: int = 0):
    buf = torch.zeros(len(data) + mis + 16, dtype=torch.uint8, device="cuda")
    if data:
        buf[mis:mis + len(data)] = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    return buf[mis:mis + len(data)]


def info_of(bsid, bc=False, cc=False, content_size=None):
    return FrameInfo(block_size=BlockSize(bsid), block_checksums=bool(bc), content_checksum=bool(cc),
                     content_size=content_size)


class Enc:
    """The C ABI of one encoder, driven directly."""

    def __init__(self, ctx, info: FrameInfo):
        self.L = _native.lib()
        h = C.c_void_p()
        ci = info.to_c()
        assert self.L.lz4b200_frame_encoder_create(ctx.handle, C.byref(ci), C.byref(h)) == OK
        self.h = h

    def bound(self, n, op):
        return self.L.lz4b200_frame_encoder_bound(self.h, n, op)

    def call(self, d_in, op, out, cap, d_written, stream=None):
        s = torch.cuda.current_stream().cuda_stream if stream is None else stream
        n = d_in.numel() if d_in is not None else 0
        return self.L.lz4b200_frame_encoder_encode_device(self.h, d_in.data_ptr() if n else None, n, op,
                                                          out.data_ptr() if out is not None else None, cap,
                                                          d_written.data_ptr() if d_written is not None else None, s)

    def checked(self, data: bytes, op, mis_in=0, mis_out=0, cap=None):
        """One call into a sentinel-filled buffer; checks the bound and the bytes past *d_written.  Returns
        (status, bytes written)."""
        n = len(data)
        b = self.bound(n, op)
        cap = b if cap is None else cap
        d_in = to_device(data, mis_in)
        buf = torch.full((mis_out + cap + 32,), SENTINEL, dtype=torch.uint8, device="cuda")
        d_w = torch.full((1,), UNSET, dtype=torch.int64, device="cuda")
        st = self.call(d_in, op, buf[mis_out:], cap, d_w)
        torch.cuda.synchronize()
        o = buf.cpu().numpy()
        w = int(d_w.item())
        if st not in (OK, CONTENT_LENGTH):
            assert w == UNSET and (o == SENTINEL).all(), "an error reported before enqueueing touched the output"
            return st, None
        assert 0 <= w <= b, (w, b)
        assert (o[:mis_out] == SENTINEL).all() and (o[mis_out + w:] == SENTINEL).all(), "bytes past *d_written written"
        return st, o[mis_out:mis_out + w].tobytes()

    def close(self):
        self.L.lz4b200_frame_encoder_destroy(self.h)


def host_encoder_run(ctx, info: FrameInfo, ops):
    """frame.FrameEncoder over the same sequence: the bytes after each call, and each call's error (or None)."""
    w = io.BytesIO()
    e = frame.FrameEncoder(w, FrameInfo(**vars(info)), ctx=ctx)
    outs, errs = [], []
    for data, op in ops:
        start = w.tell()
        err = None
        e.write_all(data)
        try:
            if op == FLUSH:
                e.flush()
            elif op == FINISH:
                e.try_finish()
        except ContentLengthError as x:
            err = (x.expected, x.actual)
        outs.append(w.getvalue()[start:])
        errs.append(err)
    return outs, errs


class OracleEncoder:
    """FrameEncoder (compress.rs:173-404) restated over oracle.FrameTable and oracle.xxh32, independent of liblz4b200."""

    def __init__(self, info: FrameInfo):
        self.bsid = int(info.block_size)
        self.bc, self.cc, self.cs = info.block_checksums, info.content_checksum, info.content_size
        self.open = self.written = False
        self.src = bytearray()
        self.content, self.clen = [], 0
        self.table = oracle.FrameTable()
        self.out = bytearray()

    def header(self):
        flg = 0x40 | 0x20 | (0x10 if self.bc else 0) | (0x08 if self.cs is not None else 0) | (0x04 if self.cc else 0)
        h = struct.pack("<IBB", 0x184D2204, flg, self.bsid << 4)
        if self.cs is not None:
            h += struct.pack("<Q", self.cs)
        return h + bytes([(oracle.xxh32(h[4:]) >> 8) & 0xFF])

    def begin(self, n):
        self.open = True
        if self.bsid == 0:
            self.bsid = 7 if n > 256 << 10 else 5 if n > 64 << 10 else 4
        self.out += self.header()
        if self.clen:
            self.content, self.clen, self.src, self.table = [], 0, bytearray(), oracle.FrameTable()

    def write_block(self):
        src = bytes(self.src)
        c = self.table.compress(src, SIZES[self.bsid])
        if len(c) < len(src):
            self.out += struct.pack("<I", len(c)) + c
            payload = c
        else:
            self.out += struct.pack("<I", len(src) | 0x80000000) + src
            payload = src
        if self.bc:
            self.out += struct.pack("<I", oracle.xxh32(payload))
        self.content.append(src)
        self.clen += len(src)
        self.src = bytearray()

    def write(self, data):
        if not self.open and data:
            self.begin(len(data))
        data = memoryview(data)
        while len(data):
            room = SIZES[self.bsid] - len(self.src)
            if room == 0:
                self.write_block()
                continue
            self.src += data[:room]
            data = data[room:]

    def flush(self):
        if self.src:
            self.write_block()

    def finish(self):
        self.flush()
        if not self.open and not self.written:
            self.begin(0)
        self.open = False
        if self.cs is not None and self.cs != self.clen:
            return (self.cs, self.clen)
        self.out += b"\0\0\0\0"
        if self.cc:
            self.out += struct.pack("<I", oracle.xxh32(b"".join(self.content)))
        self.written = True
        return None

    def run(self, ops):
        errs = []
        for data, op in ops:
            self.write(data)
            err = None
            if op == FLUSH:
                self.flush()
            elif op == FINISH:
                err = self.finish()
            errs.append(err)
        return bytes(self.out), errs


def random_ops(rng, src: bytes, bs: int, total_cap: int):
    ops, pos = [], int(rng.integers(0, 1000))
    for _ in range(int(rng.integers(1, 9))):
        r = rng.random()
        if r < 0.12:
            n = 0
        elif r < 0.22:
            n = 1
        elif r < 0.5:
            n = int(rng.choice([bs - 1, bs, bs + 1, 2 * bs + 3]))
        else:
            n = int(rng.integers(0, 3 * bs))
        n = min(n, total_cap)
        if pos + n > len(src):
            pos = 0
        data = src[pos:pos + n]
        pos += n
        q = rng.random()
        ops.append((data, WRITE if q < 0.5 else FLUSH if q < 0.75 else FINISH))
    return ops


def run_device(ctx, info, ops, **kw):
    enc = Enc(ctx, info)
    try:
        outs, errs = [], []
        for data, op in ops:
            st, got = enc.checked(data, op, **kw)
            assert st in (OK, CONTENT_LENGTH), st
            outs.append(got)
            errs.append(st == CONTENT_LENGTH)
        return outs, errs
    finally:
        enc.close()


def check_sequence(ctx, info, ops, **kw):
    if ops[-1][1] == WRITE:
        # after a write each encoder may still hold blocks the others have written: end on a flush
        ops = ops + [(b"", FLUSH)]
    outs, errs = run_device(ctx, info, ops, **kw)
    h_outs, h_errs = host_encoder_run(ctx, info, ops)
    o_bytes, o_errs = OracleEncoder(FrameInfo(**vars(info))).run(ops)
    got = b"".join(outs)
    assert errs == [e is not None for e in h_errs] == [e is not None for e in o_errs]
    assert got == b"".join(h_outs), "differs from frame.FrameEncoder"
    assert got == o_bytes, "differs from the oracle restatement"
    # at every flush or finish both have written everything
    acc_d = acc_h = b""
    for (data, op), d, h in zip(ops, outs, h_outs):
        acc_d += d
        acc_h += h
        if op != WRITE:
            assert acc_d == acc_h
    return got


# ---- sequences -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["json", "dickens", "random", "zeros"])
def test_random_sequences(ctx, sources, name):
    rng = np.random.default_rng({"json": 1, "dickens": 2, "random": 3, "zeros": 4}[name])
    small = block.Context(0)
    _native.lib().lz4b200_ctx_set_frame_budget(small.handle, 1 << 20)     # 7 blocks of 64 KiB per group
    try:
        for i in range(24):
            bsid = [0, 4, 5, 6, 7][i % 5]
            bc, cc = bool(i & 1), bool(i & 2)
            bs = SIZES[bsid] if bsid else int(rng.choice([64 << 10, 300 << 10]))
            ops = random_ops(rng, sources[name], min(bs, 1 << 20), 5 * MiB)
            total = sum(len(d) for d, _ in ops)
            cs = None
            if i % 6 == 5:
                cs = total if rng.random() < 0.5 else total + 1
            info = info_of(bsid, bc, cc, cs)
            check_sequence(small if i % 3 == 0 else ctx, info, ops)
    finally:
        small.close()


def test_quirks(ctx, sources):
    j = sources["json"]
    seqs = [
        (info_of(0, cc=True), [(b"", FINISH), (b"", FINISH), (j[:300 << 10], WRITE), (b"", FINISH), (j[:5], FINISH)]),
        (info_of(0, bc=True, content_size=10), [(b"", FINISH), (j[:10], WRITE), (b"", FINISH), (b"", FINISH),
                                                (j[:11], FINISH), (j[:10], FINISH)]),
        (info_of(5), [(b"", WRITE), (b"", FLUSH), (j[:1], WRITE), (b"", FLUSH), (b"", FLUSH), (j[:3 << 20], FINISH)]),
    ]
    for info, ops in seqs:
        check_sequence(ctx, info, ops)


def test_one_write_finish_equals_one_shot(ctx, sources):
    lens = [0, 1, 17, 65535, 65536, 65537, 262145, (1 << 20) + 7, 3 << 20]
    ins = [sources["json"][:n] for n in lens] + [sources["random"][:300000], sources["zeros"][:1 << 20],
                                                  sources["dickens"][:2 << 20]]
    L = _native.lib()
    for bsid in (0, 4, 5, 6, 7):
        for bc, cc, has_cs in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1)):
            for data in ins:
                info = info_of(bsid, bc, cc, len(data) if has_cs else None)
                enc = Enc(ctx, info)
                st, got = enc.checked(data, FINISH)
                enc.close()
                ci = info.to_c()
                cap = L.lz4b200_frame_bound(len(data), C.byref(ci))
                out = torch.empty(cap, dtype=torch.uint8, device="cuda")
                d_w = torch.empty(1, dtype=torch.int64, device="cuda")
                d_in = to_device(data)
                assert L.lz4b200_frame_compress_device(ctx.handle, d_in.data_ptr() if data else None, len(data),
                                                       C.byref(ci), len(data), out.data_ptr(), cap, d_w.data_ptr(),
                                                       torch.cuda.current_stream().cuda_stream) == OK
                assert st == OK and got == out[:int(d_w.item())].cpu().numpy().tobytes(), (bsid, bc, cc, len(data))


# ---- errors and buffers ----------------------------------------------------------------------------------------------

def test_output_too_small_changes_nothing(ctx, sources):
    j = sources["json"]
    info = info_of(4, True, True)
    ops = [(j[:100000], WRITE), (j[100000:250000], FLUSH), (j[250000:250001], WRITE), (j[250001:400000], FINISH),
           (j[:70000], FINISH)]
    enc = Enc(ctx, info)
    outs = []
    for data, op in ops:
        b = enc.bound(len(data), op)
        if b:
            st, got = enc.checked(data, op, cap=b - 1)
            assert st == TOO_SMALL and got is None
        st, got = enc.checked(data, op)
        assert st == OK
        outs.append(got)
    enc.close()
    assert b"".join(outs) == OracleEncoder(info).run(ops)[0]


def test_argument_errors_in_order(ctx):
    L = _native.lib()
    h = C.c_void_p()
    ci = info_of(4).to_c()
    assert L.lz4b200_frame_encoder_create(None, C.byref(ci), C.byref(h)) == INVALID
    assert L.lz4b200_frame_encoder_create(ctx.handle, None, C.byref(h)) == INVALID
    assert L.lz4b200_frame_encoder_create(ctx.handle, C.byref(ci), None) == INVALID
    for bad in (1, 3, 8, -1):
        b = FrameInfo(block_size=BlockSize.Max64KB).to_c()
        b.block_size_id = bad
        assert L.lz4b200_frame_encoder_create(ctx.handle, C.byref(b), C.byref(h)) == INVALID
    lk = FrameInfo(block_mode=BlockMode.Linked).to_c()
    assert L.lz4b200_frame_encoder_create(ctx.handle, C.byref(lk), C.byref(h)) == LINKED
    lk.block_size_id = 3                                              # the linked check comes first
    assert L.lz4b200_frame_encoder_create(ctx.handle, C.byref(lk), C.byref(h)) == LINKED
    with pytest.raises(LinkedBlocksUnsupported):
        frame.DeviceFrameEncoder(FrameInfo(block_mode=BlockMode.Linked), ctx=ctx)

    enc = Enc(ctx, info_of(4, cc=True))
    d_in = to_device(b"x" * 1000)
    out = torch.full((4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_w = torch.full((1,), UNSET, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    E = L.lz4b200_frame_encoder_encode_device
    assert E(None, d_in.data_ptr(), 1000, WRITE, out.data_ptr(), 4096, d_w.data_ptr(), s) == INVALID
    assert E(enc.h, d_in.data_ptr(), 1000, WRITE, out.data_ptr(), 4096, None, s) == INVALID
    assert E(enc.h, d_in.data_ptr(), 1000, WRITE, None, 4096, d_w.data_ptr(), s) == INVALID
    assert E(enc.h, None, 1000, 7, None, 4096, d_w.data_ptr(), s) == INVALID        # null d_out before the rest
    assert E(enc.h, None, 1000, 7, out.data_ptr(), 4096, d_w.data_ptr(), s) == INVALID
    assert E(enc.h, d_in.data_ptr(), 1000, 3, out.data_ptr(), 4096, d_w.data_ptr(), s) == INVALID
    assert E(enc.h, d_in.data_ptr(), 1000, -1, out.data_ptr(), 4096, d_w.data_ptr(), s) == INVALID
    assert E(enc.h, d_in.data_ptr(), 1000, FINISH, out.data_ptr(), 7, d_w.data_ptr(), s) == TOO_SMALL
    assert L.lz4b200_frame_encoder_bound(None, 10, WRITE) == 0 and L.lz4b200_frame_encoder_bound(enc.h, 10, 3) == 0
    # a WRITE that completes no group and opens no frame may have no output buffer at all
    assert E(enc.h, d_in.data_ptr(), 1000, WRITE, out.data_ptr(), 4096, d_w.data_ptr(), s) == OK
    assert enc.bound(5, WRITE) == 0
    assert E(enc.h, d_in.data_ptr(), 5, WRITE, None, 0, d_w.data_ptr(), s) == OK
    torch.cuda.synchronize()
    assert int(d_w.item()) == 0
    st, got = enc.checked(b"", FINISH)
    assert st == OK and frame.decompress_frame(out[:7].cpu().numpy().tobytes() + got) == b"x" * 1005
    enc.close()


def test_misaligned_buffers(ctx, sources):
    j = sources["json"]
    r = sources["random"]
    for k in range(1, 16):
        ops = [(j[:70001 + k], WRITE), (r[:1000 * k], FLUSH), (j[5:200000], WRITE), (j[:3 + k], FINISH)]
        check_sequence(ctx, info_of(4 if k % 2 else 0, True, True), ops, mis_in=k, mis_out=(5 * k) % 16)


# ---- asynchronous use ------------------------------------------------------------------------------------------------

def test_no_sync_input_overwritten_side_stream(ctx, sources):
    """A whole sequence enqueued without a sync: each call's output to its own region, d_in overwritten on the stream
    right after each call, the lengths read at the end; on torch's stream and on a side stream."""
    j, d = sources["json"], sources["dickens"]
    ops = [(j[:300000], WRITE), (d[:70000], FLUSH), (j[7:1 << 20], WRITE), (b"", FLUSH), (d[:5], FINISH),
           (j[:2 << 20], WRITE), (d[100:400000], FINISH)]
    info = info_of(4, True, True)
    want = OracleEncoder(FrameInfo(**vars(info))).run(ops)[0]
    small = block.Context(0)
    _native.lib().lz4b200_ctx_set_frame_budget(small.handle, 1 << 20)
    side = torch.cuda.Stream()
    for c in (ctx, small):
        for stream in (None, side):
            enc = Enc(c, info)
            caps = []
            total_cap = 2 * sum(len(data) for data, _ in ops) + 4096 * len(ops)   # each byte is in one call's bound
            srcs = [to_device(data, 3) for data, _ in ops]
            torch.cuda.synchronize()
            with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
                s = torch.cuda.current_stream()
                out = torch.full((total_cap,), SENTINEL, dtype=torch.uint8, device="cuda")
                lens = torch.full((len(ops),), UNSET, dtype=torch.int64, device="cuda")
                pos = 0
                for i, ((data, op), src) in enumerate(zip(ops, srcs)):
                    b = enc.bound(len(data), op)
                    assert enc.call(src, op, out[pos:], b, lens[i:], s.cuda_stream) == OK
                    src.fill_(0x3C)                                    # the caller reuses d_in right away
                    caps.append(b)
                    pos += b
                s.synchronize()
            got_lens = lens.cpu().tolist()
            o = out.cpu().numpy()
            pieces, pos = [], 0
            for w, b in zip(got_lens, caps):
                assert 0 <= w <= b and (o[pos + w:pos + b] == SENTINEL).all()
                pieces.append(o[pos:pos + w].tobytes())
                pos += b
            assert b"".join(pieces) == want
            enc.close()
    small.close()


def test_interleaved_encoders_decoder_and_batch(ctx, sources):
    j, d = sources["json"], sources["dickens"]
    ia, ib = info_of(4, True, True), info_of(0, False, True)
    ops_a = [(j[:200000], WRITE), (j[200000:600000], FLUSH), (j[:1], WRITE), (j[9:900000], FINISH)]
    ops_b = [(d[:400000], WRITE), (b"", FLUSH), (d[5:700000], WRITE), (d[:3], FINISH)]
    want_a, want_b = OracleEncoder(ia).run(ops_a)[0], OracleEncoder(ib).run(ops_b)[0]
    fr = oracle.frame_compress(j[:1 << 20], 4, 3)
    dec = frame.DeviceFrameDecoder(ctx)
    ea, eb = frame.DeviceFrameEncoder(FrameInfo(**vars(ia)), ctx=ctx), frame.DeviceFrameEncoder(FrameInfo(**vars(ib)), ctx=ctx)
    got_a, got_b = [], []
    d_fr = to_device(fr)
    dec_out = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    dpos = 0
    for (da, oa), (db, ob) in zip(ops_a, ops_b):
        got_a.append(ea.write(to_device(da), flush=oa == FLUSH, finish=oa == FINISH).cpu().numpy().tobytes())
        consumed, written, need, done, err = dec.decode(d_fr[dpos:dpos + 300000], dec_out)
        assert err is None
        dpos += consumed
        got_b.append(eb.write(to_device(db), flush=ob == FLUSH, finish=ob == FINISH).cpu().numpy().tobytes())
        frames, offs = frame.compress_frames_device(to_device(j[:500000]), [0, 1000], [1000, 400000],
                                                    FrameInfo(block_checksums=True), ctx=ctx)
        o1, o2 = int(offs[1]), int(offs[2])
        assert frames[o1:o2].cpu().numpy().tobytes() == frame.compress_frame(j[1000:401000],
                                                                             FrameInfo(block_checksums=True), ctx=ctx)
    assert b"".join(got_a) == want_a and b"".join(got_b) == want_b
    ea.close(); eb.close(); dec.close()


# ---- Python wrapper, errors, round trip -------------------------------------------------------------------------------

def test_content_length_error_both_ways(ctx, sources):
    j = sources["json"]
    for cs, n in ((100000, 150000), (300000, 150000)):
        info = info_of(4, True, True, cs)
        enc = frame.DeviceFrameEncoder(FrameInfo(**vars(info)), ctx=ctx)
        first = enc.write(to_device(j[:70000])).cpu().numpy().tobytes()
        with pytest.raises(ContentLengthError) as ei:
            enc.write(to_device(j[70000:n]), finish=True)
        assert (ei.value.expected, ei.value.actual) == (cs, n)
        partial = ei.value.partial.cpu().numpy().tobytes()
        h_outs, h_errs = host_encoder_run(ctx, info, [(j[:70000], WRITE), (j[70000:n], FINISH)])
        assert h_errs == [None, (cs, n)]
        assert first + partial == b"".join(h_outs)
        # the frame is closed without an EndMark: the next write opens a new frame
        tail = enc.write(to_device(j[:cs]), finish=True).cpu().numpy().tobytes()
        assert frame.decompress_frame(tail) == j[:cs]
        enc.close()


def test_round_trip_through_device_decoder(ctx, sources):
    enc = frame.DeviceFrameEncoder(FrameInfo(block_size=BlockSize.Max256KB, block_checksums=True, content_checksum=True),
                                   ctx=ctx)
    src = sources["dickens"][:5 << 20]
    pieces = []
    for a in range(0, len(src), 777777):
        pieces.append(enc.write(to_device(src[a:a + 777777]), flush=a % 3 == 0))
    pieces.append(enc.finish())
    enc.close()
    f = torch.cat(pieces)
    assert frame.decompress_frame_device(f, ctx=ctx).cpu().numpy().tobytes() == src
    chunks = iter([f[i:i + (1 << 20)] for i in range(0, f.numel(), 1 << 20)])

    def read_into(buf):
        c = next(chunks, None)
        if c is None:
            return 0
        buf[:c.numel()] = c
        return c.numel()
    got = b"".join(v.cpu().numpy().tobytes() for v, _ in frame.iter_decompress_device(read_into, ctx=ctx))
    assert got == src


# ---- the 2 GiB reposition and bounded memory --------------------------------------------------------------------------

def pattern(start: int, n: int, json_dev):
    """Bytes [start, start + n) of the JSON fixture tiled without end, generated on the device."""
    idx = (torch.arange(start, start + n, dtype=torch.int64, device="cuda") % json_dev.numel())
    return json_dev[idx]


def test_reposition_after_early_flush(ctx, sources):
    bs, first = 64 << 10, 12345
    json_dev = to_device(corpus.load("compression_66k_JSON.txt"))
    info = FrameInfo(block_size=BlockSize.Max64KB, content_checksum=True)
    enc = frame.DeviceFrameEncoder(info, ctx=ctx)
    limit = 0x7FFFFFFF
    # block 0 is short, block b >= 1 starts at stream offset first + (b - 1) * bs; block K is the first whose offset
    # reaches the reposition (compress.rs:267), which the block index alone (K % fresh_period) does not predict
    K = next(b for b in range(1, 1 << 20) if first + (b - 1) * bs + bs + 65536 >= limit)
    total = first + (K + 2) * bs + 999                               # blocks 0 .. K + 3, the last one short
    parts = [enc.write(pattern(0, first, json_dev), flush=True)]
    pos, piece = first, 256 << 20
    while pos < total:
        n = min(piece, total - pos)
        parts.append(enc.write(pattern(pos, n, json_dev)))
        pos += n
    parts.append(enc.finish())
    enc.close()
    f = torch.cat(parts)
    # walk the BlockInfo chain on the host and compare the blocks around the reposition with the oracle's table
    h = f.cpu().numpy()
    o, offs = 7, []
    while True:
        word = int.from_bytes(h[o:o + 4].tobytes(), "little")
        if word == 0:
            break
        offs.append(o)
        o += 4 + (word & 0x7FFFFFFF)
    assert len(offs) == K + 4 and (o + 8) == h.size
    table = oracle.FrameTable()
    table.offset = first + (K - 3) * bs                              # the stream offset of block K - 2
    for b in range(K - 2, K + 3):
        raw = pattern(first + (b - 1) * bs, bs, json_dev).cpu().numpy().tobytes()
        c = table.compress(raw, bs)
        word = int.from_bytes(h[offs[b]:offs[b] + 4].tobytes(), "little")
        want = (struct.pack("<I", len(c)) + c) if len(c) < len(raw) else struct.pack("<I", len(raw) | 0x80000000) + raw
        assert h[offs[b]:offs[b] + 4 + (word & 0x7FFFFFFF)].tobytes() == want, b
    assert table.offset == 3 * bs                                    # the oracle repositioned at block K as well
    del h
    out = torch.empty(total + bs, dtype=torch.uint8, device="cuda")         # room for the last block's decoded bound
    dec = frame.DeviceFrameDecoder(ctx)
    consumed_all, written_all = 0, 0
    while True:
        consumed, written, need, done, err = dec.decode(f[consumed_all:], out[written_all:], end_of_input=True)
        assert err is None
        consumed_all += consumed
        written_all += written
        if done:
            break
    dec.close()
    assert written_all == total and consumed_all == f.numel()
    for a in range(0, total, 256 << 20):
        n = min(256 << 20, total - a)
        assert torch.equal(out[a:a + n], pattern(a, n, json_dev))


def test_device_memory_does_not_grow(ctx):
    L = _native.lib()
    piece = 64 << 20
    gen = torch.arange(piece, dtype=torch.int64, device="cuda")

    def stream_bytes(bsid, total):
        fresh = block.Context(0)
        L.lz4b200_ctx_set_frame_budget(fresh.handle, 16 << 20)
        enc = frame.DeviceFrameEncoder(FrameInfo(block_size=BlockSize(bsid)), ctx=fresh)
        out = torch.empty(piece + (16 << 20), dtype=torch.uint8, device="cuda")   # the piece, a buffered group, overhead
        nframe = 0
        for a in range(0, total, piece):
            d = ((gen + a) % 251).to(torch.uint8)                    # generated piece by piece, never all resident
            nframe += enc.write(d, out=out).numel()
        nframe += enc.finish(out=out).numel()
        torch.cuda.synchronize()
        b = L.lz4b200_ctx_device_bytes(fresh.handle)
        enc.close()
        fresh.close()
        assert nframe > 0
        return b

    for bsid in (4, 7):
        small, big = stream_bytes(bsid, 64 << 20), stream_bytes(bsid, 4 << 30)
        assert small == big, (bsid, small, big)
        assert big < 3 * (16 << 20), big
