"""GPU parity of the size-prepended batch calls.  lz4b200_compress_prepend_size_batch_device writes, for every input of a
batch, the record lz4b200_compress_prepend_size writes (the oracle's compress_prepend_size), records back to back with
their offsets and the total in d_rec_off.  lz4b200_decompress_size_prepended_batch_device gives every record the status,
length, `expected` and bytes of the one-record call (the oracle's decompress_size_prepended), laid out by the running sum
of the length words, without synchronising the host.  Argument errors leave every output untouched."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, block, corpus
import vectors
from dict_cases import dict_cases

pytestmark = pytest.mark.gpu

SENT = 0xA5
UNSET = -7
TOO_SMALL, EAB, INVALID = 1, 4, 200
L = _native.lib


def _json(n: int) -> bytes:
    return corpus.tiled("compression_66k_JSON.txt", n).tobytes() if n else b""


def _kind(kind: str, n: int) -> bytes:
    if kind == "json":
        return _json(n)
    if kind == "random":
        return corpus.xorshift64star_bytes(n).tobytes() if n else b""
    if kind == "zeros":
        return bytes(n)
    return corpus.tiled("dickens.txt", n).tobytes() if n else b""


def u64(v):
    return torch.from_numpy(np.asarray(v, dtype=np.uint64).reshape(-1).view(np.int64).copy()).cuda()


def u32(v):
    return torch.from_numpy(np.asarray(v, dtype=np.int64).reshape(-1).astype(np.uint32).view(np.int32).copy()).cuda()


def pack(datas, seed: int = 0):
    """The inputs in one device buffer, each after a gap of 1..15 bytes, so they start at every alignment."""
    rng = np.random.default_rng(seed)
    parts, offs, pos = [], [], 0
    for d in datas:
        g = int(rng.integers(1, 16))
        parts.append(bytes(g))
        offs.append(pos + g)
        parts.append(bytes(d))
        pos += g + len(d)
    parts.append(bytes(16))
    return torch.from_numpy(np.frombuffer(b"".join(parts), dtype=np.uint8).copy()).cuda(), offs


def ptr(t):
    return t.data_ptr() if t is not None and t.numel() else None


def last_kernel(ctx, which: int) -> str:
    return L().lz4b200_ctx_last_kernel(ctx.handle, which).decode()


class Comp:
    """One compress call's arguments and sentinel-filled outputs; `out` is `mis` bytes into its allocation."""

    def __init__(self, datas, out_cap=None, max_in_len=None, dict_t=None, seed=0, mis=3):
        self.datas = datas
        self.n = len(datas)
        self.d_in, offs = pack(datas, seed)
        self.offs, self.lens = u64(offs), u32([len(d) for d in datas])
        self.max_in_len = max((len(d) for d in datas), default=0) if max_in_len is None else max_in_len
        bound = sum(4 + oracle.max_output_size(len(d)) for d in datas)
        self.out_cap = bound if out_cap is None else out_cap
        self.mis = mis
        self.buf = torch.full((max(bound, self.out_cap) + mis + 64,), SENT, dtype=torch.uint8, device="cuda")
        self.out = self.buf[mis:mis + self.out_cap]
        self.rec_off = torch.full((self.n + 2,), UNSET, dtype=torch.int64, device="cuda")
        self.status = torch.full((self.n + 1,), UNSET, dtype=torch.int32, device="cuda")
        self.dict_t = dict_t

    def enqueue(self, context, stream=None, **o):
        a = dict(ctx=context.handle, d_in=ptr(self.d_in), in_off=ptr(self.offs), in_len=ptr(self.lens), n=self.n,
                 max_in_len=self.max_in_len, d_out=ptr(self.out), out_cap=self.out_cap, rec_off=ptr(self.rec_off),
                 status=ptr(self.status), stream=stream if stream is not None else torch.cuda.current_stream().cuda_stream)
        a.update(o)
        head = (a["ctx"], a["d_in"], a["in_off"], a["in_len"], a["n"], a["max_in_len"])
        tail = (a["d_out"], a["out_cap"], a["rec_off"], a["status"], a["stream"])
        if self.dict_t is None and "dict" not in a:
            return L().lz4b200_compress_prepend_size_batch_device(*head, *tail)
        d = a.get("dict", (ptr(self.dict_t), self.dict_t.numel() if self.dict_t is not None else 0))
        return L().lz4b200_compress_prepend_size_batch_device_with_dict(*head, *d, *tail)

    def result(self):
        torch.cuda.synchronize()
        return (self.buf.cpu().numpy(), self.rec_off.cpu().numpy(), self.status.cpu().numpy())


def expected_record(data: bytes, dic=None) -> bytes:
    body = oracle.compress_block(data) if dic is None else oracle.compress_with_dict(data, dic)
    return len(data).to_bytes(4, "little") + body


def check_compress(c: Comp, ctx, dic=None, host=False, run=True):
    if run:
        assert c.enqueue(ctx) == 0
    buf, rec_off, status = c.result()
    n, m = c.n, c.mis
    assert (status[:n] == 0).all(), status[:n]
    assert status[n] == UNSET and rec_off[n + 1] == UNSET
    pos = 0
    for b, d in enumerate(c.datas):
        want = expected_record(d, dic)
        assert rec_off[b] == pos, b
        got = buf[m + pos: m + pos + len(want)].tobytes()
        assert got == want, (b, len(d))
        if host:
            assert got == block.compress_prepend_size(d, ctx=ctx), b
        pos += len(want)
    assert rec_off[n] == pos
    assert (buf[:m] == SENT).all() and (buf[m + pos:] == SENT).all()
    return rec_off


# ---- compress ----------------------------------------------------------------------------------------------------

LENGTHS = [0, 1, 12, 13, 15, 16, 4096, 65534, 65535, 65536, 65537, 262145, (1 << 20) + 7]


def test_compress_parity(ctx):
    datas = [_kind(k, n) for k in ("json", "random", "zeros", "dickens") for n in LENGTHS]
    check_compress(Comp(datas, seed=1), ctx, host=True)


def test_compress_small_blocks_only(ctx):
    # every block <= 64 KiB: the bound keeps the large-block encoder from running
    datas = [_kind(k, n) for k in ("json", "random", "dickens") for n in (0, 1, 13, 100, 4096, 65536)] * 3
    check_compress(Comp(datas, seed=2), ctx, host=True)


def test_compress_dict_cases(ctx):
    others = [_json(5000), _kind("random", 3000), b"", _kind("dickens", 70000)]
    for name, inp, dic in dict_cases():
        datas = [inp] + others
        dict_t = torch.from_numpy(np.frombuffer(dic, dtype=np.uint8).copy()).cuda()
        c = Comp(datas, dict_t=dict_t, seed=len(name))
        rec_off = check_compress(c, ctx, dic)
        recs = c.out[:int(rec_off[c.n])]
        out, out_off, out_len, status, exp = block.decompress_size_prepended_device(
            recs, u64(rec_off[:c.n]), u32(np.diff(rec_off[:c.n + 1])), ext_dict=dict_t, ctx=ctx)
        host = out.cpu().numpy()
        assert (status.cpu().numpy() == 0).all(), name
        offs = out_off.cpu().numpy()
        for b, d in enumerate(datas):
            assert host[offs[b]:offs[b] + len(d)].tobytes() == d, (name, b)


def test_compress_full_size_round_trip(ctx):
    n, bs = 16384, 65536
    src = torch.from_numpy(corpus.tiled("compression_66k_JSON.txt", n * bs)).cuda()
    offs = torch.arange(n, dtype=torch.int64, device="cuda") * bs
    out, rec_off, status = block.compress_prepend_size_device(src, offs, [bs] * n, ctx=ctx)
    torch.cuda.synchronize()
    assert (status.cpu().numpy() == 0).all()
    ro = rec_off.cpu().numpy()
    host_out, host_src = out.cpu().numpy(), src.cpu().numpy()
    for b in range(n):
        assert host_out[ro[b]:ro[b + 1]].tobytes() == expected_record(host_src[b * bs:(b + 1) * bs]), b
    dec, out_off, out_len, dstat, _ = block.decompress_size_prepended_device(
        out, rec_off[:n], rec_off[1:] - rec_off[:n], out=torch.empty(n * bs, dtype=torch.uint8, device="cuda"), ctx=ctx)
    torch.cuda.synchronize()
    assert (dstat == 0).all().item() and (out_len == bs).all().item()
    assert torch.equal(out_off, torch.arange(n + 1, dtype=torch.int64, device="cuda") * bs)
    assert torch.equal(dec, src)


def test_compress_capacity_edges(ctx):
    datas = [_kind(k, n) for k in ("json", "random") for n in (0, 7, 4096, 65536, 70000)]
    full = Comp(datas, seed=3)
    rec_off = check_compress(full, ctx)
    need = int(rec_off[full.n])
    for cap in (need - 1, 0, int(rec_off[4]) + 2, int(rec_off[7])):
        c = Comp(datas, out_cap=cap, seed=3)
        assert c.enqueue(ctx) == 0
        buf, ro, st = c.result()
        assert (ro[:c.n + 1] == rec_off[:c.n + 1]).all(), cap
        for b in range(c.n):
            fits = rec_off[b + 1] <= cap
            assert st[b] == (0 if fits else TOO_SMALL), (cap, b)
            region = buf[c.mis + rec_off[b]: c.mis + rec_off[b + 1]]
            if fits:
                assert region.tobytes() == expected_record(datas[b]), (cap, b)
            else:
                assert (region == SENT).all(), (cap, b)
        assert (buf[:c.mis] == SENT).all()


def test_compress_block_above_max_in_len(ctx):
    for datas, bound in (([_json(100), _json(5000), _json(70000), _json(200)], 5000),        # small encoder only
                         ([_json(100), _json(300000), _json(70000), b""], 100000)):
        c = Comp(datas, max_in_len=bound, seed=4)
        assert c.enqueue(ctx) == 0
        buf, ro, st = c.result()
        pos = 0
        for b, d in enumerate(datas):
            assert ro[b] == pos
            if len(d) > bound:
                assert st[b] == TOO_SMALL
                continue
            want = expected_record(d)
            assert st[b] == 0 and buf[c.mis + pos: c.mis + pos + len(want)].tobytes() == want
            pos += len(want)
        assert ro[len(datas)] == pos and (buf[c.mis + pos:] == SENT).all()


# ---- decompress ----------------------------------------------------------------------------------------------------

def host_one(ctx, rec: bytes, dic=None):
    """lz4b200_decompress_size_prepended(_with_dict) on one record: (status, bytes, expected)."""
    src = np.frombuffer(rec, dtype=np.uint8) if rec else np.zeros(1, np.uint8)
    want = int.from_bytes(rec[:4], "little") if len(rec) >= 4 else 0
    out = np.zeros(max(want, 1), dtype=np.uint8)
    w, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    args = (ctx.handle, src.ctypes.data, len(rec))
    tail = (out.ctypes.data, want, C.byref(w), C.byref(e1), C.byref(e2))
    if dic is None:
        st = L().lz4b200_decompress_size_prepended(*args, *tail)
    else:
        d = np.frombuffer(dic, dtype=np.uint8) if dic else np.zeros(1, np.uint8)
        st = L().lz4b200_decompress_size_prepended_with_dict(*args, d.ctypes.data, len(dic), *tail)
    return st, out[:w.value].tobytes(), e1.value


def oracle_one(rec: bytes, dic=None):
    if dic is None:
        st, out, e1, _ = oracle.decompress_size_prepended(rec)
    elif len(rec) < 4:
        st, out, e1 = EAB, b"", 0
    else:
        st, out, e1, _ = oracle.decompress_with_dict(rec[4:], int.from_bytes(rec[:4], "little"), dic)
    return st, out, (e1 if st == 2 else 0)


class Dec:
    """One decompress call over `recs`, the output `mis` bytes into a sentinel-filled allocation."""

    def __init__(self, recs, out_cap=None, dic=None, seed=0, mis=5):
        self.recs, self.n, self.dic = recs, len(recs), dic
        self.d_in, offs = pack(recs, seed)
        self.offs, self.lens = u64(offs), u32([len(r) for r in recs])
        self.sizes = [int.from_bytes(r[:4], "little") if len(r) >= 4 else 0 for r in recs]
        self.total = sum(self.sizes)
        self.out_cap = self.total if out_cap is None else out_cap
        self.mis = mis
        self.buf = torch.full((max(self.total, self.out_cap) + mis + 64,), SENT, dtype=torch.uint8, device="cuda")
        self.out = self.buf[mis:mis + self.out_cap]
        self.out_off = torch.full((self.n + 2,), UNSET, dtype=torch.int64, device="cuda")
        self.out_len = torch.full((self.n + 1,), UNSET, dtype=torch.int32, device="cuda")
        self.status = torch.full((self.n + 1,), UNSET, dtype=torch.int32, device="cuda")
        self.expected = torch.full((self.n + 1,), UNSET, dtype=torch.int64, device="cuda")
        self.dict_t = None if dic is None else torch.from_numpy(np.frombuffer(dic, dtype=np.uint8).copy()).cuda()

    def enqueue(self, context, stream=None, **o):
        a = dict(ctx=context.handle, d_in=ptr(self.d_in), rec_off=ptr(self.offs), rec_len=ptr(self.lens), n=self.n,
                 d_out=ptr(self.out), out_cap=self.out_cap, out_off=ptr(self.out_off), out_len=ptr(self.out_len),
                 status=ptr(self.status), expected=ptr(self.expected),
                 stream=stream if stream is not None else torch.cuda.current_stream().cuda_stream)
        a.update(o)
        head = (a["ctx"], a["d_in"], a["rec_off"], a["rec_len"], a["n"])
        tail = (a["d_out"], a["out_cap"], a["out_off"], a["out_len"], a["status"], a["expected"], a["stream"])
        if self.dict_t is None and "dict" not in a:
            return L().lz4b200_decompress_size_prepended_batch_device(*head, *tail)
        d = a.get("dict", (ptr(self.dict_t), self.dict_t.numel() if self.dict_t is not None else 0))
        return L().lz4b200_decompress_size_prepended_batch_device_with_dict(*head, *d, *tail)

    def result(self):
        torch.cuda.synchronize()
        return tuple(t.cpu().numpy() for t in (self.buf, self.out_off, self.out_len, self.status, self.expected))


def check_decompress(ctx, d: Dec, host=True, run=True):
    if run:
        assert d.enqueue(ctx) == 0
    buf, out_off, out_len, status, expected = d.result()
    n, m = d.n, d.mis
    assert out_off[n] == d.total and out_off[n + 1] == UNSET
    assert status[n] == UNSET and out_len[n] == UNSET and expected[n] == UNSET
    pos = 0
    for b, r in enumerate(d.recs):
        assert out_off[b] == pos, b
        end = pos + d.sizes[b]
        fits = end <= d.out_cap
        region = buf[m + pos: m + min(end, d.out_cap)]
        if len(r) >= 4 and not fits:
            assert (status[b], out_len[b], expected[b]) == (INVALID, 0, 0), b
            assert (region == SENT).all(), b
        else:
            want = oracle_one(r, d.dic)
            got = (int(status[b]), region[:out_len[b]].tobytes(), int(expected[b]))
            assert got == want, (b, r[:16], got[0], got[2], want[0], want[2])
            if host:
                assert host_one(ctx, r, d.dic) == want, b
            if status[b] == 0 or len(r) < 4:
                assert (region[out_len[b]:] == SENT).all(), b          # untouched past the decoded length
        pos = end
    assert (buf[:m] == SENT).all() and (buf[m + d.out_cap:] == SENT).all()
    return status


def decode_corpus():
    rng = np.random.default_rng(11)
    valid = [oracle.compress_prepend_size(_kind(k, n)) for k in ("json", "random", "zeros", "dickens")
             for n in (0, 1, 13, 100, 4096, 65536, 70000)]
    j = oracle.compress_block(_json(3000))
    recs = list(valid)
    recs += [b"", b"\x01", b"\x01\x02", b"\x01\x02\x03", b"\0\0\0\0"]                       # 0-4 bytes
    recs += [b"\0\0\0\0" + j, b"\0\0\0\0\x00", b"\0\0\0\0" + oracle.compress_block(b"abc")]     # prefix 0 with data
    recs += [(2999).to_bytes(4, "little") + j, (100).to_bytes(4, "little") + j]                # prefix below
    recs += [(3100).to_bytes(4, "little") + j, (1 << 16).to_bytes(4, "little") + j]            # prefix above
    for _, stream, cap, *_ in vectors.DECODE_KATS:
        recs.append(cap.to_bytes(4, "little") + bytes(stream))
    recs += [bytes(v) for v in vectors.NO_PANIC]
    recs += [oracle.compress_prepend_size(x) for x in vectors.ROUNDTRIP]
    bases = [oracle.compress_prepend_size(_kind(k, n)) for k in ("json", "dickens", "random") for n in (50, 700, 9000)]
    for i in range(2000):
        r = bytearray(bases[int(rng.integers(len(bases)))])
        op = int(rng.integers(4))
        if op == 0:                                                           # truncate
            r = r[:int(rng.integers(0, len(r) + 1))]
        elif op == 1:                                                         # flip bytes after the prefix
            for _ in range(int(rng.integers(1, 6))):
                if len(r) > 4:
                    r[int(rng.integers(4, len(r)))] = int(rng.integers(256))
        elif op == 2:                                                         # another length word
            size = int.from_bytes(r[:4], "little")
            r[:4] = int(rng.integers(0, 2 * size + 2)).to_bytes(4, "little")
        else:                                                                 # both
            r = r[:int(rng.integers(4, len(r) + 1))]
            if len(r) > 4:
                r[int(rng.integers(4, len(r)))] ^= 1 << int(rng.integers(8))
        recs.append(bytes(r))
    return recs


def test_decompress_parity(ctx):
    recs = decode_corpus()
    status = check_decompress(ctx, Dec(recs, seed=5))
    assert len(set(status[:len(recs)].tolist())) >= 5                     # OK and several errors are exercised


def test_decompress_parity_with_dict(ctx):
    for name, inp, dic in dict_cases()[::3]:
        recs = [expected_record(inp, dic), expected_record(_json(2000), dic), b"\x01\x02",
                (len(inp) + 9).to_bytes(4, "little") + oracle.compress_with_dict(inp, dic)]
        check_decompress(ctx, Dec(recs, dic=dic, seed=len(name)))


def test_decompress_capacity_edges(ctx):
    recs = decode_corpus()[:60]
    total = Dec(recs).total
    sizes = Dec(recs).sizes
    ends = np.cumsum(sizes)
    for cap in (total - 1, 0, int(ends[10]) - 1, int(ends[30])):
        check_decompress(ctx, Dec(recs, out_cap=cap, seed=6), host=False)


# ---- asynchrony ---------------------------------------------------------------------------------------------------

def test_calls_return_before_the_stream_runs(ctx):
    datas = [_json(65536)] * 64
    c = Comp(datas, seed=7)
    check_compress(c, ctx)                                             # warm: the context's scratch has its size
    hb, ro = c.buf[c.mis:].cpu().numpy(), c.rec_off.cpu().numpy()
    recs = [hb[ro[b]:ro[b + 1]].tobytes() for b in range(64)]
    d = Dec(recs, seed=7)
    check_decompress(ctx, d, host=False)
    s = torch.cuda.Stream()
    for call in (c, d):
        call.buf.fill_(SENT)
        call.status.fill_(UNSET)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(1 << 30)
            assert call.enqueue(ctx, stream=s.cuda_stream) == 0
            assert not s.query(), "the call waited for the device"
        s.synchronize()
    check_compress(c, ctx, run=False)
    check_decompress(ctx, d, host=False, run=False)


def test_back_to_back_calls_on_one_context(ctx):
    a = Comp([_json(n) for n in (100, 65536, 300000)], seed=8)
    b = Comp([_kind("dickens", n) for n in (5, 4096)] * 50, seed=9)
    check_compress(a, ctx), check_compress(b, ctx)
    sep = [x.result() for x in (a, b)]
    for x in (a, b):
        x.buf.fill_(SENT); x.rec_off.fill_(UNSET); x.status.fill_(UNSET)
    torch.cuda.synchronize()
    assert a.enqueue(ctx) == 0 and b.enqueue(ctx) == 0
    for x, y in zip((a.result(), b.result()), sep):
        assert all((p == q).all() for p, q in zip(x, y))
    da = Dec(decode_corpus()[:40], seed=10)
    db = Dec([expected_record(_json(n)) for n in (100, 70000)] * 20, seed=11)
    check_decompress(ctx, da, host=False)
    check_decompress(ctx, db, host=False)
    sep = [x.result() for x in (da, db)]
    for x in (da, db):
        x.buf.fill_(SENT); x.out_off.fill_(UNSET); x.status.fill_(UNSET)
    torch.cuda.synchronize()
    assert da.enqueue(ctx) == 0 and db.enqueue(ctx) == 0
    for x, y in zip((da.result(), db.result()), sep):
        assert all((p == q).all() for p, q in zip(x, y))


# ---- arguments and kernel choice -------------------------------------------------------------------------------------

def _untouched_comp(c: Comp):
    buf, ro, st = c.result()
    return (buf == SENT).all() and (ro == UNSET).all() and (st == UNSET).all()


def _untouched_dec(d: Dec):
    return all((x == (SENT if i == 0 else UNSET)).all() for i, x in enumerate(d.result()))


def test_argument_errors_touch_nothing(ctx):
    bad_c = [dict(ctx=None), dict(rec_off=None), dict(d_in=None), dict(in_off=None), dict(in_len=None),
             dict(status=None), dict(d_out=None), dict(n=1 << 32), dict(dict=(None, 5))]
    for o in bad_c:
        c = Comp([_json(1000), b"abc"], seed=12)
        assert c.enqueue(ctx, **o) == INVALID, o
        assert _untouched_comp(c), o
    bad_d = [dict(ctx=None), dict(out_off=None), dict(d_in=None), dict(rec_off=None), dict(rec_len=None),
             dict(out_len=None), dict(status=None), dict(d_out=None), dict(n=1 << 32), dict(dict=(None, 5))]
    for o in bad_d:
        d = Dec([expected_record(_json(1000)), b"\x03\0\0\0efg"], seed=12)
        assert d.enqueue(ctx, **o) == INVALID, o
        assert _untouched_dec(d), o


def test_empty_batch(ctx):
    c = Comp([], seed=13)
    assert c.enqueue(ctx, d_in=None, in_off=None, in_len=None, status=None, d_out=None, out_cap=0) == 0
    buf, ro, st = c.result()
    assert ro[0] == 0 and (ro[1:] == UNSET).all() and (st == UNSET).all() and (buf == SENT).all()
    d = Dec([], seed=13)
    assert d.enqueue(ctx, d_in=None, rec_off=None, rec_len=None, out_len=None, status=None, d_out=None, out_cap=0) == 0
    buf, oo, ol, st, ex = d.result()
    assert oo[0] == 0 and (oo[1:] == UNSET).all() and (st == UNSET).all() and (buf == SENT).all()


def test_null_output_with_no_room(ctx):
    # the size query of the Python wrapper: nothing fits, nothing is written, the layout is complete
    d = Dec([b"\0\0\0\0\x00", expected_record(_json(500)), b"\0\0\0\0\x00", b"ab"], out_cap=0, seed=14)
    assert d.enqueue(ctx, d_out=None) == 0
    buf, oo, ol, st, ex = d.result()
    assert list(st[:4]) == [0, INVALID, INVALID, EAB] and list(oo[:5]) == [0, 0, 500, 500, 500] and (buf == SENT).all()


def test_python_wrappers(ctx):
    datas = [_json(n) for n in (0, 50, 65536, 100000)]
    src, offs = pack(datas, 15)
    out, rec_off, status = block.compress_prepend_size_device(src, offs, [len(x) for x in datas], ctx=ctx)
    ro = rec_off.cpu().numpy()
    assert (status.cpu().numpy() == 0).all()
    host = out.cpu().numpy()
    assert [host[ro[b]:ro[b + 1]].tobytes() for b in range(4)] == [expected_record(x) for x in datas]
    dec, out_off, out_len, st, ex = block.decompress_size_prepended_device(out, rec_off[:4], np.diff(ro), ctx=ctx)
    assert dec.numel() == max(sum(map(len, datas)), 1) and (st.cpu().numpy() == 0).all()
    assert dec[:int(out_off[4])].cpu().numpy().tobytes() == b"".join(datas)
    with pytest.raises(ValueError):
        block.compress_prepend_size_device(src, [src.numel()], [1], ctx=ctx)


@pytest.mark.parametrize("sizes,with_dict", [((100,) * 8, False), ((4096,) * 4000, False), ((300000,) * 4, False),
                                             ((0, 70000), False), ((2000,) * 50, True), ((30000, 50000), True)])
def test_kernel_choice_matches_block_batch(ctx, sizes, with_dict):
    datas = [_json(n) for n in sizes]
    dic = _kind("dickens", 40000) if with_dict else None
    dict_t = torch.from_numpy(np.frombuffer(dic, dtype=np.uint8).copy()).cuda() if dic else None
    c = Comp(datas, dict_t=dict_t, seed=16)
    rec_off = check_compress(c, ctx, dic)
    mine = last_kernel(ctx, 0)
    n = len(datas)
    slot = oracle.max_output_size(max(sizes))
    outs = torch.empty(n * slot, dtype=torch.uint8, device="cuda")
    lens = torch.empty(n, dtype=torch.int32, device="cuda")
    st = torch.empty(n, dtype=torch.int32, device="cuda")
    out_off, caps = u64([b * slot for b in range(n)]), u32([slot] * n)
    args = (ctx.handle, ptr(c.d_in), ptr(c.offs), ptr(c.lens))
    tail = (ptr(outs), ptr(out_off), ptr(caps), ptr(lens), ptr(st), n, max(sizes), 0)
    if dic:
        assert L().lz4b200_compress_batch_device_with_dict(*args, ptr(dict_t), dict_t.numel(), *tail) == 0
    else:
        assert L().lz4b200_compress_batch_device(*args, None, *tail) == 0
    torch.cuda.synchronize()
    assert last_kernel(ctx, 0) == mine
    hb = c.buf.cpu().numpy()
    recs = [hb[c.mis + a: c.mis + b].tobytes() for a, b in zip(rec_off[:n], rec_off[1:n + 1])]
    d = Dec(recs, dic=dic, seed=16)
    check_decompress(ctx, d, host=False)
    mine = last_kernel(ctx, 1)
    dl = torch.empty(n, dtype=torch.int32, device="cuda")
    dout = torch.empty(sum(sizes) + 1, dtype=torch.uint8, device="cuda")
    doff = u64(np.concatenate([[0], np.cumsum(sizes)[:-1]]))
    din_off = d.offs + 4
    din_len = u32([len(r) - 4 for r in recs])
    dcap = u32(sizes)
    dargs = (ctx.handle, ptr(d.d_in), ptr(din_off), ptr(din_len))
    dtail = (ptr(dout), ptr(doff), ptr(dcap), ptr(dl), ptr(st), None, n, 0)
    if dic:
        assert L().lz4b200_decompress_batch_device_with_dict(*dargs, ptr(dict_t), dict_t.numel(), *dtail) == 0
    else:
        assert L().lz4b200_decompress_batch_device(*dargs, *dtail) == 0
    torch.cuda.synchronize()
    assert last_kernel(ctx, 1) == mine
    assert (st.cpu().numpy() == 0).all()
