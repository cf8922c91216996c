"""CPU tests of the linked-frame encoder's ground truth: the per-block chain plan (lz4_flex_b200/csrc/lz4b200_frame_chain.cuh,
compiled for the host by g++ under AddressSanitizer and UndefinedBehaviorSanitizer through tests/cpp/frame_chain_host.cpp)
against a restatement of FrameEncoder's buffer moves, and the BlockMode::Linked frames of the linked-frame reference
(tests/cpp/linked_frame_ref.c, through tests/linked_ref.py): they decode to their
input through the oracle and through the system liblz4's LZ4F decoder, their sequences obey the ext_dict / prefix rules
of compress_internal, and they are smaller than independent frames.  No GPU needed."""
import ctypes
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import linked_ref
import oracle
from lz4_flex_b200 import corpus

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "frame_chain_host.cpp")
HDRS = [os.path.join(os.path.dirname(HERE), "lz4_flex_b200", "csrc", h)
        for h in ("lz4b200_frame_chain.cuh", "lz4b200_frame_walk.cuh")]
API = os.path.join(os.path.dirname(HERE), "include", "lz4b200.h")
EXE = os.path.join(HERE, "cpp", "_build", "frame_chain_host")

WINDOW = 65536
BLOCK_SIZES = [64 << 10, 256 << 10, 1 << 20, 4 << 20]
FLAG_SETS = [0, 1, 2, 4, 7]                     # block checksums, content checksum, content size, all


@pytest.fixture(scope="module")
def chain():
    if shutil.which("g++") is None:
        pytest.fail("g++ is required to build the host chain plan")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [SRC, API] + HDRS):
        tmp = f"{EXE}.tmp{os.getpid()}"
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-fno-omit-frame-pointer", "-o", tmp, SRC], check=True)
        os.replace(tmp, EXE)

    def run(cases):
        blob = b"".join(struct.pack("<QQQQI", bs, s, e, st, len(lens)) + np.asarray(lens, dtype=np.uint64).tobytes()
                        for bs, s, e, st, lens in cases)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        r = subprocess.run([EXE], input=blob, capture_output=True, env=env)
        assert r.returncode == 0 and not r.stderr, r.stderr.decode(errors="replace")[-4000:]
        return [tuple(map(int, ln.split())) for ln in r.stdout.decode().splitlines()]
    return run


def py_chain(bs, lens, stream=0, ext=0, start=0):
    """FrameEncoder::write_block in linked mode (frame/compress.rs:261-371), written with the names of the reference:
    per block (stream, ext_dict_len, input_pos, repositioned, shift, frame position of input[0] - stream, first)."""
    src_start, ext_len, src_stream_offset, consumed = start, ext, stream, start
    out = []
    for n in lens:
        rep = src_stream_offset + bs + WINDOW >= 0xFFFFFFFF // 2
        shift = 0
        if rep:
            shift = src_stream_offset - ext_len
            src_stream_offset = ext_len
        first = src_start == 0 and src_stream_offset == 0
        out.append((src_stream_offset, ext_len, src_start, int(rep), shift,
                    consumed - src_start - src_stream_offset, int(first)))
        consumed += n
        src_start += n
        src_end = src_start
        if src_start >= bs + WINDOW:
            ext_len = WINDOW
            src_stream_offset += src_end
            src_start = 0
        elif src_start + ext_len > WINDOW:
            ext_len -= min(ext_len, src_start + ext_len - WINDOW)
    return out


def random_lengths(rng, bs):
    nb = int(rng.integers(1, 40))
    style = int(rng.integers(0, 3))
    if style == 0:                                   # whole-input frame: full blocks and a short last one
        return [bs] * (nb - 1) + [int(rng.integers(1, bs + 1))]
    if style == 1:                                   # a flush every so often: short blocks anywhere
        return [bs if rng.random() < 0.5 else int(rng.integers(1, bs + 1)) for _ in range(nb)]
    return [int(rng.integers(1, min(bs, 3 * WINDOW) + 1)) for _ in range(nb)]   # mostly short blocks


def test_plan_matches_restatement(chain):
    rng = np.random.default_rng(11)
    cases = []
    for _ in range(1500):
        bs = int(rng.choice(BLOCK_SIZES))
        cases.append((bs, 0, 0, 0, random_lengths(rng, bs)))
    # synthetic states whose stream offset nears 2^31 - 1: the reposition fires within the sequence
    for _ in range(300):
        bs = int(rng.choice(BLOCK_SIZES))
        lim = 0x7FFFFFFF - WINDOW - bs
        ext = int(rng.choice([0, WINDOW, int(rng.integers(1, WINDOW))]))
        start = 0 if ext == WINDOW else int(rng.integers(0, bs + WINDOW))
        stream = max(ext, lim - int(rng.integers(0, 6 * bs)))
        cases.append((bs, stream, ext, start, random_lengths(rng, bs)))
    got = chain(cases)
    want = [row for bs, s, e, st, lens in cases for row in py_chain(bs, lens, s, e, st)]
    assert got == want
    assert sum(r[3] for r in want) > 100                    # the reposition is exercised
    assert sum(1 for r in want if r[1] and r[2]) > 100      # so are blocks with both an ext_dict and a prefix


def test_whole_input_period_two(chain):
    """Whole-input frames: blocks 0 and 1 have no ext_dict (block 1's prefix is block 0); from block 2 on, even blocks
    have a 64 KiB ext_dict and no prefix, odd blocks have block k-1 as prefix and no ext_dict."""
    for bs in BLOCK_SIZES:
        rows = chain([(bs, 0, 0, 0, [bs] * 9 + [7])])
        for k, (s, e, pre, rep, shift, to_frame, first) in enumerate(rows):
            assert (rep, shift, first) == (0, 0, int(k == 0))
            assert s + to_frame + pre == k * bs                  # the block starts at frame position k * bs
            if k < 2:
                assert (s, e, pre) == (0, 0, k * bs)
            elif k % 2 == 0:
                assert (s, e, pre) == (k * bs, WINDOW, 0)
            else:
                assert (s, e, pre) == ((k - 1) * bs, 0, bs)


def test_reposition_epochs(chain):
    """With 4 MiB blocks the stream offset steps by 8 MiB every two blocks; the first reposition falls before the
    first block whose offset S has S + 4 MiB + 64 KiB >= 2^31 - 1, and sets S to the ext_dict length."""
    bs = 4 << 20
    rows = chain([(bs, 0, 0, 0, [bs] * 600)])
    reps = [k for k, r in enumerate(rows) if r[3]]
    assert reps and reps[0] % 2 == 0
    k = reps[0]
    assert rows[k - 2][0] + bs + WINDOW < 0x7FFFFFFF <= rows[k - 2][0] + 2 * bs + bs + WINDOW
    assert rows[k][0] == WINDOW and rows[k][4] == k * bs - WINDOW
    for k2, r in enumerate(rows):
        assert r[0] + r[5] + r[2] == k2 * bs


# ---- the reference's linked frames ---------------------------------------------------------------------------------

def _lz4f():
    try:
        L = ctypes.CDLL("liblz4.so.1")
    except OSError:
        return None
    L.LZ4F_createDecompressionContext.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint]
    L.LZ4F_freeDecompressionContext.argtypes = [ctypes.c_void_p]
    L.LZ4F_decompress.restype = ctypes.c_size_t
    L.LZ4F_decompress.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t), ctypes.c_void_p,
                                  ctypes.POINTER(ctypes.c_size_t), ctypes.c_void_p]
    L.LZ4F_isError.argtypes = [ctypes.c_size_t]
    return L


LZ4F = _lz4f()


def lz4f_decompress(frame: bytes, n: int) -> bytes:
    dctx = ctypes.c_void_p()
    assert LZ4F.LZ4F_createDecompressionContext(ctypes.byref(dctx), 100) == 0
    try:
        src = ctypes.create_string_buffer(frame, len(frame))
        dst = ctypes.create_string_buffer(max(n, 1))
        out, ip, op = [], 0, 0
        while True:
            ds, ss = ctypes.c_size_t(len(dst) - op), ctypes.c_size_t(len(frame) - ip)
            r = LZ4F.LZ4F_decompress(dctx, ctypes.addressof(dst) + op, ctypes.byref(ds), ctypes.addressof(src) + ip,
                                     ctypes.byref(ss), None)
            assert not LZ4F.LZ4F_isError(r), r
            ip += ss.value
            op += ds.value
            if r == 0 or (ss.value == 0 and ds.value == 0):
                break
        assert ip == len(frame)
        return dst.raw[:op]
    finally:
        LZ4F.LZ4F_freeDecompressionContext(dctx)


def corpora():
    dk = corpus.load("dickens.txt")
    return {"json": corpus.load("compression_66k_JSON.txt") * 40, "dickens": dk[:3_000_000],
            "hdfs": corpus.load("hdfs.json")[:2_000_000], "small": corpus.load("compression_1k.txt")}


def test_reference_linked_frames_decode():
    cases = []
    for name, d in corpora().items():
        for bsid in (4, 5, 6, 7, 0):
            for fl in FLAG_SETS:
                cases.append((name, d, bsid, fl, 0))
    d = corpora()["dickens"][:1_000_000]
    for fe in (13, 1000, 40_000, 70_000, 200_000):         # flushes: short blocks, ext_dict and prefix together
        cases.append(("flush", d, 4, 7, fe))
    for name, d, bsid, fl, fe in cases:
        f = linked_ref.frame_compress(d, bsid, fl, fe)
        assert f[4] & 0x20 == 0                              # the header says linked
        st, out, _ = oracle.frame_decompress(f, len(d) + 16)
        assert st == 0 and out == d, (name, bsid, fl, fe)
        if LZ4F is not None:
            assert lz4f_decompress(f, len(d)) == d, (name, bsid, fl, fe)
    if LZ4F is None:
        pytest.skip("liblz4.so.1 not present: decoded by the C oracle only")


def iter_blocks(frame: bytes):
    """(block index, stored, payload) of a frame with no checksums and no content size."""
    assert frame[4] & 0x1D == 0
    pos, k = 7, 0
    while True:
        info = struct.unpack_from("<I", frame, pos)[0]
        pos += 4
        if info == 0:
            return
        n = info & 0x7FFFFFFF
        yield k, bool(info >> 31), frame[pos:pos + n]
        pos += n
        k += 1


def sequences(payload: bytes):
    """(literal length, offset, match length) per sequence; the last one has offset 0."""
    i, out = 0, []
    while i < len(payload):
        tok = payload[i]; i += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                b = payload[i]; i += 1; lit += b
                if b != 255:
                    break
        i += lit
        if i >= len(payload):
            out.append((lit, 0, 0))
            break
        off = payload[i] | payload[i + 1] << 8; i += 2
        ml = (tok & 15) + 4
        if tok & 15 == 15:
            while True:
                b = payload[i]; i += 1; ml += b
                if b != 255:
                    break
        out.append((lit, off, ml))
    return out


def test_sequence_walk():
    """Whole-input frames: offsets are at most 65 535; block 0 does not start with a match; in every even block k >= 2
    (ext_dict = the 64 KiB before the block, no prefix) no match whose source starts before the block runs past the
    block's start; odd blocks (block k-1 as prefix) do have such matches on repetitive data."""
    period = bytes(np.random.default_rng(3).integers(0, 256, 3000, dtype=np.uint8))
    data = {"dickens": corpus.load("dickens.txt")[:2_000_000], "period": period * 200}
    crossing_odd = 0
    for name, d in data.items():
        for bsid in (4, 5):
            bs = {4: 64 << 10, 5: 256 << 10}[bsid]
            f = linked_ref.frame_compress(d, bsid)
            for k, stored, payload in iter_blocks(f):
                if stored:
                    continue
                seqs = sequences(payload)
                start = k * bs
                if k == 0:
                    assert seqs[0][0] > 0 or seqs[0][1] == 0
                pos = start
                for lit, off, ml in seqs:
                    pos += lit
                    if off == 0:
                        break
                    assert 1 <= off <= 65535
                    src = pos - off
                    if src < start:
                        if k >= 2 and k % 2 == 0:
                            assert src + ml <= start, (name, bsid, k)
                        elif src + ml > start:
                            crossing_odd += 1
                    pos += ml
                assert pos == min(start + bs, len(d))
    assert crossing_odd > 0


def test_linked_smaller_than_independent():
    d = corpus.load("dickens.txt")
    ind = oracle.frame_compress(d, 4, 0)
    lnk = linked_ref.frame_compress(d, 4)
    assert len(lnk) < len(ind)
    assert oracle.frame_decompress(lnk, len(d))[:2] == (0, d)
