"""CPU tests of the sync-free batch frame encoder's planner (lz4b200_frame_batch.cuh, run frame after frame by
tests/cpp/frame_batch_async_host.cpp under AddressSanitizer and UndefinedBehaviorSanitizer): on random length lists and
capacities, every frame's plan, status, the empty plans past capacity and the device block count against a Python
restatement of the capacity rule; the shared header writer against the oracle's; and the Python defaults of
compress_frames_device_async() (block capacity, out_cap helper) against the oracle's frames.  No GPU needed."""
import ctypes as C
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import oracle
from lz4_flex_b200 import corpus, frame

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "frame_batch_async_host.cpp")
HDRS = [os.path.join(os.path.dirname(HERE), "lz4_flex_b200", "csrc", h)
        for h in ("lz4b200_frame_batch.cuh", "lz4b200_frame_walk.cuh")]
API = os.path.join(os.path.dirname(HERE), "include", "lz4b200.h")
EXE = os.path.join(HERE, "cpp", "_build", "frame_batch_async_host")

BS = {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20}
OK, TOO_SMALL, INVALID = 0, 1, 200
U64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def planner():
    if shutil.which("g++") is None:
        pytest.fail("g++ is required to build the host planner")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [SRC, API] + HDRS):
        tmp = f"{EXE}.tmp{os.getpid()}"
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-fno-omit-frame-pointer", "-o", tmp, SRC], check=True)
        os.replace(tmp, EXE)

    def run(blob: bytes):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        r = subprocess.run([EXE], input=blob, capture_output=True, env=env)
        assert r.returncode == 0 and not r.stderr, (r.returncode, r.stderr.decode(errors="replace")[-4000:])
        return r.stdout.decode().splitlines()
    return run


def _info(bsid, bc, cc, cs, linked):
    return struct.pack("<5i", bsid, bc, cc, cs, linked)


def fresh_period(bs):
    return -(-(0x7FFFFFFF - 65536 - bs) // bs)


def slot(n):
    return (20 + n * 110 // 100 + 15) & ~15


def auto_id(n):
    return 7 if n > 256 << 10 else 5 if n > 64 << 10 else 4


def hdr_len(cs):
    return 15 if cs else 7


def py_plan(bsid, cc, cs, limits, frames):
    """The capacity rule and placement, restated: frames 0..f must together fit (blocks, input bytes, frame bound);
    the first limit passed, in that order, gives the status; a frame past capacity has no input, no header and adds
    nothing to the places after it."""
    max_blocks, max_in, out_cap = limits
    tail = 8 if cc else 4
    rows = []
    sb = si = sbound = 0
    nb = slots = ovh = 0
    for off, n in frames:
        bs = BS[bsid or auto_id(n)]
        k = -(-n // bs)
        sb, si, sbound = sb + k, si + n, sbound + 27 + n + 8 * k
        st = INVALID if sb > max_blocks or si > max_in else TOO_SMALL if sbound > out_cap else OK
        if st == OK:
            rows.append((OK, off, n, bs, fresh_period(bs), nb, slots, ovh, hdr_len(cs)))
            nb += k
            slots += sum(slot(min(bs, n - i * bs)) for i in range(k))
            ovh += hdr_len(cs) + tail
        else:
            rows.append((st, off, 0, bs, fresh_period(bs), nb, slots, ovh, 0))
    return rows, nb


def batch_record(bsid, bc, cc, cs, linked, limits, frames):
    return (struct.pack("<I", 0) + _info(bsid, bc, cc, cs, linked) + struct.pack("<QQQI", *limits, len(frames)) +
            b"".join(struct.pack("<QQ", o, n) for o, n in frames))


def random_case(rng):
    nf = int(rng.integers(0, 30))
    style = int(rng.integers(0, 3))
    frames, off = [], int(rng.integers(0, 64))
    for _ in range(nf):
        if style == 0:
            n = 0 if rng.random() < 0.5 else int(rng.integers(1, 5000))
        elif style == 1:
            n = int(rng.integers(0, 3 * 65536))
        else:
            n = int(rng.integers(0, 9 << 20))
        frames.append((off, n))
        off += n + int(rng.integers(0, 17))
    bsid = int(rng.choice([0, 4, 5, 6, 7]))
    cc, cs = int(rng.integers(0, 2)), int(rng.integers(0, 2))
    total_b = sum(-(-n // BS[bsid or auto_id(n)]) for _, n in frames)
    total_in = sum(n for _, n in frames)
    total_bound = sum(27 + n + 8 * -(-n // BS[bsid or auto_id(n)]) for _, n in frames)

    def pick(total):
        r = rng.random()
        if r < 0.4:
            return total + int(rng.integers(0, 3))
        if r < 0.5:
            return 0
        if r < 0.6:
            return U64
        return int(rng.integers(0, total + 2))
    return bsid, int(rng.integers(0, 2)), cc, cs, int(rng.integers(0, 2)), (pick(total_b), pick(total_in),
                                                                          pick(total_bound)), frames


def test_planner_matches_restatement(planner):
    rng = np.random.default_rng(11)
    cases = [random_case(rng) for _ in range(1200)]
    # edges: each limit at 0, at the total - 1 and at the total, one at a time; a frame past 2^62 bytes
    frames = [(0, 70000), (70000, 0), (70000, 300000), (370000, 5 << 20), (0, 10)]
    for bsid in (0, 4, 7):
        tb = sum(-(-n // BS[bsid or auto_id(n)]) for _, n in frames)
        ti = sum(n for _, n in frames)
        tbound = sum(27 + n + 8 * -(-n // BS[bsid or auto_id(n)]) for _, n in frames)
        for i, t in enumerate((tb, ti, tbound)):
            for cap in (0, t - 1, t):
                lim = [U64, U64, U64]
                lim[i] = cap
                cases.append((bsid, 1, 1, 1, 0, tuple(lim), frames))
    # frames whose sums pass 2^64: past the largest block capacity the C ABI takes, whatever the other limits
    cases.append((0, 0, 0, 1, 0, ((1 << 32) - 1, U64, U64), [(0, 100), (5, (1 << 63) + 7), (0, 1)]))
    cases.append((4, 0, 0, 0, 0, ((1 << 32) - 1, U64, U64), [(0, U64), (0, 0), (0, U64)]))
    out = planner(b"".join(batch_record(*c) for c in cases))
    pos, statuses = 0, set()
    for bsid, bc, cc, cs, linked, limits, frames in cases:
        want, want_nb = py_plan(bsid, cc, cs, limits, frames)
        got = [tuple(int(x) for x in ln.split()) for ln in out[pos:pos + len(frames)]]
        assert got == want, (bsid, cc, cs, limits, frames)
        assert int(out[pos + len(frames)]) == want_nb
        pos += len(frames) + 1
        statuses |= {r[0] for r in got}
        # a prefix rule: once a frame is past capacity, so is every frame after it
        st = [r[0] for r in got]
        first_out = next((i for i, s in enumerate(st) if s != OK), len(st))
        assert all(s != OK for s in st[first_out:])
    assert pos == len(out)
    assert statuses == {OK, TOO_SMALL, INVALID}


def _oracle_header(bsid, flags, content_size):
    L = oracle.lib()
    L.lz4o_frame_header.restype = C.c_size_t
    L.lz4o_frame_header.argtypes = [C.c_void_p, C.c_int, C.c_uint, C.c_uint64]
    buf = (C.c_uint8 * 32)()
    n = L.lz4o_frame_header(buf, bsid, flags, content_size)
    return bytes(buf[:n])


def test_header_writer_matches_oracle(planner):
    combos, blob = [], b""
    for bsid in (4, 5, 6, 7):
        for bc in (0, 1):
            for cc in (0, 1):
                for cs in (0, 1):
                    for linked in (0, 1):
                        for size in (0, 1, (1 << 32) - 1, (1 << 32) + 5):
                            combos.append((bsid, bc, cc, cs, linked, size))
                            blob += struct.pack("<I", 1) + _info(bsid, bc, cc, cs, linked) + struct.pack("<Q", size)
    out = planner(blob)
    assert len(out) == len(combos)
    for (bsid, bc, cc, cs, linked, size), hexed in zip(combos, out):
        flags = (bc * oracle.F_BLOCK_CHECKSUMS) | (cc * oracle.F_CONTENT_CHECKSUM) | (cs * oracle.F_CONTENT_SIZE) | \
            (linked * 8)
        got = bytes.fromhex(hexed)
        assert got == _oracle_header(bsid, flags, size)
        if size <= 1 and not linked:                      # the first bytes of a whole frame of that many bytes
            f = oracle.frame_compress(b"\x5a" * size, bsid, flags)
            assert f[:len(got)] == got


def _inputs(n):
    j = corpus.tiled("compression_66k_JSON.txt", n).tobytes()
    return {"zeros": bytes(n), "json": j, "random": corpus.xorshift64star_bytes(n).tobytes()}


@pytest.mark.parametrize("bsid", [0, 4, 5, 6, 7])
@pytest.mark.parametrize("flags", [0, oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM | oracle.F_CONTENT_SIZE])
def test_python_defaults_hold_oracle_frames(bsid, flags):
    """For inputs laid back to back in d_in: the default block capacity holds every block of the oracle's frames, and
    compress_out_cap() is at least their summed lz4b200_frame_bound, which is at least what they take."""
    rng = np.random.default_rng(bsid * 7 + flags)
    info = frame.FrameInfo(block_size=frame.BlockSize(bsid), block_checksums=bool(flags & 1),
                           content_checksum=bool(flags & 2), content_size=0 if flags & 4 else None)
    for lens in ([0], [1], [65535, 65536, 65537], [0] * 5, [3 << 20], [int(x) for x in rng.integers(0, 300000, 12)],
                 [65536] * 16 + [1]):
        total = sum(lens)
        blocks = bound = taken = 0
        for i, n in enumerate(lens):
            d = _inputs(n)["json" if i % 3 else "zeros"] if n else b""
            f = oracle.frame_compress(d, bsid, flags)
            bs = BS[bsid or auto_id(n)]
            blocks += -(-n // bs)
            bound += 27 + n + 8 * -(-n // bs)
            taken += len(f)
        assert frame.default_compress_max_blocks(total, len(lens)) >= blocks, lens
        assert frame.compress_out_cap(len(lens), total, info) >= bound >= taken, lens


def test_out_cap_helper_is_the_frame_bound_sum():
    """compress_out_cap() against lz4b200_frame_bound itself, on the worst split of T bytes into F frames."""
    from lz4_flex_b200 import _native
    L = _native.lib()
    for bsid in (0, 4, 5, 6, 7):
        info = frame.FrameInfo(block_size=frame.BlockSize(bsid))
        for F, T in ((1, 0), (3, 1), (4, 65536 * 4 + 3), (10, 1 << 20), (1, 5 << 20)):
            lens = [T // F + (1 if i < T % F else 0) for i in range(F)]
            s = 0
            for n in lens:
                ci = frame.FrameInfo(block_size=frame.BlockSize(bsid or auto_id(n))).to_c()
                s += L.lz4b200_frame_bound(n, C.byref(ci))
            assert frame.compress_out_cap(F, T, info) >= s
