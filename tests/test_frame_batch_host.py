"""CPU tests of the batch frame encoder's plan (lz4_flex_b200/csrc/lz4b200_frame_batch.cuh), compiled for the host by
g++ under AddressSanitizer and UndefinedBehaviorSanitizer (tests/cpp/frame_batch_host.cpp): on random lists of frame
lengths, block sizes and first FRESH blocks, every block's frame, frame-local index, input range, scratch slot, FRESH/CONT
mode and packed destination, and every frame's place in the packed output, against a Python restatement.  No GPU needed."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "frame_batch_host.cpp")
HDRS = [os.path.join(os.path.dirname(HERE), "lz4_flex_b200", "csrc", h)
        for h in ("lz4b200_frame_batch.cuh", "lz4b200_frame_walk.cuh")]
API = os.path.join(os.path.dirname(HERE), "include", "lz4b200.h")
EXE = os.path.join(HERE, "cpp", "_build", "frame_batch_host")

CONT, HASH5_ALWAYS = 1, 2
BLOCK_SIZES = [64 << 10, 256 << 10, 1 << 20, 4 << 20]


@pytest.fixture(scope="module")
def planner():
    if shutil.which("g++") is None:
        pytest.fail("g++ is required to build the host frame plan")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [SRC, API] + HDRS):
        tmp = f"{EXE}.tmp{os.getpid()}"
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-fno-omit-frame-pointer", "-o", tmp, SRC], check=True)
        os.replace(tmp, EXE)

    def run(blob: bytes):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        r = subprocess.run([EXE], input=blob, capture_output=True, env=env)
        assert r.returncode == 0 and not r.stderr, r.stderr.decode(errors="replace")[-4000:]
        return [tuple(map(int, ln.split())) for ln in r.stdout.decode().splitlines()]
    return run


def fresh_period(bs):
    """FrameEncoder repositions its table at the first block whose offset off has off + bs + 64 KiB >= 2^31 - 1
    (frame/compress.rs:266-271); block k of a frame is FRESH iff k >= first_fresh and k - first_fresh is a multiple of
    the period."""
    limit = 0x7FFFFFFF - 65536 - bs
    return -(-limit // bs)


def slot(n):
    return (20 + n * 110 // 100 + 15) & ~15                 # lz4b200_max_output_size(n), rounded up to 16


def py_plan(frames, tail, seg):
    """frames: [(in_off, in_len, bs, hdr_len, first_fresh)]; seg: every block's segment size.  Returns (blocks,
    places)."""
    blocks, places = [], []
    seg_off = np.concatenate([[0], np.cumsum(np.asarray(seg, dtype=np.int64))]).tolist()
    b, slot_base, ovh = 0, 0, 0
    for f, (in_off, n, bs, hdr_len, ff) in enumerate(frames):
        nb = -(-n // bs)
        first = b
        for k in range(nb):
            ln = min(bs, n - k * bs)
            flags = HASH5_ALWAYS | (0 if k >= ff and (k - ff) % fresh_period(bs) == 0 else CONT)
            blocks.append((f, k, in_off + k * bs, ln, slot_base, slot(ln), flags, seg_off[b] + ovh + hdr_len))
            slot_base += slot(ln)
            b += 1
        places.append((seg_off[first] + ovh, seg_off[b] + ovh + hdr_len))
        ovh += hdr_len + tail
    return blocks, places, slot_base


def record(frames, tail, seg):
    head = struct.pack("<II", len(frames), tail)
    body = b"".join(struct.pack("<QQIIIB", o, n, bs, fresh_period(bs), ff, h) for o, n, bs, h, ff in frames)
    return head + body + np.asarray(seg, dtype=np.uint32).tobytes()


def random_batch(rng):
    nf = int(rng.integers(0, 40))
    style = int(rng.integers(0, 3))                        # empty-heavy, small, or spanning several blocks
    frames, off = [], int(rng.integers(0, 64))
    for _ in range(nf):
        bs = int(rng.choice(BLOCK_SIZES))
        if style == 0:
            n = 0 if rng.random() < 0.6 else int(rng.integers(1, 5000))
        elif style == 1:
            n = int(rng.integers(0, 3 * 65536))
        else:
            n = int(rng.integers(0, 5 * bs + 2))
            if rng.random() < 0.3:
                n = bs * int(rng.integers(0, 4))           # a whole number of blocks
        ff = 0 if rng.random() < 0.5 else int(rng.integers(0, 6))   # a streaming group's blocks after a flush
        frames.append((off, n, bs, int(rng.choice([7, 15])), ff))
        off += n + int(rng.integers(0, 17))
    return frames


def test_plan_matches_restatement(planner):
    rng = np.random.default_rng(7)
    cases = []
    for _ in range(1500):
        frames = random_batch(rng)
        nb = sum(-(-n // bs) for _, n, bs, _, _ in frames)
        seg = rng.integers(8, 1 << 20, size=nb).tolist()
        cases.append((frames, int(rng.choice([4, 8])), seg))
    out = planner(b"".join(record(*c) for c in cases))
    pos, nonfresh_after_first = 0, 0
    for frames, tail, seg in cases:
        want_blocks, want_places, want_slots = py_plan(frames, tail, seg)
        nb, slots = out[pos]
        assert (nb, slots) == (len(want_blocks), want_slots)
        got_blocks = out[pos + 1:pos + 1 + nb]
        got_places = out[pos + 1 + nb:pos + 1 + nb + len(frames)]
        pos += 1 + nb + len(frames)
        assert got_blocks == want_blocks
        assert got_places == want_places
        # packed: every frame starts where the one before it ends
        for f in range(1, len(frames)):
            assert got_places[f][0] == got_places[f - 1][1] + tail
        nonfresh_after_first += sum(1 for blk in got_blocks
                                    if blk[1] != frames[blk[0]][4] and blk[0] and not blk[6] & CONT)
    assert pos == len(out)
    assert nonfresh_after_first == 0


def test_slot_is_max_output_size():
    from lz4_flex_b200 import _native
    for n in [0, 1, 15, 16, 4096, 65535, 65536, 65537, 262144, 1 << 20, 4 << 20]:
        assert slot(n) == (_native.lib().lz4b200_max_output_size(n) + 15) & ~15


def test_fresh_is_frame_local(planner):
    """A 513-block frame of 4 MiB blocks after frames with blocks: its block 511 is FRESH by its frame-local index.  A
    frame whose first FRESH block is 1 (a streaming group after a flush) repositions at its block 512."""
    bs = 4 << 20
    frames = [(0, 3 * 65536 + 5, 64 << 10, 7, 0), (3 * 65536 + 5, 10, bs, 15, 0), (3 * 65536 + 15, 513 * bs, bs, 15, 0),
              (0, 513 * bs, bs, 0, 1)]
    nb = 4 + 1 + 513 + 513
    seg = [100] * nb
    out = planner(record(frames, 8, seg))
    blocks = out[1:1 + nb]
    big = [blk for blk in blocks if blk[0] == 2]
    assert len(big) == 513
    fresh = [blk[1] for blk in big if not blk[6] & CONT]
    assert fresh == [0, 511]
    assert [blk[1] for blk in blocks if blk[0] == 3 and not blk[6] & CONT] == [1, 512]
    assert fresh_period(bs) == 511
    assert py_plan(frames, 8, seg)[0] == blocks
