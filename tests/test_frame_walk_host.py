"""CPU tests of the frame walk and XXH32 shared by the host and device frame decoders
(lz4_flex_b200/csrc/lz4b200_frame_walk.cuh), compiled for the host by g++ under AddressSanitizer and
UndefinedBehaviorSanitizer (tests/cpp/frame_walk_host.cpp): XXH32 against the library's at every short length and
several seeds, the recorded block list of valid frames against a short Python parse, and the walk's status on
mutated and truncated frames against the oracle frame decoder.  No GPU needed."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import oracle
from lz4_flex_b200 import corpus, frame

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "frame_walk_host.cpp")
HDR = os.path.join(os.path.dirname(HERE), "lz4_flex_b200", "csrc", "lz4b200_frame_walk.cuh")
API = os.path.join(os.path.dirname(HERE), "include", "lz4b200.h")
EXE = os.path.join(HERE, "cpp", "_build", "frame_walk_host")

# the statuses the walk itself decides (header errors, BlockTooBig, block checksum, end of input)
WALK_STATUSES = {oracle.FERR_WRONG_MAGIC, oracle.FERR_RESERVED_BITS, oracle.FERR_UNSUPPORTED_VERSION,
                 oracle.FERR_UNSUPPORTED_BLOCKSIZE, oracle.FERR_HEADER_CHECKSUM, oracle.FERR_SKIPPABLE,
                 oracle.FERR_DICTIONARY, oracle.FERR_BLOCK_TOO_BIG, oracle.FERR_BLOCK_CHECKSUM, oracle.FERR_IO_EOF}


@pytest.fixture(scope="module")
def walker():
    if shutil.which("g++") is None:
        pytest.fail("g++ is required to build the host frame walk")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in (SRC, HDR, API)):
        tmp = f"{EXE}.tmp{os.getpid()}"
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-fno-omit-frame-pointer", "-o", tmp, SRC], check=True)
        os.replace(tmp, EXE)

    def run(records):
        """records: (op, arg, bytes) -> the program's output lines; fails on any sanitizer report."""
        blob = b"".join(struct.pack("<BIQ", op, arg, len(b)) + bytes(b) for op, arg, b in records)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        r = subprocess.run([EXE], input=blob, capture_output=True, env=env)
        assert r.returncode == 0 and not r.stderr, r.stderr.decode(errors="replace")[-4000:]
        return r.stdout.decode().splitlines()
    return run


def walk_all(run, frames, chunk=65536):
    """(status, consumed, blocks, flg, closed) per frame; blocks as (payload_off, word, checksum)."""
    lines = run([(1, chunk, f) for f in frames])
    out, i = [], 0
    for _ in frames:
        st, consumed, nb, flg, closed = map(int, lines[i].split())
        blocks = [tuple(map(int, ln.split())) for ln in lines[i + 1:i + 1 + nb]]
        out.append((st, consumed, blocks, flg, closed))
        i += 1 + nb
    assert i == len(lines)
    return out


def py_blocks(f: bytes):
    """The block list of a well-formed frame, straight from its BlockInfo words."""
    u32 = lambda p: int.from_bytes(f[p:p + 4], "little")
    if u32(0) == 0x184C2102:                                               # legacy: words until the end of the input
        flg, pos = 0, 4
    else:
        flg = f[4]
        pos = 7 + (8 if flg & 0x08 else 0)
    blocks = []
    while pos + 4 <= len(f):
        word = u32(pos)
        pos += 4
        if word == 0:
            pos += 4 if flg & 0x04 else 0
            break
        ln = word & 0x7FFFFFFF
        cs = u32(pos + ln) if flg & 0x10 else 0
        blocks.append((pos, word, cs))
        pos += ln + (4 if flg & 0x10 else 0)
    return blocks, pos


def test_xxh32_every_short_length_and_seed(walker):
    rng = np.random.default_rng(9)
    data = rng.integers(0, 256, 300, dtype=np.uint8).tobytes()
    seeds = [0, 1, 0x9E3779B1, 0xFFFFFFFF, 12345]
    recs = [(0, s, data[:n]) for s in seeds for n in range(301)]
    lines = walker(recs)
    assert len(lines) == len(recs)
    for (_, s, d), ln in zip(recs, lines):
        want = frame.xxh32(d, s)
        assert want == oracle.xxh32(d, s)
        assert [int(v) for v in ln.split()] == [want] * 5, (len(d), s)


def _valid_frames():
    j = corpus.tiled("compression_66k_JSON.txt", 600000).tobytes()
    rnd = corpus.xorshift64star_bytes(70000).tobytes()
    d = corpus.load("dickens.txt")[: (4 << 20) + 300000]
    frames = []
    for bsid, data in ((4, j + rnd + j[:1000]), (5, j + rnd), (6, j[:300000] * 4), (7, d)):
        for flags in range(8):
            frames.append(oracle.frame_compress(data, bsid, flags))
    frames.append(oracle.frame_compress(j, 4, 7, 1000))                    # flushed short blocks
    frames.append(oracle.frame_compress(b"", 4, 7))
    frames.append(oracle.frame_compress(b"a", 4, 7))
    frames.append(corpus.load("dickens.lz4"))                              # legacy
    gdir = os.path.join(HERE, "golden", "linked")
    frames += [open(os.path.join(gdir, f), "rb").read() for f in sorted(os.listdir(gdir)) if f.endswith(".lz4")]
    return frames


def test_valid_frames_record_every_block(walker):
    frames = _valid_frames()
    for chunk in (65536, 3):
        for f, (st, consumed, blocks, flg, closed) in zip(frames, walk_all(walker, frames, chunk)):
            want, end = py_blocks(f)
            assert st == 0 and blocks == want, (len(f), chunk)
            assert consumed == end == len(f)
            assert closed == (f[:4] != b"\x02\x21\x4c\x18")


def test_mutated_frames_match_oracle_status(walker):
    """2 000 seeded byte flips and truncations: the walk stays inside the input (the sanitizer checks every read)
    and reports the oracle's status whenever that status is one the walk decides."""
    rng = np.random.default_rng(2024)
    j = corpus.tiled("compression_66k_JSON.txt", 400000).tobytes()
    bases = [oracle.frame_compress(j, 4, 7), oracle.frame_compress(j, 4, 5), oracle.frame_compress(j, 5, 0),
             oracle.frame_compress(j[:5000], 4, 7, 700)]
    cases = []
    for i in range(2000):
        f = bytearray(bases[i % len(bases)])
        kind = i % 3
        if kind != 1:                                                      # byte flips, often in the header / BlockInfo
            for _ in range(int(rng.integers(1, 4))):
                p = int(rng.integers(0, 24)) if rng.random() < 0.4 else int(rng.integers(0, len(f)))
                f[p] ^= 1 << int(rng.integers(0, 8))
        if kind != 0:
            f = f[:int(rng.integers(0, len(f) + 1))]
        cases.append(bytes(f))
    results = walk_all(walker, cases)
    decided = 0
    for t, (f, (st, consumed, blocks, _, _)) in enumerate(zip(cases, results)):
        assert consumed <= len(f)
        want, _, _ = oracle.frame_decompress(f, 4 << 20)
        if want in WALK_STATUSES:
            decided += 1
            assert st == want, (t, len(f), st, want)
    assert decided > 800
