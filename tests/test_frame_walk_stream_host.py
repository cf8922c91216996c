"""CPU tests of the streaming frame walk (fw::frame_walk_stream in lz4_flex_b200/csrc/lz4b200_frame_walk.cuh), the walk
lz4b200_frame_decoder runs on the GPU over each presented chunk.  tests/cpp/frame_walk_stream_host.cpp, compiled by g++
under AddressSanitizer and UndefinedBehaviorSanitizer, presents every frame of the corpus in many chunkings: all at once,
at every unit boundary, in random chunks and in 1-byte steps, with 1, 3 or 65 536 blocks per call.  For each, the
streaming walk must record the blocks fw::frame_walk records on the whole input and end in the same FrameWalk; it must
take whole units only, stop for input without a status and with a `need` past the bytes it had, and never read at or
past the bytes presented.  No GPU needed."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from stream_frames import broken_frames, byte_steps, random_splits, unit_ends, valid_frames

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "frame_walk_stream_host.cpp")
HDR = os.path.join(os.path.dirname(HERE), "lz4_flex_b200", "csrc", "lz4b200_frame_walk.cuh")
API = os.path.join(os.path.dirname(HERE), "include", "lz4b200.h")
EXE = os.path.join(HERE, "cpp", "_build", "frame_walk_stream_host")


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

    def run(cases):
        """cases: (max_blocks, frame, splits) -> (ok, status, ip, nblocks, calls) each; fails on any sanitizer report."""
        blob = b"".join(struct.pack("<IQ", mb, len(f)) + f + struct.pack("<I", len(s)) + struct.pack(f"<{len(s)}Q", *s)
                        for mb, f, s in cases)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        r = subprocess.run([EXE], input=blob, capture_output=True, env=env)
        assert r.returncode == 0 and not r.stderr, r.stderr.decode(errors="replace")[-4000:]
        lines = r.stdout.decode().splitlines()
        assert len(lines) == len(cases)
        return [tuple(map(int, ln.split())) for ln in lines]
    return run


def check_all(walker, named_cases):
    results = walker([c for _, c in named_cases])
    for (name, (mb, f, s)), (ok, st, ip, nb, calls) in zip(named_cases, results):
        assert ok == 1, (name, mb, len(f), len(s), st, ip, nb)
    return results


def test_valid_frames_every_split(walker):
    rng = np.random.default_rng(11)
    cases = []
    for name, f in valid_frames():
        n = len(f)
        cases.append((name + " whole", (65536, f, [n])))
        cases.append((name + " whole 3", (3, f, [n])))
        ends = unit_ends(f)
        if ends[-1] != n:
            ends.append(n)
        cases.append((name + " units", (1, f, ends)))
        cases.append((name + " units shifted", (2, f, sorted({min(n, e + 1) for e in ends} | {n}))))
        cases.append((name + " random", (int(rng.choice([1, 3, 65536])), f, random_splits(n, rng, 300000))))
        if n < (3 << 20):                                                  # each call copies up to a whole block
            cases.append((name + " small random", (65536, f, random_splits(n, rng, 5000))))
        cases.append((name + " bytes", (65536, f, byte_steps(n))))
    results = check_all(walker, cases)
    for (name, _), (_, st, ip, nb, _) in zip(cases, results):
        assert st == 0, name


def test_broken_frames_every_split(walker):
    rng = np.random.default_rng(12)
    cases = []
    for name, f in broken_frames():
        n = len(f)
        cases.append((name + " whole", (65536, f, [n])))
        cases.append((name + " random", (int(rng.choice([1, 3, 65536])), f, random_splits(n, rng, 40000))))
        cases.append((name + " bytes", (1, f, byte_steps(n, 120, 20))))
    results = check_all(walker, cases)
    assert len({r[1] for r in results}) >= 6                              # header errors, EOF, too big, OK, ...


def test_every_byte_step_of_small_frames(walker):
    from stream_frames import linked_frame
    import oracle
    from lz4_flex_b200 import corpus
    d = corpus.load("dickens.txt")[:30000]
    frames = [oracle.frame_compress(d, 4, flags, 3000) for flags in range(8)]
    frames.append(linked_frame(d, [5000, 300, 12000], 4, True, True, True))
    cases = [(f"small {i}", (mb, f, list(range(1, len(f) + 1)))) for i, f in enumerate(frames) for mb in (1, 65536)]
    check_all(walker, cases)
