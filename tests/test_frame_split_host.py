"""CPU tests of the frame split (lz4_flex_b200/csrc/lz4b200_frame_split.cuh): its four phases, compiled for the host by
g++ under AddressSanitizer and UndefinedBehaviorSanitizer (tests/cpp/frame_split_host.cpp) and run one after another,
give the regions the serial decode loop visits (a Python model of that loop), for every max_frames edge and through the
serial fallback; the hop count on converging fake headers stays linear; and the bound rule over the regions equals
lz4b200_frame_decoded_bound.  No GPU needed."""
import ctypes as C
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import split_cases
from lz4_flex_b200 import _native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "frame_split_host.cpp")
CSRC = os.path.join(os.path.dirname(HERE), "lz4_flex_b200", "csrc")
HDRS = [os.path.join(CSRC, "lz4b200_frame_split.cuh"), os.path.join(CSRC, "lz4b200_frame_walk.cuh"),
        os.path.join(os.path.dirname(HERE), "include", "lz4b200.h")]
EXE = os.path.join(HERE, "cpp", "_build", "frame_split_host")
HOPS = 64                                                   # kSplitHops


@pytest.fixture(scope="module")
def splitter():
    if shutil.which("g++") is None:
        pytest.fail("g++ is required to build the host frame split")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [SRC] + HDRS):
        tmp = f"{EXE}.tmp{os.getpid()}"
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-fno-omit-frame-pointer", "-o", tmp, SRC], check=True)
        os.replace(tmp, EXE)

    def run(records):
        """records: (max_frames, max_candidates, bytes) -> per record (regions, covered, candidates, hops, bound,
        [(offset, length)]); fails on any sanitizer report."""
        blob = b"".join(struct.pack("<QQQ", mf, mc, len(b)) + bytes(b) for mf, mc, b in records)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        r = subprocess.run([EXE], input=blob, capture_output=True, env=env)
        assert r.returncode == 0 and not r.stderr, (r.returncode, r.stderr.decode(errors="replace")[-4000:])
        lines, out, i = r.stdout.decode().splitlines(), [], 0
        for _ in records:
            nreg, covered, cand, hops, bound = map(int, lines[i].split())
            regs = [tuple(map(int, ln.split())) for ln in lines[i + 1:i + 1 + nreg]]
            out.append((nreg, covered, cand, hops, bound, regs))
            i += 1 + nreg
        assert i == len(lines)
        return out
    return run


@pytest.fixture(scope="module")
def cases():
    return split_cases.cases()


def host_bound(b: bytes) -> int:
    src = np.frombuffer(b, np.uint8)
    bound = C.c_size_t(0)
    assert _native.lib().lz4b200_frame_decoded_bound(src.ctypes.data if len(b) else None, len(b), C.byref(bound)) == 0
    return bound.value


def default_candidates(n: int) -> int:
    return n // 128 + 1024


def test_regions_match_the_serial_loop(splitter, cases):
    names = list(cases) + ["nothing"]
    inputs = list(cases.values()) + [b""]
    got = splitter([(1 << 40, default_candidates(len(b)), b) for b in inputs])
    for name, b, (nreg, covered, cand, _, bound, regs) in zip(names, inputs, got):
        want = split_cases.regions(b)
        assert regs == want, name
        assert covered == len(b), name
        if name != "highway":                                          # a fake header every 15 bytes
            assert cand <= default_candidates(len(b)), name            # the parallel path, not the fallback
        assert bound == host_bound(b), name
    assert len(split_cases.regions(cases["mixed"])) == 33
    assert got[names.index("nothing")][0] == 0


def test_max_frames_edges(splitter, cases):
    for name in ("mixed", "junk_tail_3", "linked_golden", "skippable_middle"):
        b = cases[name]
        want = split_cases.regions(b)
        R = len(want)
        limits = sorted({0, 1, max(R - 1, 0), R, R + 1})
        got = splitter([(m, default_candidates(len(b)), b) for m in limits])
        for m, (nreg, covered, _, _, _, regs) in zip(limits, got):
            k = min(m, R)
            assert nreg == k and regs == want[:k], (name, m)
            assert covered == (want[k][0] if k < R else len(b)), (name, m)


def test_too_many_candidates_walk_serially(splitter, cases):
    """max_candidates below the candidate count: the chain walk walks every frame itself and gives the same regions."""
    for name in ("mixed_then_legacy", "small_frames", "nested_frames", "header_checksum_middle", "junk_tail_7"):
        b = cases[name]
        want = split_cases.regions(b)
        (_, _, cand, _, _, _), = splitter([(1 << 40, 1 << 30, b)])
        assert cand >= len(want) - 1
        for mc in (0, cand - 1):
            (nreg, covered, _, _, bound, regs), = splitter([(1 << 40, mc, b)])
            assert regs == want and covered == len(b), (name, mc)
            assert bound == host_bound(b)


def test_false_candidates_inside_stored_blocks(splitter, cases):
    """Whole .lz4 files stored inside a frame's blocks are candidates whose walks succeed; they are not regions."""
    b = cases["nested_frames"]
    (nreg, _, cand, _, _, regs), = splitter([(1 << 40, default_candidates(len(b)), b)])
    assert regs == split_cases.regions(b) and nreg == 3
    assert cand >= 3 + 2 * 2                                          # the first stored copy of both inner frames


def test_converging_walks_stay_linear(splitter):
    """Fake headers inside every payload of one long frame: each candidate's walk stops after kSplitHops BlockInfo
    words and the chain walk reads the long frame once, so hops grow linearly with the frame, not quadratically."""
    sizes = (500, 1000, 2000, 4000, 8000)
    got = splitter([(1 << 40, 1 << 20, split_cases.highway(k)) for k in sizes])
    for k, (nreg, covered, cand, hops, _, regs) in zip(sizes, got):
        assert regs == split_cases.regions(split_cases.highway(k)) and nreg == 2
        assert cand == k + 2
        assert hops <= HOPS * cand + 2 * (k + 1) + 16, (k, hops)
    assert got[-1][3] < 20 * got[0][3]                               # 16x the blocks: about 16x the hops
