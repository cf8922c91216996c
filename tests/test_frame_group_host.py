"""CPU tests of the batch frame decoder's planning step (lz4_flex_b200/csrc/lz4b200_frame_walk.cuh), compiled for the
host by g++ under AddressSanitizer and UndefinedBehaviorSanitizer (tests/cpp/frame_group_host.cpp): the one-group rule
(`group_cut`, which the one-frame group loop also runs) against a Python restatement of that loop's cut on random block
lists, and the count walk on real frames against their block lists.  No GPU needed."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import oracle
from lz4_flex_b200 import corpus

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "frame_group_host.cpp")
HDR = os.path.join(os.path.dirname(HERE), "lz4_flex_b200", "csrc", "lz4b200_frame_walk.cuh")
API = os.path.join(os.path.dirname(HERE), "include", "lz4b200.h")
EXE = os.path.join(HERE, "cpp", "_build", "frame_group_host")


@pytest.fixture(scope="module")
def counter():
    if shutil.which("g++") is None:
        pytest.fail("g++ is required to build the host frame count")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in (SRC, HDR, API)):
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


def list_record(budget, bs, blocks):
    return (struct.pack("<BQQI", 0, budget, bs, len(blocks))
            + b"".join(struct.pack("<QI", off, word) for off, word in blocks))


def frame_record(budget, f: bytes):
    return struct.pack("<BQQ", 1, budget, len(f)) + f


def cap(word, bs):
    return 0 if word & 0x80000000 else min(bs, (word & 0x7FFFFFFF) * 255 + 16)


def py_groups(blocks, bs, budget):
    """The group loop of decode_frame_blocks, restated: [(g0, g1)] for an independent-block frame."""
    groups, g0 = [], 0
    while g0 < len(blocks):
        g1, slot_total = g0, 0
        while g1 < len(blocks):
            c = cap(blocks[g1][1], bs)
            in_span = blocks[g1][0] + (blocks[g1][1] & 0x7FFFFFFF) - blocks[g0][0]
            if g1 > g0 and (slot_total + c > budget or in_span > budget):
                break
            slot_total += (c + 15) & ~15
            g1 += 1
        groups.append((g0, g1))
        g0 = g1
    return groups


def random_blocks(rng, bs):
    nb = int(rng.integers(0, 200))
    style = int(rng.integers(0, 3))                      # tiny payloads (caps of 255 x), full blocks, or a mix
    blocks, off = [], int(rng.integers(7, 20))
    for _ in range(nb):
        off += 4
        if style == 0:
            ln = int(rng.integers(1, 64))
        elif style == 1:
            ln = int(rng.integers(bs // 2, bs + 1))
        else:
            ln = int(rng.integers(1, bs + 1))
        word = ln | (0x80000000 if rng.random() < 0.2 else 0)
        blocks.append((off, word))
        off += ln + (4 if rng.random() < 0.5 else 0)
    return blocks


def test_one_group_rule_matches_group_loop(counter):
    rng = np.random.default_rng(31)
    cases = []
    for _ in range(3000):
        bs = int(rng.choice([64 << 10, 256 << 10, 1 << 20, 4 << 20, 8 << 20]))
        budget = int(rng.choice([1 << 20, 3 << 20, 16 << 20, 256 << 20])) + int(rng.integers(0, 17))
        cases.append((budget, bs, random_blocks(rng, bs)))
    got = counter(b"".join(list_record(*c) for c in cases))
    assert len(got) == len(cases)
    kinds = set()
    for (budget, bs, blocks), (slot_total, nb, one_group, linked, _, _) in zip(cases, got):
        groups = py_groups(blocks, bs, budget)
        assert nb == len(blocks) and linked == 0
        assert slot_total == sum((cap(w, bs) + 15) & ~15 for _, w in blocks)
        assert one_group == (len(groups) <= 1), (budget, bs, len(blocks), groups[:3])
        kinds.add((one_group, len(blocks) > 1))
    assert kinds == {(0, True), (1, True), (1, False)}


def test_count_walk_on_frames(counter):
    j = corpus.tiled("compression_66k_JSON.txt", 600000).tobytes()
    gdir = os.path.join(HERE, "golden", "linked")
    linked = [open(os.path.join(gdir, f), "rb").read() for f in sorted(os.listdir(gdir)) if f.endswith(".lz4")]
    frames = [oracle.frame_compress(j, 4, 7), oracle.frame_compress(j, 5, 0), oracle.frame_compress(j, 4, 7, 700),
              oracle.frame_compress(b"", 4, 7), corpus.load("dickens.lz4")] + linked
    frames += [f[:len(f) // 2] for f in frames[:3]]
    for budget in (1 << 20, 256 << 20):
        got = counter(b"".join(frame_record(budget, f) for f in frames))
        for f, (slot_total, nb, one_group, lnk, status, consumed) in zip(frames, got):
            assert consumed <= len(f)
            is_linked = f[:4] == b"\x04\x22\x4d\x18" and not (f[4] & 0x20)
            assert lnk == int(is_linked and nb > 1)
            if is_linked:
                assert one_group == 1
            if f[:4] == b"\x04\x22\x4d\x18":
                flg, bs = f[4], (64 << 10) << (2 * (((f[5] >> 4) & 7) - 4))
                pos = 7 + (8 if flg & 0x08 else 0)
                blocks = []
                while pos + 4 <= len(f):
                    w = int.from_bytes(f[pos:pos + 4], "little")
                    if w == 0 or pos + 4 + (w & 0x7FFFFFFF) + (4 if flg & 0x10 else 0) > len(f):
                        break
                    blocks.append((pos + 4, w))
                    pos += 4 + (w & 0x7FFFFFFF) + (4 if flg & 0x10 else 0)
                assert nb == len(blocks)
                assert slot_total == sum((cap(w, bs) + 15) & ~15 for _, w in blocks)
                if not is_linked:
                    assert one_group == (len(py_groups(blocks, bs, budget)) <= 1)
