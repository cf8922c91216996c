"""Frames for the streaming frame decoder's tests (test_frame_walk_stream_host.py, test_gpu_frame_decoder_device.py):
oracle frames for every block size and option, the legacy and linked fixtures, linked frames with real cross-block
matches, and broken frames of every kind; plus the ways to split a frame into presented chunks."""
import os

import numpy as np

import oracle
from lz4_flex_b200 import corpus, frame

HERE = os.path.dirname(os.path.abspath(__file__))
MAGIC = b"\x04\x22\x4d\x18"


def linked_frame(data: bytes, block_lens, bsid: int = 4, block_checksums=False, content_checksum=False,
                 content_size=False) -> bytes:
    """A BlockMode::Linked frame of `data`, cut into blocks of the lengths `block_lens` gives in turn (capped at the
    block size).  Block k is compressed with the last 64 KiB of content before it as its dictionary, so its matches
    reach into earlier blocks, several of them when blocks are short; it is stored when that does not shrink it."""
    bs = 65536 << (2 * (bsid - 4))
    flg = 0x40 | (0x10 if block_checksums else 0) | (0x08 if content_size else 0) | (0x04 if content_checksum else 0)
    hdr = bytes([flg, bsid << 4]) + (len(data).to_bytes(8, "little") if content_size else b"")
    parts = [MAGIC, hdr, bytes([(frame.xxh32(hdr) >> 8) & 0xFF])]
    pos, i = 0, 0
    while pos < len(data):
        ln = min(block_lens[i % len(block_lens)], bs, len(data) - pos)
        i += 1
        blk = data[pos:pos + ln]
        c = oracle.compress_with_dict(blk, data[max(0, pos - 65536):pos])
        word, payload = (len(c), c) if len(c) < ln else (ln | 0x80000000, blk)
        parts.append(word.to_bytes(4, "little") + payload)
        if block_checksums:
            parts.append(frame.xxh32(payload).to_bytes(4, "little"))
        pos += ln
    parts.append(b"\0\0\0\0")
    if content_checksum:
        parts.append(frame.xxh32(data).to_bytes(4, "little"))
    return b"".join(parts)


def unit_ends(f: bytes):
    """The ends of the units of a well-formed frame at f[0:]: header, each block (BlockInfo, payload, checksum), and
    the EndMark with its content checksum."""
    u32 = lambda p: int.from_bytes(f[p:p + 4], "little")
    if u32(0) == 0x184C2102:
        flg, pos = 0, 4
    else:
        flg = f[4]
        pos = 7 + (8 if flg & 0x08 else 0)
    ends = [pos]
    while pos + 4 <= len(f):
        word = u32(pos)
        pos += 4
        if word == 0:
            pos += 4 if flg & 0x04 else 0
            ends.append(pos)
            break
        pos += (word & 0x7FFFFFFF) + (4 if flg & 0x10 else 0)
        ends.append(pos)
    return [e for e in ends if e <= len(f)]


def valid_frames():
    """(name, frame) of well-formed frames: oracle frames for every block size and option combination, short flushed
    blocks, empty and one-byte content, the legacy fixture, the linked fixtures and linked frames built here."""
    j = corpus.tiled("compression_66k_JSON.txt", 600000).tobytes()
    rnd = corpus.xorshift64star_bytes(70000).tobytes()
    d = corpus.load("dickens.txt")[: (4 << 20) + 300000]
    out = []
    for bsid, data in ((4, j + rnd + j[:1000]), (5, j + rnd), (6, j[:300000] * 4), (7, d)):
        for flags in range(8):
            out.append((f"oracle bs{bsid} flags{flags}", oracle.frame_compress(data, bsid, flags)))
    out.append(("flushed", oracle.frame_compress(j, 4, 7, 1000)))
    out.append(("empty", oracle.frame_compress(b"", 4, 7)))
    out.append(("one byte", oracle.frame_compress(b"a", 4, 7)))
    out.append(("legacy dickens", corpus.load("dickens.lz4")))
    gdir = os.path.join(HERE, "golden", "linked")
    out += [(f, open(os.path.join(gdir, f), "rb").read()) for f in sorted(os.listdir(gdir)) if f.endswith(".lz4")]
    dk = corpus.load("dickens.txt")[:700000]
    out.append(("linked short blocks", linked_frame(dk, [65536, 20000, 7000, 1000, 40000], 4, True, True, True)))
    out.append(("linked 256k", linked_frame(dk + rnd, [262144, 5000], 5, False, True)))
    return out


def broken_frames(seed: int = 5, mutations: int = 200):
    """(name, bytes) of inputs that are not one clean frame: concatenated frames, a frame truncated in every region,
    corrupted headers, skippable and wrong magic, and seeded byte flips and truncations."""
    j = corpus.tiled("compression_66k_JSON.txt", 300000).tobytes()
    f = oracle.frame_compress(j, 4, 7)
    lf = linked_frame(corpus.load("dickens.txt")[:200000], [65536, 3000, 30000], 4, True, True, True)
    out = [("concatenated", f + oracle.frame_compress(j[:5000], 5, 2)), ("linked + trailing", lf + f[:40])]
    ends = unit_ends(f)
    for c in sorted(set(range(0, 24)) | {e + d for e in ends[:3] + ends[-3:] for d in (-3, -1, 0, 1, 2)}):
        if 0 <= c < len(f):
            out.append((f"truncated at {c}", f[:c]))
    out += [("magic only", MAGIC), ("legacy magic only", b"\x02\x21\x4c\x18"),
            ("skippable", b"\x50\x2a\x4d\x18" + (4).to_bytes(4, "little") + b"abcd" + f),
            ("wrong magic", bytes([f[0] ^ 1]) + f[1:]), ("header checksum", f[:14] + bytes([f[14] ^ 1]) + f[15:]),
            ("block too big", f[:15] + (65537).to_bytes(4, "little") + f[19:]),
            ("content checksum", f[:-1] + bytes([f[-1] ^ 1])), ("linked content checksum", lf[:-1] + bytes([lf[-1] ^ 1])),
            ("short", b"\x04\x22"), ("header cut", f[:9])]
    rng = np.random.default_rng(seed)
    bases = [f, lf, oracle.frame_compress(j, 5, 0), oracle.frame_compress(j[:20000], 4, 7, 700)]
    for i in range(mutations):
        g = bytearray(bases[i % len(bases)])
        kind = i % 3
        if kind != 1:
            for _ in range(int(rng.integers(1, 4))):
                p = int(rng.integers(0, 24)) if rng.random() < 0.4 else int(rng.integers(0, len(g)))
                g[p] ^= 1 << int(rng.integers(0, 8))
        if kind != 0:
            g = g[:int(rng.integers(0, len(g) + 1))]
        out.append((f"mutated {i}", bytes(g)))
    return out


def random_splits(n: int, rng, max_step: int):
    """Increasing chunk ends of random sizes in [1, max_step], the last one n."""
    ends, p = [], 0
    while p < n:
        p = min(n, p + int(rng.integers(1, max_step + 1)))
        ends.append(p)
    return ends or [0]


def byte_steps(n: int, head: int = 400, tail: int = 40):
    """Chunk ends one byte apart over the first `head` and the last `tail` bytes, one chunk in between."""
    if n <= head + tail:
        return list(range(1, n + 1)) or [0]
    return list(range(1, head + 1)) + list(range(n - tail, n + 1))
