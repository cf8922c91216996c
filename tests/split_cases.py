"""Inputs of concatenated LZ4 frames for the frame split's tests (tests/test_frame_split_host.py on the CPU,
tests/test_gpu_frame_split.py on the GPU), and a Python model of the regions the serial decode loop
(lz4b200_frame_decompress_next, called again at in + consumed) visits."""
import os

import numpy as np

import oracle
from lz4_flex_b200 import corpus, frame

HERE = os.path.dirname(os.path.abspath(__file__))
FRAME_MAGIC, LEGACY_MAGIC = 0x184D2204, 0x184C2102


def _u32(b, p):
    return int.from_bytes(b[p:p + 4], "little")


def walk(b: bytes, p: int):
    """(ok, consumed) of the header and BlockInfo walk of the frame at b[p:] (no block checksums): ok is the walk's
    status being OK, consumed the bytes it took (lz4b200_frame_walk.cuh, frame/decompress.rs:109-342)."""
    n = len(b) - p
    if n < 4:
        return False, n
    magic = _u32(b, p)
    if magic == LEGACY_MAGIC:
        bs, flg, ip = 8 << 20, 0x20, 4
    else:
        if n == 4:
            return True, 4
        if n < 7 or magic != FRAME_MAGIC:
            return False, 0
        flg, bd = b[p + 4], b[p + 5]
        o = 6 + (8 if flg & 0x08 else 0) + (4 if flg & 0x01 else 0)
        if n < o + 1 or (flg & 0xC0) != 0x40 or flg & 0x02 or bd & 0x8F or (bd >> 4) & 7 < 4:
            return False, 0
        if (frame.xxh32(b[p + 4:p + o]) >> 8) & 0xFF != b[p + o] or flg & 0x01:
            return False, 0
        bs, ip = (64 << 10) << (2 * (((bd >> 4) & 7) - 4)), o + 1
    while True:
        if n - ip < 4:
            return True, n                                    # the input ends where a BlockInfo is due
        word = _u32(b, p + ip)
        ip += 4
        if word == 0:
            if flg & 0x04:
                if n - ip < 4:
                    return False, n
                ip += 4
            return True, ip
        ln = word & 0x7FFFFFFF
        if ln > bs or n - ip < ln:
            return False, n
        ip += ln
        if flg & 0x10:
            if n - ip < 4:
                return False, n
            ip += 4


def regions(b: bytes):
    """[(offset, length)] of the regions the serial loop visits."""
    out, p = [], 0
    while p < len(b):
        ok, c = walk(b, p)
        if ok and p + c < len(b):
            out.append((p, c))
            p += c
        else:
            out.append((p, len(b) - p))
            break
    return out


def skippable(payload: bytes) -> bytes:
    return (0x184D2A53).to_bytes(4, "little") + len(payload).to_bytes(4, "little") + payload


def highway(nblocks: int) -> bytes:
    """A frame of nblocks stored blocks of 11 bytes, each payload a junk word and then a valid frame header whose walk
    continues into the real frame's next BlockInfo word: every fake header's unbounded walk would run to the end of the
    chain, so unbounded walks would cost nblocks^2 / 2 hops.  A small frame follows."""
    flg, bd = 0x60, 0x40
    hdr = FRAME_MAGIC.to_bytes(4, "little") + bytes([flg, bd, (frame.xxh32(bytes([flg, bd])) >> 8) & 0xFF])
    blk = (0x80000000 | 11).to_bytes(4, "little") + b"\x11\x22\x33\x44" + hdr
    return hdr + blk * nblocks + b"\0\0\0\0" + oracle.frame_compress(b"tail" * 100, 4, 7)


def cases():
    """name -> bytes: concatenations of valid frames, concatenations whose last region ends in an error, and
    concatenations with a frame in the middle that fails its block or content checksum."""
    j = corpus.tiled("compression_66k_JSON.txt", 300000).tobytes()
    rnd = corpus.xorshift64star_bytes(90000).tobytes()
    d = corpus.load("dickens.txt")[:300000]
    gdir = os.path.join(HERE, "golden", "linked")
    golden = [open(os.path.join(gdir, f), "rb").read() for f in sorted(os.listdir(gdir)) if f.endswith(".lz4")]
    legacy = corpus.load("dickens.lz4")
    mixed = []
    for bsid, data in ((4, j + rnd[:70000]), (5, j[:200000] + rnd), (6, d), (7, j)):
        for flags in range(8):
            mixed.append(oracle.frame_compress(data[:(bsid - 3) * 40000 + flags * 3000], bsid, flags))
    mixed.append(oracle.frame_compress(j[:50000], 4, 7, 1000))               # flushed short blocks
    empty = oracle.frame_compress(b"", 4, 7)
    small = [oracle.frame_compress(j[i * 300:i * 300 + 200 + i], 4, i % 8) for i in range(64)]
    inner = oracle.frame_compress(rnd[:3000], 4, 0) + oracle.frame_compress(rnd[3000:5000], 4, 5)
    nested = oracle.frame_compress(rnd[:20000] + inner + rnd[20000:40000] + inner + inner, 4, 0)
    good = b"".join(mixed)
    bad_hc = bytearray(small[3])
    bad_hc[6] ^= 0x5A
    c = {
        "mixed": good,
        "mixed_then_legacy": good + legacy,
        "empty_frames": empty * 5 + small[0] + empty * 3,
        "one_empty": empty,
        "linked_golden": b"".join(golden) + b"".join(golden[:2]),
        "small_frames": b"".join(small) * 3,
        "nested_frames": nested + small[1] + nested,
        "highway": highway(3000) + small[2],
        "skippable_middle": small[0] + small[1] + skippable(b"x" * 40) + small[2],
        "truncated_last": good[:len(good) - 1000],
        "header_checksum_middle": small[0] + bytes(bad_hc) + small[1],
        "block_too_big": small[0] + small[1][:7] + (0x00200000).to_bytes(4, "little") + b"z" * 64,
        "magic_only_tail": small[0] + FRAME_MAGIC.to_bytes(4, "little"),
    }
    bad_content = bytearray(oracle.frame_compress(j[5000:90000], 4, 2))   # content checksum
    bad_content[-1] ^= 0x01
    bad_block = bytearray(oracle.frame_compress(j[5000:200000], 4, 1))    # block checksums: the second block fails
    bad_block[7 + 4 + (int.from_bytes(bad_block[7:11], "little") & 0x7FFFFFFF) + 4 + 4 + 10] ^= 0x01
    c["content_checksum_middle"] = small[0] + bytes(bad_content) + small[1]
    c["block_checksum_middle"] = small[0] + bytes(bad_block) + small[1]
    for k in range(1, 8):
        c[f"junk_tail_{k}"] = small[4] + small[5] + b"\x07\x01\x02\x03\x04\x05\x06"[:k]
    return c
