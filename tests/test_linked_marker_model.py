"""A numpy model of the linked-frame range decoder (lz4b200_frame_decompress_ranges_device on linked frames), checked
against slices of the oracle's whole-frame decode.

A block of a linked frame decodes without the 64 KiB before it when each output byte is an entry: its value, or a marker
naming the earlier content byte it copies.  The model marker-decodes the blocks of a segment (consecutive touched
blocks and a look-back before them), resolves the markers in two passes as the kernels do (each block's last 64 KiB in
block order, then every other entry with one lookup), and doubles a segment's look-back, in blocks, while a requested
byte still copies content before it.  Segments whose look-backs meet merge.  The number of block decodes it runs is
the number lz4b200_ctx_last_range_blocks reports; tests/test_gpu_frame_range_linked.py compares the two."""
import json
import os

import numpy as np
import pytest

import oracle
from lz4_flex_b200 import corpus
from stream_frames import linked_frame

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "linked")
CARRY = 65536
POISON = -(1 << 62)          # a byte that copies content before its segment


def walk(f: bytes):
    """(payload_off, word) of every block of the frame at f[0:]."""
    flg = f[4]
    pos = 7 + (8 if flg & 0x08 else 0)
    out = []
    while True:
        word = int.from_bytes(f[pos:pos + 4], "little")
        pos += 4
        if word == 0:
            return out
        out.append((pos, word))
        pos += (word & 0x7FFFFFFF) + (4 if flg & 0x10 else 0)


def marker_decode(payload: bytes, stored: bool, decoded_off: int, cap: int):
    """The block's entries: values >= 0, markers -1 - p for a copy of content byte p before the block.  None where the
    block decoder fails (a copy before content byte 0 included) or the length is not cap."""
    if stored:
        return np.frombuffer(payload, dtype=np.uint8).astype(np.int64) if len(payload) == cap else None
    src, n = payload, len(payload)
    out = np.zeros(cap, dtype=np.int64)
    ip = op = 0
    if n == 0:
        return None
    while True:
        tok = src[ip]
        ip += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                if ip >= n:
                    return None
                b = src[ip]
                ip += 1
                lit += b
                if b != 255:
                    break
        if lit:
            if lit > n - ip or lit > cap - op:
                return None
            out[op:op + lit] = np.frombuffer(src, dtype=np.uint8, count=lit, offset=ip)
            ip += lit
            op += lit
        if ip >= n:
            break
        if n - ip < 2:
            return None
        dist = src[ip] | (src[ip + 1] << 8)
        ip += 2
        if dist == 0:
            return None
        m = 4 + (tok & 15)
        if m == 19:
            while True:
                if ip >= n:
                    return None
                b = src[ip]
                ip += 1
                m += b
                if b != 255:
                    break
        if dist > op and dist - op > decoded_off:
            return None
        if m > cap - op:
            return None
        if dist > op:
            pre = min(m, dist - op)
            out[op:op + pre] = -1 - (decoded_off + op - dist + np.arange(pre, dtype=np.int64))
            op += pre
            m -= pre
        if m:
            out[op:op + m] = np.resize(out[op - dist:op], m) if dist < m else out[op - dist:op - dist + m]
            op += m
        if ip >= n:
            return None
    return out if op == cap else None


def build_index(f: bytes):
    """The index entries (payload_off, decoded_off, word, decoded_len) of a valid linked frame, lengths from the oracle's
    block decoder with the content before the block as dictionary."""
    ent, content = [], b""
    for off, word in walk(f):
        payload = f[off:off + (word & 0x7FFFFFFF)]
        if word & 0x80000000:
            b = payload
        else:
            st, b, _, _ = oracle.decompress_with_dict(payload, 4 << 20, content[-65536:])
            assert st == 0
        ent.append((off, len(content), word, len(b)))
        content += b
    return ent, content


def block_at(offs, x):
    return int(np.searchsorted(offs, x, side="right")) - 1


def clip(s, ln, c):
    s = min(s, c)
    return s, s + min(ln, c - s)


def decode_ranges(f: bytes, ent, ranges, content_len: int):
    """The model of the range call: (bytes of every range, block decodes run, look-backs in blocks of the last round)."""
    nb = len(ent)
    offs = np.array([e[1] for e in ent], dtype=np.int64)
    touch = np.zeros(nb + 1, dtype=np.int64)
    clipped = [clip(s, ln, content_len) for s, ln in ranges]
    for s, e in clipped:
        if e > s:
            touch[block_at(offs, s)] += 1
            touch[block_at(offs, e - 1) + 1] -= 1
    run = np.cumsum(touch[:nb])
    act = []
    for b in range(nb):
        if run[b] <= 0:
            continue
        if act and act[-1][2] + 1 == b:
            act[-1][2] = b
            continue
        d = ent[b][1]
        act.append([block_at(offs, d - CARRY) if d > CARRY else 0, b, b])
    out = [None] * len(ranges)
    decodes, lookbacks = 0, []
    while act:
        merged = []
        for g in act:
            if merged and g[0] <= merged[-1][2] + 1:
                merged[-1][0] = min(merged[-1][0], g[0])
                merged[-1][2] = g[2]
            else:
                merged.append(list(g))
        act, nxt = merged, []
        for j, a, b in act:
            decodes += b - j + 1
            lookbacks.append(a - j)
            base = ent[j][1]
            parts = []
            for k in range(j, b + 1):
                off, d0, word, ln = ent[k]
                e = marker_decode(f[off:off + (word & 0x7FFFFFFF)], bool(word & 0x80000000), d0, ln)
                if e is None:
                    raise ValueError(f"block {k} fails")
                parts.append(e)
            E = np.concatenate(parts) if parts else np.zeros(0, np.int64)

            def look(v):
                p = -1 - v
                return np.where(p >= base, E[np.maximum(p - base, 0)], POISON)

            tail = np.zeros(E.size, dtype=bool)
            for k in range(j, b + 1):                      # serial pass: block tails in order
                d0, ln = ent[k][1] - base, ent[k][3]
                t = np.arange(d0 + ln - min(ln, CARRY), d0 + ln)
                v = E[t]
                mk = (v < 0) & (v != POISON)
                E[t[mk]] = look(v[mk])
                tail[t] = True
            v = E.copy()                                   # parallel pass: every other entry, one lookup
            mk = (v < 0) & (v != POISON) & ~tail
            E[mk] = look(v[mk])
            assert not ((E < 0) & (E != POISON)).any()
            c0, c1 = base, ent[b][1] + ent[b][3]
            unresolved = False
            for i, (s, e) in enumerate(clipped):
                if e > s and s >= c0 and e <= c1 and s >= ent[a][1]:
                    seg = E[s - c0:e - c0]
                    if (seg == POISON).any():
                        unresolved = True
                    else:
                        out[i] = seg.astype(np.uint8).tobytes()
            if unresolved:
                assert j > 0
                back = 2 * (a - j)
                nxt.append([0 if back >= a else a - back, a, b])
        act = nxt
    for i, (s, e) in enumerate(clipped):
        if e == s:
            out[i] = b""
    return out, decodes, lookbacks


def edges(ent, c):
    """The range shapes of the GPU tests' _edges: whole content, inside a block, on block boundaries, across stored and
    short blocks, empty ranges and ranges past the end."""
    r = [(0, c), (0, c + 10), (c, 5), (c + 7, 3), (0, 0), (c // 2, 0), (max(c - 1, 0), 100)]
    for _, d, _, L in ent:
        r += [(d, L), (d, 1), (d + L // 3, L // 3), (max(d - 1, 0), 2), (d + L, 0)]
        if len(r) > 600:
            break
    return r


def check(f: bytes, ranges):
    ent, content = build_index(f)
    assert oracle.frame_decompress(f, len(content) + 1)[1] == content
    got, decodes, lookbacks = decode_ranges(f, ent, ranges, len(content))
    for (s, ln), g in zip(ranges, got):
        assert g == content[s:s + ln], (s, ln)
    return decodes, lookbacks


def golden_frames():
    man = json.load(open(os.path.join(GOLDEN, "manifest.json")))
    return [(e["file"], open(os.path.join(GOLDEN, e["file"]), "rb").read()) for e in man]


def model_frames():
    """Linked frames of the model and GPU tests: short and mixed block lengths (matches reach across several blocks),
    stored blocks, every block size, and self-copying data."""
    json1 = corpus.load("compression_66k_JSON.txt")
    dick = corpus.load("dickens.txt")[:1 << 20]
    rnd = np.random.default_rng(5).integers(0, 256, 60 << 10, dtype=np.uint8).tobytes()
    zeros = bytes(600 << 10)
    return [
        ("json short blocks", linked_frame(json1, [1000, 5000, 300, 17, 40000])),
        ("dickens 64k", linked_frame(dick[:400000], [65536])),
        ("dickens mixed", linked_frame(dick[:300000], [70, 20000, 65536, 3, 9000])),
        ("stored and random", linked_frame(rnd[:20000] + json1[:30000] + rnd[20000:40000] + json1[30000:], [7000])),
        ("json 256k", linked_frame(corpus.tiled("compression_66k_JSON.txt", 700000).tobytes(), [1 << 20], bsid=5)),
        ("dickens 1m", linked_frame(dick, [1 << 20], bsid=6)),
        ("dickens 4m", linked_frame(dick + dick[:300000], [4 << 20], bsid=7)),
        ("random 60k repeated", linked_frame(rnd * 10, [65536])),
        ("zeros", linked_frame(zeros, [65536])),
    ]


@pytest.fixture(scope="module")
def frames():
    return golden_frames() + model_frames()


def test_model_on_edges(frames):
    for name, f in frames:
        ent, content = build_index(f)
        c = len(content)
        rng = np.random.default_rng(len(f))
        ranges = edges(ent, c) + [(int(rng.integers(0, c + 1)), int(rng.integers(0, 300000))) for _ in range(50)]
        decodes, _ = check(f, ranges)
        assert decodes > 0 or c == 0, name


def test_single_ranges_record_block_counts(frames):
    """A 4 KiB range at the start, the middle and the end of each frame: the model's bytes, and where the look-back
    went.  Data that repeats a random 60 KiB pattern copies itself from block to block, so its look-back reaches block
    0.  All-zero content resolves after one block: every block ends in literals."""
    rounds = {}
    for name, f in frames:
        ent, content = build_index(f)
        c = len(content)
        for where in (0, c // 2, max(c - 4096, 0)):
            rounds[(name, where)] = check(f, [(where, 4096)])[1]
    for name, f in frames:
        if name in ("random 60k repeated", "zeros"):
            ent, content = build_index(f)
            last = len(content) - 4096
            k = block_at(np.array([e[1] for e in ent]), last)
            assert rounds[(name, last)][-1] == (k if name != "zeros" else 1), (name, rounds[(name, last)])


def test_text_look_back_is_bounded():
    """6 MiB of dickens in 64 KiB linked blocks: a 4 KiB range in the last blocks decodes a few blocks, not 96."""
    f = linked_frame(corpus.load("dickens.txt")[:6 << 20], [65536])
    ent, content = build_index(f)
    c = len(content)
    for where in (c - 4096, c - 70000, c // 2):
        decodes, lookbacks = check(f, [(where, 4096)])
        assert decodes <= 12 and lookbacks[-1] <= 4, (where, decodes, lookbacks)


def test_overlapping_copies_keep_markers():
    """A match with offset < length whose source starts before the block copies markers byte by byte: a run that
    repeats the last 3 bytes of the previous block for 40 bytes."""
    prev = b"0123456789abc"
    blk = bytes([0x0F | (0 << 4)]) + (3).to_bytes(2, "little") + bytes([40 - 19]) + bytes([0x10]) + b"Z"
    e = marker_decode(blk, False, len(prev), 41)
    assert e is not None
    want = [-1 - (len(prev) - 3 + (i % 3)) for i in range(40)] + [ord("Z")]
    assert e.tolist() == want
    # one byte further back than content byte 0 fails the block
    assert marker_decode(bytes([0x00]) + (14).to_bytes(2, "little") + bytes([0x00]), False, 13, 4) is None
