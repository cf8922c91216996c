"""The linked-block decoder (lz4_decompress_blocks_linked) against the oracle, on frames built here from explicit
sequences, so every offset and match length is exactly what the case asks for.

Linked frames (what `lz4`, LZ4F and pyarrow write by default) are decoded by one kernel on every frame decoder path:
the host call, the device call, the batch call and the streaming decoder, which adds the frame's last <= 64 KiB of
output as a stored pseudo-block ahead of each group.  The cases aim at what only that kernel does: the walk back over
earlier blocks, the copy that switches between stored payloads and decoded slots inside one match, overlapping matches
whose source starts in an earlier block, the frame's first byte as the furthest legal source, the order of
OffsetOutOfBounds before OutputTooSmall, the block size as every block's capacity, a block that ends on a match,
zero-length stored blocks, and failing blocks that later blocks reference.  Each path is compared with
oracle.frame_decompress (status, block status, bytes) and with the host call on every result field; nothing past
`written` may change.

Two differences from the reference are pinned, not replicated (include/lz4b200.h, SURVEY.md): OutputTooSmall's
expected / actual are relative to the block (expected = the block's output so far + the run, actual = the block size),
and a block that decodes to more than the block size fails with OutputTooSmall even where the reference's buffer has
wrapped and would let it through."""
from __future__ import annotations

import numpy as np
import pytest

import oracle
from lz4_flex_b200 import frame
from test_gpu_launch_shapes import seq

BSID = 4
BS = 65536
MAGIC = b"\x04\x22\x4d\x18"
DEC_ERR = oracle.FERR_DECOMPRESSION
OTS, LIT_OOB, EAB, OFF0, OFF_OOB = (oracle.ERR_OUTPUT_TOO_SMALL, oracle.ERR_LITERAL_OOB, oracle.ERR_EXPECTED_ANOTHER_BYTE,
                                    oracle.ERR_OFFSET_ZERO, oracle.ERR_OFFSET_OOB)
BOUNDARIES = {"stored->compressed", "compressed->stored", "stored->stored", "compressed->compressed", "through_zero"}


# ---- blocks and frames ---------------------------------------------------------------------------------------------

def S(data: bytes):
    """A stored block (any length, 0 included)."""
    return ("s", bytes(data), len(data), None)


def C(*seqs):
    """A compressed block of sequences (literals, dist, mlen); the last one may be (literals,) alone.  Its decoded
    length assumes every sequence decodes."""
    payload = b"".join(seq(*s) for s in seqs)
    return ("c", payload, sum(len(s[0]) + (s[2] if len(s) > 1 else 0) for s in seqs), seqs)


def RAW(payload: bytes):
    """A compressed block given as its exact payload (truncated or malformed streams)."""
    return ("c", bytes(payload), None, None)


def Z():
    return S(b"")


def _r(rng, n: int) -> bytes:
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def frame_bytes(blocks, flags: int = 0, content: bytes = b"", bad_sum=None) -> bytes:
    """A linked frame of `blocks`.  flags: oracle.F_BLOCK_CHECKSUMS | F_CONTENT_CHECKSUM | F_CONTENT_SIZE (over
    `content`); block `bad_sum` gets a wrong checksum."""
    flg = (0x40 | (0x10 if flags & oracle.F_BLOCK_CHECKSUMS else 0) | (0x08 if flags & oracle.F_CONTENT_SIZE else 0)
           | (0x04 if flags & oracle.F_CONTENT_CHECKSUM else 0))
    hdr = bytes([flg, BSID << 4]) + (len(content).to_bytes(8, "little") if flags & oracle.F_CONTENT_SIZE else b"")
    out = bytearray(MAGIC + hdr + bytes([(frame.xxh32(hdr) >> 8) & 0xFF]))
    for k, (kind, payload, _, _) in enumerate(blocks):
        out += (len(payload) | (0x80000000 if kind == "s" else 0)).to_bytes(4, "little") + payload
        if flags & oracle.F_BLOCK_CHECKSUMS:
            out += (frame.xxh32(payload) ^ (k == bad_sum)).to_bytes(4, "little")
    out += bytes(4)
    if flags & oracle.F_CONTENT_CHECKSUM:
        out += frame.xxh32(content).to_bytes(4, "little")
    return bytes(out)


def decoded_bound(blocks) -> int:
    return sum(len(p) if k == "s" else min(BS, 255 * len(p) + 16) for k, p, _, _ in blocks)


def block_ob(b) -> int:
    """What the streaming decoder reserves of out_cap for a block (decoder_step)."""
    return len(b[1]) if b[0] == "s" else min(BS, 255 * len(b[1]) + 16)


class Case:
    """One frame: its blocks, bytes, the status it was built for (None: the oracle decides), the oracle's
    (status, block_status, bytes delivered before the first failing block), and what it covers."""

    def __init__(self, name, blocks, want=None, err=None, flags=0, bad_sum=None, stream_cap=None, edge=None):
        self.name, self.blocks, self.want, self.err, self.flags, self.bad_sum = name, blocks, want, err, flags, bad_sum
        self.edge = edge                        # index of the block whose match reaches frame byte 0 (or one further)
        self.cap = decoded_bound(blocks) + BS   # room for a full block after any output: the oracle sees OutputTooSmall
        plain = frame_bytes(blocks)
        st, out, _ = oracle.frame_decompress(plain, self.cap)
        self.fail = None                        # the first block that fails to decode
        content = out
        if st != 0:
            for k in range(len(blocks)):
                if oracle.frame_decompress(frame_bytes(blocks[:k + 1]), self.cap)[0] != 0:
                    self.fail = k
                    content = oracle.frame_decompress(frame_bytes(blocks[:k]), self.cap)[1]
                    break
        self.frame = frame_bytes(blocks, flags, content, bad_sum)
        self.ost, out, self.obst = oracle.frame_decompress(self.frame, self.cap)
        stop = min(x for x in (self.fail, bad_sum, len(blocks)) if x is not None)
        self.data = out if self.ost == 0 else oracle.frame_decompress(frame_bytes(blocks[:stop]), self.cap)[1]
        self.stream_cap = max([stream_cap or BS] + [block_ob(b) for b in blocks])
        self.tags = coverage(blocks)

    def __repr__(self):
        return f"<{self.name}: {len(self.blocks)} blocks, oracle {self.ost}/{self.obst}>"


def coverage(blocks):
    """What the frame's matches exercise: 'spanN' (the source lies in N earlier non-empty blocks), the kinds of block
    boundary inside a source (the current block counts as compressed; 'through_zero': zero-length blocks sit on it),
    'overlap_cross' (dist < mlen, source starting in an earlier block) and 'byte0' (the source starts at frame byte 0
    from a later block)."""
    tags = set()
    starts, pos = [], 0
    for b in blocks:
        starts.append(pos)
        pos += b[2] or 0
    for j, (kind, _, _, seqs) in enumerate(blocks):
        if kind != "c" or seqs is None:
            continue
        base, op = starts[j], starts[j]
        for s in seqs:
            op += len(s[0])
            if len(s) == 1:
                break
            dist, mlen = s[1], s[2]
            src = op - dist
            if dist == 0 or src < 0:
                break
            if src < base:
                hi = src + min(mlen, dist)           # the distinct source bytes
                touched = [k for k in range(j) if blocks[k][2] and starts[k] < min(hi, base) and
                           starts[k] + blocks[k][2] > src]
                tags.add(f"span{len(touched)}")
                if dist < mlen:
                    tags.add("overlap_cross")
                if src == 0:
                    tags.add("byte0")
                for p in sorted({starts[k] for k in range(1, j + 1)}):
                    if not src < p < hi:
                        continue
                    before = [k for k in range(j) if blocks[k][2] and starts[k] + blocks[k][2] == p]
                    after = [k for k in range(j + 1) if (blocks[k][2] or k == j) and starts[k] == p]
                    if any(starts[k] == p and not blocks[k][2] for k in range(j)):
                        tags.add("through_zero")
                    name = lambda k: "stored" if blocks[k][0] == "s" else "compressed"
                    if before and after:
                        tags.add(f"{name(before[-1])}->{name(after[0])}")
            op += mlen
    return tags


# ---- hand-built cases ----------------------------------------------------------------------------------------------

def span_cases():
    """Matches whose source spans 1, 2, 3 and 8 earlier blocks of 1..20 bytes (stored, compressed, zero-length), each
    source starting and ending at block edges and inside blocks, plus overlapping matches (dist 1..40) whose source
    starts in an earlier block and runs on into the current one."""
    rng = np.random.default_rng(11)
    r = lambda n: _r(rng, n)
    prefixes = [
        [S(r(7)), C((r(9),))],
        [C((r(5), 3, 6), (r(2),)), S(r(6))],
        [S(r(5)), Z(), C((r(8),))],
        [C((r(6),)), Z(), S(r(4))],
        [C((r(6),)), Z(), Z(), C((r(1), 1, 6), (r(1),))],
        [S(r(3)), Z(), S(r(9)), C((r(2),))],
        [S(r(3)), C((r(4),)), Z(), S(r(2)), C((r(14), 9, 6), (r(1),)), S(r(1)), Z(), C((r(5),)), S(r(6)), C((r(7),))],
        [C((r(20),)), S(r(20)), C((r(1), 1, 15), (r(4),)), S(r(1)), Z(), S(r(13)), C((r(3),)), S(r(2)), C((r(19),))],
    ]
    out = []
    for pi, pre in enumerate(prefixes):
        ends = np.cumsum([0] + [b[2] for b in pre])
        total = int(ends[-1])
        nz = [k for k, b in enumerate(pre) if b[2]]
        for nspan in (1, 2, 3, 8):
            if nspan > len(nz):
                continue
            first, last = nz[-nspan], nz[-1]
            for lit in (0, 3):
                for s_at in {int(ends[first]), int(ends[first]) + pre[first][2] - 1, int(ends[first]) + pre[first][2] // 2}:
                    # the source ends in the last earlier block, at its end, or runs into the current block's literals
                    for e_at in {int(ends[last]) + 1, total, total + lit}:
                        m = e_at - s_at
                        if m < 4 or e_at <= int(ends[last]) and nspan > 1:
                            continue
                        d = total + lit - s_at
                        out.append(Case(f"span{nspan} p{pi}", pre + [C((r(lit), d, m), (r(2),)), S(r(3))], (0, 0)))
        for dist in range(1, 41):                    # overlap across the boundary into the current block
            lit = dist % 4
            if dist > total + lit or dist <= lit:
                continue
            m = dist + 1 + dist % 7 + (dist % 3) * 20
            out.append(Case(f"overlap p{pi} d{dist}", pre + [C((r(lit), dist, m), (r(1),))], (0, 0)))
    return out


def byte0_cases():
    """dist = the frame's output so far reaches frame byte 0 (OK); one more is OFFSET_OUT_OF_BOUNDS.  In the first
    block, the second block, after a stored block, after zero-length blocks, and at dist 65 535 after exactly 65 535
    bytes and after more than 64 KiB."""
    rng = np.random.default_rng(12)
    r = lambda n: _r(rng, n)
    out = []
    for extra, st in ((0, (0, 0)), (1, (DEC_ERR, OFF_OOB))):
        for lit in (0, 1, 5):
            pres = {"first": [], "second": [C((r(9),))], "after_stored": [C((r(4),)), S(r(6))],
                    "after_zero": [S(r(5)), Z(), Z()], "zero_first": [Z(), C((r(3),))]}
            for where, pre in pres.items():
                total = sum(b[2] for b in pre)
                if total + lit == 0:
                    continue
                blk = C((r(lit), total + lit + extra, 4 + lit * 3), (r(2),))
                out.append(Case(f"byte0+{extra} {where} lit{lit}", pre + [blk, S(r(2))], st, edge=len(pre)))
        # dist 65 535 at exactly 65 535 bytes of output (and 65 534: one byte further than the frame)
        pre = [S(r(35535 - extra)), C((r(29990), 1, 8), (r(2),))]
        out.append(Case(f"dist65535+{extra}", pre + [C((b"", 65535, 9), (r(1),))], st, edge=2))
    big = [S(r(40000)), C((r(30000),))]                  # 70 000 bytes: 65 535 reaches byte 4 465
    out.append(Case("dist65535 after 70000", big + [C((r(2), 65535, 30), (r(1),)), S(r(1))], (0, 0)))
    out.append(Case("dist65535 overlap after 70000", big + [C((r(2), 65535, 65530), (r(1),))], (0, 0)))
    return out


def edge_cases():
    """Order of errors, the block size as capacity, streams that end badly, and failing blocks that later blocks
    reference.  `err`: the (err_expected, err_actual) every path reports for OutputTooSmall."""
    rng = np.random.default_rng(13)
    r = lambda n: _r(rng, n)
    pre = [S(r(7)), C((r(3),))]                          # 10 bytes before a later block
    out = []
    for name, p in (("first", []), ("later", pre)):
        t = sum(b[2] for b in p)
        tail = [S(r(3))]
        # exactly the block size: OK
        out.append(Case(f"bs exact match {name}", p + [C((r(5), 1, BS - 6), (r(1),))] + tail, (0, 0)))
        out.append(Case(f"bs exact literals {name}", p + [C((r(100), 1, BS - 200), (r(100),))] + tail, (0, 0)))
        # bs + 1 by a match, by literals after a match, by a match from earlier blocks (a payload holds at most the block
        # size, so a literal run alone cannot pass it)
        out.append(Case(f"bs+1 match {name}", p + [C((r(5), 1, BS - 4), (r(3),))] + tail, (DEC_ERR, OTS), (BS + 1, BS)))
        out.append(Case(f"bs+1 literals {name}", p + [C((r(5), 1, BS - 5), (r(1),))] + tail, (DEC_ERR, OTS), (BS + 1, BS)))
        if t:
            out.append(Case(f"bs+1 cross-block match {name}", p + [C((r(2), t + 2, BS - 1), (r(1),))] + tail,
                            (DEC_ERR, OTS), (BS + 1, BS)))
        # offset out of bounds and output too small at once: the offset wins (SURVEY.md, "Exact-decode specification")
        for lit in (0, 2, 10):
            if t + lit == 0:
                continue
            out.append(Case(f"oob before ots {name} lit{lit}", p + [C((r(lit), t + lit + 1, BS + 1), (r(1),))] + tail,
                            (DEC_ERR, OFF_OOB)))
            out.append(Case(f"byte0 with ots {name} lit{lit}", p + [C((r(lit), t + lit, BS + 1), (r(1),))] + tail,
                            (DEC_ERR, OTS), (lit + BS + 1, BS)))
        # streams that end badly
        for k, (kind, payload, st) in enumerate((
                ("ends on match", seq(r(3), 2, 5), EAB),
                ("ends on cross-block match", seq(r(1), t + 1, 6), EAB),
                ("offset 0", seq(r(3), 0, 5) + seq(r(2)), OFF0),
                ("truncated offset", bytes([0x30]) + r(3) + b"\x01", EAB),
                ("truncated match length", bytes([0x3F]) + r(3) + b"\x02\x00" + b"\xff" * 2, EAB),
                ("truncated literal length", bytes([0xF0]) + b"\xff", EAB),
                ("literals past the payload", bytes([0x50]) + r(3), LIT_OOB),
                ("token and one offset byte", bytes([0x04, 0x01]), EAB))):
            out.append(Case(f"{kind} {name}", p + [RAW(payload)] + tail, (DEC_ERR, st)))
        # a compressed block of one token and nothing else decodes to 0 bytes; the next block reaches over it
        out.append(Case(f"empty compressed block {name}", p + [RAW(b"\x00"), C((r(1), t + 1, 4), (r(1),))] + tail,
                        (0, 0)))
    # a failing block mid-frame, then blocks that reference it and each other, and a later failure of another kind
    body = [S(r(6)), C((r(4), 3, 9), (r(2),)), Z(), S(r(5))]
    later = [C((r(1), 12, 8), (r(1),)), S(r(3)), C((b"", 20, 30), (r(2),)), C((r(2), 0, 4), (r(1),))]
    for fk, (bad, st) in enumerate(((C((r(3), 40, 6), (r(1),)), OFF_OOB), (RAW(bytes([0x60]) + r(2)), LIT_OOB),
                                     (C((r(2), 1, BS), (r(1),)), OTS), (RAW(seq(r(2), 7, 7)), EAB))):
        err = (2 + BS, BS) if st == OTS else None
        out.append(Case(f"mid-frame failure {fk}", body + [bad] + later, (DEC_ERR, st), err))
    # a block with a bad checksum mid-frame: later blocks reference it, nothing of it or after it is decoded
    bl = body + [C((r(3), 5, 12), (r(1),))] + later[:3]
    out.append(Case("bad checksum mid-frame", bl, (oracle.FERR_BLOCK_CHECKSUM, 0), flags=oracle.F_BLOCK_CHECKSUMS,
                    bad_sum=4))
    out.append(Case("checksums, content size and checksum", bl, (0, 0), flags=7))
    return out


def window_cases():
    """Edge offsets in a later group of the streaming decoder, while its window is shorter than 64 KiB: small blocks
    under a small out_cap (a group every block or two), and 18 blocks of 64 KiB slots under a 1 MiB frame budget (a
    cut after 16).  The last block's match reaches frame byte 0 through the window, or one byte further."""
    rng = np.random.default_rng(14)
    r = lambda n: _r(rng, n)
    out = []
    small = [C((r(10 + k),)) if k % 3 else S(r(1 + 3 * k)) for k in range(9)] + [Z()]
    budget = [C((r(300),)) for _ in range(18)]
    for extra, st in ((0, (0, 0)), (1, (DEC_ERR, OFF_OOB))):
        for lit in (0, 3):
            for name, pre, cap in (("small out_cap", small, 4000), ("budget", budget, 8 << 20)):
                total = sum(b[2] for b in pre)
                blk = C((r(lit), total + lit + extra, 5 + lit), (r(1),))
                out.append(Case(f"window {name} +{extra} lit{lit}", pre + [blk], st, stream_cap=cap, edge=len(pre)))
    return out


def random_cases(count: int = 2000, seed: int = 21):
    """Seeded frames of 1..8 short blocks: stored (also empty) and compressed blocks of 1..4 sequences with random
    literals, dist and mlen (a few offsets past the frame's start, a few zero, a few blocks ending on a match)."""
    rng = np.random.default_rng(seed)
    r = lambda n: _r(rng, n)
    out = []
    for i in range(count):
        blocks, total = [], 0
        for _ in range(int(rng.integers(1, 9))):
            u = rng.random()
            if u < 0.12:
                blocks.append(Z())
            elif u < 0.35:
                blocks.append(S(r(int(rng.integers(1, 21)))))
            else:
                seqs, op = [], 0
                for _ in range(int(rng.integers(1, 5))):
                    lit = r(int(rng.integers(0, 8)))
                    avail = total + op + len(lit)
                    v = rng.random()
                    dist = (0 if v < 0.02 else avail + int(rng.integers(1, 3)) if v < 0.08 or not avail
                            else int(rng.integers(1, avail + 1)))
                    mlen = int(rng.integers(4, 41))
                    seqs.append((lit, dist, mlen))
                    op += len(lit) + mlen
                if rng.random() < 0.92:
                    seqs.append((r(int(rng.integers(1, 6))),))
                blocks.append(C(*seqs))
            total += blocks[-1][2]
        flags = int(rng.integers(0, 8)) if rng.random() < 0.3 else 0
        out.append(Case(f"random {i}", blocks, flags=flags & 7, stream_cap=int(rng.integers(2000, 20000))))
    return out


def hand_cases():
    return span_cases() + byte0_cases() + edge_cases() + window_cases()


_CACHE = {}


def all_cases():
    if not _CACHE:
        _CACHE["hand"] = hand_cases()
        _CACHE["random"] = random_cases()
    return _CACHE["hand"], _CACHE["random"]


def stream_groups(case, out_cap: int, budget: int):
    """The groups the streaming decoder decodes the whole frame in (presented at once): decoder_step takes the longest
    prefix of blocks whose reserved output fits out_cap and that fw::group_cut would not cut.  Returns the first block
    of each group."""
    blocks = case.blocks
    hdr = 7 + (8 if case.flags & oracle.F_CONTENT_SIZE else 0)
    csum = 4 if case.flags & oracle.F_BLOCK_CHECKSUMS else 0
    offs, p = [], hdr
    for b in blocks:
        offs.append(p + 4)
        p += 4 + len(b[1]) + csum
    firsts, g0 = [], 0
    while g0 < len(blocks):
        firsts.append(g0)
        t, bound, slots = g0, 0, 0
        while t < len(blocks):
            b = blocks[t]
            cap = 0 if b[0] == "s" else block_ob(b)
            if bound + block_ob(b) > out_cap:
                break
            if t > g0 and (slots + cap > budget or offs[t] + len(b[1]) - offs[g0] > budget):
                break
            bound += block_ob(b)
            slots += (cap + 15) & ~15
            t += 1
        assert t > g0, "the next block alone does not fit out_cap"
        g0 = t
    return firsts


# ---- the generator itself (CPU) ------------------------------------------------------------------------------------

def test_generator_builds_what_it_claims():
    """Every hand-built frame decodes (oracle) to the status it was built for; the cases hold every decoder status,
    every kind of block boundary inside a match source and sources over 1, 2, 3 and 8 blocks; the window cases really
    put their edge block in a later group of the streaming decoder than frame byte 0, while its window is shorter than
    64 KiB."""
    hand, rnd = all_cases()
    for c in hand:
        got = (c.ost, c.obst if c.ost == DEC_ERR else 0)
        assert got == c.want, (c.name, got, c.want)
        if c.err:                                    # the failing block alone, with the frame so far as dictionary
            blk = oracle.decompress_with_dict(c.blocks[c.fail][1], BS, c.data)
            assert got == (DEC_ERR, OTS) and (blk[0],) + blk[2:] == (OTS,) + c.err, (c.name, blk[0], blk[2:], c.err)
    tags = set().union(*(c.tags for c in hand))
    assert BOUNDARIES | {"span1", "span2", "span3", "span8", "overlap_cross", "byte0"} <= tags, sorted(tags)
    statuses = {(c.ost, c.obst) for c in hand}
    assert {(0, 0), (oracle.FERR_BLOCK_CHECKSUM, 0)} | {(DEC_ERR, s) for s in (OTS, LIT_OOB, EAB, OFF0, OFF_OOB)} <= statuses
    rstat = [(c.ost, c.obst) for c in rnd]
    for s in {(0, 0)} | {(DEC_ERR, s) for s in (EAB, OFF0, OFF_OOB)}:
        assert rstat.count(s) >= 20, (s, {x: rstat.count(x) for x in set(rstat)})
    rtags = set().union(*(c.tags for c in rnd))
    assert BOUNDARIES | {"span1", "span2", "span3", "overlap_cross", "byte0"} <= rtags, sorted(rtags)
    # the window cases: the edge block opens a later group, with less than 64 KiB of output before it
    win = [c for c in hand if c.name.startswith("window")]
    assert len(win) == 8
    for c in win:
        budget = 1 << 20 if "budget" in c.name else 256 << 20
        firsts = stream_groups(c, c.stream_cap, budget)
        g = max(i for i, f in enumerate(firsts) if f <= c.edge)
        assert g > 0, (c.name, firsts)                   # frame byte 0 lies in the window, not in the group
        assert sum(b[2] for b in c.blocks[:firsts[g]]) < BS, c.name
    # the budget cut: on the default 256 MiB budget the same frame is one group under that out_cap
    c = next(c for c in win if "budget" in c.name)
    assert stream_groups(c, c.stream_cap, 256 << 20) == [0] and stream_groups(c, c.stream_cap, 1 << 20)[1] == 16


# ---- the GPU paths -------------------------------------------------------------------------------------------------

def _host(ctx, c):
    from test_gpu_frame_batch_device import host_next
    return host_next(ctx, c.frame, c.cap)


def _device(ctx, c):
    from test_gpu_frame_group_cuts import device_next
    return device_next(ctx, c.frame, c.cap)


def check_host(c, got):
    """A path's ((status, consumed, written, block_status, err_expected, err_actual), bytes) against the oracle."""
    (st, consumed, written, bst, e1, e2), data = got
    assert st == c.ost, (c.name, st, c.ost, bst, c.obst)
    if st == DEC_ERR:
        assert bst == c.obst, (c.name, bst, c.obst)
    assert written == len(data) and data == c.data, (c.name, written, len(c.data))
    if st == 0:
        assert consumed == len(c.frame), c.name
    if c.err:
        assert (e1, e2) == c.err, (c.name, e1, e2, c.err)
    elif bst == OTS:
        assert e2 == BS and e1 > BS, (c.name, e1, e2)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["hand", "random"])
def test_host_and_device_calls(ctx, which):
    hand, rnd = all_cases()
    for c in hand if which == "hand" else rnd:
        h = _host(ctx, c)
        check_host(c, h)
        assert _device(ctx, c) == h, c.name


@pytest.mark.gpu
def test_batch_call(ctx):
    """All cases in batches: linked chains side by side with independent frames (good and failing), in two orders."""
    from test_gpu_frame_batch_device import host_next, run_batch
    hand, rnd = all_cases()
    j = bytes(range(256)) * 40
    ind = [oracle.frame_compress(j[:1000 + 37 * i], 4, i % 8) for i in range(6)]
    ind += [ind[5][:len(ind[5]) // 2], ind[2][:-1] + bytes([ind[2][-1] ^ 1])]    # truncated; bad content checksum
    want_ind = [host_next(ctx, f, 20000) for f in ind]
    assert [w[0][0] for w in want_ind[-2:]] == [oracle.frame_decompress(f, 20000)[0] for f in ind[-2:]] != [0, 0]
    cases = hand + rnd
    for order in (1, -1):
        seq_ = cases[::order]
        for lo in range(0, len(seq_), 700):
            frames, caps, kinds = [], [], []
            for i, c in enumerate(seq_[lo:lo + 700]):
                frames.append(c.frame)
                caps.append(c.cap)
                kinds.append(c)
                if i % 3 == 0:
                    k = (lo + i) % len(ind)
                    frames.append(ind[k])
                    caps.append(20000)
                    kinds.append(k)
            got = run_batch(ctx, frames, caps, seed=2 * lo + (order < 0))
            for g, k in zip(got, kinds):
                if isinstance(k, int):
                    assert g == want_ind[k], k
                else:
                    check_host(k, g)
                    assert g == _host(ctx, k), k.name


def _splits(c, mode: str):
    from stream_frames import byte_steps, unit_ends
    n = len(c.frame)
    if mode == "whole":
        return [n]
    if mode == "units":
        e = unit_ends(c.frame)
        return e if e[-1] == n else e + [n]
    return byte_steps(n, head=120, tail=20)


def _stream(dec, ctx, c, mode: str, cap: int):
    from test_gpu_frame_decoder_device import stream_decode
    h = _host(ctx, c)
    data, r, consumed, _ = stream_decode(dec, c.frame, _splits(c, mode), lambda i: cap)
    assert data == h[1], (c.name, mode, cap, len(data), len(h[1]))
    assert r[1] == consumed
    if h[0][0] == DEC_ERR:                   # consumed: the end of the failing block and its checksum
        assert r[0] == DEC_ERR and r[2:] == h[0][2:], (c.name, mode, r, h[0])
    else:
        assert r == h[0], (c.name, mode, r, h[0])


@pytest.mark.gpu
def test_streaming_decoder(ctx):
    """Every hand-built frame whole and at its units under its small out_cap, whole under the block size, and in
    one-byte steps (one in eight of the span and overlap frames); every fourth random frame at its units."""
    from test_gpu_frame_decoder_device import Decoder
    hand, rnd = all_cases()
    dec = Decoder(ctx)
    try:
        for i, c in enumerate(hand):
            bulk = c.name.startswith(("span", "overlap"))          # one in eight of these in one-byte steps
            for mode in ("whole", "units") + (("bytes",) if not bulk or i % 8 == 0 else ()):
                _stream(dec, ctx, c, mode, c.stream_cap)
            _stream(dec, ctx, c, "whole", max(BS, c.stream_cap))
        for c in rnd[::4]:
            _stream(dec, ctx, c, "units", c.stream_cap)
    finally:
        dec.close()


@pytest.fixture(scope="module")
def small_ctx():
    from lz4_flex_b200 import _native, block
    c = block.Context(0)
    _native.lib().lz4b200_ctx_set_frame_budget(c.handle, 1 << 20)
    yield c
    c.close()


@pytest.mark.gpu
def test_one_mib_budget(small_ctx):
    """The window cases and the edge cases on a context with a 1 MiB frame budget: the streaming decoder cuts the
    budget frames after 16 blocks; every path still agrees with the oracle."""
    from test_gpu_frame_decoder_device import Decoder
    hand, _ = all_cases()
    dec = Decoder(small_ctx)
    try:
        for c in hand:
            if not c.name.startswith(("window", "byte0", "dist65535", "mid-frame", "bs+1", "oob", "bad checksum")):
                continue
            h = _host(small_ctx, c)
            check_host(c, h)
            assert _device(small_ctx, c) == h, c.name
            _stream(dec, small_ctx, c, "whole", c.stream_cap)
            _stream(dec, small_ctx, c, "units", c.stream_cap)
    finally:
        dec.close()
