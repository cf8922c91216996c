"""The encoder's parse at the two places natural content never decides: the 64 KiB match window's edge and deep in the
probe ladder, on every encoder kernel of the product library, against the oracle.

* Window plants: `zeros | S (48 random bytes) | zeros | S` with the copy D = 65 533 .. 65 537 bytes after its source,
  at every source alignment 0..3, near the block start, more than 1 MiB in, and 12..20 bytes before the last probe
  position n - 12.  The reference takes the copy at offset D while D <= 65 535 and emits it as literals above that.
* Empty-slot plants: 16 random bytes, zeros up to position p = 65 533 .. 65 537, the same 16 bytes: in a FRESH block
  above 64 KiB the candidate is position 0.
* Dictionary plants: the used dictionary (its last 64 KiB) holds a 24-byte segment S at position 0, 1 or 2 (init_dict's
  three residues) and zeros elsewhere; the input is j random bytes then S, so the offset is (used length - r + j).
* Ladder plants: `zeros | S (600 random) | R (r random) | S'`, S' a copy of S with every m-th byte flipped, its first
  byte included: the first probe of the ladder that lands on an unflipped word of S' decides where the match starts,
  and backward extension stops at the flip before it, so a ladder one probe off changes the bytes.  Past 64 KiB of literals (where S' is out
  of reach) a periodic strip does the same: the first probe whose phase repeats an earlier probe's lands, and the
  match's offset is the distance between the two probes.
* Ring plants for the one-chain-per-CTA kernel: window plants with D swept over the reach of its 64 KiB shared-memory
  ring (25..26 chunks of 2 KiB behind the cursor's chunk) at all 16 input address residues.

test_plants_reach_the_edges checks on the CPU that every plant reaches its edge in the oracle's output, so a plant that
stops doing so fails there rather than becoming a weaker GPU test.  The GPU tests run one device-pointer launch per
batch, assert the kernel the launcher records, compare every block with the oracle and decode the output again on the
device.  Last, hand-built streams whose match reads exactly 65 535 bytes back (and one byte further) run through the
decoder at G = 32, 16 and 8, with match lengths that the 8-lane decoder defers (up to 64) and longer ones.
"""
from __future__ import annotations

import concurrent.futures as cf
import contextlib
import functools
import io
import os
from typing import NamedTuple

import numpy as np
import pytest

import oracle
from lz4_flex_b200 import block
from test_gpu_enc_path import _pad
from test_gpu_launch_shapes import (FL_CONT, FL_FRESH_H5, GTAB, ORACLE_BY_MODE, SPLIT16, SPLIT32, DecodeLayout,
                                    EncodeLayout, collect_decode, collect_encode, dec_count, dec_name, decode_tensors,
                                    enqueue_decode, enqueue_encode, encode_tensors, layout_decode_tensors,
                                    oracle_decode, seq, sm_count)

MODES = (0, FL_FRESH_H5, FL_CONT)
EDGE = range(65533, 65538)                                   # 65 535 is the largest offset the format has
SOLO2 = "lz4_compress_blocks_solo2"
GTABG = {62: "lz4_compress_blocks_gtabg<16, 6, 2>", 71: "lz4_compress_blocks_gtabg<16, 7, 1>",
         862: "lz4_compress_blocks_gtabg<8, 6, 2>", 871: "lz4_compress_blocks_gtabg<8, 7, 1>"}


class Plant(NamedTuple):
    kind: str          # window | slot | dict | ladder | strip
    at: int            # where the copy (or the strip) starts in the block
    dist: int          # the distance back to its source (strip: 0, any)
    flipped: bool = False


class Case(NamedTuple):
    data: bytes
    mode: int
    plants: tuple


def _rand(rng, n: int) -> bytes:
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def _window(rng, lead: int, D: int, copy_len: int = 48):
    """zeros(lead) | S | zeros(D - 48) | S[:copy_len]: (bytes, where the copy starts)."""
    s = _rand(rng, 48)
    return bytes(lead) + s + bytes(D - 48) + s[:copy_len], lead + D


def _flip(s: bytes, m: int | None) -> bytes:
    if m is None:
        return s
    b = bytearray(s)
    b[::m] = bytes(x ^ 0xFF for x in b[::m])
    return bytes(b)


def _ladder(rng, r: int, m: int | None):
    """zeros(64) | S | R (r) | S' | 64 random: (bytes, plant)."""
    s = _rand(rng, 600)
    head = bytes(64) + s + _rand(rng, r)
    return head + _flip(s, m) + _rand(rng, 64), Plant("ladder", len(head), 600 + r, m is not None)


def _strip(rng, r: int, period: int):
    """zeros(64) | R (r) | 8 KiB of a random unit of `period` bytes repeated | 64 random: (bytes, plant)."""
    head = bytes(64) + _rand(rng, r)
    unit = _rand(rng, period)
    return head + (unit * (8192 // period + 1))[:8192] + _rand(rng, 64), Plant("strip", len(head), 0, True)


# ---- generators ----------------------------------------------------------------------------------------------------

R_SMALL = (0, 1, 4, 16, 64, 256, 1000, 3000, 8000, 20000, 40000, 60000, 64000)
M_ALL = (None, 3, 5, 9, 17, 33)


@functools.lru_cache(maxsize=None)
def small_ladders() -> tuple:
    """Ladder and strip plants in blocks of at most 64 KiB (the u16-table kernels), a mode per block."""
    rng = np.random.default_rng(11)
    out = []
    for rep in range(2):
        for r in R_SMALL:
            for m in M_ALL:
                d, p = _ladder(rng, r, m)
                out.append(Case(d, MODES[(len(out) + len(out) // 6) % 3], (p,)))    # each m in every mode
    for r in (0, 300, 3000, 20000, 45000):
        for period in (7, 11, 13):
            d, p = _strip(rng, r, period)
            out.append(Case(d, MODES[len(out) % 3], (p,)))
    assert max(len(c.data) for c in out) <= 65536
    return tuple(out)


@functools.lru_cache(maxsize=None)
def window_blocks() -> tuple:
    """Window plants in blocks of 65 537 .. 300 000 bytes, near the start and 12..20 bytes before n - 12, every D,
    source alignment and mode."""
    rng = np.random.default_rng(12)
    out = []
    for D in EDGE:
        for align in range(4):
            for mode in MODES:
                w, at = _window(rng, 100 + align, D)
                w += _rand(rng, 64)
                n = int(rng.integers(max(65537, len(w)), 300001))
                out.append(Case(w + bytes(n - len(w)), mode, (Plant("window", at, D),)))
                k = 24 + (D + align + mode) % 9                    # the copy: the block's last 24..32 bytes
                w, at = _window(rng, 100 + align, D, k)
                assert 12 <= len(w) - 12 - at <= 20
                out.append(Case(w, mode, (Plant("window", at, D),)))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def slot_blocks() -> tuple:
    """Empty-slot plants: FRESH blocks (block API above 64 KiB, FRESH with hash5) whose copy's candidate is position
    0, p = 65 533 .. 65 537 bytes back."""
    rng = np.random.default_rng(13)
    out = []
    for p in EDGE:
        for mode in (0, FL_FRESH_H5):
            s = _rand(rng, 16)
            out.append(Case(s + bytes(p - 16) + s + _rand(rng, 32), mode, (Plant("slot", p, p),)))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def big_ladders() -> tuple:
    """Ladders whose copy lies 65 533 .. 65 537 bytes back (ladder depth and window edge at once), and strips behind
    70 KiB .. 1 MiB of literals: blocks above 64 KiB."""
    rng = np.random.default_rng(14)
    out = []
    for r in (x - 600 for x in EDGE):
        for m in (None, 5, 9, 17):
            d, p = _ladder(rng, r, m)
            out.append(Case(d, MODES[len(out) % 3], (p,)))
    for r in (70000, 150000, 300000, 600000, 1 << 20):
        for period in (7, 11, 13):
            d, p = _strip(rng, r, period)
            out.append(Case(d, MODES[len(out) % 3], (p,)))
    assert min(len(c.data) for c in out) > 65536
    return tuple(out)


@functools.lru_cache(maxsize=None)
def huge_block() -> Case:
    """One 4 MiB block: a window plant of every D and alignment more than 1 MiB in, then a strip behind 200 KiB of
    literals."""
    rng = np.random.default_rng(15)
    parts, plants, pos = [bytes(1 << 20)], [], 1 << 20
    for D in EDGE:
        for align in range(4):
            w, at = _window(rng, 100 + align, D)
            w += _rand(rng, 64)
            parts.append(w)
            plants.append(Plant("window", pos + at, D))
            pos += len(w)
    d, p = _strip(rng, 200000, 11)
    parts.append(d)
    plants.append(p._replace(at=pos + p.at))
    pos += len(d)
    parts.append(bytes((4 << 20) - pos))
    return Case(b"".join(parts), 0, tuple(plants))


@functools.lru_cache(maxsize=None)
def ring_blocks() -> tuple:
    """Window plants with D swept through 51 150 .. 53 300 (the reach of the 64 KiB ring), 16 blocks per D: in a batch
    that starts with them, block b's input lies at address residue b mod 16."""
    rng = np.random.default_rng(16)
    out = []
    for D in range(51150, 53301, 50):
        for res in range(16):
            w, at = _window(rng, 100, D)
            w += _rand(rng, 64)
            out.append(Case(w + bytes(66000 - len(w)), MODES[(D // 50 + res) % 3], (Plant("window", at, D),)))
    return tuple(out)


DICT_LENS = (65533, 65534, 65535, 65536, 70000)
DICT_SMALL = 65496                                            # dictionary + input <= 64 KiB: the u16-table kernel


@functools.lru_cache(maxsize=None)
def dict_batch(dlen: int, r: int):
    """(dictionary, cases): the used window holds S at position r and zeros elsewhere (the zeros keep init_dict's
    entries of S in the table); inputs j random bytes | S | random, for j = 0..4 and the j that put the offset at
    65 533 .. 65 537."""
    rng = np.random.default_rng(17 + dlen + r)
    used = min(dlen, 65536)
    s = _rand(rng, 24)
    dct = _rand(rng, dlen - used) + bytes(r) + s + bytes(used - r - 24)
    if dlen == DICT_SMALL:                                    # inputs of 40 bytes: dictionary + input = 64 KiB
        js = range(5)
        return dct, tuple(Case(_rand(rng, j) + s + _rand(rng, 16 - j), 0, (Plant("dict", j, used - r + j),)) for j in js)
    js = sorted(set(range(5)) | {t - (used - r) for t in EDGE if t >= used - r})
    return dct, tuple(Case(_rand(rng, j) + s + _rand(rng, 24), 0, (Plant("dict", j, used - r + j),)) for j in js)


def dict_residues(dlen: int):
    return (0,) if dlen == DICT_SMALL else (0, 1, 2)


# ---- the oracle and its sequences ----------------------------------------------------------------------------------

def walk(stream: bytes):
    """The sequences of an LZ4 block: (literal start, literal length, match start, offset, match length); the last
    sequence has offset and length 0."""
    out, i, op, n = [], 0, 0, len(stream)
    while i < n:
        t = stream[i]
        i += 1
        ll = t >> 4
        if ll == 15:
            while True:
                b = stream[i]
                i += 1
                ll += b
                if b != 255:
                    break
        anchor = op
        i += ll
        op += ll
        if i >= n:
            out.append((anchor, ll, op, 0, 0))
            break
        off = stream[i] | (stream[i + 1] << 8)
        i += 2
        ml = t & 15
        if ml == 15:
            while True:
                b = stream[i]
                i += 1
                ml += b
                if b != 255:
                    break
        out.append((anchor, ll, op, off, ml + 4))
        op += ml + 4
    return out


def _oracle(case: Case, dct: bytes = b"") -> bytes:
    return oracle.compress_with_dict(case.data, dct) if dct else ORACLE_BY_MODE[case.mode](case.data)


def oracle_all(cases, dct: bytes = b""):
    with cf.ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        return list(ex.map(lambda c: _oracle(c, dct), cases))


def _covering(seqs, x: int):
    """The sequence whose match covers byte x, or None if x is a literal."""
    for s in seqs:
        if s[4] and s[2] <= x < s[2] + s[4]:
            return s
        if s[2] > x:
            return None
    return None


def plant_outcome(seqs, p: Plant):
    """What the oracle did with plant p: ("match", offset, match start, literal run before it) for the first match that
    reaches into the copy (or strip), or ("literals",) if none does before its end."""
    span = 48 if p.kind in ("window", "slot") else 24 if p.kind == "dict" else 600 if p.kind == "ladder" else 8192
    for s in seqs:
        if s[4] and s[2] + s[4] > p.at:
            if s[2] >= p.at + span:
                break
            return "match", s[3], s[2], s[1]
    return ("literals",)


DEPTHS = ((0, 1024), (1024, 8192), (8192, 32768), (32768, 65536), (65536, 1 << 30))


def test_plants_reach_the_edges():
    """Each plant, compressed by the oracle in its mode, does what the GPU tests rely on: a copy within 65 535 bytes is
    taken at exactly its distance (offsets 65 535 and 65 534 occur in every mode and with a dictionary), one further
    back is literals, the empty slot matches only at p <= 65 535, ladder first hits come after literal runs in five
    depth ranges up to beyond 64 KiB, and most flipped copies are entered past their start."""
    offsets = {m: set() for m in MODES}
    dict_offsets, depth_hits, flipped = set(), [0] * len(DEPTHS), [0, 0]
    groups = [(c, b"") for c in small_ladders() + window_blocks() + slot_blocks() + big_ladders() + ring_blocks()
              + (huge_block(),)]
    for dlen in DICT_LENS + (DICT_SMALL,):
        for r in dict_residues(dlen):
            dct, cases = dict_batch(dlen, r)
            groups += [(c, dct) for c in cases]
    with cf.ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        streams = list(ex.map(lambda g: _oracle(*g), groups))
    for (case, dct), stream in zip(groups, streams):
        seqs = walk(stream)
        where = f"{case.plants[0].kind} plant, n {len(case.data)}, mode {case.mode}, dict {len(dct)}"
        for p in case.plants:
            got = plant_outcome(seqs, p)
            if p.kind in ("window", "slot", "dict"):
                if p.dist <= 65535:
                    assert got[:3] == ("match", p.dist, p.at), (where, p, got)
                else:
                    assert got == ("literals",) and _covering(seqs, p.at) is None, (where, p, got)
                (dict_offsets if dct else offsets[case.mode]).add(got[1] if got[0] == "match" else None)
            elif p.kind == "ladder" and p.dist > 65535:
                assert got == ("literals",), (where, p, got)
            elif got[0] == "match":                          # ladder within reach, strip
                assert p.kind == "strip" or got[1] == p.dist, (where, p, got)
                depth_hits[next(i for i, (lo, hi) in enumerate(DEPTHS) if lo <= got[3] < hi)] += 1
                if p.kind == "ladder" and p.flipped:
                    flipped[got[2] > p.at] += 1
    for m in MODES:
        assert {65534, 65535} <= offsets[m], (m, sorted(o for o in offsets[m] if o))
    assert {65534, 65535} <= dict_offsets, sorted(o for o in dict_offsets if o)
    assert all(depth_hits), depth_hits
    assert flipped[1] > 2 * flipped[0], flipped


# ---- GPU -----------------------------------------------------------------------------------------------------------

def _first_difference(got: bytes, want: bytes) -> str:
    g, w = walk(got), walk(want)
    for i, (a, b) in enumerate(zip(g, w)):
        if a != b:
            return f"sequence {i}: GPU {a} != oracle {b}"
    return f"sequence {min(len(g), len(w))}: GPU has {len(g)} sequences, the oracle {len(w)}"


class DictLayout(EncodeLayout):
    """An EncodeLayout whose batch has the dictionary `dct` (EncodeLayout's own dictionary batches always use the
    shape tests' 30 000-byte JSON dictionary): the oracle, the tensors and the round trip all read `self.dct`, so the
    base class's assignment of its default is ignored."""

    def __init__(self, blocks, dct: bytes):
        self._dct = dct
        super().__init__(blocks, 1)

    @property
    def dct(self) -> bytes:
        return self._dct

    @dct.setter
    def dct(self, _default):
        pass


def _run(ctx, cases, name: str, max_in_len: int | None = None, dct: bytes = b""):
    """One launch of `cases` (max_in_len None: the exact bound), its kernel record, every block against the oracle
    (naming the first differing sequence), the layout's canary gaps, and a round trip through the device decoder."""
    import torch
    blocks = [(c.data, 0 if dct else c.mode, block.get_maximum_output_size(len(c.data))) for c in cases]
    lay = DictLayout(blocks, dct) if dct else EncodeLayout(blocks, 0)
    t = encode_tensors(lay)
    bound = int(lay.in_len.max()) if max_in_len is None else max_in_len
    assert enqueue_encode(ctx, t, bound) == name, len(cases)
    torch.cuda.synchronize()
    got = collect_encode(t)
    buf, st, ol = got
    for b in range(len(cases)):
        o = int(lay.out_off[b])
        want = lay.want_bytes[o: o + int(lay.want_len[b])].tobytes()
        mine = buf[o: o + max(int(ol[b]), 0)].tobytes()
        assert st[b] == 0 and mine == want, (f"{lay.where(b)} {cases[b].plants}: status {st[b]}, length {ol[b]} != "
                                             f"{len(want)}; " + (_first_difference(mine, want) if st[b] == 0 else ""))
    lay.check(got)
    td = decode_tensors(buf, lay.out_off, ol.astype(np.uint32), np.zeros(lay.src.size, dtype=np.uint8), lay.in_off,
                        lay.in_len, lay.dct)
    enqueue_decode(ctx, td)
    out, dst, dol, _ = collect_decode(td)
    assert not dst.any() and np.array_equal(dol, lay.in_len.astype(np.int64))
    assert np.array_equal(out, lay.src[: out.size]), "round trip differs"


def _padded(cases, sm: int, seed: int):
    """`cases` and short JSON blocks up to 24 blocks per SM + 1: the global-table kernels."""
    pads = _pad([], 24 * sm + 1 - len(cases), seed)
    return list(cases) + [Case(bytes(p), MODES[i % 3], ()) for i, p in enumerate(pads)]


@contextlib.contextmanager
def env_context(env: dict):
    """A fresh Context created with exactly the LZ4B200_ switches in `env` (it reads them once, at creation); the
    environment is restored before the body runs and the context closed after it."""
    saved = {k: v for k, v in os.environ.items() if k.startswith("LZ4B200_")}
    for k in saved:
        del os.environ[k]
    os.environ.update(env)
    try:
        c = block.Context(0)
    finally:
        for k in env:
            os.environ.pop(k, None)
        os.environ.update(saved)
    try:
        yield c
    finally:
        c.close()


@pytest.mark.gpu
def test_split16_ladders(ctx):
    _run(ctx, small_ladders(), SPLIT16.format(0))


@pytest.mark.gpu
def test_gtab_ladders(ctx):
    _run(ctx, _padded(small_ladders(), sm_count(), 21), GTAB)


@pytest.mark.gpu
@pytest.mark.parametrize("g16", list(GTABG), ids=list(GTABG.values()))
def test_gtabg_ladders(g16):
    with env_context({"LZ4B200_ENC_G16": str(g16)}) as c:
        _run(c, _padded(small_ladders(), sm_count(), 22), GTABG[g16])


def _big_cases():
    return window_blocks() + slot_blocks() + big_ladders() + (huge_block(),)


@pytest.mark.gpu
def test_split32_window_slot_and_deep_ladders(ctx):
    _run(ctx, _big_cases(), SPLIT32.format(0))


@pytest.mark.gpu
def test_unknown_bound_runs_both_kernels(ctx):
    """max_in_len 0: the u16-table kernel takes the blocks up to 64 KiB, the u32-table kernel the rest."""
    cases = small_ladders() + window_blocks() + slot_blocks() + big_ladders()
    assert len(cases) <= 24 * sm_count()
    _run(ctx, cases, SPLIT16.format(0) + " + " + SPLIT32.format(0), max_in_len=0)


@pytest.mark.gpu
@pytest.mark.parametrize("dlen", DICT_LENS + (DICT_SMALL,))
def test_dictionary_window_edge(ctx, dlen):
    for r in dict_residues(dlen):
        dct, cases = dict_batch(dlen, r)
        both = max(len(c.data) for c in cases) + min(dlen, 65536) > 65536
        _run(ctx, cases, SPLIT16.format(1) + (" + " + SPLIT32.format(1) if both else ""), dct=dct)


@pytest.mark.gpu
def test_solo2_ring_window_and_ladders():
    """The one-chain-per-CTA kernel over its shared-memory ring: ring plants first (block b at residue b mod 16), then
    window, empty-slot and deep ladder plants and the 4 MiB block."""
    cases = ring_blocks() + _big_cases()
    with env_context({"LZ4B200_ENC_SOLO": "2"}) as c:
        _run(c, cases, SOLO2)


# ---- frames --------------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def frame_input(bsize: int) -> bytes:
    """Two blocks and a bit of `bsize`: a copy 2 000 bytes after its source across the first block boundary (an
    independent block must not take it), window plants at 65 535 and 65 536 inside the second block, a ladder."""
    rng = np.random.default_rng(bsize)
    s = _rand(rng, 48)
    parts = [bytes(bsize - 1000), s, bytes(2000 - 48), s, _rand(rng, 64)]
    for D in (65535, 65536):
        parts.append(_window(rng, 101, D)[0] + _rand(rng, 64))
    parts.append(_ladder(rng, 20000, 9)[0])
    n = sum(len(p) for p in parts)
    parts.append(bytes(max(2 * bsize + 12345 - n, 0)))
    return b"".join(parts)


FRAME_SIZES = {5: 256 << 10, 6: 1 << 20, 7: 4 << 20}


def test_frame_copy_across_blocks_is_literals():
    """In the oracle's frame the copy whose source lies in the previous block is literals (independent blocks), and
    the second block takes the window plant at 65 535."""
    for bsid, bsize in FRAME_SIZES.items():
        f = oracle.frame_compress(frame_input(bsize), bsid)
        pos, blocks = 7, []                                   # magic, FLG, BD, HC
        while True:
            ln = int.from_bytes(f[pos: pos + 4], "little")
            pos += 4
            if ln == 0:
                break
            assert not ln & 0x80000000
            blocks.append(f[pos: pos + (ln & 0x7FFFFFFF)])
            pos += ln & 0x7FFFFFFF
        seqs = walk(blocks[1])
        assert all(_covering(seqs, x) is None for x in range(1000, 1048)), bsid    # the copy: block 2 at 1 000
        assert 65535 in {s[3] for s in seqs} and 65536 not in {s[3] for s in seqs}, bsid


@pytest.mark.gpu
@pytest.mark.parametrize("bsid", list(FRAME_SIZES))
def test_frames_across_the_window_edge(ctx, bsid):
    import torch

    from lz4_flex_b200 import _native, frame
    data = frame_input(FRAME_SIZES[bsid])
    want = oracle.frame_compress(data, bsid)
    info = frame.FrameInfo(block_size=frame.BlockSize(bsid))
    d_in = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    got = frame.compress_frame_device(d_in, info, ctx=ctx)
    assert _native.lib().lz4b200_ctx_last_kernel(ctx.handle, 0).decode() == SPLIT32.format(0)
    assert got.cpu().numpy().tobytes() == want
    enc = frame.FrameEncoder(io.BytesIO(), info, ctx=ctx)
    enc.write(data)
    assert enc.finish().getvalue() == want


# ---- the decoder at the same edge ----------------------------------------------------------------------------------

MLENS = tuple(range(4, 201))


@functools.lru_cache(maxsize=None)
def edge_streams() -> tuple:
    """(stream, cap, status): a match at offset 65 535 once the output holds op = 65 535 bytes (it reads the first
    byte: decodes) and op = 65 534 bytes (one byte before the output: OffsetOutOfBounds), reached by one literal run or
    after an earlier match, at every match length 4..200, then literals."""
    rng = np.random.default_rng(18)
    out = []
    for mlen in MLENS:
        for lead in (False, True):
            for op in (65535, 65534):
                head = (seq(_rand(rng, 20), 10, 40) + seq(_rand(rng, op - 60), 65535, mlen)) if lead else \
                    seq(_rand(rng, op), 65535, mlen)
                tail = 5 + mlen % 11
                out.append((head + seq(_rand(rng, tail)), op + mlen + tail, 0 if op == 65535 else oracle.ERR_OFFSET_OOB))
    return tuple(out)


def test_decoder_edge_streams_decode_as_built():
    for s, cap, st in edge_streams():
        got = oracle.decompress_block(s, cap)
        assert got[0] == st and (st or len(got[1]) == cap), (len(s), cap, st, got[0])


def _dec_blocks(count: int):
    """The edge streams, then short valid streams up to `count` blocks: (kind, stream, cap, status)."""
    rng = np.random.default_rng(19)
    blocks = [("edge", s, cap, st) for s, cap, st in edge_streams()]
    i = 0
    while len(blocks) < count:
        k, tail = 8 + i % 20, 6 + i % 5
        s = seq(_rand(rng, k), 1 + i % 8, 4 + i % 30) + seq(_rand(rng, tail))
        blocks.append(("filler", s, k + 4 + i % 30 + tail, 0))
        i += 1
    return blocks


@pytest.mark.gpu
@pytest.mark.parametrize("g", (32, 16, 8))
def test_decoder_offset_65535(ctx, g):
    import torch
    sm = sm_count()
    w = 1 if dec_count(g, 1, 0, sm) else 4
    blocks = _dec_blocks(dec_count(g, w, 0, sm))
    lay = DecodeLayout(blocks, oracle_decode(blocks))
    assert all(st == lay.want_status[b] for b, (_, _, _, st) in enumerate(blocks))
    for fill in (0x00, 0xFF):
        t = layout_decode_tensors(lay, fill)
        assert enqueue_decode(ctx, t) == dec_name(g, w, 0), len(blocks)
        torch.cuda.synchronize()
        lay.check(collect_decode(t), fill)
