"""Single blocks from 8 MiB to the largest one the host entry points accept (about 3.64 GiB), built so that the oracle's
parse reaches the places 32-bit positions go wrong: literal runs longer than 2^24, table entries and matches past 2^31, a
match at offset 65 535 past 2^31 (and a copy one byte further back left as literals), a match longer than 2^20, and the
end-of-block rules at the last 12 bytes.  tests/test_gpu_big_blocks.py compares the GPU codec with the oracle on them.

* text: hdfs / JSON / dickens tiled, 8 MiB + 1, 16 MiB - 3, 64 MiB and 256 MiB (about 23 ms of GPU parse per MiB, so
  nothing larger is text).
* sparse: xorshift64* noise, which the parse crosses with a growing step, and islands it must stop in.  Every island
  starts with 64 KiB of zeros, so whatever step the noise before it left, some probe lands in the zeros, matches, and
  the step starts again at 1.  Islands: 1 MiB of dickens on each side of 2^24 (and of 2^31); a row of window plants
  `zeros | S | zeros | S` whose copy lies D = 65 530 .. 65 540 bytes after its source (past 2^31 where the block is that
  large); and a last island of period-11 content that ends exactly 12 bytes before the block's end (1 GiB and
  2^31 + 2^20 + 7) or runs through it (top), so the last match ends at n - 12 or is cut at n - 6 (END_OFFSET).
* long match: a 256 MiB zero run between short noise: a match-length extension of about a million 0xFF bytes.
* top: the largest n with lz4b200_max_output_size(n) <= 0xffffffff, built as sparse.

test_plants_reach_their_edges walks the oracle's sequences of every plant and asserts the edge each was built for,
and that the oracle's decoder round-trips it, so the GPU tests are never the first to run the oracle on a block this
large.  The two largest text plants have ~6 M and ~25 M sequences; their walk stops at the first length extension
(what the decoder tests cut), and only the round trip covers the rest.
"""
from __future__ import annotations

import ctypes as C
import functools
import gc
import re
from typing import NamedTuple

import numpy as np
import pytest

import oracle
from lz4_flex_b200 import corpus
from test_gpu_launch_shapes import seq

KiB, MiB, GiB = 1 << 10, 1 << 20, 1 << 30
FL_FRESH_H5 = 2                                  # block.BLOCK_HASH5_ALWAYS
FL_CONT = 3                                      # block.BLOCK_HASH5_ALWAYS | block.BLOCK_CONT
ORACLE_BY_MODE = {0: oracle.compress_block, FL_FRESH_H5: oracle.compress_block_fresh_h5,
                  FL_CONT: oracle.compress_block_cont}


def max_output_size(n: int) -> int:
    return 16 + 4 + n * 110 // 100


# the largest block the host entry points accept: the batch planner refuses a bound above 0xffffffff
TOP = ((0xFFFFFFFF - 20 + 1) * 100 - 1) // 110
assert max_output_size(TOP) <= 0xFFFFFFFF < max_output_size(TOP + 1)

NOISE_PERIOD = MiB + 4093                         # tiled noise: its repeats lie far outside the 64 KiB window
ZLEAD = 64 * KiB                                  # zeros before every island: more than the largest step of the parse
WINDOW_D = tuple(range(65530, 65541))             # 65 535 is the largest offset the format has
PERIOD = 11                                       # the last island's period


class Plant(NamedTuple):
    name: str
    n: int
    modes: tuple            # encoder modes the GPU tests run (FRESH / FRESH_H5 / CONT on text only)
    edges: tuple            # what test_plants_reach_their_edges asserts
    windows: tuple = ()     # (copy start, D) of each window plant
    tail: str = ""          # "n-12": the last match ends at n - 12; "cut": it is cut at n - 6


# ---- building ------------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _noise_unit() -> np.ndarray:
    return corpus.xorshift64star_bytes(NOISE_PERIOD, seed=0x243F6A8885A308D3)


def _fill_noise(buf: np.ndarray):
    """buf[i] = unit[i mod NOISE_PERIOD], doubling the filled prefix (the period stays a divisor of it)."""
    u = _noise_unit()
    k = min(u.size, buf.size)
    buf[:k] = u[:k]
    while k < buf.size:
        m = min(k, buf.size - k)
        buf[k: k + m] = buf[:m]
        k += m


@functools.lru_cache(maxsize=None)
def _dickens() -> np.ndarray:
    return np.frombuffer(corpus.load("dickens.txt"), dtype=np.uint8)


def _text_island(buf, start: int, end: int, seed: int):
    """zeros(ZLEAD) then dickens from a seeded offset, over [start, end)."""
    buf[start: start + ZLEAD] = 0
    t = _dickens()
    a = (seed * 1_000_003) % (t.size - (end - start))
    buf[start + ZLEAD: end] = t[a: a + end - start - ZLEAD]


def _window_row(buf, start: int, lead: int, seed: int):
    """zeros(lead) then, for every D in WINDOW_D: S (48 random) | zeros(D - 48) | S | 64 random | zeros(64).  Returns
    ((copy start, D) ..., end)."""
    rng = np.random.default_rng(seed)
    pos = start
    buf[pos: pos + lead] = 0
    pos += lead
    out = []
    for d in WINDOW_D:
        s = rng.integers(0, 256, 48, dtype=np.uint8)
        buf[pos: pos + 48] = s
        buf[pos + 48: pos + d] = 0
        buf[pos + d: pos + d + 48] = s
        buf[pos + d + 48: pos + d + 112] = rng.integers(0, 256, 64, dtype=np.uint8)
        buf[pos + d + 112: pos + d + 176] = 0
        out.append((pos + d, d))
        pos += d + 176
    return tuple(out), pos


def _periodic_island(buf, start: int, end: int, seed: int):
    rng = np.random.default_rng(seed)
    unit = rng.integers(0, 256, PERIOD, dtype=np.uint8)
    buf[start: start + ZLEAD] = 0
    k = end - start - ZLEAD
    buf[start + ZLEAD: end] = np.resize(unit, k)


TEXT = {"text_8m+1": ("hdfs.json", 8 * MiB + 1), "text_16m-3": ("compression_66k_JSON.txt", 16 * MiB - 3),
        "text_64m": ("dickens.txt", 64 * MiB), "text_256m": ("hdfs.json", 256 * MiB)}
SPARSE = {"sparse_1g": GiB, "sparse_2g+1m+7": (1 << 31) + MiB + 7, "top": TOP}
LONG = "long_256m_match"
NAMES = tuple(TEXT) + (LONG,) + tuple(SPARSE)


@functools.lru_cache(maxsize=None)
def plant(name: str):
    """(Plant, data as a read-only uint8 array)."""
    if name in TEXT:
        f, n = TEXT[name]
        d = corpus.tiled(f, n)
        p = Plant(name, n, (0, FL_FRESH_H5, FL_CONT), ("tail",))
    elif name == LONG:
        n = 256 * MiB + 128 * KiB
        d = np.empty(n, dtype=np.uint8)
        _fill_noise(d)
        d[64 * KiB: n - 64 * KiB] = 0
        p = Plant(name, n, (0,), ("match_len>2^20", "tail"))
    else:
        n = SPARSE[name]
        d = np.empty(n, dtype=np.uint8)
        _fill_noise(d)
        _text_island(d, (1 << 24) - MiB, (1 << 24) + MiB, 1)
        if name == "sparse_1g":
            win, _ = _window_row(d, 1 << 29, ZLEAD, 2)
            _periodic_island(d, n - 12 - MiB, n - 12, 3)
            p = Plant(name, n, (0,), ("lit>2^24", "window", "tail"), win, "n-12")
        elif name == "top":
            _text_island(d, (1 << 31) - MiB, (1 << 31) + MiB, 4)
            win, _ = _window_row(d, 3 * GiB, ZLEAD, 5)
            _periodic_island(d, n - MiB, n, 6)
            p = Plant(name, n, (0,), ("lit>2^24", "match>2^31", "window>2^31", "tail"), win, "cut")
        else:                                                    # 2^31 + 2^20 + 7: little room past 2^31
            _text_island(d, (1 << 31) - MiB, (1 << 31) + 64 * KiB, 7)
            win, end = _window_row(d, (1 << 31) + 64 * KiB, 64, 8)
            assert end + 64 * KiB < n - 12 - 2 * ZLEAD
            _periodic_island(d, n - 12 - 2 * ZLEAD, n - 12, 9)
            p = Plant(name, n, (0,), ("lit>2^24", "match>2^31", "window>2^31", "tail"), win, "n-12")
    d.flags.writeable = False
    assert d.size == p.n
    return p, d


@functools.lru_cache(maxsize=None)
def oracle_stream(name: str, mode: int = 0) -> bytes:
    return ORACLE_BY_MODE[mode](plant(name)[1])


def oracle_decode_into(stream, out: np.ndarray):
    """block::decompress_into into `out` (no copy of the output): (status, written, expected)."""
    a = np.frombuffer(stream, dtype=np.uint8)
    w, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    st = oracle.lib().lz4o_decompress_block(a.ctypes.data, a.size, out.ctypes.data, out.size, C.byref(w), C.byref(e1),
                                            C.byref(e2))
    return st, w.value, e1.value


def release():
    """Drop every cached plant and oracle output (about 15 GiB of host memory for the whole set)."""
    for f in (plant, oracle_stream, dict_plant, dict_oracle, huge_length_streams):
        f.cache_clear()
    gc.collect()


@pytest.fixture(scope="module", autouse=True)
def _release_at_end():
    """The plants stay cached while this module runs and are released after it, so the rest of the session does not
    carry them."""
    yield
    release()


# ---- walking -------------------------------------------------------------------------------------------------------

_FF = re.compile(rb"\xff*")


class Seq(NamedTuple):
    anchor: int      # output position of the literals
    lit: int
    at: int          # output position of the match (or the end, for the last sequence)
    off: int         # 0: the last sequence
    mlen: int
    ext: tuple       # (stream position, length of its 0xFF run) of each length extension


def _ext(stream: bytes, i: int):
    """A length extension at i: (its value, the index after it, the length of its 0xFF run)."""
    j = _FF.match(stream, i).end()
    return 255 * (j - i) + stream[j], j + 1, j - i


def walk(stream: bytes, stop=None):
    """The sequences of an LZ4 block (0xFF runs skipped in C, not byte by byte); `stop(seq)` true ends the walk."""
    out, i, op, n = [], 0, 0, len(stream)
    while i < n:
        t = stream[i]
        i += 1
        ll, ext = t >> 4, []
        if ll == 15:
            v, j, r = _ext(stream, i)
            ll += v
            ext.append((i, r))
            i = j
        anchor = op
        i += ll
        op += ll
        if i >= n:
            out.append(Seq(anchor, ll, op, 0, 0, tuple(ext)))
            break
        off = stream[i] | (stream[i + 1] << 8)
        i += 2
        ml = t & 15
        if ml == 15:
            v, j, r = _ext(stream, i)
            ml += v
            ext.append((i, r))
            i = j
        out.append(Seq(anchor, ll, op, off, ml + 4, tuple(ext)))
        op += ml + 4
        if stop and stop(out[-1]):
            break
    return out


def first_ff_run(stream: bytes, at_least: int = 1):
    """(stream position, length) of the first length extension whose 0xFF run is at least `at_least` bytes long."""
    hit = []
    walk(stream, lambda s: bool([hit.append(e) for e in s.ext if e[1] >= at_least]))
    assert hit, "no length extension that long"
    return hit[0]


def longest_ff_run(seqs):
    return max((e for s in seqs for e in s.ext), key=lambda e: e[1])


def covering(seqs, x: int):
    """The sequence whose match covers output byte x, or None if x is a literal (seqs in order)."""
    lo, hi = 0, len(seqs)
    while lo < hi:                                              # the last sequence whose match starts at or before x
        mid = (lo + hi) // 2
        if seqs[mid].at <= x:
            lo = mid + 1
        else:
            hi = mid
    s = seqs[lo - 1] if lo else None
    return s if s and s.mlen and x < s.at + s.mlen else None


def check_tail(seqs, n: int):
    """The end-of-block rules (block/mod.rs:46-61): the last sequence is literals only, at least LAST_LITERALS = 5 of
    them, and no match starts after n - MFLIMIT = n - 12."""
    last = seqs[-1]
    assert last.off == 0 and last.at == n and last.lit >= 5, last[:5]
    if len(seqs) > 1:
        m = seqs[-2]
        assert m.at <= n - 12 and m.at + m.mlen <= n - 5, m[:5]
    return seqs[-2] if len(seqs) > 1 else None


WALKED = ("text_8m+1", "text_16m-3", LONG) + tuple(SPARSE)


def test_plant_sizes_and_top():
    assert [TEXT[k][1] for k in TEXT] == [8 * MiB + 1, 16 * MiB - 3, 64 * MiB, 256 * MiB]
    assert SPARSE["sparse_2g+1m+7"] == 2**31 + 2**20 + 7 and TOP == 3904515705


def test_plants_reach_their_edges():
    for name in NAMES:
        p, data = plant(name)
        stream = oracle_stream(name)
        out = np.zeros(p.n, dtype=np.uint8)
        st, w, _ = oracle_decode_into(stream, out)
        assert st == 0 and w == p.n and np.array_equal(out, data), name
        del out
        if name not in WALKED:
            assert first_ff_run(stream)[1] >= 1, name
            continue
        seqs = walk(stream)
        assert seqs[-1].at == p.n, name
        last = check_tail(seqs, p.n)
        if "lit>2^24" in p.edges:
            assert max(s.lit for s in seqs) > 1 << 24, name
        if "match_len>2^20" in p.edges:
            assert max(s.mlen for s in seqs) > 1 << 20 and longest_ff_run(seqs)[1] > 4000, name
        if "match>2^31" in p.edges:
            past = [s for s in seqs if s.off and s.at > 1 << 31]
            assert len(past) > 1000, (name, len(past))
        for at, d in p.windows:
            s = covering(seqs, at)
            if d <= 65535:
                assert s is not None and (s.at, s.off) == (at, d), (name, at, d, s)
            else:
                assert s is None, (name, at, d, s)                  # a copy one byte out of reach: literals
            if "window>2^31" in p.edges:
                assert at > 1 << 31
        if p.tail == "n-12":
            assert last.at + last.mlen == p.n - 12 and last.off == PERIOD, (name, last)
        elif p.tail == "cut":
            assert last.at + last.mlen == p.n - 6 and last.off == PERIOD, (name, last)
        del seqs


@pytest.mark.parametrize("name", ("text_8m+1", "text_16m-3", "text_64m", "text_256m"))
def test_text_plants_in_every_mode(name):
    """The oracle's FRESH_H5 and CONT parses (the frame encoder's), which the GPU tests compare with, round-trip."""
    p, data = plant(name)
    for mode in (FL_FRESH_H5, FL_CONT):
        s = oracle_stream(name, mode)
        out = np.zeros(p.n, dtype=np.uint8)
        st, w, _ = oracle_decode_into(s, out)
        assert st == 0 and w == p.n and np.array_equal(out, data), (name, mode)


# ---- the dictionary plant and length fields past 2^32 ---------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def dict_plant():
    """(dictionary, input): 64 KiB of dickens; 64 MiB of hdfs whose byte 0 starts a copy of dictionary bytes 100..
    (offset 65 436, in reach) and whose byte 65 536 starts a copy of dictionary bytes 30 000.. (65 536 + 35 536 back:
    out of reach, so literals or matches inside the input only)."""
    dct = np.frombuffer(corpus.load("dickens.txt"), dtype=np.uint8)[1 << 20: (1 << 20) + 65536].copy()
    d = corpus.tiled("hdfs.json", 64 * MiB)
    d[:4096] = dct[100: 4196]
    d[65536: 65536 + 4096] = dct[30000: 34096]
    return dct.tobytes(), d


@functools.lru_cache(maxsize=None)
def dict_oracle() -> bytes:
    dct, d = dict_plant()
    return oracle.compress_with_dict(d, dct)


def test_dictionary_plant_reaches_its_edges():
    """The oracle's first match, a few bytes in, copies the dictionary; no match covering byte 65 536 reaches before
    the input."""
    dct, d = dict_plant()
    seqs = walk(dict_oracle(), lambda s: s.at > 70000)
    assert seqs[0].at < 16 and seqs[0].off > seqs[0].at, seqs[0][:5]         # a match into the dictionary
    for s in seqs:
        if s.off and s.at <= 65536 < s.at + s.mlen:
            assert s.off <= s.at, s[:5]
    st, out, _, _ = oracle.decompress_with_dict(dict_oracle(), d.size, dct)
    assert st == 0 and out == d.tobytes()


LIT8 = bytes(range(1, 9))
SMALL_DICT = bytes(range(256)) * 4


def _ext_bytes(v: int) -> bytes:
    return b"\xff" * (v // 255) + bytes([v % 255])


@functools.lru_cache(maxsize=None)
def huge_length_streams():
    """(label, stream, cap, status, expected): about 17 MiB each, most of it 0xFF extension bytes.  A literal length
    of 2^32 + 5 with 16 literals behind it; 8 literals and a match of 2^32 + 3 bytes at capacity 1 000; 8 literals and a
    match of 2^32 - 8 bytes (ending at exactly 2^32) at capacity 2^32 - 1."""
    return (
        ("literal 2^32+5", bytes([0xF0]) + _ext_bytes((1 << 32) + 5 - 15) + bytes(16), 64, oracle.ERR_LITERAL_OOB, 0),
        ("match 2^32+3", seq(LIT8, 1, (1 << 32) + 3) + seq(bytes(6)), 1000, oracle.ERR_OUTPUT_TOO_SMALL,
         8 + (1 << 32) + 3),
        ("match to 2^32", seq(LIT8, 8, (1 << 32) - 8) + seq(bytes(6)), (1 << 32) - 1, oracle.ERR_OUTPUT_TOO_SMALL,
         1 << 32),
    )


def test_huge_length_streams_in_the_oracle():
    """The oracle gives each stream the status and `expected` it was built for, with and without a dictionary."""
    for label, s, cap, status, expected in huge_length_streams():
        assert 16 << 20 < len(s) < 18 << 20, label
        for r in (oracle.decompress_block(s, cap), oracle.decompress_with_dict(s, cap, SMALL_DICT)):
            assert (r[0], r[2] if r[0] == oracle.ERR_OUTPUT_TOO_SMALL else 0) == (status, expected), (label, r[0], r[2])
