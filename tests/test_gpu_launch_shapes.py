"""Every kernel instantiation the block launchers pick, each reached by ONE device-pointer launch whose size comes from
this GPU's SM count, with the launcher's record of what ran asserted exactly and every block of the batch compared with
the CPU oracle.

The decoder picks its lanes per block G (32 / 16 / 8) from the batch size, one- or four-warp CTAs from the batch size
and the SM count, and a separate instantiation when the batch has a dictionary; only G <= 8 defers the stores of short
matches, and at G < 32 several blocks share a warp.  The encoder picks the global-table kernel above 24 blocks per SM,
the shared-memory-table kernel at or below that and with a dictionary, and adds the kernel for blocks above 64 KiB when
the batch may hold one.  The hard cases of the other GPU tests run in batches of fewer than 4 096 blocks, which reach
only the 32-lane decoder and the shared-memory-table encoder, so the same hard cases are run here at every shape:

* decode: the reference's KATs, hand-built streams aimed at the deferred match stores, every overlap distance 1..70
  at match lengths around 4*G, mutated and truncated good streams of five kinds of content, garbage; capacities 0,
  exact - 1, exact and random.  Output slots lie between canary gaps; every batch runs once into a 0x00-filled and once
  into a 0xFF-filled buffer.
* encode: eight kinds of content, lengths 0..64, 65 533..65 536 and ragged, a mode per block, capacities one byte
  short, input and output offsets at all 16 residues; a round trip through the decoder.
"""
from __future__ import annotations

import concurrent.futures as cf
import functools
import os

import numpy as np
import pytest

import oracle
from dict_cases import dict_cases
from lz4_flex_b200 import _native, block, corpus
from vectors import DECODE_KATS

FL_FRESH_H5 = block.BLOCK_HASH5_ALWAYS
FL_CONT = block.BLOCK_HASH5_ALWAYS | block.BLOCK_CONT
ORACLE_BY_MODE = {0: oracle.compress_block, FL_FRESH_H5: oracle.compress_block_fresh_h5, FL_CONT: oracle.compress_block_cont}
DEC_STATUSES = {0, 2, 3, 4, 5, 6}          # every decoder status (1 is the encoder's CompressOutputTooSmall)
DICT = dict((c[0], c[2]) for c in dict_cases())["json_small_u16"]   # 30 000 bytes of JSON

GTAB = "lz4_compress_blocks_gtab<unsigned short, 7, 1, 7, 3>"
SPLIT16 = "lz4_compress_blocks_split<unsigned short, 3, {}>"
SPLIT32 = "lz4_compress_blocks_split<unsigned int, 2, {}>"


# ---- LZ4 stream building -------------------------------------------------------------------------------------------

def _ext(v: int) -> bytes:
    if v < 15:
        return b""
    v -= 15
    return b"\xff" * (v // 255) + bytes([v % 255])


def seq(lit: bytes = b"", dist: int | None = None, mlen: int = 4) -> bytes:
    """One LZ4 sequence: the literals, then a match of `mlen` bytes at `dist` (none for the last sequence)."""
    ml = mlen - 4 if dist is not None else 0
    s = bytes([(min(len(lit), 15) << 4) | min(ml, 15)]) + _ext(len(lit)) + bytes(lit)
    if dist is not None:
        s += dist.to_bytes(2, "little") + _ext(ml)
    return s


def defer_cases(rng, dlen: int = 0, per_kind: int = 40):
    """Streams aimed at the deferred match stores of the 8-lane decoder: a literal run and a short non-overlapping match
    (mlen <= 32, dist >= mlen, both on the fast path: its bytes stay in registers until the next flush), followed at once
    by the event that must flush them first or must not disturb them.  `dlen` > 0: the batch has a dictionary of that
    many bytes.  Returns (kind, stream, cap, status, expected) with the status the stream was built for."""
    r = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    out = []
    for i in range(per_kind):
        k, m, j = i % 15, 4 + i % 29, i % 5                  # literals before the match, its length, literals after
        head = seq(r(14), 1, 18)                             # 32 bytes of output (an overlapping match: not deferred)
        d = int(rng.integers(m, 32 + k + 1))
        pre = head + seq(r(k), d, m)                         # the deferred match
        op = 32 + k + m                                      # output length once it is stored
        tail = seq(r(9 + i % 6))                             # >= 8 bytes behind every offset: the fast path
        big = op + 400
        out.append(("defer_offset0", pre + seq(r(j), 0, 4 + i % 8) + tail, big, 5, 0))
        out.append(("defer_offset_oob", pre + seq(r(j), op + j + dlen + 1 + i % 7, 4) + tail, big, 6, 0))
        out.append(("defer_trunc_literal_len", pre + bytes([0xF0]) + b"\xff" * (i % 3), big, 4, 0))
        out.append(("defer_trunc_match_len", pre + bytes([(j << 4) | 15]) + r(j) + (1 + i % 8).to_bytes(2, "little")
                    + b"\xff" * (i % 2), big, 4, 0))
        out.append(("defer_ends_on_match", pre + seq(r(j), 1 + i % 20, 4 + i % 10), big, 4, 0))
        m2 = 4 + i % 12
        s = pre + seq(r(j), 1 + i % 30, m2) + tail
        out.append(("defer_cap_at_match", s, op + j + m2 - 1, 2, op + j + m2))
        if j:
            out.append(("defer_cap_at_literals", s, op + j - 1, 2, op + j))
        u = i % m                                            # the next match reads the pending bytes from p_at + u
        out.append(("defer_source_pending", pre + seq(r(j), m + j - u, 4 + i % 40) + tail, op + j + 4 + i % 40 + len(tail) - 1, 0, 0))
        nl = 15 + (i * 37) % 300                             # a long literal run: the checked path
        out.append(("defer_long_literals", pre + seq(r(nl), 1 + i % 50, 4 + i % 20) + tail, big + nl, 0, 0))
        if dlen:
            # the deferred match starts at p_at = a; the next match starts kk bytes into the dictionary and runs on into
            # the output's first a + v bytes, the last v of which are still pending
            a = 4 + i % 11
            m = 4 + i % (a - 3)
            pre = seq(r(a), int(rng.integers(m, a + 1)), m)
            l, kk, v = i % 3, 1 + int(rng.integers(0, min(dlen, 200))), 1 + i % m
            ml = kk + a + v
            s = pre + seq(r(l), a + m + l + kk, ml) + tail
            out.append(("defer_dict_into_pending", s, a + m + l + ml + len(tail) - 1 + i % 3, 0, 0))
    return out


def overlap_cases(rng):
    """Every overlap distance 1..70 at match lengths around 4*G (G = 8, 16, 32), on the fast path."""
    out = []
    r = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    for dist in range(1, 71):
        for mlen in (31, 32, 33, 63, 64, 65, 127, 128, 129):
            s = seq(r(14), 5, 40) + seq(r(14), 31, 30) + seq(r(dist % 5), dist, mlen) + seq(r(10))
            out.append(("overlap", s, 98 + dist % 5 + mlen + 10, 0, 0))
    return out


# ---- decoder batches -----------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _texts():
    t = {name: corpus.tiled(f, 4 << 20) for name, f in (("json", "compression_66k_JSON.txt"), ("dickens", "dickens.txt"),
                                                         ("hdfs", "hdfs.json"))}
    return t


def _content(rng, kind: str, n: int) -> bytes:
    if kind in ("json", "dickens", "hdfs"):
        t = _texts()[kind]
        a = int(rng.integers(0, t.size - n))
        return t[a: a + n].tobytes()
    if kind == "noise":                                      # small alphabet
        return (rng.integers(0, int(rng.integers(2, 9)), n, dtype=np.uint8) + 97).tobytes()
    if kind == "alphabet":                                   # 2..34 symbols
        return (rng.integers(0, int(rng.integers(2, 35)), n, dtype=np.uint8) + 60).tobytes()
    if kind == "periodic":
        p = int(rng.integers(1, 300))
        return (rng.integers(0, 256, p, dtype=np.uint8).tobytes() * (n // p + 1))[:n]
    if kind == "words":
        vocab = _vocab()
        idx = rng.integers(0, len(vocab), n // 3 + 2)
        s = b" ".join(vocab[i] for i in idx)
        return (s * (n // max(len(s), 1) + 1))[:n]
    if kind == "zeros":
        return bytes(n)
    assert kind == "random"
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


@functools.lru_cache(maxsize=None)
def _vocab():
    rng = np.random.default_rng(99)
    return [(rng.integers(97, 123, int(rng.integers(2, 11)), dtype=np.uint8)).tobytes() for _ in range(300)]


def _filler(rng, dct):
    """One generated block: (kind, stream, cap); status and bytes come from the oracle."""
    u = rng.random()
    if u < 0.15:
        return "garbage", rng.integers(0, 256, int(rng.integers(0, 200)), dtype=np.uint8).tobytes(), int(rng.integers(0, 900))
    if u < 0.25:
        return "garbage_small_symbols", rng.integers(0, 32, int(rng.integers(1, 200)), dtype=np.uint8).tobytes(), int(rng.integers(0, 900))
    src = ("json", "dickens", "hdfs", "noise", "periodic")[int(rng.integers(0, 5))]
    n = int(rng.integers(16, 2000)) if rng.random() < 0.85 else int(rng.integers(2000, 16000))
    data = _content(rng, src, n)
    good = oracle.compress_with_dict(data, dct) if dct else oracle.compress_block(data)
    cap = (0, n - 1, n, int(rng.integers(0, n + 100)))[int(rng.integers(0, 4))]
    if u < 0.5:
        return f"good_{src}", good, cap
    s = bytearray(good)
    kind = "truncated"
    if u < 0.85:
        for _ in range(int(rng.integers(1, 4))):
            s[int(rng.integers(0, len(s)))] = int(rng.integers(0, 256))
        kind = "mutated"
    if u >= 0.7:
        s = s[: int(rng.integers(0, len(s)))]
        kind += "_truncated" if kind == "mutated" else ""
    return f"{kind}_{src}", bytes(s), cap


def hand_built(dct: bytes = b""):
    """The KATs, the deferral streams and the overlap streams: (kind, stream, cap, status, expected)."""
    rng = np.random.default_rng(1234 + len(dct))
    kats = [("kat", bytes(s), cap, st, exp or 0) for (_, s, cap, st, _, exp) in DECODE_KATS]
    if dct:                                                  # with a dictionary the oracle decides the KATs' status
        kats = [("kat", s, cap, None, None) for (_, s, cap, _, _) in kats]
    return kats + defer_cases(rng, len(dct)) + overlap_cases(rng)


def decode_blocks(count: int, dct: bytes = b""):
    """`count` distinct (kind, stream, cap, built_status) blocks, the same prefix for every count: the hand-built
    streams at the even positions of the first part, generated blocks everywhere else."""
    special = hand_built(dct)
    rng = np.random.default_rng(4321 + len(dct))
    seen, out = set(), []
    si = 0
    while len(out) < count:
        if len(out) % 2 == 0 and si < len(special):
            kind, s, cap, st, _ = special[si]
            si += 1
        else:
            kind, s, cap = _filler(rng, dct)
            st = None
        if (s, cap) in seen:
            assert st is None, kind
            continue
        seen.add((s, cap))
        out.append((kind, s, cap, st))
    return out


def oracle_decode(blocks, dct: bytes = b""):
    """(status, bytes, expected) of every block, from the oracle on all host cores (ctypes releases the GIL)."""
    def one(b):
        st, o, e1, _ = oracle.decompress_with_dict(b[1], b[2], dct) if dct else oracle.decompress_block(b[1], b[2])
        return st, o, e1 if st == oracle.ERR_OUTPUT_TOO_SMALL else 0
    with cf.ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        return list(ex.map(one, blocks, chunksize=256))


# ---- shapes --------------------------------------------------------------------------------------------------------

def sm_count() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


DEC_SHAPES = [(32, 1, 0), (32, 4, 0), (16, 1, 0), (16, 4, 0), (8, 1, 0), (8, 4, 0), (32, 4, 1), (16, 4, 1), (8, 4, 1)]


def dec_name(g: int, w: int, d: int) -> str:
    return f"lz4_decompress_blocks<{g}, 0, {d}, {w}>"


def dec_count(g: int, w: int, d: int, sm: int):
    """A block count at which the decoder launcher picks <g, 0, d, w> on `sm` SMs, or None if no count does: G = 32
    below 4 096 blocks, 16 below 12 288, else 8; one-warp CTAs while ceil(nblocks / (32 / G)) <= 32 * sm and there is no
    dictionary."""
    lo, hi = {32: (1, 4095), 16: (4096, 12287), 8: (12288, None)}[g]
    if d:
        return {32: 2500, 16: 4500, 8: 12400}[g]
    one = 32 * sm * (32 // g)                                # the largest batch that still runs as one-warp CTAs
    if w == 1:
        hi = one if hi is None else min(hi, one)
    else:
        lo = max(lo, one + 1)
    if hi is None:
        return lo + 257
    if lo > hi:
        return None
    return min(hi, 3000) if (g, w) == (32, 1) else (lo + hi) // 2


@functools.lru_cache(maxsize=None)
def _dec_master(d: int, count: int):
    dct = DICT if d else b""
    blocks = decode_blocks(count, dct)
    return blocks, oracle_decode(blocks, dct)


def dec_batch(d: int, count: int, sm: int):
    """The first `count` blocks of the largest batch any shape of this kind needs on `sm` SMs (generated and run
    through the oracle once)."""
    top = max(c for (g, w, dd) in DEC_SHAPES if dd == d for c in [dec_count(g, w, dd, sm)] if c)
    blocks, want = _dec_master(d, top)
    return blocks[:count], want[:count]


class DecodeLayout:
    """A decode batch in memory: input streams at every residue mod 16, output slots between canary gaps of 1..16
    bytes, and what the output buffer must hold afterwards (oracle bytes in the slots of blocks that succeed; the rest
    of those slots and every gap unchanged; failed blocks' slots are not specified)."""

    def __init__(self, blocks, want, dct: bytes = b""):
        rng = np.random.default_rng(len(blocks))
        nb = len(blocks)
        self.blocks, self.dct = blocks, dct
        self.in_len = np.array([len(b[1]) for b in blocks], dtype=np.uint32)
        self.out_cap = np.array([b[2] for b in blocks], dtype=np.uint32)
        self.in_off = _place(self.in_len, np.arange(nb) % 16)
        self.out_off = _place(self.out_cap, (np.arange(nb) * 7 + 3) % 16, gap=True)
        self.src = np.zeros(int(self.in_off[-1]) + int(self.in_len[-1]) + 16, dtype=np.uint8)
        for o, b in zip(self.in_off, blocks):
            self.src[int(o): int(o) + len(b[1])] = np.frombuffer(b[1], dtype=np.uint8)
        self.size = int(self.out_off[-1]) + int(self.out_cap[-1]) + 16
        self.canary = rng.integers(0, 256, self.size, dtype=np.uint8)
        self.slot = np.zeros(self.size, dtype=bool)
        self.checked = np.ones(self.size, dtype=bool)
        self.want_status = np.array([w[0] for w in want], dtype=np.int32)
        self.want_len = np.array([len(w[1]) if w[0] == 0 else 0 for w in want], dtype=np.int64)
        self.want_expected = np.array([w[2] for w in want], dtype=np.int64)
        self.want_bytes = self.canary.copy()
        for b, (o, c) in enumerate(zip(self.out_off, self.out_cap)):
            o, c = int(o), int(c)
            self.slot[o: o + c] = True
            if want[b][0] == 0:
                self.want_bytes[o: o + len(want[b][1])] = np.frombuffer(want[b][1], dtype=np.uint8)
                self.slot[o: o + len(want[b][1])] = False       # holds oracle bytes, not the fill
            else:
                self.checked[o: o + c] = False

    def initial(self, fill: int) -> np.ndarray:
        buf = self.canary.copy()
        buf[self.slot] = fill
        return buf

    def expected(self, fill: int) -> np.ndarray:
        buf = self.want_bytes.copy()
        buf[self.slot] = fill
        return buf

    def where(self, b: int) -> str:
        kind, s, cap, _ = self.blocks[b]
        return f"block {b} ({kind}, cap {cap}, stream {s[:48].hex()}{'...' if len(s) > 48 else ''})"

    def check(self, res, fill: int):
        buf, status, out_len, expected = res
        bad = np.nonzero(status != self.want_status)[0]
        assert not bad.size, f"{bad.size} statuses differ; first: {self.where(bad[0])}: {status[bad[0]]} != {self.want_status[bad[0]]}"
        bad = np.nonzero(out_len != self.want_len)[0]
        assert not bad.size, f"{bad.size} out_len differ; first: {self.where(bad[0])}: {out_len[bad[0]]} != {self.want_len[bad[0]]}"
        bad = np.nonzero(expected != self.want_expected)[0]
        assert not bad.size, f"{bad.size} `expected` differ; first: {self.where(bad[0])}: {expected[bad[0]]} != {self.want_expected[bad[0]]}"
        diff = (buf != self.expected(fill)) & self.checked
        if diff.any():
            i = int(np.argmax(diff))
            b = int(np.searchsorted(self.out_off, i, side="right")) - 1
            part = "in its slot" if b >= 0 and i < int(self.out_off[b]) + int(self.out_cap[b]) else "in the canary gap after it"
            pytest.fail(f"{int(diff.sum())} output bytes differ (fill 0x{fill:02x}); first at {i}, {part}: "
                        f"{self.where(max(b, 0))}")


def _place(lens, residues, gap: bool = False):
    """Offsets of back-to-back regions of `lens` bytes, region b at residue residues[b] mod 16 and (with `gap`) at
    least one byte after the previous region."""
    off = np.zeros(len(lens), dtype=np.uint64)
    pos = 0
    for b, n in enumerate(lens):
        pos += 1 if gap else 0
        pos += (int(residues[b]) - pos) % 16
        off[b] = pos
        pos += int(n)
    return off


def _t(a):
    """numpy descriptor array -> torch CUDA tensor of the same bytes."""
    import torch
    a = np.ascontiguousarray(a)
    view = {np.dtype(np.uint64): np.int64, np.dtype(np.uint32): np.int32}.get(a.dtype, a.dtype)
    return torch.from_numpy(a.view(view)).cuda()


def decode_tensors(src, in_off, in_len, out_init, out_off, out_cap, dct: bytes = b""):
    """The device buffers of one decode batch (statuses and `expected` start at -1: a block the kernel skips shows)."""
    import torch
    nb = len(in_len)
    t = dict(nb=nb, dlen=len(dct), src=_t(src), ioff=_t(in_off), ilen=_t(in_len), out=_t(out_init), ooff=_t(out_off),
             ocap=_t(out_cap), olen=torch.full((nb,), -1, dtype=torch.int32, device="cuda"),
             st=torch.full((nb,), -1, dtype=torch.int32, device="cuda"),
             exp=torch.full((nb,), -1, dtype=torch.int64, device="cuda"))
    if dct:
        t["dict"] = _t(np.frombuffer(dct, dtype=np.uint8).copy())
    return t


def enqueue_decode(ctx, t) -> str:
    """One lz4b200_decompress_batch_device[_with_dict] call on torch's current stream, no synchronisation.  Returns the
    kernel the launcher recorded."""
    import torch
    L, s = _native.lib(), torch.cuda.current_stream().cuda_stream
    p = {k: v.data_ptr() for k, v in t.items() if hasattr(v, "data_ptr")}
    if t["dlen"]:
        rc = L.lz4b200_decompress_batch_device_with_dict(ctx.handle, p["src"], p["ioff"], p["ilen"], p["dict"], t["dlen"],
                                                         p["out"], p["ooff"], p["ocap"], p["olen"], p["st"], p["exp"],
                                                         t["nb"], s)
    else:
        rc = L.lz4b200_decompress_batch_device(ctx.handle, p["src"], p["ioff"], p["ilen"], p["out"], p["ooff"], p["ocap"],
                                               p["olen"], p["st"], p["exp"], t["nb"], s)
    assert rc == 0, ctx.last_cuda_error()
    return L.lz4b200_ctx_last_kernel(ctx.handle, 1).decode()


def layout_decode_tensors(lay: DecodeLayout, fill: int):
    return decode_tensors(lay.src, lay.in_off, lay.in_len, lay.initial(fill), lay.out_off, lay.out_cap, lay.dct)


def collect_decode(t):
    return (t["out"].cpu().numpy(), t["st"].cpu().numpy(), t["olen"].cpu().numpy().astype(np.int64),
            t["exp"].cpu().numpy())


def _dec_case(g, w, d, sm):
    n = dec_count(g, w, d, sm)
    if n is None:
        pytest.skip(f"no batch size reaches {dec_name(g, w, d)} on {sm} SMs")
    blocks, want = dec_batch(d, n, sm)
    return DecodeLayout(blocks, want, DICT if d else b"")


@pytest.mark.gpu
@pytest.mark.parametrize("g,w,d", DEC_SHAPES, ids=[dec_name(*s) for s in DEC_SHAPES])
def test_decoder_shape_adversarial_batch(ctx, g, w, d):
    import torch
    lay = _dec_case(g, w, d, sm_count())
    for fill in (0x00, 0xFF):
        t = layout_decode_tensors(lay, fill)
        assert enqueue_decode(ctx, t) == dec_name(g, w, d), len(lay.blocks)
        torch.cuda.synchronize()
        lay.check(collect_decode(t), fill)


# ---- encoder batches -----------------------------------------------------------------------------------------------

CONTENT = ("json", "dickens", "hdfs", "alphabet", "words", "zeros", "random", "periodic")

# (label, blocks as a function of the SM count, lengths: small | span | big | mixed (see _bound_class), max_in_len:
# "exact" | 0 (unknown), dictionary)
ENC_CASES = [
    ("24sm", lambda sm: 24 * sm, "small", "exact", 0),
    ("24sm+1", lambda sm: 24 * sm + 1, "small", "exact", 0),
    ("64sm+5", lambda sm: 64 * sm + 5, "small", "exact", 0),
    ("24sm+1", lambda sm: 24 * sm + 1, "small", 0, 0),
    ("48", lambda sm: 48, "big", "exact", 0),
    ("24sm", lambda sm: 24 * sm, "mixed", "exact", 0),
    ("24sm", lambda sm: 24 * sm, "mixed", 0, 0),
    ("24sm+1", lambda sm: 24 * sm + 1, "mixed", "exact", 0),
    ("24sm+1", lambda sm: 24 * sm + 1, "mixed", 0, 0),
    ("24sm+1", lambda sm: 24 * sm + 1, "small", "exact", 1),
    ("300", lambda sm: 300, "span", "exact", 1),
    ("600", lambda sm: 600, "mixed", 0, 1),
]


def enc_name(nblocks: int, sm: int, max_in_len: int, d: int) -> str:
    """What the encoder launcher records: above 24 blocks per SM without a dictionary the global-table kernel, else the
    shared-memory-table one; a bound above 64 KiB names the kernel of the larger blocks instead; an unknown bound (0),
    or one that the dictionary takes above 64 KiB, runs both and names both."""
    if max_in_len > 65536:
        return SPLIT32.format(d)
    first = GTAB if not d and nblocks > 24 * sm else SPLIT16.format(d)
    both = max_in_len == 0 or max_in_len + (len(DICT) if d else 0) > 65536
    return first + (" + " + SPLIT32.format(d) if both else "")


def _bound_class(lengths: str, d: int) -> int:
    """A bound of the class encode_blocks() produces for `lengths`: small <= 64 KiB - len(DICT) (dictionary + input
    <= 64 KiB), span <= 64 KiB < dictionary + input, big and mixed > 64 KiB."""
    return {"small": 65536 - (len(DICT) if d else 0), "span": 65536}.get(lengths, 65537)


def _enc_id(c):
    label, count, lengths, mil, d = c
    bound = _bound_class(lengths, d) if mil == "exact" else 0
    return f"{enc_name(count(132), 132, bound, d)} | nb={label} {lengths}{' dict' if d else ''} max_in_len={mil}"


def encode_blocks(count: int, lengths: str, d: int, seed: int):
    """(data, mode, cap) per block: one kind of content per block, lengths 0..64 and 65 533..65 536 (with a dictionary:
    the same sums of dictionary and input) plus ragged ones, a mode per block (block API without a dictionary), every
    tenth capacity one byte short."""
    rng = np.random.default_rng(seed)
    dl = len(DICT) if d else 0
    if lengths == "big":
        ns = [65537, 65538, 65548, 70000, 131072, 131073] + [int(x) for x in rng.integers(65537, 300000, count)]
    else:
        ns = list(range(65)) + [x - dl for x in range(65533, 65537) for _ in range(6)]
        if lengths != "small":
            ns += [x - dl for x in (65537, 65538, 65540)]
        top = 65536 - dl if lengths == "small" else 65536
        while len(ns) < count:
            u = rng.random()
            if lengths == "mixed" and u < 0.03:
                ns.append(int(rng.integers(65537 - dl, 140000)))
            else:
                ns.append(int(rng.integers(65, 3000)) if u < 0.75 else int(rng.integers(3000, 12000)) if u < 0.95
                          else int(rng.integers(12000, top + 1)))
    ns = [ns[i] for i in rng.permutation(len(ns))][:count]
    out = []
    for b, n in enumerate(ns):
        data = _content(rng, CONTENT[int(rng.integers(0, len(CONTENT)))], n)
        mode = 0 if d else (0, FL_FRESH_H5, FL_CONT)[int(rng.integers(0, 3))]
        cap = block.get_maximum_output_size(n) - (1 if b % 10 == 7 else 0) + (int(rng.integers(0, 40)) if b % 10 == 3 else 0)
        out.append((data, mode, cap))
    return out


class EncodeLayout:
    def __init__(self, blocks, d: int):
        rng = np.random.default_rng(len(blocks) + 7)
        nb = len(blocks)
        self.blocks, self.dct = blocks, DICT if d else b""
        self.in_len = np.array([len(b[0]) for b in blocks], dtype=np.uint32)
        self.flags = None if d else np.array([b[1] for b in blocks], dtype=np.uint8)
        self.out_cap = np.array([b[2] for b in blocks], dtype=np.uint32)
        self.in_off = _place(self.in_len, np.arange(nb) % 16)
        self.out_off = _place(self.out_cap, (np.arange(nb) * 5 + 9) % 16, gap=True)
        self.src = np.zeros(int(self.in_off[-1]) + int(self.in_len[-1]) + 16, dtype=np.uint8)
        for o, b in zip(self.in_off, blocks):
            self.src[int(o): int(o) + len(b[0])] = np.frombuffer(b[0], dtype=np.uint8)
        self.size = int(self.out_off[-1]) + int(self.out_cap[-1]) + 16
        self.init = rng.integers(0, 256, self.size, dtype=np.uint8)
        short = np.array([b[2] < block.get_maximum_output_size(len(b[0])) for b in blocks])

        def one(b):
            return None if short[b] else (oracle.compress_with_dict(blocks[b][0], self.dct) if d
                                          else ORACLE_BY_MODE[blocks[b][1]](blocks[b][0]))
        with cf.ThreadPoolExecutor(os.cpu_count() or 1) as ex:
            want = list(ex.map(one, range(nb), chunksize=16))
        self.want_status = np.where(short, 1, 0).astype(np.int32)
        self.want_len = np.array([0 if w is None else len(w) for w in want], dtype=np.int64)
        self.want_bytes = self.init.copy()
        self.checked = np.ones(self.size, dtype=bool)        # the bytes a block wrote past its length are not specified
        for b, w in enumerate(want):
            if w is not None:
                o = int(self.out_off[b])
                self.want_bytes[o: o + len(w)] = np.frombuffer(w, dtype=np.uint8)
                self.checked[o + len(w): o + int(self.out_cap[b])] = False

    def where(self, b: int) -> str:
        data, mode, cap = self.blocks[b]
        return f"block {b} (n {len(data)}, mode {mode}, cap {cap}, in_off {int(self.in_off[b])}, out_off {int(self.out_off[b])})"

    def check(self, res):
        buf, status, out_len = res
        bad = np.nonzero(status != self.want_status)[0]
        assert not bad.size, f"{bad.size} statuses differ; first: {self.where(bad[0])}: {status[bad[0]]}"
        bad = np.nonzero(out_len != self.want_len)[0]
        assert not bad.size, f"{bad.size} lengths differ; first: {self.where(bad[0])}: {out_len[bad[0]]} != {self.want_len[bad[0]]}"
        diff = (buf != self.want_bytes) & self.checked
        if diff.any():
            i = int(np.argmax(diff))
            b = int(np.searchsorted(self.out_off, i, side="right")) - 1
            part = "in its slot" if b >= 0 and i < int(self.out_off[b]) + int(self.out_cap[b]) else "in the canary gap after it"
            pytest.fail(f"{int(diff.sum())} output bytes differ; first at {i}, {part}: {self.where(max(b, 0))}")


def encode_tensors(lay: EncodeLayout):
    import torch
    nb = len(lay.blocks)
    t = dict(nb=nb, dlen=len(lay.dct), src=_t(lay.src), ioff=_t(lay.in_off), ilen=_t(lay.in_len), out=_t(lay.init),
             ooff=_t(lay.out_off), ocap=_t(lay.out_cap), olen=torch.full((nb,), -1, dtype=torch.int32, device="cuda"),
             st=torch.full((nb,), -1, dtype=torch.int32, device="cuda"))
    if lay.dct:
        t["dict"] = _t(np.frombuffer(lay.dct, dtype=np.uint8).copy())
    else:
        t["flags"] = _t(lay.flags)
    return t


def enqueue_encode(ctx, t, max_in_len: int) -> str:
    """One lz4b200_compress_batch_device[_with_dict] call on torch's current stream, no synchronisation.  Returns the
    kernel(s) the launcher recorded."""
    import torch
    L, s = _native.lib(), torch.cuda.current_stream().cuda_stream
    p = {k: v.data_ptr() for k, v in t.items() if hasattr(v, "data_ptr")}
    if t["dlen"]:
        rc = L.lz4b200_compress_batch_device_with_dict(ctx.handle, p["src"], p["ioff"], p["ilen"], p["dict"], t["dlen"],
                                                       p["out"], p["ooff"], p["ocap"], p["olen"], p["st"], t["nb"],
                                                       max_in_len, s)
    else:
        rc = L.lz4b200_compress_batch_device(ctx.handle, p["src"], p["ioff"], p["ilen"], p["flags"], p["out"], p["ooff"],
                                             p["ocap"], p["olen"], p["st"], t["nb"], max_in_len, s)
    assert rc == 0, ctx.last_cuda_error()
    return L.lz4b200_ctx_last_kernel(ctx.handle, 0).decode()


def collect_encode(t):
    return t["out"].cpu().numpy(), t["st"].cpu().numpy(), t["olen"].cpu().numpy().astype(np.int64)


@functools.lru_cache(maxsize=None)
def _enc_layout(i: int, sm: int):
    _, count, lengths, _, d = ENC_CASES[i]
    return EncodeLayout(encode_blocks(count(sm), lengths, d, seed=100 + i), d)


def _enc_run(i: int, sm: int):
    """(layout, max_in_len to pass, kernel name to expect) of encoder case i."""
    _, count, lengths, mil, d = ENC_CASES[i]
    lay = _enc_layout(i, sm)
    bound = int(lay.in_len.max()) if mil == "exact" else 0
    if bound:                                                # the generator produced the class of bound the id names
        cls = _bound_class(lengths, d)
        assert (bound > 65536) == (cls > 65536) and (bound + len(lay.dct) > 65536) == (cls + len(lay.dct) > 65536)
    return lay, bound, enc_name(count(sm), sm, bound, d)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(ENC_CASES)), ids=[_enc_id(c) for c in ENC_CASES])
def test_encoder_shape_adversarial_batch(ctx, i):
    import torch
    lay, max_in_len, name = _enc_run(i, sm_count())
    t = encode_tensors(lay)
    assert enqueue_encode(ctx, t, max_in_len) == name, len(lay.blocks)
    torch.cuda.synchronize()
    got = collect_encode(t)
    lay.check(got)
    # round trip: what the GPU wrote, back through the device decoder into the input's layout
    ok = np.nonzero(lay.want_status == 0)[0]
    td = decode_tensors(got[0], lay.out_off[ok], got[2][ok].astype(np.uint32), np.zeros(lay.src.size, dtype=np.uint8),
                        lay.in_off[ok], lay.in_len[ok], lay.dct)
    enqueue_decode(ctx, td)
    out, st, ol, _ = collect_decode(td)
    assert not st.any() and np.array_equal(ol, lay.in_len[ok].astype(np.int64))
    for b in ok:
        o = int(lay.in_off[b])
        assert out[o: o + int(lay.in_len[b])].tobytes() == lay.blocks[b][0], lay.where(b)


# ---- back to back --------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_all_shapes_back_to_back_on_one_stream(ctx):
    """Every shape above enqueued on one stream with no synchronisation between the launches: each kernel re-arms the
    ticket counters it shares with the next launch of its kind (split-u16 and gtab share one pair, the decoders
    another), so a counter left behind would skip or repeat blocks of the next batch."""
    import itertools

    import torch
    sm = sm_count()
    dec = [("dec", s) for s in DEC_SHAPES if dec_count(*s, sm)]
    enc = [("enc", i) for i in range(len(ENC_CASES))]
    order = [k for pair in itertools.zip_longest(dec, enc) for k in pair if k]     # decoders and encoders interleaved
    runs = []
    for kind, arg in order:                                  # every buffer uploaded first: nothing waits in between
        if kind == "dec":
            lay = _dec_case(*arg, sm)
            runs.append((kind, lay, layout_decode_tensors(lay, 0xFF), dec_name(*arg), None))
        else:
            lay, max_in_len, name = _enc_run(arg, sm)
            runs.append((kind, lay, encode_tensors(lay), name, max_in_len))
    torch.cuda.synchronize()
    for kind, lay, t, name, max_in_len in runs:
        got = enqueue_decode(ctx, t) if kind == "dec" else enqueue_encode(ctx, t, max_in_len)
        assert got == name
    torch.cuda.synchronize()
    for kind, lay, t, _, _ in runs:
        if kind == "dec":
            lay.check(collect_decode(t), 0xFF)
        else:
            lay.check(collect_encode(t))


# ---- the generator itself (CPU) ------------------------------------------------------------------------------------

def test_generator_builds_what_it_claims():
    """Every hand-built stream decodes (oracle) to the status it was built for; each decoder batch, even the smallest
    one any shape uses, holds every decoder status, the deferral patterns in useful numbers and only distinct blocks."""
    for dct, count in ((b"", dec_count(32, 1, 0, 132)), (DICT, dec_count(32, 4, 1, 132))):
        for kind, s, cap, st, exp in hand_built(dct):
            if st is None:
                continue
            got = oracle.decompress_with_dict(s, cap, dct) if dct else oracle.decompress_block(s, cap)
            assert got[0] == st, (kind, s.hex(), cap, got[0])
            if st == oracle.ERR_OUTPUT_TOO_SMALL:
                assert got[2] == exp, (kind, s.hex(), cap)
            if st == 0 and kind.startswith("defer"):
                assert got[0] == 0 and len(got[1]) <= cap
        blocks = decode_blocks(count, dct)
        assert len({(b[1], b[2]) for b in blocks}) == count
        want = oracle_decode(blocks, dct)
        assert {w[0] for w in want} >= DEC_STATUSES, sorted({w[0] for w in want})
        kinds = {}
        for b in blocks:
            kinds[b[0]] = kinds.get(b[0], 0) + 1
        defer = [k for k in kinds if k.startswith("defer")]
        assert len(defer) == (10 if dct else 9) and all(kinds[k] >= 24 for k in defer), kinds
        assert kinds["overlap"] == 630 and kinds["kat"] == len(DECODE_KATS)
        for src in ("json", "dickens", "hdfs", "noise", "periodic"):
            assert kinds.get(f"mutated_{src}", 0) >= 5 and kinds.get(f"good_{src}", 0) >= 5, (src, kinds)
        assert sum(v for k, v in kinds.items() if k.startswith("garbage")) >= 50
    # the shape table: every range the launcher has, on a few SM counts
    for sm in (8, 66, 114, 132, 144, 200):
        for g, w, d in DEC_SHAPES:
            n = dec_count(g, w, d, sm)
            if n is None:
                continue
            G = 8 if n >= 12288 else 16 if n >= 4096 else 32
            one = not d and -(-n // (32 // G)) <= 32 * sm
            assert (G, 1 if one else 4) == (g, w), (sm, g, w, d, n)
    assert dec_count(32, 4, 0, 132) is None and dec_count(32, 4, 0, 100) is not None
