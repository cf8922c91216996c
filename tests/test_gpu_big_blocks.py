"""The block codec on single blocks from 8 MiB to the largest one the host entry points accept, and on length fields
whose extension bytes sum past 2^32, against the oracle.

The plants (tests/test_big_block_plants.py, which checks on the CPU that each reaches its edge) put literal runs
longer than 2^24, table entries and matches past 2^31, a match at offset 65 535 past 2^31, a match longer than 2^20
and the end-of-block rules in front of the u32-table encoder (`lz4_compress_blocks_split<unsigned int, 2, {0,1}>`)
and the decoders (`lz4_decompress_blocks<G, 0, d, w>`), whose positions and sizes are all 32 bits wide.

* encode: block.compress, compress_prepend_size and one DeviceBatch with max_in_len exact and 0 (the launcher's record
  names the kernels that ran), byte for byte against the oracle; the text plants also in FRESH_H5 and CONT; the
  dictionary form on a 64 MiB plant.  A mismatch names the first differing sequence.
* the largest accepted block, and one byte more: InvalidArgument with nothing written.
* decode: block.decompress, decompress_size_prepended and decompress_into (G = 32, one-warp CTA); the 64 MiB text
  and 2^31 + 2^20 + 7 sparse plants inside batches the launcher runs at G = 16 and 8, one- and four-warp CTAs.  Each
  with the exact capacity, one byte less (OutputTooSmall with the oracle's `expected`) and the stream cut inside a
  0xFF run (ExpectedAnotherByte), canaries after every output slot, outputs compared on the device.
* hand-built streams of about 17 MiB whose length fields sum past 2^32, through every decoder path: a literal length
  of 2^32 + 5 without the input (LiteralOutOfBounds), a match length of 2^32 + 3 (OutputTooSmall, expected
  op + 2^32 + 3), and a match ending exactly at 2^32 with a capacity of 2^32 - 1 (OutputTooSmall, expected 2^32),
  which a 32-bit sum would wrap to 0.
"""
from __future__ import annotations

import functools
import gc
import warnings

import numpy as np
import pytest

import oracle
from lz4_flex_b200 import _native, block, errors
from test_big_block_plants import (NAMES, SMALL_DICT, TOP, dict_oracle, dict_plant, first_ff_run, huge_length_streams,
                                   max_output_size, oracle_decode_into, oracle_stream, plant, release, walk)
from test_gpu_launch_shapes import (SPLIT16, SPLIT32, DecodeLayout, _t, dec_batch, dec_count, dec_name, enqueue_decode,
                                    sm_count)

pytestmark = pytest.mark.gpu

CANARY = 0x5A
GAP = 64                                          # canary bytes after every output slot


@pytest.fixture(scope="module")
def ctx():
    """This module's own context.  Blocks of up to 3.64 GiB grow a context's device scratch by more than 12 GiB and
    torch's cached allocations by about 25 GiB; closing the context, dropping the cached plants and tensors and
    emptying torch's cache at the end hands all of it back to the tests that run after this module."""
    import torch
    c = block.Context(0)
    yield c
    c.close()
    _dev_plant.cache_clear()
    short_expected.cache_clear()
    release()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _empty_torch_cache():
    """Each test's buffers are sized to its block; handing them back after every test keeps torch from caching a new
    set of tens of GiB per block size."""
    import torch
    yield
    torch.cuda.empty_cache()


def _dev(a):
    """bytes / read-only uint8 array -> CUDA uint8 tensor (a copy; the source is never written)."""
    import torch
    a = np.frombuffer(a, dtype=np.uint8) if isinstance(a, (bytes, bytearray, memoryview)) else a
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                    # torch warns about read-only arrays
        return torch.from_numpy(a).cuda()


@functools.lru_cache(maxsize=2)
def _dev_plant(name: str):
    return _dev(plant(name)[1])


def _first_difference(got, want) -> str:
    g, w = walk(bytes(got)), walk(bytes(want))
    for i, (a, b) in enumerate(zip(g, w)):
        if a[:5] != b[:5]:
            return f"sequence {i}: GPU {a[:5]} != oracle {b[:5]}"
    return f"sequence {min(len(g), len(w))}: GPU has {len(g)} sequences, the oracle {len(w)}"


def _same_stream(got: np.ndarray, want: bytes, where: str):
    w = np.frombuffer(want, dtype=np.uint8)
    if got.size != w.size or not np.array_equal(got, w):
        pytest.fail(f"{where}: {got.size} bytes, the oracle {w.size}; " + _first_difference(got, w))


def _kernel(ctx, which: int) -> str:
    return _native.lib().lz4b200_ctx_last_kernel(ctx.handle, which).decode()


# ---- encode --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", NAMES)
def test_block_api_encode(ctx, name):
    p, data = plant(name)
    want = oracle_stream(name)
    got = block.compress(data, ctx=ctx)
    assert SPLIT32.format(0) in _kernel(ctx, 0)
    _same_stream(np.frombuffer(got, dtype=np.uint8), want, f"{name} compress")
    del got
    got = np.frombuffer(block.compress_prepend_size(data, ctx=ctx), dtype=np.uint8)
    assert got[:4].tobytes() == p.n.to_bytes(4, "little")
    _same_stream(got[4:], want, f"{name} compress_prepend_size")


@pytest.mark.parametrize("bound", ("exact", 0))
@pytest.mark.parametrize("name", NAMES)
def test_device_batch_encode(ctx, name, bound):
    """One DeviceBatch: the plant once per mode (text: FRESH, FRESH_H5 and CONT, all reading the same input), slots
    followed by canaries."""
    import torch
    p, _ = plant(name)
    d_in = _dev_plant(name)
    nb, cap = len(p.modes), max_output_size(p.n)
    stride = (cap + GAP + 15) // 16 * 16 + 16
    out_off = [b * stride + 3 * b for b in range(nb)]               # slots at residues 0, 3, 6 mod 16
    d_out = torch.full((out_off[-1] + cap + GAP,), CANARY, dtype=torch.uint8, device="cuda")
    bt = block.DeviceBatch([0] * nb, [p.n] * nb, out_off, [cap] * nb, flags=list(p.modes))
    bt.max_in_len = p.n if bound == "exact" else 0
    bt.compress(d_in, d_out, ctx)
    torch.cuda.synchronize()
    assert _kernel(ctx, 0) == (SPLIT32.format(0) if bound else SPLIT16.format(0) + " + " + SPLIT32.format(0))
    st = bt.status.cpu().numpy()
    ol = bt.out_len.cpu().numpy().view(np.uint32)
    for b, mode in enumerate(p.modes):
        want = oracle_stream(name, mode)
        o = out_off[b]
        assert st[b] == 0 and ol[b] == len(want), (name, mode, st[b], ol[b], len(want))
        if not torch.equal(d_out[o: o + len(want)], _dev(want)):
            _same_stream(d_out[o: o + len(want)].cpu().numpy(), want, f"{name} mode {mode}")
        assert bool((d_out[o + cap: o + cap + GAP] == CANARY).all()), (name, mode, "canary")


def test_dictionary_u32_kernel(ctx):
    dct, d = dict_plant()
    want = dict_oracle()
    got = block.compress_with_dict(d, dct, ctx=ctx)
    assert SPLIT32.format(1) in _kernel(ctx, 0)
    _same_stream(np.frombuffer(got, dtype=np.uint8), want, "compress_with_dict")
    out = np.empty(d.size + GAP, dtype=np.uint8)
    out[d.size:] = CANARY
    assert block.decompress_into_with_dict(want, out[: d.size], dct, ctx=ctx) == d.size
    assert np.array_equal(out[: d.size], d) and (out[d.size:] == CANARY).all()


def test_largest_accepted_block_and_one_more(ctx):
    """n = TOP is encoded (test_block_api_encode[top]); n = TOP + 1 needs a bound above 0xffffffff: InvalidArgument,
    with the output untouched (zero pages that are never committed unless written)."""
    src = np.zeros(TOP + 1, dtype=np.uint8)
    out = np.zeros(max_output_size(TOP + 1), dtype=np.uint8)
    with pytest.raises(ValueError):
        block.compress_into(src, out, ctx=ctx)
    assert not out.any()


# ---- decode --------------------------------------------------------------------------------------------------------

def _cut(name: str):
    """The oracle stream cut inside a length extension: halfway through a long 0xFF run (a literal run through noise,
    the long match) where the plant has one, else in the first extension of a text plant."""
    s = oracle_stream(name)
    pos, r = first_ff_run(s, 0 if name.startswith("text") else 200)
    return s[: pos + (r + 1) // 2]


@functools.lru_cache(maxsize=None)
def short_expected(name: str) -> int:
    """The oracle's OutputTooSmall `expected` at capacity n - 1."""
    p, _ = plant(name)
    st, _, e = oracle_decode_into(oracle_stream(name), np.empty(p.n - 1, dtype=np.uint8))
    assert st == oracle.ERR_OUTPUT_TOO_SMALL
    return e


@pytest.mark.parametrize("name", NAMES)
def test_single_block_decode(ctx, name):
    p, data = plant(name)
    s = oracle_stream(name)
    got = np.frombuffer(block.decompress(s, p.n, ctx=ctx), dtype=np.uint8)
    assert _kernel(ctx, 1) == dec_name(32, 1, 0)
    assert got.size == p.n and np.array_equal(got, data), name
    del got
    got = np.frombuffer(block.decompress_size_prepended(p.n.to_bytes(4, "little") + s, ctx=ctx), dtype=np.uint8)
    assert got.size == p.n and np.array_equal(got, data), name
    del got
    buf = np.empty(p.n + GAP, dtype=np.uint8)
    buf[p.n:] = CANARY
    assert block.decompress_into(s, buf[: p.n], ctx=ctx) == p.n
    assert np.array_equal(buf[: p.n], data) and (buf[p.n:] == CANARY).all(), name
    buf[p.n - 1:] = CANARY
    with pytest.raises(errors.OutputTooSmall) as e:
        block.decompress_into(s, buf[: p.n - 1], ctx=ctx)
    assert (e.value.expected, e.value.actual) == (short_expected(name), p.n - 1)
    assert (buf[p.n - 1:] == CANARY).all(), name
    cut = _cut(name)
    assert oracle.decompress_block(cut, 1 << 20)[0] == oracle.ERR_EXPECTED_ANOTHER_BYTE
    buf[p.n:] = CANARY
    with pytest.raises(errors.ExpectedAnotherByte):
        block.decompress_into(cut, buf[: p.n], ctx=ctx)
    assert (buf[p.n:] == CANARY).all(), name


class Big:
    """A block of a decode batch that is not one of the shape tests' small blocks: its stream (bytes or a CUDA
    tensor), capacity, the status and `expected` the oracle gives, and the bytes its slot must hold on success."""

    def __init__(self, stream, cap: int, status: int, expected: int = 0, want=None, fill_checked: int = -1):
        self.stream, self.cap, self.status, self.expected, self.want = stream, cap, status, expected, want
        self.fill_checked = fill_checked            # >= 0: the slot from this byte on must still hold the fill


def _run_batch(ctx, g: int, w: int, bigs, dct: bytes = b""):
    """One device batch of dec_count(g, w) blocks: the shape tests' small blocks (checked as they check them) with the
    `bigs` placed among them (at the start, the middle and the end of the descriptors), their streams after the small
    ones' and their slots after the small ones' slots, each followed by GAP canary bytes."""
    import torch
    sm = sm_count()
    count = dec_count(g, w, 0, sm)
    if count is None:
        pytest.skip(f"no batch size reaches {dec_name(g, w, 0)} on {sm} SMs")
    small, want = dec_batch(0, count - len(bigs), sm)
    lay = DecodeLayout(small, want)
    fill = 0x00
    where = np.linspace(0, count - 1, len(bigs)).astype(np.int64)
    streams = [b.stream if hasattr(b.stream, "data_ptr") else _dev(b.stream) for b in bigs]
    ilens = [int(s.numel()) for s in streams]
    in_off, pos = [], lay.src.size + 16
    for n in ilens:
        pos += (5 - pos) % 16                                      # streams at residue 5
        in_off.append(pos)
        pos += n
    src = torch.zeros(pos + 16, dtype=torch.uint8, device="cuda")
    src[: lay.src.size] = _dev(lay.src)
    for o, s in zip(in_off, streams):
        src[o: o + s.numel()] = s
    out_off, pos = [], lay.size + GAP
    for b in bigs:
        pos += (9 - pos) % 16
        out_off.append(pos)
        pos += b.cap + GAP
    out = torch.full((pos,), CANARY, dtype=torch.uint8, device="cuda")
    out[: lay.size] = _dev(lay.initial(fill))
    for o, b in zip(out_off, bigs):
        out[o: o + b.cap] = fill

    def merge(small_vals, big_vals, dt):
        a = np.insert(np.asarray(small_vals, dtype=dt), where - np.arange(len(bigs)), np.asarray(big_vals, dtype=dt))
        assert a.size == count
        return a
    ioff = merge(lay.in_off, in_off, np.uint64)
    ilen = merge(lay.in_len, ilens, np.uint32)
    ooff = merge(lay.out_off, out_off, np.uint64)
    ocap = merge(lay.out_cap, [b.cap for b in bigs], np.uint32)
    assert np.array_equal(ilen[where], np.array(ilens, dtype=np.uint32))
    t = dict(nb=count, dlen=len(dct), src=src, ioff=_t(ioff), ilen=_t(ilen), out=out, ooff=_t(ooff), ocap=_t(ocap),
             olen=torch.full((count,), -1, dtype=torch.int32, device="cuda"),
             st=torch.full((count,), -1, dtype=torch.int32, device="cuda"),
             exp=torch.full((count,), -1, dtype=torch.int64, device="cuda"))
    assert enqueue_decode(ctx, t) == dec_name(g, w, 0), count
    torch.cuda.synchronize()
    st, olen, exp = (t["st"].cpu().numpy(), t["olen"].cpu().numpy().view(np.uint32).astype(np.int64),
                     t["exp"].cpu().numpy())
    rest = np.setdiff1d(np.arange(count), where)
    lay.check((out[: lay.size].cpu().numpy(), st[rest], olen[rest], exp[rest]), fill)
    for k, (i, o, b) in enumerate(zip(where, out_off, bigs)):
        what = f"big block {k} at {i} (cap {b.cap})"
        assert (st[i], exp[i]) == (b.status, b.expected), (what, st[i], exp[i], b.status, b.expected)
        assert olen[i] == (b.cap if b.status == 0 else 0), (what, olen[i])
        if b.want is not None:
            assert torch.equal(out[o: o + b.cap], b.want), what
        if b.fill_checked >= 0:
            assert bool((out[o + b.fill_checked: o + b.cap] == fill).all()), (what, "written past what it decoded")
        assert bool((out[o + b.cap: o + b.cap + GAP] == CANARY).all()), (what, "canary")


BATCH_SHAPES = ((16, 1), (16, 4), (8, 1), (8, 4))


@pytest.mark.parametrize("g,w", BATCH_SHAPES, ids=[dec_name(g, w, 0) for g, w in BATCH_SHAPES])
@pytest.mark.parametrize("name", ("text_64m", "sparse_2g+1m+7"))
def test_big_block_in_batch_shapes(ctx, name, g, w):
    """The plant three times in one batch of small blocks: exact capacity, one byte less, and cut inside a 0xFF run."""
    p, _ = plant(name)
    s = _dev(oracle_stream(name))
    bigs = [Big(s, p.n, 0, want=_dev_plant(name)),
            Big(s, p.n - 1, oracle.ERR_OUTPUT_TOO_SMALL, short_expected(name)),
            Big(_cut(name), p.n, oracle.ERR_EXPECTED_ANOTHER_BYTE)]
    _run_batch(ctx, g, w, bigs)


# ---- length fields past 2^32 ---------------------------------------------------------------------------------------

EXC = {oracle.ERR_LITERAL_OOB: errors.LiteralOutOfBounds, oracle.ERR_OUTPUT_TOO_SMALL: errors.OutputTooSmall}


def _host_out(cap: int):
    """A zero-filled buffer of cap + GAP bytes, committed only where written, with canaries after the slot."""
    buf = np.zeros(cap + GAP, dtype=np.uint8)
    buf[cap:] = CANARY
    return buf


@pytest.mark.parametrize("path", ("decompress_into", "decompress_into_with_dict", "decompress_batch"))
def test_huge_lengths_host_paths(ctx, path):
    for label, s, cap, status, expected in huge_length_streams():
        buf = _host_out(cap)
        if path == "decompress_batch":
            _, st, exp = block.decompress_batch(np.frombuffer(s, dtype=np.uint8), [0], [len(s)], buf, [0], [cap],
                                                ctx=ctx, raise_on_error=False)
            got = (int(st[0]), int(exp[0]) if st[0] == oracle.ERR_OUTPUT_TOO_SMALL else 0)
        else:
            with pytest.raises(EXC[status]) as e:
                if path == "decompress_into":
                    block.decompress_into(s, buf[:cap], ctx=ctx)
                else:
                    block.decompress_into_with_dict(s, buf[:cap], SMALL_DICT, ctx=ctx)
            got = (status, e.value.expected if status == oracle.ERR_OUTPUT_TOO_SMALL else 0)
            if status == oracle.ERR_OUTPUT_TOO_SMALL:
                assert e.value.actual == cap, label
        assert got == (status, expected), (path, label, got)
        assert (buf[cap:] == CANARY).all(), (path, label, "canary")
        del buf


@pytest.mark.parametrize("g", (32, 16, 8))
def test_huge_lengths_device_batch(ctx, g):
    """The three streams among small blocks at G = g: statuses, `expected`, and nothing written past the 8 literals
    (the 4 GiB slot of the last stream included) or after any slot."""
    w = 1 if dec_count(g, 1, 0, sm_count()) else 4
    bigs = [Big(s, cap, status, expected, fill_checked=0 if status == oracle.ERR_LITERAL_OOB else 8)
            for _, s, cap, status, expected in huge_length_streams()]
    _run_batch(ctx, g, w, bigs)
