"""GPU parity tests of the block path: every call goes through the C ABI (include/lz4b200.h) into the
sm_90a kernels and is compared with the CPU oracle — bit-exact for compressed bytes, decoded bytes, error
codes and OutputTooSmall fields.  Structure follows the reference's tests/tests.rs."""
import hashlib
import json
import os

import numpy as np
import pytest

import oracle
from lz4_flex_b200 import block, corpus, errors
from vectors import DECODE_KATS, NO_PANIC, ROUNDTRIP

pytestmark = pytest.mark.gpu
GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "known_answers.json")))
FL_FRESH_H5 = block.BLOCK_HASH5_ALWAYS
FL_CONT = block.BLOCK_HASH5_ALWAYS | block.BLOCK_CONT


def sha(b):
    return hashlib.sha256(b).hexdigest()


def _golden_input(name):
    gen = {"json_tiled_block0": lambda: corpus.tiled("compression_66k_JSON.txt", 131072).tobytes()[:65536],
           "json_tiled_block1": lambda: corpus.tiled("compression_66k_JSON.txt", 131072).tobytes()[65536:],
           "zeros_65536": lambda: bytes(65536),
           "hdfs_first_4MiB": lambda: corpus.load("hdfs.json")[: 4 << 20],
           "xorshift_65536": lambda: corpus.xorshift64star_bytes(65536).tobytes()}
    return gen[name]() if name in gen else corpus.load(name)


def test_native_library_is_what_runs(ctx):
    # the loaded shared object is the in-tree CUDA library, and it sees the device
    from lz4_flex_b200 import _native
    assert os.path.samefile(_native.lib()._name, os.path.join(os.path.dirname(block.__file__), "liblz4b200.so"))
    assert ctx.handle


@pytest.mark.parametrize("entry", GOLDEN["block"], ids=[e["name"] for e in GOLDEN["block"]])
def test_known_answers(ctx, entry):
    data = _golden_input(entry["name"])
    for mode, fl in (("block_api", None), ("frame_fresh", [FL_FRESH_H5]), ("frame_cont", [FL_CONT])):
        c = block.compress_blocks([data], fl, ctx)[0]
        assert (len(c), sha(c)) == (entry[mode]["len"], entry[mode]["sha256"]), mode
    assert block.decompress(block.compress(data, ctx), len(data), ctx) == data


def test_single_block_api(ctx):
    # config 1: compress_prepend_size + decompress_size_prepended on compression_66k_JSON.txt
    j = corpus.load("compression_66k_JSON.txt")
    p = block.compress_prepend_size(j, ctx)
    assert p == oracle.compress_prepend_size(j) and len(p) == 4 + 15268
    assert block.decompress_size_prepended(p, ctx) == j
    out = np.zeros(block.get_maximum_output_size(len(j)), dtype=np.uint8)
    n = block.compress_into(j, out, ctx)
    assert out[:n].tobytes() == oracle.compress_block(j)
    with pytest.raises(errors.CompressOutputTooSmall):                 # compress.rs:338-340
        block.compress_into(j, np.zeros(block.get_maximum_output_size(len(j)) - 1, dtype=np.uint8), ctx)
    back = np.zeros(len(j) + 100, dtype=np.uint8)                      # larger capacity is fine
    assert block.decompress_into(p[4:], back, ctx) == len(j) and back[: len(j)].tobytes() == j


@pytest.mark.parametrize("name,stream,cap,status,out,expected", DECODE_KATS, ids=[str(i) for i in range(len(DECODE_KATS))])
def test_decode_kats(ctx, name, stream, cap, status, out, expected):
    outs, st, exp = block.decompress_blocks([bytes(stream)], [cap], ctx, raise_on_error=False)
    assert st[0] == status, name
    if out is not None:
        assert outs[0] == out
    if expected is not None:
        assert int(exp[0]) == expected


def test_decode_errors_raise_reference_variants(ctx):
    with pytest.raises(errors.ExpectedAnotherByte):
        block.decompress_into(b"", np.zeros(8, dtype=np.uint8), ctx)
    with pytest.raises(errors.LiteralOutOfBounds):
        block.decompress_into(bytes([0x40, 97, 1, 0]), np.zeros(4, dtype=np.uint8), ctx)
    with pytest.raises(errors.OutputTooSmall) as e:
        block.decompress_into(bytes([0x20, 97, 97, 1, 0]), np.zeros(1, dtype=np.uint8), ctx)
    assert (e.value.expected, e.value.actual) == (2, 1)
    with pytest.raises(errors.OutputTooSmall) as e:
        block.decompress_into(bytes([0x10, 97, 1, 0]), np.zeros(4, dtype=np.uint8), ctx)
    assert (e.value.expected, e.value.actual) == (5, 4)
    with pytest.raises(errors.OffsetOutOfBounds):
        block.decompress_into(bytes([0x0E, 255] + [0] * 18), np.zeros(256, dtype=np.uint8), ctx)
    with pytest.raises(errors.OffsetZero):
        block.decompress_into(bytes([0x0E, 0, 0, 0x70] + [0] * 20), np.zeros(256, dtype=np.uint8), ctx)
    with pytest.raises(errors.ExpectedAnotherByte):
        block.decompress_size_prepended(b"\x01\x00", ctx)


def test_roundtrip_vectors_all_modes(ctx):
    for fl, ref in ((None, oracle.compress_block), ([FL_FRESH_H5] * len(ROUNDTRIP), oracle.compress_block_fresh_h5),
                    ([FL_CONT] * len(ROUNDTRIP), oracle.compress_block_cont)):
        comp = block.compress_blocks(ROUNDTRIP, fl, ctx)
        for d, c in zip(ROUNDTRIP, comp):
            assert c == ref(d), len(d)
        outs, st, _ = block.decompress_blocks(comp, [max(len(d), 1) for d in ROUNDTRIP], ctx)
        assert outs == list(ROUNDTRIP)


def test_edge_lengths_and_hash_switch(ctx):
    """Every length around MFLIMIT/LZ4_MIN_LENGTH, warp-width multiples, extension-byte boundaries
    (15+255k) and the 65 535-byte hash4->hash5 / u16->u32 switch (compress.rs:559)."""
    rng = np.random.default_rng(3)
    lens = list(range(0, 40)) + [63, 64, 65, 269, 270, 271, 272, 524, 525, 526, 1000, 4095, 4096, 4097,
                                  65533, 65534, 65535, 65536, 65537, 65548, 70000, 131072, 200001]
    cases = []
    for n in lens:
        cases.append(rng.integers(0, 3, n, dtype=np.uint8).tobytes())
        cases.append((b"abcdefgh" * (n // 8 + 1))[:n])
        cases.append(bytes(n))
    comp = block.compress_blocks(cases, None, ctx)
    for d, c in zip(cases, comp):
        assert c == oracle.compress_block(d), len(d)
    outs, st, _ = block.decompress_blocks(comp, [max(len(d), 1) for d in cases], ctx)
    assert outs == cases
    comp = block.compress_blocks(cases, [FL_CONT] * len(cases), ctx)
    for d, c in zip(cases, comp):
        assert c == oracle.compress_block_cont(d), len(d)


def test_overlapping_matches_and_long_runs(ctx):
    """Periodic data with every period 1..40 (overlapping back-copies: duplicate_overlapping,
    decompress.rs:57-82; offset 1 = fill) and literal/match lengths crossing 15+255k."""
    cases = []
    rng = np.random.default_rng(5)
    for period in list(range(1, 41)) + [63, 64, 65, 255, 256, 257, 1000]:
        seed = rng.integers(0, 256, period, dtype=np.uint8).tobytes()
        for total in (period * 3 + 20, 300, 5000, 66000):
            cases.append((seed * (total // period + 1))[:total])
    comp = block.compress_blocks(cases, None, ctx)
    for d, c in zip(cases, comp):
        assert c == oracle.compress_block(d)
    outs, st, _ = block.decompress_blocks(comp, [len(d) for d in cases], ctx)
    assert outs == cases
    # hand-built streams with long extension chains
    for lit in (14, 15, 16, 269, 270, 271, 525, 5000):
        body = bytes(rng.integers(0, 256, lit, dtype=np.uint8))
        ext = b"" if lit < 15 else b"\xff" * ((lit - 15) // 255) + bytes([(lit - 15) % 255])
        stream = bytes([min(lit, 15) << 4]) + ext + body
        assert oracle.decompress_block(stream, lit)[:2] == (0, body)
        assert block.decompress(stream, lit, ctx) == body


def test_foreign_streams_liblz4(ctx):
    """Any valid LZ4 stream must decode bit-exact: blocks produced by the C library (different parse)."""
    import ctypes
    try:
        L = ctypes.CDLL("liblz4.so.1")
    except OSError:
        pytest.skip("liblz4 not present")
    L.LZ4_compress_default.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_int]
    L.LZ4_compressBound.argtypes = [ctypes.c_int]
    srcs = [corpus.load(f) for f in ("compression_1k.txt", "compression_34k.txt", "compression_65k.txt",
                                     "compression_66k_JSON.txt")]
    d = corpus.load("dickens.txt")
    srcs += [d[i * 65536:(i + 1) * 65536] for i in range(24)] + [d[: 1 << 20], bytes(100000)]
    comp = []
    for s in srcs:
        cap = L.LZ4_compressBound(len(s))
        buf = ctypes.create_string_buffer(cap)
        n = L.LZ4_compress_default(s, buf, len(s), cap)
        comp.append(buf.raw[:n])
    outs, st, _ = block.decompress_blocks(comp, [len(s) for s in srcs], ctx)
    assert outs == srcs


def test_no_panic_corpus(ctx):
    for data in NO_PANIC:
        data = bytes(data)
        size = int.from_bytes(data[:4], "little")
        if size > 20_000_000:
            continue
        s, o, e1, e2 = oracle.decompress_size_prepended(data)
        try:
            got = block.decompress_size_prepended(data, ctx)
            assert s == 0 and got == o
        except errors.DecompressError as e:
            assert s != 0 and type(e) is type(errors.block_error(s, e1, e2))


def test_garbage_matches_oracle(ctx):
    """fuzz_decomp_corrupt_block: random and mutated streams, arbitrary capacities — same status, same
    bytes on success, same `expected` on OutputTooSmall; neighbours in the batch unaffected."""
    rng = np.random.default_rng(11)
    streams, caps = [], []
    good = oracle.compress_block(corpus.load("compression_1k.txt"))
    for i in range(1500):
        kind = i % 3
        if kind == 0:
            s = rng.integers(0, 256, int(rng.integers(0, 64)), dtype=np.uint8).tobytes()
        elif kind == 1:
            b = bytearray(good)
            for _ in range(int(rng.integers(1, 4))):
                b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
            s = bytes(b[: int(rng.integers(1, len(b) + 1))])
        else:
            s = rng.integers(0, 32, int(rng.integers(1, 200)), dtype=np.uint8).tobytes()
        streams.append(s)
        caps.append(int(rng.integers(0, 900)))
    outs, st, exp = block.decompress_blocks(streams, [max(c, 0) for c in caps], ctx, raise_on_error=False)
    for i, (s, cap) in enumerate(zip(streams, caps)):
        es, eo, e1, e2 = oracle.decompress_block(s, cap)
        assert st[i] == es, (i, s.hex(), cap)
        if es == 0:
            assert outs[i] == eo
        if es == 2:
            assert int(exp[i]) == e1


def test_no_output_leak(ctx):
    """fuzz_decomp_no_output_leak.rs: decoding into a zero-filled and a 0xFF-filled buffer gives the same
    (len, bytes)."""
    rng = np.random.default_rng(13)
    streams = [rng.integers(0, 256, int(rng.integers(1, 80)), dtype=np.uint8).tobytes() for _ in range(400)]
    lens = np.array([len(s) for s in streams], dtype=np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens[:-1])]).astype(np.uint64)
    src = np.frombuffer(b"".join(streams), dtype=np.uint8)
    caps = np.full(len(streams), 300, dtype=np.uint32)
    ooff = (np.arange(len(streams)) * 300).astype(np.uint64)
    res = []
    for fill in (0, 255):
        out = np.full(300 * len(streams), fill, dtype=np.uint8)
        ol, st, _ = block.decompress_batch(src, offs, lens, out, ooff, caps, ctx, raise_on_error=False)
        res.append([(int(st[i]), out[i * 300: i * 300 + int(ol[i])].tobytes()) for i in range(len(streams))])
    assert res[0] == res[1]


def test_big_blocks(ctx):
    """4 MiB frame-sized blocks (u32 table path) in all three modes, an 8 MiB legacy-sized block, and an
    unaligned sub-buffer."""
    h = corpus.load("hdfs.json")
    d = corpus.load("dickens.txt")
    cases = [h[: 4 << 20], d[: 4 << 20], d[1: (1 << 20) + 7], h[3: 3 + (8 << 20)], bytes(4 << 20)]
    for fl, ref in ((None, oracle.compress_block), ([FL_FRESH_H5] * len(cases), oracle.compress_block_fresh_h5),
                    ([FL_CONT] * len(cases), oracle.compress_block_cont)):
        comp = block.compress_blocks(cases, fl, ctx)
        for x, c in zip(cases, comp):
            assert c == ref(x), len(x)
    outs, st, _ = block.decompress_blocks(comp, [len(x) for x in cases], ctx)
    assert outs == cases


def _oracle_compress_all(data, nb, B, slot):
    """Every block of a batch through the oracle (all host cores): (slot buffer, lengths)."""
    comp = np.zeros(nb * slot, dtype=np.uint8)
    offs = np.arange(nb, dtype=np.uint64) * B
    lens = np.full(nb, B, dtype=np.uint32)
    soff = np.arange(nb, dtype=np.uint64) * slot
    clen, st = oracle.compress_batch(data, offs, lens, comp, soff, np.full(nb, slot, dtype=np.uint32), os.cpu_count())
    assert not st.any()
    return comp, clen


def _assert_slots_equal(got, glen, want, wlen, nb, slot):
    """Byte-for-byte comparison of ALL blocks (vectorised: mask out each slot's unused tail)."""
    assert np.array_equal(glen.astype(np.int64), wlen.astype(np.int64))
    g = got[: nb * slot].reshape(nb, slot)
    w = want[: nb * slot].reshape(nb, slot)
    used = np.arange(slot, dtype=np.uint32)[None, :] < wlen.astype(np.uint32)[:, None]
    diff = (g != w) & used
    assert not diff.any(), f"first differing block {int(np.argmax(diff.any(axis=1)))}"


def test_config2_full_size_properties(ctx):
    """BASELINE config 2 at full size: 16 384 x 64 KiB JSON blocks on the device-pointer path.  EVERY block's bytes
    equal the oracle's, exact round trip, and the GPU decodes the oracle's stream."""
    import torch
    nb, B, slot = 16384, 65536, 72112
    data = corpus.tiled("compression_66k_JSON.txt", nb * B)
    dev = torch.device("cuda", 0)
    d_in = torch.from_numpy(data).to(dev)
    d_comp = torch.zeros(nb * slot, dtype=torch.uint8, device=dev)
    d_back = torch.zeros(nb * B, dtype=torch.uint8, device=dev)
    offs = np.arange(nb, dtype=np.uint64) * B
    lens = np.full(nb, B, dtype=np.uint32)
    soff = np.arange(nb, dtype=np.uint64) * slot
    enc = block.DeviceBatch(offs, lens, soff, np.full(nb, slot, dtype=np.uint32), None, dev)
    dec = block.DeviceBatch(soff, lens, offs, lens, None, dev)
    enc.compress(d_in, d_comp, ctx)
    dec.in_len = enc.out_len
    dec.decompress(d_comp, d_back, ctx)
    torch.cuda.synchronize()
    assert int(enc.status.abs().sum()) == 0 and int(dec.status.abs().sum()) == 0
    assert torch.equal(d_back, d_in)
    clen = enc.out_len.cpu().numpy()
    want, wlen = _oracle_compress_all(data, nb, B, slot)
    _assert_slots_equal(d_comp.cpu().numpy(), clen, want, wlen, nb, slot)
    assert 0.22 < clen.astype(np.uint64).sum() / (nb * B) < 0.24


def test_config3_dickens_decompress(ctx):
    """BASELINE config 3 at full size (16 384 x 64 KiB): dickens tiled, compressed by the ORACLE, decompressed on the
    GPU; and the GPU encoder agrees with the oracle on every one of these blocks."""
    nb, B = 16384, 65536
    data = corpus.tiled("dickens.txt", nb * B)
    slot = 72112
    offs = np.arange(nb, dtype=np.uint64) * B
    lens = np.full(nb, B, dtype=np.uint32)
    soff = np.arange(nb, dtype=np.uint64) * slot
    comp, clen = _oracle_compress_all(data, nb, B, slot)
    out = np.zeros(nb * B, dtype=np.uint8)
    ol, st, _ = block.decompress_batch(comp, soff, clen, out, offs, lens, ctx)
    assert (ol == B).all() and np.array_equal(out, data)
    gout, goff, glen = block.compress_batch(data, offs, lens, ctx=ctx)
    assert np.array_equal(glen, clen)
    # packed GPU stream == packed oracle stream (every block)
    packed = np.concatenate([comp[b * slot: b * slot + int(clen[b])] for b in range(nb)])
    assert np.array_equal(goff[1:], np.cumsum(glen[:-1].astype(np.uint64)))
    assert np.array_equal(gout[: packed.size], packed)


def test_config5_adversarial(ctx):
    """BASELINE config 5: zero blocks (268 bytes, one offset-1 match of 65 529) interleaved with
    incompressible blocks (65 794 bytes), every zero fraction, 4 096 blocks per fraction (the size at which the
    launcher uses the thread-per-block kernels), every block compared with the oracle."""
    B, nb, slot = 65536, 4096, 72112
    for frac in (0.0, 0.25, 0.5, 0.75, 1.0):
        data = corpus.adversarial_blocks(nb, frac)
        offs = np.arange(nb, dtype=np.uint64) * B
        lens = np.full(nb, B, dtype=np.uint32)
        out, ooff, olen = block.compress_batch(data, offs, lens, ctx=ctx)
        want, wlen = _oracle_compress_all(data, nb, B, slot)
        assert np.array_equal(olen, wlen)
        zero = ~data.reshape(nb, B).any(axis=1)
        assert np.array_equal(wlen, np.where(zero, 268, 65794))
        packed = np.concatenate([want[b * slot: b * slot + int(wlen[b])] for b in range(nb)])
        assert np.array_equal(out[: packed.size], packed)
        back = np.zeros(nb * B, dtype=np.uint8)
        block.decompress_batch(out, ooff, olen, back, offs, lens, ctx)
        assert np.array_equal(back, data)


def test_host_batch_many_small_blocks_global_table_path(ctx):
    """More blocks per launch than the shared-memory-table kernel keeps in flight (24 per SM): the launcher picks the
    global-table kernel, here from two pipeline lanes at once (each lane owns its own table region).  Ragged block
    lengths around the interesting sizes; bytes identical to the oracle, exact round trip."""
    src = corpus.tiled("compression_66k_JSON.txt", 48 << 20)
    rng = np.random.default_rng(21)
    lens = rng.integers(1500, 3000, 20000).astype(np.uint32)
    lens[:64] = np.arange(64, dtype=np.uint32)                        # 0..63: tiny blocks, the n < 13 path included
    offs = np.zeros(lens.size, dtype=np.uint64)
    offs[1:] = np.cumsum(lens[:-1].astype(np.uint64))
    assert int(offs[-1]) + int(lens[-1]) <= src.size
    out, ooff, olen = block.compress_batch(src, offs, lens, ctx=ctx)
    for b in list(range(0, 64)) + list(range(64, lens.size, 397)) + [lens.size - 1]:
        a, n = int(offs[b]), int(lens[b])
        got = out[int(ooff[b]): int(ooff[b]) + int(olen[b])].tobytes()
        assert got == oracle.compress_block(src[a: a + n].tobytes()), b
    back = np.zeros(int(offs[-1]) + int(lens[-1]), dtype=np.uint8)
    ol, st, _ = block.decompress_batch(out, ooff, olen, back, offs, lens, ctx=ctx)
    assert not st.any() and np.array_equal(ol, lens)
    assert np.array_equal(back, src[: back.size])

