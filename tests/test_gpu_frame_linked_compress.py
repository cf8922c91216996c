"""GPU parity of the linked batch frame encoder: lz4b200_frame_compress_linked_batch_device (frame.compress_linked_frames_device)
writes, for every input of a batch, the BlockMode::Linked frame the linked-frame reference (tests/cpp/linked_frame_ref.c:
lz4_flex's FrameEncoder with linked blocks, restated in C) writes for the same bytes, frames back to back with their offsets.  Every frame made here also decodes back to its input
through frame.decompress_frames_device, and through frame.index_frames_device with frame.decompress_frames_ranges_device;
the one frame past 2 GiB is decoded by the C oracle.
Covered: the corpora at every block size and flag set, lengths at the block and window edges, planted matches at the
ext_dict / prefix boundaries and the 64 KiB window edge, a stored block mid-chain, thousands of mixed frames, a frame past
the table reposition, and the order of argument errors."""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import linked_ref
import oracle
from lz4_flex_b200 import _native, corpus, frame
from lz4_flex_b200.frame import BlockMode, BlockSize, FrameInfo

pytestmark = pytest.mark.gpu

ALL = oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM | oracle.F_CONTENT_SIZE
FLAGS = {"none": 0, "block": oracle.F_BLOCK_CHECKSUMS, "content": oracle.F_CONTENT_CHECKSUM,
         "content_size": oracle.F_CONTENT_SIZE, "all": ALL}
BLOCK_SIZES = [BlockSize.Auto, BlockSize.Max64KB, BlockSize.Max256KB, BlockSize.Max1MB, BlockSize.Max4MB]
INVALID, TOO_SMALL = 200, 1
SENTINEL, UNSET = 0xA5, -7


def info_of(bs, flags: int) -> FrameInfo:
    return FrameInfo(block_size=BlockSize(int(bs)), block_mode=BlockMode.Linked,
                     block_checksums=bool(flags & oracle.F_BLOCK_CHECKSUMS),
                     content_checksum=bool(flags & oracle.F_CONTENT_CHECKSUM),
                     content_size=0 if flags & oracle.F_CONTENT_SIZE else None)


def noise(n: int, seed: int) -> bytes:
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def pack(datas, seed=0):
    """The inputs in one device buffer, each after an odd gap (most start unaligned)."""
    gaps = np.random.default_rng(seed).integers(0, 16, size=len(datas))
    offs, pos = [], 0
    for d, g in zip(datas, gaps):
        pos += int(g)
        offs.append(pos)
        pos += len(d)
    host = np.zeros(pos + 16, dtype=np.uint8)
    for d, o in zip(datas, offs):
        host[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
    return torch.from_numpy(host).cuda(), np.array(offs, dtype=np.int64), np.array([len(d) for d in datas], np.int64)


def check_decodes(ctx, out, offs, datas):
    """Every frame decodes to its input through the batch decoder, and through the index + range decoder."""
    offs_h = offs.cpu().numpy()
    starts, lens = offs_h[:-1], np.diff(offs_h)
    dec = frame.decompress_frames_device(out, starts, lens, ctx=ctx)
    for i, d in enumerate(datas):
        got, consumed, err = dec.frame(i)
        assert err is None and consumed == lens[i], (i, err)
        assert got.cpu().numpy().tobytes() == d, f"frame {i} does not decode to its input"
    idx = frame.index_frames_device(out, starts, lens, ctx=ctx)
    rng = np.random.default_rng(len(datas))
    fr, st, ln = [], [], []
    for i, d in enumerate(datas):
        fr.append(i); st.append(0); ln.append(len(d))                  # the whole content
        if len(d) > 2:
            a = int(rng.integers(0, len(d)))
            fr.append(i); st.append(a); ln.append(int(rng.integers(1, 70000)))
    got, got_off, written = frame.decompress_frames_ranges_device(out, idx, fr, st, ln, ctx=ctx)
    g, go, w = got.cpu().numpy(), got_off.cpu().numpy(), written.cpu().numpy()
    for j, (i, a, n) in enumerate(zip(fr, st, ln)):
        assert g[go[j]:go[j] + w[j]].tobytes() == datas[i][a:a + n], (j, i, a, n)


def run(ctx, datas, bs, flags, decode=True, seed=0):
    d_in, off, lens = pack(datas, seed)
    out, offs = frame.compress_linked_frames_device(d_in, off, lens, info_of(bs, flags), ctx=ctx)
    torch.cuda.synchronize()
    host = out.cpu().numpy().tobytes()
    o = offs.cpu().numpy()
    want_sizes = []
    for i, d in enumerate(datas):
        want = linked_ref.frame_compress(d, int(bs), flags)
        assert host[o[i]:o[i + 1]] == want, f"frame {i} ({len(d)} bytes, bs {bs}, flags {flags}) differs from the reference"
        want_sizes.append(len(want))
    assert o[0] == 0 and (o[1:] == np.cumsum(want_sizes)).all()
    if len(lens) and lens.max() > 0:
        assert _native.lib().lz4b200_ctx_last_kernel(ctx.handle, 0) == b"lz4_compress_frames_linked"
    if decode:
        check_decodes(ctx, out, offs, datas)
    return out, offs


@pytest.fixture(scope="module")
def corpora():
    dk = corpus.load("dickens.txt")
    return [corpus.tiled("compression_66k_JSON.txt", 1_500_000).tobytes(), dk[:1_800_000],
            corpus.load("hdfs.json")[:1_200_000], corpus.load("compression_34k.txt"), corpus.load("compression_1k.txt"),
            b"", noise(300_000, 1)]


@pytest.mark.parametrize("flags", list(FLAGS.values()), ids=list(FLAGS))
@pytest.mark.parametrize("bs", BLOCK_SIZES, ids=[b.name for b in BLOCK_SIZES])
def test_corpora(ctx, corpora, bs, flags):
    run(ctx, corpora, bs, flags)


@pytest.mark.parametrize("bs", BLOCK_SIZES[1:], ids=[b.name for b in BLOCK_SIZES[1:]])
def test_edge_lengths(ctx, bs):
    b = bs.get_size()
    lens = [0, 1, 12, 13, b - 1, b, b + 1, 2 * b, 2 * b + 65535, 2 * b + 65536, 2 * b + 65537]
    src = corpus.tiled("compression_66k_JSON.txt", max(lens)).tobytes()
    run(ctx, [src[:n] for n in lens], bs, ALL)


def planted(bs: int) -> list:
    rng = np.random.default_rng(5)
    out = []
    # a period shorter than 64 KiB over five blocks: matches into block 1 are cut at block 2's start (ext_dict),
    # matches into block 2 from block 3 are not (prefix)
    per = noise(3001, 2)
    out.append((per * (5 * bs // len(per) + 2))[:5 * bs - 77])
    # 32-byte islands copied exactly 65 535 and 65 536 bytes later, across the boundaries 0|1, 1|2 and 2|3
    base = bytearray(noise(4 * bs + 100, 3))
    for edge in (bs, 2 * bs, 3 * bs):
        for dist in (65535, 65536):
            at = edge + 40 + (dist - 65535) * 200
            base[at:at + 32] = base[at - dist:at - dist + 32]
    out.append(bytes(base))
    # an incompressible block mid-chain, then a block that matches into it
    txt = corpus.tiled("compression_66k_JSON.txt", bs).tobytes()
    nz = noise(bs, 4)
    out.append(txt + nz + nz[-60000:] + nz[:bs - 60000] + txt[:5000])
    # a final block under 13 bytes
    out.append(txt + txt[:bs] + b"tail-bytes!")
    out.append(bytes(rng.integers(0, 4, 3 * bs + 12, dtype=np.uint8)))
    return out


@pytest.mark.parametrize("bs", BLOCK_SIZES[1:3], ids=[b.name for b in BLOCK_SIZES[1:3]])
def test_planted(ctx, bs):
    for flags in (0, ALL):
        run(ctx, planted(bs.get_size()), bs, flags)


def test_many_mixed_frames(ctx):
    """A few thousand frames of mixed lengths, empty ones included, Auto block size: each frame picks its own."""
    rng = np.random.default_rng(9)
    src = corpus.load("dickens.txt")
    lens = np.where(rng.random(3000) < 0.9, rng.integers(0, 20000, 3000), rng.integers(0, 600_000, 3000))
    lens[rng.random(3000) < 0.05] = 0
    starts = rng.integers(0, len(src) - 600_000, 3000)
    datas = [src[s:s + n] for s, n in zip(starts, lens)]
    run(ctx, datas, BlockSize.Auto, oracle.F_CONTENT_SIZE | oracle.F_CONTENT_CHECKSUM)


def test_past_reposition(ctx):
    """One frame of 2^31 + 3 x 4 MiB + 12 345 bytes in 4 MiB blocks: the table is repositioned before block 512, where
    the stream offset reaches 2^31 (frame/compress.rs:266-271).  The input is a text period with a noise byte every
    ~1 MiB, so the chain and the CPU reference stay fast.  On an H100 80GB HBM3 at 700 W the chain took 23 s and
    the whole test about 30 s."""
    bs = BlockSize.Max4MB
    n = (1 << 31) + 3 * bs.get_size() + 12345
    per = np.frombuffer(corpus.load("compression_34k.txt")[:4099], dtype=np.uint8)
    host = np.resize(per, n)
    rng = np.random.default_rng(13)
    at = rng.integers(0, n, n >> 20)
    host[at] = rng.integers(0, 256, at.size, dtype=np.uint8)
    data = host.tobytes()
    d_in = torch.from_numpy(host).cuda()
    del host
    t0 = time.perf_counter()
    out, offs = frame.compress_linked_frames_device(d_in, [0], [n], info_of(bs, ALL), ctx=ctx)
    torch.cuda.synchronize()
    print(f"\n{n} bytes: GPU chain {time.perf_counter() - t0:.1f} s", end="")
    t0 = time.perf_counter()
    want = linked_ref.frame_compress(data, int(bs), ALL)
    print(f", reference {time.perf_counter() - t0:.1f} s")
    assert out.cpu().numpy().tobytes() == want
    assert offs.cpu().tolist() == [0, len(want)]
    # the decode goes through the C oracle: the device decoders are not run on a linked frame past 2 GiB here
    st, back, _ = oracle.frame_decompress(want, n)
    assert st == 0 and back == data
    del d_in, out
    torch.cuda.empty_cache()


def test_argument_errors_in_order(ctx):
    js = corpus.tiled("compression_66k_JSON.txt", 100000).tobytes()
    datas = [js, b"", js[:70000]]
    info = info_of(BlockSize.Max64KB, ALL)
    lib = _native.lib()
    d_in, off, lens = pack(datas)
    need = sum(lib.lz4b200_frame_bound(len(d), C.byref(info.to_c())) for d in datas)

    def status(finfo=info, cap=None, **override):
        cap = need if cap is None else cap
        buf = torch.full((cap + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
        d_off = torch.full((len(datas) + 1,), UNSET, dtype=torch.int64, device="cuda")
        ci = finfo.to_c()
        a = dict(ctx=ctx.handle, d_in=d_in.data_ptr(), in_off=off.ctypes.data, in_len=lens.ctypes.data, info=C.byref(ci),
                 d_out=buf.data_ptr(), out_cap=cap, d_frame_off=d_off.data_ptr(), nframes=len(datas),
                 stream=torch.cuda.current_stream().cuda_stream)
        a.update(override)
        st = lib.lz4b200_frame_compress_linked_batch_device(*a.values())
        torch.cuda.synchronize()
        if st != 0:
            assert (buf.cpu().numpy() == SENTINEL).all() and (d_off.cpu().numpy() == UNSET).all()
        return st, buf, d_off

    independent = FrameInfo(block_size=BlockSize.Max64KB)
    assert status(ctx=None)[0] == INVALID
    assert status(info=None)[0] == INVALID
    assert status(d_frame_off=None)[0] == INVALID
    for k in ("in_off", "in_len", "d_out"):
        assert status(**{k: None})[0] == INVALID, k
    assert status(d_in=None)[0] == INVALID
    assert status(independent)[0] == INVALID                        # where the independent call says LINKED_UNSUPPORTED
    ci = independent.to_c()
    ci.block_size_id = 3
    assert status(independent, info=C.byref(ci))[0] == INVALID
    for bad in (1, 3, 8):
        ci = info.to_c()
        ci.block_size_id = bad
        assert status(info=C.byref(ci), out_cap=0)[0] == INVALID, bad   # the block size before the capacity
    assert status(nframes=1 << 32, out_cap=0)[0] == INVALID
    huge = np.array([1 << 47, 1 << 47], dtype=np.int64)
    zeros = np.zeros(3, dtype=np.int64)
    assert status(in_len=huge.ctypes.data, in_off=zeros.ctypes.data, nframes=2, out_cap=0)[0] == INVALID
    assert status(cap=need - 1)[0] == TOO_SMALL
    st, buf, d_off = status()
    assert st == 0
    o = d_off.cpu().numpy()
    b = buf.cpu().numpy()
    for i, d in enumerate(datas):
        assert b[o[i]:o[i + 1]].tobytes() == linked_ref.frame_compress(d, 4, ALL)
    assert (b[o[-1]:] == SENTINEL).all()
    assert status(nframes=0)[0] == 0
    with pytest.raises(ValueError):
        frame.compress_linked_frames_device(d_in, off, lens, independent, ctx=ctx)
