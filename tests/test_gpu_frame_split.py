"""GPU tests of concatenated frames in device memory: split_frames_device (lz4b200_frame_split_device) finds exactly the
frames the batch encoders packed back to back; decompress_frame_device (lz4b200_frame_decompress_device) gives what a
loop of decompress_next_frame_device gives (bytes, exception type and fields) on every input of the CPU tests, at
misaligned bases and with the output one byte short of each frame boundary; decoded_bound_device equals the host
bound; the split runs inside a CUDA graph; and its regions feed the batch index and range reads."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import split_cases
from lz4_flex_b200 import _native, corpus, frame

pytestmark = pytest.mark.gpu


def dev(b: bytes, shift: int = 0):
    """b as a CUDA uint8 tensor whose first byte sits `shift` bytes past an aligned allocation."""
    t = torch.zeros(len(b) + shift, dtype=torch.uint8, device="cuda")
    if b:
        t[shift:] = torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
    return t[shift:]


def err_key(e):
    if e is None:
        return None
    inner = e.args[0] if e.args and isinstance(e.args[0], Exception) else None
    return (type(e).__name__, str(e), getattr(e, "expected", None), getattr(e, "actual", None),
            None if inner is None else (type(inner).__name__, str(inner)))


def loop_decode(d_in, out, ctx):
    """The serial loop: decompress_next_frame_device at d_in + consumed into out + written."""
    pos, total = 0, 0
    while pos < d_in.numel():
        used, w, err = frame.decompress_next_frame_device(d_in[pos:], out[total:], ctx)
        total += w
        if err is not None:
            return out[:total].cpu().numpy().tobytes(), err
        if used == 0:
            break
        pos += used
    return out[:total].cpu().numpy().tobytes(), None


def new_decode(d_in, out, ctx, delivered=None):
    """(decoded bytes, exception or None).  On an exception the bytes are out[:delivered]: the partial output, which
    the caller knows from the loop."""
    try:
        return frame.decompress_frame_device(d_in, out, ctx).cpu().numpy().tobytes(), None
    except Exception as e:                                              # noqa: BLE001 - compared field by field
        return out[:delivered].cpu().numpy().tobytes(), e


def host_bound(b: bytes) -> int:
    src = np.frombuffer(b, np.uint8)
    bound = C.c_size_t(0)
    assert _native.lib().lz4b200_frame_decoded_bound(src.ctypes.data if len(b) else None, len(b), C.byref(bound)) == 0
    return bound.value


@pytest.fixture(scope="module")
def cases():
    return split_cases.cases()


def regions_of(sp):
    torch.cuda.synchronize()
    k, covered = (int(v) for v in sp.counts.cpu())
    return list(zip(sp.offsets[:k].cpu().tolist(), sp.lengths[:k].cpu().tolist())), covered


def test_split_matches_the_serial_loop(ctx, cases):
    for name, b in cases.items():
        for shift in (0, 3):
            regs, covered = regions_of(frame.split_frames_device(dev(b, shift), ctx=ctx))
            assert regs == split_cases.regions(b) and covered == len(b), (name, shift)
    regs, covered = regions_of(frame.split_frames_device(dev(b""), ctx=ctx))
    assert regs == [] and covered == 0
    b = cases["mixed"]
    R = len(split_cases.regions(b))
    for mf in (0, 1, R - 1, R, R + 1):
        regs, covered = regions_of(frame.split_frames_device(dev(b), max_frames=mf, ctx=ctx))
        assert regs == split_cases.regions(b)[:mf], mf
    regs, _ = regions_of(frame.split_frames_device(dev(cases["nested_frames"]), max_candidates=2, ctx=ctx))
    assert regs == split_cases.regions(cases["nested_frames"])               # the serial fallback


def test_split_finds_the_batch_encoders_frames(ctx):
    rng = np.random.default_rng(5)
    j = corpus.tiled("compression_66k_JSON.txt", 24 << 20)
    sizes = rng.integers(0, 20000, 3000)
    sizes[::97] = rng.integers(100000, 300000, sizes[::97].size)
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]) % (j.size - 300000)
    d_j = torch.from_numpy(j.copy()).cuda()
    info = frame.FrameInfo(block_size=frame.BlockSize.Max64KB, content_checksum=True)
    for fn in (frame.compress_frames_device, frame.compress_linked_frames_device):
        fi = frame.FrameInfo(block_size=frame.BlockSize.Max64KB, content_checksum=True,
                             block_mode=frame.BlockMode.Linked) if fn is frame.compress_linked_frames_device else info
        out, fo = fn(d_j, offs, sizes, fi, ctx=ctx)
        fo = fo.cpu().numpy()
        sp = frame.split_frames_device(out, ctx=ctx)
        regs, covered = regions_of(sp)
        assert covered == out.numel()
        assert [r[0] for r in regs] == fo[:-1].tolist()
        assert [r[1] for r in regs] == np.diff(fo).tolist()


def test_decompress_matches_the_loop(ctx, cases):
    for name, b in cases.items():
        bound = max(host_bound(b), 1)
        for shift in (0, 1, 2, 3):
            d_in = dev(b, shift)
            want, werr = loop_decode(d_in, torch.zeros(bound, dtype=torch.uint8, device="cuda"), ctx)
            got, gerr = new_decode(d_in, torch.zeros(bound, dtype=torch.uint8, device="cuda"), ctx, len(want))
            assert err_key(gerr) == err_key(werr), (name, shift)
            assert got == want, (name, shift)                           # the partial output too, on an error
            if shift == 0 and gerr is None:
                assert frame.decompress_frame_device(d_in, ctx=ctx).cpu().numpy().tobytes() == want


def test_output_one_byte_short_of_each_boundary(ctx, cases):
    for name in ("small_frames", "mixed", "linked_golden", "empty_frames"):
        b = cases[name]
        d_in = dev(b, 1)
        ends, total = [], 0
        for p, ln in split_cases.regions(b)[:40]:
            _, w, _ = frame.decompress_next_frame_device(d_in[p:p + ln], torch.empty(max(host_bound(b[p:p + ln]), 1),
                                                         dtype=torch.uint8, device="cuda"), ctx)
            total += w
            ends.append(total)
        for cap in sorted({e - 1 for e in ends if e > 0}):
            want, werr = loop_decode(d_in, torch.zeros(cap, dtype=torch.uint8, device="cuda"), ctx)
            out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
            got, gerr = new_decode(d_in, out, ctx, len(want))
            assert werr is not None and err_key(gerr) == err_key(werr), (name, cap)
            assert got == want, (name, cap)


def test_context_counts_the_split_scratch(cases):
    """The split's scratch, which a decode of several frames leaves on the context, is in lz4b200_ctx_device_bytes."""
    from lz4_flex_b200 import block
    c = block.Context(0)
    b = cases["mixed"]
    L = _native.lib()
    before = L.lz4b200_ctx_device_bytes(c.handle)
    frame.decompress_frame_device(dev(b), ctx=c)
    n = len(b) - split_cases.regions(b)[1][0]
    grown = L.lz4b200_ctx_device_bytes(c.handle) - before
    assert grown >= L.lz4b200_frame_split_device_scratch(n, frame.default_max_candidates(n))
    c.close()


def test_decoded_bound_matches_host(ctx, cases):
    for name, b in list(cases.items()) + [("nothing", b"")]:
        assert frame.decoded_bound_device(dev(b, 2), ctx) == host_bound(b), name


def test_ten_thousand_small_frames_round_trip(ctx):
    rng = np.random.default_rng(11)
    j = corpus.tiled("compression_66k_JSON.txt", 4 << 20).tobytes()
    parts, frames = [], []
    for i in range(12000):
        a = int(rng.integers(0, len(j) - 2000))
        d = j[a:a + int(rng.integers(0, 1500))]
        parts.append(d)
        frames.append(oracle.frame_compress(d, 4, i % 8))
    b = b"".join(frames)
    assert frame.decompress_frame_device(dev(b, 1), ctx=ctx).cpu().numpy().tobytes() == b"".join(parts)
    regs, _ = regions_of(frame.split_frames_device(dev(b), ctx=ctx))
    assert len(regs) == 12000


def test_cuda_graph_split_bound_decode(ctx):
    """split -> per-region bound -> cumsum -> sync-free batch decode, captured once and replayed after the input buffer
    is overwritten with another concatenation of the same length."""
    j = corpus.tiled("compression_66k_JSON.txt", 2 << 20).tobytes()

    def concat(seed):
        r = np.random.default_rng(seed)
        parts, frames = [], []
        while sum(map(len, frames)) < 150000:
            a = int(r.integers(0, len(j) - 40000))
            d = j[a:a + int(r.integers(0, 40000))]
            parts.append(d)
            frames.append(oracle.frame_compress(d, 4, int(r.integers(0, 8))))
        return b"".join(frames), b"".join(parts)

    (b1, p1), (b2, p2) = concat(1), concat(2)
    r = np.random.default_rng(4)
    while not 15 <= abs(len(b1) - len(b2)) <= 60000:                # grow the shorter one until a filler fits
        a = int(r.integers(0, len(j) - 20000))
        d = j[a:a + 20000]
        if len(b1) <= len(b2):
            b1, p1 = b1 + oracle.frame_compress(d, 4, 0), p1 + d
        else:
            b2, p2 = b2 + oracle.frame_compress(d, 4, 0), p2 + d
    junk = r.integers(0, 256, abs(len(b1) - len(b2)) - 15, dtype=np.uint8).tobytes()
    filler = oracle.frame_compress(junk, 4, 0)                       # one stored block: 15 + len(junk) bytes
    if len(b1) < len(b2):
        b1, p1 = b1 + filler, p1 + junk
    else:
        b2, p2 = b2 + filler, p2 + junk
    n = len(b1)
    assert len(b2) == n and b1 != b2
    out_cap = max(host_bound(b1), host_bound(b2))
    d_in = torch.zeros(n, dtype=torch.uint8, device="cuda")
    out = torch.zeros(out_cap + (1 << 20), dtype=torch.uint8, device="cuda")
    maxf = frame.default_max_candidates(n) + 1
    L = _native.lib()

    def call():
        sp = frame.split_frames_device(d_in, ctx=ctx)
        # only regions below counts[0] are frames: the rest are masked to empty regions on the device before any call
        # reads them (split_frames_device also leaves them empty)
        live = torch.arange(maxf, device="cuda") < sp.counts[0]
        lens = torch.where(live, sp.lengths, torch.zeros_like(sp.lengths))
        offs = torch.where(live, sp.offsets, torch.zeros_like(sp.offsets))
        bound = torch.zeros(maxf, dtype=torch.int64, device="cuda")
        L.lz4b200_frame_decoded_bound_batch_device(ctx.handle, d_in.data_ptr(), offs.data_ptr(), lens.data_ptr(),
                                                   bound.data_ptr(), maxf, torch.cuda.current_stream().cuda_stream)
        ends = torch.cumsum(bound, 0)
        r = frame.decompress_frames_device_async(d_in, offs, lens, out, ends - bound, bound, ctx=ctx)
        return sp, r

    d_in.copy_(dev(b1))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="global"):
        sp, r = call()
    for b, p in ((b2, p2), (b1, p1), (b2, p2)):
        d_in.copy_(dev(b))
        g.replay()
        torch.cuda.synchronize()
        k = int(sp.counts[0])
        assert k == len(split_cases.regions(b))
        assert not sp.offsets[k:].any() and not sp.lengths[k:].any()
        res = r.results[:k].cpu().numpy()
        assert (res[:, 4] == 0).all()
        oo = r.out_offsets[:k].cpu().numpy()
        got = b"".join(out[int(o):int(o) + int(w)].cpu().numpy().tobytes() for o, w in zip(oo, res[:, 1]))
        assert got == p


def test_index_and_ranges_over_split_regions(ctx, cases):
    b = cases["mixed"] + cases["linked_golden"]
    d_in = dev(b, 2)
    full = frame.decompress_frame_device(d_in, ctx=ctx).cpu().numpy().tobytes()
    sp = frame.split_frames_device(d_in, ctx=ctx)
    k = int(sp.counts[0])
    idx = frame.index_frames_device(d_in, sp.offsets[:k], sp.lengths[:k], ctx=ctx)
    content = idx.content_lens()
    starts_of = np.concatenate([[0], np.cumsum(content)[:-1]])
    assert int(content.sum()) == len(full)
    rng = np.random.default_rng(8)
    fr = rng.integers(0, k, 300)
    st = np.array([int(rng.integers(0, max(int(content[f]), 1))) for f in fr])
    ln = rng.integers(0, 100000, 300)
    out, oo, written = frame.decompress_frames_ranges_device(d_in, idx, fr, st, ln, ctx=ctx)
    oo, written = oo.cpu().numpy(), written.cpu().numpy()
    for i in range(300):
        a = int(starts_of[fr[i]]) + int(st[i])
        want = full[a:a + min(int(ln[i]), int(content[fr[i]]) - int(st[i]))]
        assert out[int(oo[i]):int(oo[i]) + int(written[i])].cpu().numpy().tobytes() == want, i
