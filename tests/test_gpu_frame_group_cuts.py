"""GPU parity at the group loop's cuts: on a context with a 1 MiB frame budget a frame of 48 independent 64 KiB blocks
decodes as three groups of 16 blocks.  Errors in a later group (a block that fails to decode or to fit its slot, a bad
block checksum) and output caps at the end of the first group give the same result, field for field, and the same
bytes from the host call, the device call, the batch call (where the frame is decoded alone, since it does not fit one
group) and the streaming decoder (consumed excepted after a block decode error, where the decoder stands after the
failing block)."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from lz4_flex_b200 import _native, block, corpus, frame
from test_gpu_frame_batch_device import run_batch
from test_gpu_frame_decoder_device import Decoder, stream_decode, to_device

pytestmark = pytest.mark.gpu

BS = 65536
NB = 48
GROUP = 16                                       # blocks per group: 16 slots of 64 KiB fill the 1 MiB budget
DATA = corpus.tiled("compression_66k_JSON.txt", NB * BS).tobytes()
FLG_BLOCK, FLG_SIZE, FLG_CONTENT = 0x10, 0x08, 0x04


def assemble(payloads, flg=FLG_BLOCK | FLG_SIZE | FLG_CONTENT, bad_sum=None):
    """An independent 64 KiB-block frame of the given block payloads over DATA; block `bad_sum` gets a wrong checksum."""
    h = bytes([0x60 | flg, 4 << 4]) + (len(DATA).to_bytes(8, "little") if flg & FLG_SIZE else b"")
    out = bytearray(b"\x04\x22\x4d\x18" + h + bytes([(frame.xxh32(h) >> 8) & 0xFF]))
    for k, p in enumerate(payloads):
        out += len(p).to_bytes(4, "little") + p
        if flg & FLG_BLOCK:
            out += (frame.xxh32(p) ^ (k == bad_sum)).to_bytes(4, "little")
    out += bytes(4)
    if flg & FLG_CONTENT:
        out += frame.xxh32(DATA).to_bytes(4, "little")
    return bytes(out)


def payloads():
    return [oracle.compress_block(DATA[k * BS:(k + 1) * BS]) for k in range(NB)]


def host_next(ctx, f: bytes, cap: int):
    src = np.frombuffer(f, dtype=np.uint8)
    out = np.zeros(cap, dtype=np.uint8)
    used, w, bs, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_uint64(0), C.c_uint64(0)
    st = _native.lib().lz4b200_frame_decompress_next(ctx.handle, src.ctypes.data, src.size, out.ctypes.data, cap,
                                                     C.byref(used), C.byref(w), C.byref(bs), C.byref(e1), C.byref(e2))
    return (st, used.value, w.value, bs.value, e1.value, e2.value), out[:w.value].tobytes()


def device_next(ctx, f: bytes, cap: int):
    d_in = to_device(f)
    d_out = torch.full((cap + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    used, w, bs, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_uint64(0), C.c_uint64(0)
    st = _native.lib().lz4b200_frame_decompress_next_device(ctx.handle, d_in.data_ptr(), len(f), d_out.data_ptr(), cap,
                                                            C.byref(used), C.byref(w), C.byref(bs), C.byref(e1),
                                                            C.byref(e2), torch.cuda.current_stream().cuda_stream)
    assert bool((d_out[w.value:] == 0xA5).all()), "bytes past written were modified"
    return (st, used.value, w.value, bs.value, e1.value, e2.value), d_out[:w.value].cpu().numpy().tobytes()


@pytest.fixture(scope="module")
def small_ctx():
    c = block.Context(0)
    _native.lib().lz4b200_ctx_set_frame_budget(c.handle, 1 << 20)
    yield c
    c.close()


def check_all(ctx, f: bytes, cap: int, stream: bool = True):
    """Every decoder against the host call; returns the host result."""
    want = host_next(ctx, f, cap)
    assert device_next(ctx, f, cap) == want
    small = oracle.frame_compress(DATA[:1000], 4, oracle.F_CONTENT_CHECKSUM)
    got = run_batch(ctx, [small, f, small], [1000, cap, 1000], seed=3)
    assert got[1] == want and got[0][0][0] == got[2][0][0] == 0
    if stream:
        dec = Decoder(ctx)
        try:
            for out_cap in (BS, 1 << 20):
                data, r, consumed, _ = stream_decode(dec, f, [len(f)], lambda _: out_cap)
                assert data == want[1] and r[1] == consumed
                if want[0][0] == 101:                       # FRAME_DECOMPRESSION_ERROR: consumed is the decoder's own
                    assert r[0] == 101 and r[2:] == want[0][2:]
                else:
                    assert r == want[0]
        finally:
            dec.close()
    return want[0]


def test_decode_error_opens_second_group(small_ctx):
    p = payloads()
    p[GROUP] = b"\xff" * len(p[GROUP])                     # literal-length bytes that run past the payload
    r = check_all(small_ctx, assemble(p), len(DATA))
    assert r[0] == 101 and r[2] == GROUP * BS and r[3] != 0


def test_output_too_small_in_later_group(small_ctx):
    p = payloads()
    p[GROUP + 4] = oracle.compress_block(DATA[:2 * BS])   # decodes to twice the block size
    r = check_all(small_ctx, assemble(p), len(DATA))
    assert r[0] == 101 and r[3] == 2 and r[2] == (GROUP + 4) * BS and r[5] == BS   # DEC_OUTPUT_TOO_SMALL


def test_bad_checksum_opens_third_group(small_ctx):
    r = check_all(small_ctx, assemble(payloads(), bad_sum=2 * GROUP), len(DATA))
    assert r[0] == 107 and r[2] == 2 * GROUP * BS                                  # BLOCK_CHECKSUM


@pytest.mark.parametrize("extra", [0, 1])
def test_cap_at_first_group_end(small_ctx, extra):
    f = assemble(payloads())
    assert check_all(small_ctx, f, len(DATA))[0] == 0
    r = check_all(small_ctx, f, GROUP * BS + extra, stream=False)
    assert r[0] == 115 and r[2] == GROUP * BS                                      # OUTPUT_FULL
