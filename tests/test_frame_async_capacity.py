"""The default block capacity of decompress_frames_device_async, in_len // 256 + nframes, holds for every frame written
with full blocks: no block of 64 KiB (the smallest block size) compresses below 256 bytes with its BlockInfo word, so a
frame of k bytes holds at most k // 256 full blocks and one short last block.  Pinned with the oracle's encoder on the
most compressible inputs; frames flushed with short blocks can pass it, as the docstring says."""
import numpy as np
import pytest

import oracle
from lz4_flex_b200 import corpus, frame
from stream_frames import linked_frame

BS = {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20}


def _inputs(n):
    j = corpus.tiled("compression_66k_JSON.txt", n).tobytes()
    return {"zeros": bytes(n), "one byte": b"\xab" * n, "period 2": b"ab" * (n // 2) + b"a" * (n % 2),
            "period 4": (b"abcd" * (n // 4 + 1))[:n], "json": j, "random": corpus.xorshift64star_bytes(n).tobytes()}


def test_densest_block_takes_256_bytes():
    for name, d in _inputs(BS[4]).items():
        assert len(oracle.compress_block(d)) + 4 >= 256, name


@pytest.mark.parametrize("bsid", sorted(BS))
@pytest.mark.parametrize("flags", [0, oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM | oracle.F_CONTENT_SIZE])
def test_default_capacity_holds_full_block_frames(bsid, flags):
    bs = BS[bsid]
    nblocks = {4: 64, 5: 16, 6: 5, 7: 3}[bsid]
    for extra in (0, 1, bs // 2):
        n = nblocks * bs + extra
        frames, blocks = [], []
        for name, d in _inputs(n).items():
            f = oracle.frame_compress(d, bsid, flags)
            k = -(-n // bs)
            assert frame.default_max_blocks(len(f), 1) >= k, (name, len(f), k)
            frames.append(f)
            blocks.append(k)
        assert frame.default_max_blocks(sum(len(f) for f in frames), len(frames)) >= sum(blocks)


def test_default_capacity_holds_linked_frames():
    """Linked blocks compressed with the 64 KiB before them as dictionary: still no block below 256 bytes."""
    for name, d in _inputs(40 * BS[4] + 1000).items():
        f = linked_frame(d, [BS[4]], 4, True, True, True)
        assert frame.default_max_blocks(len(f), 1) >= 41, name


def test_flushed_frames_can_pass_it():
    d = bytes(200000)
    f = oracle.frame_compress(d, 4, 0, 1000)                             # a block per 1000 bytes of zeros
    assert frame.default_max_blocks(len(f), 1) < 200
    assert np.ceil(len(d) / 1000) == 200
