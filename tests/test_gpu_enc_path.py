"""The many-block encoder's per-sequence path (lz4_compress_blocks_gtab: match_block_view under matcher warps whose role
the compiler sees as warp-uniform) against the oracle, on every block of batches large enough to reach it.

Every batch gives each block one of the three modes (FRESH, FRESH with hash5 always, CONT) and places inputs at all 16
address residues, so candidate and cursor fetches meet every word alignment.  Contents: the bench workload (16 384
blocks of 64 KiB JSON), dickens at 16 384 blocks, zero / random mixes, every block length 0..40 and 65 533..65 536,
blocks whose last match ends at n - 6 or whose last repeat starts around the last probe position n - 12, planted
matches of 4..16 bytes at every candidate alignment 0..3 (the mismatch falls on each of the first 12 extension bytes),
and low-entropy blocks whose probe batches collide on table slots, so that in-batch forwarding (the `!exact` path) runs
in most batches.
"""
from __future__ import annotations

import numpy as np
import pytest

from lz4_flex_b200 import corpus
from test_gpu_launch_shapes import (FL_CONT, FL_FRESH_H5, GTAB, EncodeLayout, collect_encode, enqueue_encode,
                                    encode_tensors, sm_count)
from lz4_flex_b200 import block

MODES = (0, FL_FRESH_H5, FL_CONT)
B = 65536


def _with_modes(datas, seed: int):
    rng = np.random.default_rng(seed)
    out = []
    for b, d in enumerate(datas):
        out.append((bytes(d), MODES[(b + int(rng.integers(0, 3))) % 3], block.get_maximum_output_size(len(d))))
    return out


def _pad(blocks, count: int, seed: int):
    """Fill the batch up to `count` blocks (beyond 24 per SM: the global-table kernel) with short JSON blocks."""
    rng = np.random.default_rng(seed)
    j = corpus.load("compression_66k_JSON.txt")
    while len(blocks) < count:
        n = int(rng.integers(13, 4000))
        o = int(rng.integers(0, len(j) - n))
        blocks.append(j[o:o + n])
    return blocks


def _tiled(name: str, nb: int):
    data = corpus.tiled(name, nb * B)
    return [data[i * B:(i + 1) * B].tobytes() for i in range(nb)]


def _mixes(nb: int, seed: int):
    rng = np.random.default_rng(seed)
    out = []
    for b in range(nb):
        n = B if b % 2 == 0 else int(rng.integers(13, B))
        kind = b % 4
        if kind == 0:
            d = np.zeros(n, dtype=np.uint8)
        elif kind == 1:
            d = rng.integers(0, 256, n, dtype=np.uint8)
        else:                                                   # zero and random runs interleaved
            d = np.zeros(n, dtype=np.uint8)
            pos = 0
            while pos < n:
                run = int(rng.integers(1, 3000))
                if rng.random() < 0.5:
                    d[pos:pos + run] = rng.integers(0, 256, min(run, n - pos), dtype=np.uint8)
                pos += run
        out.append(d.tobytes())
    return out


def _edges(seed: int):
    rng = np.random.default_rng(seed)
    j = corpus.load("compression_66k_JSON.txt")
    out = []
    for n in list(range(41)) + [65533, 65534, 65535, 65536] * 4:
        out.append(j[:n] if n <= len(j) else (j * 2)[:n])
        out.append(rng.integers(0, 4, n, dtype=np.uint8).tobytes())
    for n in range(13, 300):
        period = int(rng.integers(1, 20))
        unit = rng.integers(0, 256, period, dtype=np.uint8)
        out.append(np.resize(unit, n).tobytes())               # one match that runs into n - 6
        for d in range(-3, 4):                                  # a repeat of the first bytes starting near n - 12
            r = rng.integers(0, 256, n, dtype=np.uint8)
            at = n - 12 + d
            if 0 < at and at + 4 <= n:
                r[at:at + min(8, n - at)] = r[:min(8, n - at)]
            out.append(r.tobytes())
    return out


def _planted(seed: int):
    """Random bytes with one earlier copy of a segment of 4..16 bytes, the copy's source at every alignment 0..3 (from
    the block start; the block's own address residue varies as well), with and without a byte of backward extension."""
    rng = np.random.default_rng(seed)
    out = []
    for L in range(4, 17):
        for align in range(4):
            for back in (False, True):
                for rep in range(3):
                    n = int(rng.integers(200, 3000))
                    r = rng.integers(0, 256, n, dtype=np.uint8)
                    c = 4 * int(rng.integers(1, 8)) + align
                    m = c + L + int(rng.integers(8, 60))
                    r[m:m + L] = r[c:c + L]
                    r[m + L] = r[c + L] ^ 0x5A                  # the match ends after exactly L bytes
                    r[m - 1] = r[c - 1] ^ (0 if back else 0xA5)  # one byte of backward extension, or none
                    out.append(r.tobytes())
    return out


def _colliding(nb: int, seed: int):
    """Low-entropy blocks: within a 32-probe batch many probes share a 4-byte value or a table slot."""
    rng = np.random.default_rng(seed)
    out = []
    for b in range(nb):
        n = int(rng.integers(100, 20000))
        alpha = 2 + b % 5
        syms = rng.integers(0, 256, alpha, dtype=np.uint8)
        out.append(syms[rng.integers(0, alpha, n)].tobytes())
    return out


def _run(ctx, blocks):
    import torch
    lay = EncodeLayout(blocks, 0)
    t = encode_tensors(lay)
    assert enqueue_encode(ctx, t, int(lay.in_len.max())) == GTAB, len(blocks)
    torch.cuda.synchronize()
    lay.check(collect_encode(t))


def _count():
    return max(4096, 24 * sm_count() + 1)


@pytest.mark.gpu
def test_bench_workload_every_block(ctx):
    _run(ctx, _with_modes(_tiled("compression_66k_JSON.txt", 16384), 1))


@pytest.mark.gpu
def test_dickens_every_block(ctx):
    _run(ctx, _with_modes(_tiled("dickens.txt", 16384), 2))


@pytest.mark.gpu
def test_zero_random_mixes(ctx):
    _run(ctx, _with_modes(_mixes(_count(), 3), 3))


@pytest.mark.gpu
def test_length_and_limit_edges(ctx):
    _run(ctx, _with_modes(_pad(_edges(4), _count(), 4), 4))


@pytest.mark.gpu
def test_short_matches_at_every_alignment(ctx):
    _run(ctx, _with_modes(_pad(_planted(5), _count(), 5), 5))


@pytest.mark.gpu
def test_colliding_probe_batches(ctx):
    _run(ctx, _with_modes(_colliding(_count(), 6), 6))
