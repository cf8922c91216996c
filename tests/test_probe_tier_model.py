"""The block encoder's probe batch with its candidates in two tiers (tests/probe_tiers.py) against the sequential parse.

The kernel decides a batch from lanes 0..T-1's candidates whenever the first of them that hits is exact, and reads the
other lanes' candidates only otherwise.  These tests run that scheme lane by lane in plain Python, with tier 2 unknown
until it is read, and require the oracle's bytes in all three parse modes (block API, frame FRESH, frame CONT) at
T = 2, 4 and 8: on the corpus, on adversarial streams, and on the seeded blocks that the GPU test aims at the boundary.
The kernel itself runs T = 4 (tests/test_gpu_enc_probe_tiers.py).
"""
import numpy as np
import pytest

import oracle
from lz4_flex_b200 import corpus
from probe_tiers import G, boundary_blocks, tiered_encode

TIERS = (2, 4, 8)


def _corpus_cases():
    rng = np.random.default_rng(11)
    cases = [(f, corpus.load(f)) for f in ("compression_1k.txt", "compression_34k.txt", "compression_65k.txt")]
    cases.append(("json_block", corpus.tiled("compression_66k_JSON.txt", 65536).tobytes()))
    cases.append(("zeros", bytes(20000)))
    cases.append(("period7", (b"abcdefg" * 3000)[:20000]))
    for k in range(6):
        a = int(rng.integers(2, 6))
        cases.append((f"low_entropy_{k}", rng.integers(0, a, int(rng.integers(13, 6000)), dtype=np.uint8).tobytes()))
    cases.append(("random", rng.integers(0, 256, 5000, dtype=np.uint8).tobytes()))
    for n in (0, 1, 12, 13, 14, 20, 64):
        cases.append((f"tiny_{n}", (b"xyxyzxyxyz" * 10)[:n]))
    return cases


CASES = _corpus_cases()
BOUNDARY = boundary_blocks()


def _all_modes(data: bytes, T: int, stats=None):
    assert tiered_encode(data, T, stats=stats) == oracle.compress_block(data)
    assert tiered_encode(data, T, cont=True, h5=True, stats=stats) == oracle.compress_block_cont(data)
    assert tiered_encode(data, T, cont=False, h5=True, stats=stats) == oracle.compress_block_fresh_h5(data)


@pytest.mark.parametrize("T", TIERS)
@pytest.mark.parametrize("name,data", CASES, ids=[c[0] for c in CASES])
def test_tiered_probe_equals_sequential_parse(name, data, T):
    _all_modes(data, T)


@pytest.mark.parametrize("T", TIERS)
def test_boundary_blocks_keep_the_parse_and_reach_every_case(T):
    st = {}
    for name, data in BOUNDARY:
        _all_modes(data, T, st)
    fh = st["first_hit"]
    for k in (T - 1, T, T + 1):                                  # first real hit just before, at and after the boundary
        assert fh[k] >= 20, (k, fh[: 2 * T + 2])
    assert st["straddle"] >= 20, st
    assert st["invalidated"] >= (10 if T >= 4 else 1), st           # at T = 2 only lane 1 can lose its hit
    assert st["end_in_tier2"] >= 10, st
    assert st["tier1_decided"] >= 1000 and st["tier2_read"] >= 1000, st


def test_tier1_decides_most_json_batches():
    """The point of the tiers: on JSON most batches never need lanes 4..31's candidates."""
    data = corpus.tiled("compression_66k_JSON.txt", 65536).tobytes()
    st = {}
    assert tiered_encode(data, 4, h5=True, stats=st) == oracle.compress_block_fresh_h5(data)
    assert st["tier1_decided"] > 0.8 * st["batches"], st
    assert sum(st["first_hit"][:4]) + st["tier2_read"] >= st["batches"]


def test_first_hits_spread_over_all_lanes():
    """The batched scheme is only exercised if winners reach deep lanes too (a no-hit batch counts at lane 32)."""
    st = {}
    for name, data in BOUNDARY[:20]:
        tiered_encode(data, 4, stats=st)
    fh = st["first_hit"]
    assert sum(1 for w in range(G) if fh[w]) >= 16, fh
