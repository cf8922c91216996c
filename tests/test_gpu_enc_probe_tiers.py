"""The default block encoder against the oracle on blocks aimed at its probe batch's tier boundary.

`lz4_compress_blocks_gtab<unsigned short, 7, 1, 7, 3>` loads a probe batch's candidates in two tiers, lanes 0..3 and the
rest, and decides from lanes 0..3 alone when the first of them that hits is exact (lz4b200_enc_split.cuh,
match_block_view).  The blocks of tests/probe_tiers.py put the first real hit at lanes 3, 4 and 5 (and around 2 and 8),
slot collisions across the boundary, tier-1 hits that a collision takes away, and block ends in every lane; the CPU
model counts each of those at T = 4 (test_probe_tier_model.py).  Here every block runs in all three parse modes in one
launch of that kernel, padded past 24 blocks per SM, and must equal the oracle byte for byte and round-trip through the
device decoder.  The same blocks also run unpadded, through the shared-memory-table kernel, which shares the matcher.
"""
import pytest

from probe_tiers import boundary_blocks
from test_gpu_enc_window import MODES, Case, _padded, _run
from test_gpu_launch_shapes import GTAB, SPLIT16, sm_count

CASES = [Case(data, mode, (name,)) for name, data in boundary_blocks() for mode in MODES]


@pytest.mark.gpu
def test_tier_boundary_blocks_on_the_default_encoder(ctx):
    _run(ctx, _padded(CASES, sm_count(), 31), GTAB)


@pytest.mark.gpu
def test_tier_boundary_blocks_on_the_shared_table_encoder(ctx):
    _run(ctx, CASES, SPLIT16.format(0))
