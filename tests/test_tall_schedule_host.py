"""Host-side replay of the balanced schedule of the tall-A CQT kernel (csrc/tct_kernels.cu: TallSched<true>):
the same integer arithmetic in Python, checked for the properties the kernel relies on — every (tile, chunk)
unit is visited exactly once, a tile is shared by at most two CTAs (`pairs` below counts CTAs), the one
holding a tile's LAST chunks is `reader + 1` and meets the tile as its FIRST piece (so its parked sums exist
long before the reader, which meets the tile as its LAST piece, asks for them: no cyclic wait)."""
import pytest


def pieces(pair, num_pairs, total_tiles, n_cols):
    U = total_tiles * n_cols
    u, u_end = U * pair // num_pairs, U * (pair + 1) // num_pairs
    out = []
    while u < u_end:
        tile = u // n_cols
        ci_lo = u - tile * n_cols
        rem = u_end - tile * n_cols
        ci_hi = rem if rem < n_cols else n_cols
        out.append((tile, ci_lo, ci_hi))
        u = tile * n_cols + ci_hi
    return out


@pytest.mark.parametrize("tiles,pairs,n_cols", [(463, 74, 8), (170, 74, 8), (8, 3, 8), (8, 5, 8), (75, 74, 8),
                                                (147, 74, 1), (149, 66, 4), (1000, 74, 16), (5, 5, 8), (7, 2, 3),
                                                (926, 132, 8), (29, 7, 8), (133, 132, 8)])
def test_balanced_ranges_cover_once_and_share_tiles_pairwise(tiles, pairs, n_cols):
    assert pairs <= tiles  # the launcher's condition: a range is at least one tile long
    seen = {}
    for p in range(pairs):
        ps = pieces(p, pairs, tiles, n_cols)
        for i, (tile, lo, hi) in enumerate(ps):
            assert 0 <= lo < hi <= n_cols
            assert not (lo > 0 and hi < n_cols), "a middle piece would need a three-way sum"
            if lo > 0:
                assert i == 0, "parked sums are produced by the FIRST piece of the range"
            if hi < n_cols:
                assert i == len(ps) - 1, "and consumed by the LAST piece of the neighbour's range"
            for c in range(lo, hi):
                assert (tile, c) not in seen
                seen[(tile, c)] = p
    assert len(seen) == tiles * n_cols
    for tile in range(tiles):
        owners = sorted({seen[(tile, c)] for c in range(n_cols)})
        assert len(owners) <= 2
        if len(owners) == 2:
            assert owners[1] == owners[0] + 1
            assert seen[(tile, 0)] == owners[0] and seen[(tile, n_cols - 1)] == owners[1]
    # balance: no pair carries more than one unit above the mean
    loads = [sum(hi - lo for _, lo, hi in pieces(p, pairs, tiles, n_cols)) for p in range(pairs)]
    assert max(loads) - min(loads) <= 1
