"""CPU: the tile order of the chained launches (chain.cuh `locate`), restated in Python: it must enumerate every tile of every
phase exactly once, and every dependency must point to a tile that comes EARLIER in the list -- that is what makes the in-kernel
waits deadlock-free (all CTAs resident, every role walks the list in order)."""
import itertools

import pytest


def locate(g, num_mp, n_of, lag0, lag1):
    """Mirror of the lambda in gemm_chain_wgmma (keep the two in step); num_mp counts 128-row blocks."""
    lag0, lag1 = min(lag0, num_mp), min(lag1, num_mp)
    wave0 = num_mp * (n_of[0] + n_of[1])
    w1 = g >= wave0
    gg = g - wave0 if w1 else g
    na, nbb = (n_of[2], n_of[3]) if w1 else (n_of[0], n_of[1])
    lag = num_mp if nbb == 0 else (lag1 if w1 else lag0)
    pa = 2 if w1 else 0
    head = na * lag
    mid = (num_mp - lag) * (na + nbb)
    if gg < head:
        return pa, gg // na, gg % na
    if gg < head + mid:
        q = gg - head
        s, r = lag + q // (na + nbb), q % (na + nbb)
        return (pa, s, r) if r < na else (pa + 1, s - lag, r - na)
    q = gg - head - mid
    return pa + 1, num_mp - lag + q // nbb, q % nbb


@pytest.mark.parametrize("num_mp,n_of,lags", [
    (48, (3, 12, 3, 9), (16, 22)), (48, (3, 12, 3, 9), (0, 0)), (48, (3, 12, 3, 9), (100, 100)), (1, (3, 12, 3, 9), (16, 22)),
    (7, (3, 12, 3, 9), (16, 22)), (24, (5, 20, 5, 15), (16, 22)), (48, (3, 9, 0, 0), (16, 22)), (48, (3, 12, 3, 0), (16, 22)),
    (3, (3, 12, 3, 9), (2, 1)), (33, (4, 16, 4, 12), (5, 31))])
def test_order_is_a_permutation_with_backward_dependencies(num_mp, n_of, lags):
    total = num_mp * sum(n_of)
    seen = {}
    for g in range(total):
        ph, mp, nb = locate(g, num_mp, n_of, *lags)
        assert 0 <= ph < 4 and 0 <= mp < num_mp and 0 <= nb < n_of[ph], (g, ph, mp, nb)
        assert (ph, mp, nb) not in seen
        seen[(ph, mp, nb)] = g
    assert len(seen) == total
    # phase 1 (fc1 / qkv0) of pair mp needs LayerNorm of pair mp <- every phase-0 tile of pair mp; phase 2 (fc2) needs every
    # phase-1 tile of pair mp; phase 3 (next qkv) needs every phase-2 tile of pair mp
    for (ph, mp, nb), g in seen.items():
        if ph >= 1:
            for n in range(n_of[ph - 1]):
                assert seen[(ph - 1, mp, n)] < g, (ph, mp, nb)
