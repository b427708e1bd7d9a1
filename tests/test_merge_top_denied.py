"""merge_top_denied: the global top k of per-rank top-denied lists (no GPU needed)."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from throttlecrab_b200.sharded import merge_top_denied  # noqa: E402


def test_merge_orders_by_count_then_hash():
    a = [(50, 9), (7, 3), (3, 1)]
    b = [(40, 9), (8, 3), (2, 2)]
    assert merge_top_denied([a, b], 10) == [(40, 9), (50, 9), (7, 3), (8, 3), (2, 2), (3, 1)]
    assert merge_top_denied([a, b], 3) == [(40, 9), (50, 9), (7, 3)]       # k cuts through a tie: smaller hash first
    assert merge_top_denied([a, [], b], 0) == []
    assert merge_top_denied([], 5) == []


def test_merge_of_each_ranks_top_k_is_the_global_top_k():
    import random
    rng = random.Random(7)
    keys = sorted({rng.getrandbits(64) | 1 for _ in range(2000)})
    counts = {k: rng.randint(1, 30) for k in keys}
    ranks = [[k for k in keys if (k >> 1) % 3 == r] for r in range(3)]

    def top(ks, k):
        return sorted(((h, counts[h]) for h in ks), key=lambda hc: (-hc[1], hc[0]))[:k]
    for k in (1, 17, 100, 1999, 2000, 2500):
        assert merge_top_denied([top(r, k) for r in ranks], k) == top(keys, k)


def test_a_key_on_two_ranks_is_an_error():
    with pytest.raises(ValueError):
        merge_top_denied([[(5, 1)], [(5, 2)]], 2)
