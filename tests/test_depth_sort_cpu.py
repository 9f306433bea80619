"""CPU: the depth-sort key sets of tests/golden/sort_cases.py.  The std::sort restatement there must equal the compiled
std::sort of the association oracle and torch.sort(stable=False) on every set, and the sets together must reach every
branch of the introsort that group_kernel replays on ties: insertion sort only (n <= 16), partitions (n > 16), the
heap-sort fallback, NaN-NaN ties and +0.0/-0.0 ties.  tests/test_assoc_limits_gpu.py feeds the same sets to the device."""
import numpy as np
import pytest
import torch

import sort_cases
from oracle import assoc


@pytest.fixture(scope="module")
def key_sets():
    return sort_cases.key_sets()


def test_restatement_equals_std_sort_and_torch(key_sets):
    print()
    for name, k in key_sets.items():
        order, st = sort_cases.introsort(k.tolist())
        print("%-12s n=%3d %s" % (name, len(k), st))
        assert np.array_equal(order, assoc.depth_order(k)), name
        _, idx = torch.from_numpy(k.copy()).sort(0, False)
        assert np.array_equal(order, idx.numpy()), name
        assert sorted(order.tolist()) == list(range(len(k)))


def test_restatement_on_random_ties():
    rng = np.random.default_rng(11)
    for t in range(200):
        n = int(rng.integers(1, 128))
        k = rng.integers(0, max(2, n // 4), n).astype(np.float32)
        if t % 5 == 0:
            k[rng.choice(n, int(rng.integers(1, n + 1)), replace=False)] = np.nan
        if t % 7 == 0:
            k[k == 0] = -0.0
        assert np.array_equal(sort_cases.introsort(k.tolist())[0], assoc.depth_order(k))


def test_every_set_has_a_tie(key_sets):
    """group_kernel takes the replay only when two keys tie; every named set must send it there."""
    for name, k in key_sets.items():
        assert sort_cases.has_tie(k), name


def test_sets_reach_every_branch(key_sets):
    stats = {name: sort_cases.introsort(k.tolist())[1] for name, k in key_sets.items()}
    assert any(s.insertion_only for name, s in stats.items() if len(key_sets[name]) <= 16)
    assert all(s.insertion_only == (len(key_sets[name]) <= 16) for name, s in stats.items())
    assert any(s.partitions > 0 for s in stats.values())
    assert stats["heap_n127"].heap_sorts >= 1
    assert any(s.nan_ties > 0 for s in stats.values())
    assert any(s.zero_ties > 0 for s in stats.values())
    for n in sort_cases.N_SIZES:  # NaN and +-0 ties at every size
        assert stats["nans_n%d" % n].nan_ties > 0 and stats["pm0_n%d" % n].zero_ties > 0


def test_heap_sort_set():
    k = sort_cases.heap_sort_keys()
    order, st = sort_cases.introsort(k.tolist())
    vals = np.unique(k)
    print("\nheap_n127: %d keys, %d distinct values, %s" % (len(k), len(vals), st))
    assert len(k) == 127 and len(vals) < len(k) // 4 and st.heap_sorts >= 1
    assert np.array_equal(k, sort_cases.heap_sort_keys())  # deterministic
    assert not np.array_equal(order, np.argsort(k, kind="stable"))
    # the adversary's distinct-key killer alone goes deeper than the depth limit
    assert sort_cases.introsort(sort_cases.antiqsort_ranks(127).astype(np.float64).tolist())[1].heap_sorts >= 1


def test_unstable_order_differs_from_stable_where_the_device_test_relies_on_it(key_sets):
    """For n > 16 the order of equal keys is not the stable one, so a stable sort on the device would be caught; for
    n <= 16 the final insertion sort is stable and the two agree."""
    for name, k in key_sets.items():
        order = sort_cases.introsort(k.tolist())[0]
        stable = np.argsort(k, kind="stable")
        if len(k) > 16:
            assert not np.array_equal(order, stable), name
        else:
            assert np.array_equal(order, stable), name
