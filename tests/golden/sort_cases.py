"""Depth-sort key sets for the grouping's tie-order replay (association.cpp:144, `predRootDepth.sort(0, false)`).

The reference sorts root depths with an unstable at::sort: libstdc++ std::sort over (key, index) pairs with the
comparator comp(a, b) = (!isnan(a) && isnan(b)) || a < b (ATen KeyValueCompAsc).  Equal keys (exact ties, two NaNs,
+0.0 against -0.0) come out in whatever order the introsort leaves, and that order decides which person is row 0 and
which person claims a contested limb first.  group_kernel replays the algorithm step by step when any two keys tie.

This module holds
  * `introsort`: a restatement of that std::sort (bits/stl_algo.h: median-of-3 pivot moved to the front, unguarded
    partition, threshold 16, heap-sort fallback at depth 2*floor(log2 n), final insertion sort), instrumented to report
    which branches a key set reaches.  It is a coverage probe, not the oracle: the tests pin it against the compiled
    std::sort of oracle/assoc_oracle.cpp and against torch.sort(stable=False) on every set it is used for.
  * `key_sets()`: named key sets for n in N_SIZES (ties, few values, NaNs, +-0, +-inf and negative depths) and a
    127-key set with ties that drives the sort into its heap-sort fallback (`heap_sort_keys`, built from McIlroy's
    "A Killer Adversary for Quicksort" against the restatement, then with adjacent ranks merged).
Pure numpy / Python, no reference and no oracle code."""
import math

import numpy as np

N_SIZES = (2, 3, 16, 17, 18, 33, 64, 127)
THRESHOLD = 16  # libstdc++ _S_threshold


def kv_comp(a, b):
    """KeyValueCompAsc on float keys: NaN sorts last, NaNs tie with each other, +0.0 ties with -0.0."""
    return (not math.isnan(a) and math.isnan(b)) or a < b


class Stats:
    def __init__(self):
        self.partitions = 0      # passes of __unguarded_partition_pivot
        self.heap_sorts = 0      # entries into the __partial_sort fallback
        self.nan_ties = 0        # comparisons of two NaN keys
        self.zero_ties = 0       # comparisons of +0.0 with -0.0

    @property
    def insertion_only(self):
        return self.partitions == 0 and self.heap_sorts == 0

    def __repr__(self):
        return "partitions=%d heap_sorts=%d insertion_only=%s nan_ties=%d zero_ties=%d" % (
            self.partitions, self.heap_sorts, self.insertion_only, self.nan_ties, self.zero_ties)


def introsort(keys, comp=None):
    """std::sort restated over (key, index) pairs.  keys: sequence of floats (or of anything `comp` orders).
    Returns (order, Stats): order[i] = index of the i-th element of the sorted sequence."""
    st = Stats()
    if comp is None:
        def comp(a, b):
            if a != a and b != b:
                st.nan_ties += 1
            elif a == 0.0 and b == 0.0 and math.copysign(1.0, a) != math.copysign(1.0, b):
                st.zero_ties += 1
            return kv_comp(a, b)
    a = [(k, i) for i, k in enumerate(keys)]
    n = len(a)

    def lt(x, y):
        return comp(x[0], y[0])

    def adjust_heap(base, hole, length, value):  # std::__adjust_heap + __push_heap
        top = hole
        child = hole
        while child < (length - 1) // 2:
            child = 2 * (child + 1)
            if lt(a[base + child], a[base + child - 1]):
                child -= 1
            a[base + hole] = a[base + child]
            hole = child
        if (length & 1) == 0 and child == (length - 2) // 2:
            child = 2 * (child + 1)
            a[base + hole] = a[base + child - 1]
            hole = child - 1
        parent = (hole - 1) // 2
        while hole > top and lt(a[base + parent], value):
            a[base + hole] = a[base + parent]
            hole = parent
            parent = (hole - 1) // 2
        a[base + hole] = value

    def heap_sort(first, last):  # std::__partial_sort(first, last, last): __make_heap, empty __heap_select, __sort_heap
        length = last - first
        if length >= 2:
            parent = (length - 2) // 2
            while True:
                adjust_heap(first, parent, length, a[first + parent])
                if parent == 0:
                    break
                parent -= 1
        while last - first > 1:
            last -= 1
            value = a[last]
            a[last] = a[first]
            adjust_heap(first, 0, last - first, value)

    def move_median_to_first(result, x, y, z):
        if lt(a[x], a[y]):
            if lt(a[y], a[z]):
                m = y
            elif lt(a[x], a[z]):
                m = z
            else:
                m = x
        elif lt(a[x], a[z]):
            m = x
        elif lt(a[y], a[z]):
            m = z
        else:
            m = y
        a[result], a[m] = a[m], a[result]

    def unguarded_partition(lo, hi, pivot):
        while True:
            while lt(a[lo], a[pivot]):
                lo += 1
            hi -= 1
            while lt(a[pivot], a[hi]):
                hi -= 1
            if not lo < hi:
                return lo
            a[lo], a[hi] = a[hi], a[lo]
            lo += 1

    def introsort_loop(first, last, depth):
        while last - first > THRESHOLD:
            if depth == 0:
                st.heap_sorts += 1
                heap_sort(first, last)
                return
            depth -= 1
            st.partitions += 1
            mid = first + (last - first) // 2
            move_median_to_first(first, first + 1, mid, last - 1)
            cut = unguarded_partition(first + 1, last, first)
            introsort_loop(cut, last, depth)
            last = cut

    def unguarded_linear_insert(last):
        val = a[last]
        nxt = last - 1
        while lt(val, a[nxt]):
            a[last] = a[nxt]
            last = nxt
            nxt -= 1
        a[last] = val

    def insertion_sort(first, last):
        if first == last:
            return
        for i in range(first + 1, last):
            if lt(a[i], a[first]):
                val = a[i]
                a[first + 1:i + 1] = a[first:i]
                a[first] = val
            else:
                unguarded_linear_insert(i)

    if n > 0:
        introsort_loop(0, n, 2 * (n.bit_length() - 1))
        if n > THRESHOLD:
            insertion_sort(0, THRESHOLD)
            for i in range(THRESHOLD, n):
                unguarded_linear_insert(i)
        else:
            insertion_sort(0, n)
    return np.array([i for _, i in a], np.int32), st


def has_tie(keys):
    """group_kernel's own condition for the replay: two keys that neither compares below the other."""
    k = [float(x) for x in keys]
    return any(not kv_comp(k[i], k[j]) and not kv_comp(k[j], k[i]) for i in range(len(k)) for j in range(i))


def antiqsort_ranks(n):
    """McIlroy's adversary run against `introsort`: values are assigned lazily so that every pivot is as bad as the
    comparisons seen so far allow.  Returns distinct integer ranks [n] that drive the sort deep."""
    gas = n
    val = [gas] * n
    state = {"solid": 0, "candidate": -1}

    def freeze(i):
        val[i] = state["solid"]
        state["solid"] += 1

    def comp(x, y):  # x, y: element indices (the sort's keys are the indices themselves)
        if val[x] == gas and val[y] == gas:
            freeze(x if x == state["candidate"] else y)
        if val[x] == gas:
            state["candidate"] = x
        elif val[y] == gas:
            state["candidate"] = y
        return val[x] < val[y]

    introsort(list(range(n)), comp)
    for i in range(n):  # anything never frozen takes the remaining values
        if val[i] == gas:
            freeze(i)
    return np.array(val, np.int64)


def heap_sort_keys(n=127):
    """Float32 keys with ties that still reach the heap-sort fallback: the adversary's ranks, then adjacent ranks merged
    greedily (lowest first) while the restatement still enters heap sort.  Deterministic."""
    ranks = antiqsort_ranks(n)
    assert introsort(ranks.astype(np.float64))[1].heap_sorts > 0
    group = np.arange(n)  # group[r] = merged value of rank r (non-decreasing)
    for r in range(1, n):
        trial = group.copy()
        trial[r:] -= 1  # merge rank r into rank r - 1's value
        if introsort(trial[ranks].astype(np.float64))[1].heap_sorts > 0:
            group = trial
    vals = group[ranks]
    return (0.75 + 0.125 * vals).astype(np.float32)  # exact in float32, depths of a plausible scale


def key_sets():
    """-> {name: float32 keys}.  Names are '<kind>_n<n>'; every set except 'distinct*' contains a tie."""
    out = {}
    for n in N_SIZES:
        rng = np.random.default_rng(7000 + n)
        out["equal_n%d" % n] = np.full(n, 1.25, np.float32)
        for k in range(2, 6):
            if k < n:  # every value appears and at least one repeats
                out["few%d_n%d" % (k, n)] = (0.5 + 0.25 * rng.permutation(np.arange(n) % k)).astype(np.float32)
        if n >= 3:
            one = (0.5 + 0.25 * rng.permutation(np.arange(n) % max(1, min(3, n - 2)))).astype(np.float32)
            one[rng.integers(0, n)] = np.nan
            out["nan1_n%d" % n] = one
        many = rng.permutation(np.linspace(0.5, 3.0, n)).astype(np.float32)  # distinct apart from the NaNs
        many[rng.choice(n, max(2, n // 4), replace=False)] = np.nan
        out["nans_n%d" % n] = many
        z = np.where(rng.permutation(np.arange(n) % 2) == 0, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
        if n > 4:
            z[rng.choice(n, n // 4, replace=False)] = np.linspace(0.5, 2.0, n // 4)
        out["pm0_n%d" % n] = z
        if n >= 3:
            vals = np.array([-np.inf, -1.5, -0.5, 0.75, np.inf], np.float32)
            out["infneg_n%d" % n] = vals[rng.permutation(np.arange(n) % min(5, n - 1))]
    out["heap_n127"] = heap_sort_keys(127)
    return out
