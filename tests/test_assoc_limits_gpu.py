"""GPU: the data-dependent paths behind the association that only crowded frames or tied depths reach.

  * Grouping on tied root depths.  group_kernel rank-sorts the root depths in parallel when they are distinct and has one
    thread replay libstdc++'s std::sort otherwise (association.cpp:144 is an unstable sort, so the order of equal depths is
    the introsort's).  Frames whose root channel holds exactly the key sets of tests/golden/sort_cases.py (ties, few
    values, NaNs, +-0, +-inf, negative depths, a set that reaches the heap-sort fallback) are connected with both roots
    and both dist_flag values, bit-exact against the oracle.  PAFs that point along +x make most pairs score, so persons
    compete for candidates and the processing order changes the bodies: a stable-order oracle gives other bodies.
  * The lift at capacity.  lift_kernel strides NP*NL (person, limb) items, NP*NJ body entries and, with ground truth, G*P
    distances over 256 threads; frames of up to 127 persons and 127 GT persons take several passes, the GT arg-min sees
    several entries per thread and exact distance ties across warps.  Bit-exact against oracle/lift_numpy.py.
  * RefineNet's records mode at 0 ... 127 persons per frame (empty frame, full and partial CTAs, the last CTA) and
    refine_mlp, against a float64 evaluation of the same network, under a bound tight enough that a wrong BN epsilon, a
    dropped output bias or a bias without its mean shift are flagged.
`-s` prints persons per frame and loop passes of the lift, the tied distances that decided a GT match and the worst
refine error relative to max|r|."""
import numpy as np
import pytest
import torch

import sort_cases
from cases import GEOMS, refine_state_dict
from oracle import assoc, lift_numpy, refine_torch

pytestmark = pytest.mark.gpu
H, W = 128, 208
NJ, NL, MAXP = 15, 14, 127
LIFT_THREADS = 256  # lift_kernel's block: its per-item loops stride by this
WARP = 32


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=8, in_h=512, in_w=832)
    e.load_refine_state_dict(refine_state_dict())
    yield e
    e.close()


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---------------------------------------------------------------------------------------------------------------------
# grouping on tied depths
# ---------------------------------------------------------------------------------------------------------------------
_GY, _GX = np.meshgrid(np.arange(6, 118, 15), np.arange(6, 196, 12), indexing="ij")
PAIR_CENTRES = np.stack([_GY.ravel(), _GX.ravel()], 1)  # 8 x 16, raster order


def root_positions(n):
    """n (y, x) pixels in raster order (the order NMS lists peaks in): pairs 4 px apart, so that two persons reach the
    same candidates, spread over the map.  At least 4 px between peaks: each 7x7 centroid window sees one pixel."""
    m = (n + 1) // 2
    c = PAIR_CENTRES[np.round(np.linspace(0, len(PAIR_CENTRES) - 1, m)).astype(int)]
    return np.stack([c, c + (0, 4)], 1).reshape(-1, 2)[:n]


def tie_frame(keys, root_ch, seed):
    """-> (hms [43,H,W], rd [H,W]): the root channel holds exactly len(keys) isolated single-pixel peaks, peak i (raster
    order) on a root depth of keys[i]; the other keypoint channels are noise with many peaks, the PAFs point along +x."""
    rng = np.random.default_rng(seed)
    lo = rng.normal(0, 1, (43, H // 4, W // 4)).astype(np.float32)
    hms = np.kron(lo, np.ones((1, 4, 4), np.float32)) * 0.4 + rng.normal(0, 0.15, (43, H, W)).astype(np.float32)
    hms[15::2] = 0.6 + 0.1 * hms[15::2]
    hms[16::2] *= 0.1
    hms[root_ch] = 0
    pos = root_positions(len(keys))
    hms[root_ch, pos[:, 0], pos[:, 1]] = rng.uniform(0.5, 0.9, len(keys))
    rd = rng.uniform(0.5, 3, (H, W)).astype(np.float32)
    rd[pos[:, 0], pos[:, 1]] = keys
    return hms.astype(np.float32), rd


def stable_keys(keys):
    """The keys with each run of equal values nudged up by 0, 1, 2 ... ulps in index order: the sort then yields the
    stable order of the original keys (the values are otherwise unchanged)."""
    k = keys.copy()
    for v in np.unique(keys):
        for j, i in enumerate(np.flatnonzero(keys == v)):
            for _ in range(j):
                k[i] = np.nextafter(k[i], np.float32(np.inf))
    return k


def canonical(bodies):
    """Rows ordered by root position: two body sets that differ only in row order compare equal."""
    return bodies[np.lexsort((bodies[:, 2, 0], bodies[:, 2, 1], bodies[:, 0, 0], bodies[:, 0, 1]))]


def connect_batch(eng, hms, rd, root_idx, dist_flag):
    bodies, counts = eng.connect(dev(hms), dev(rd), root_idx, dist_flag)
    torch.cuda.synchronize()
    return bodies.cpu().numpy(), counts.cpu().numpy()


@pytest.mark.parametrize("dist_flag", [True, False])
@pytest.mark.parametrize("root_idx", [2, 0])
def test_grouping_on_tied_depths_bit_exact(eng, root_idx, dist_flag):
    sets = sort_cases.key_sets()
    names = list(sets)
    for c in range(0, len(names), 8):
        chunk = names[c:c + 8]  # several key sets mixed in one batch
        frames = [tie_frame(sets[nm], root_idx, 100 + c + i) for i, nm in enumerate(chunk)]
        hms, rd = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
        bodies, counts = connect_batch(eng, hms, rd, root_idx, dist_flag)
        for b, nm in enumerate(chunk):
            keys = sets[nm]
            assert sort_cases.has_tie(keys), nm  # the kernel's own condition for the std::sort replay
            ob = assoc.connect(hms[b], rd[b], root_idx, dist_flag)
            assert counts[b] == len(ob) == len(keys), nm
            assert np.array_equal(bodies[b, :len(ob)], ob), "bodies differ: %s" % nm
            assert not bodies[b, len(ob):].any(), nm


@pytest.mark.parametrize("root_idx", [2, 0])
def test_tie_order_decides_the_bodies(eng, root_idx):
    """The check above can fail: where the std::sort order of ties differs from the stable one, an oracle given the
    stable order builds other bodies than the device, and not only in another row order."""
    sets = sort_cases.key_sets()
    names = ["heap_n127", "few3_n127"]
    frames = [tie_frame(sets[nm], root_idx, 200 + i) for i, nm in enumerate(names)]
    hms, rd = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    bodies, counts = connect_batch(eng, hms, rd, root_idx, True)
    for b, nm in enumerate(names):
        keys = sets[nm]
        nudged = stable_keys(keys)
        assert np.array_equal(assoc.depth_order(nudged), np.argsort(keys, kind="stable"))
        assert not np.array_equal(assoc.depth_order(keys), np.argsort(keys, kind="stable"))
        rd_stable = rd[b].copy()
        pos = root_positions(len(keys))
        rd_stable[pos[:, 0], pos[:, 1]] = nudged
        ob = assoc.connect(hms[b], rd_stable, root_idx, True)
        got = bodies[b, :counts[b]]
        assert np.array_equal(got, assoc.connect(hms[b], rd[b], root_idx, True)), nm
        assert len(ob) == len(got)
        assert not np.array_equal(got, ob), nm
        assert not np.array_equal(canonical(got), canonical(ob)), nm


# ---------------------------------------------------------------------------------------------------------------------
# the lift at capacity
# ---------------------------------------------------------------------------------------------------------------------
LIFT_PERSONS = (18, 19, 64, 126, 127)


def capacity_bodies(P, seed, drop_roots):
    """float32 [P,15,4] as connect returns them (heat-map px): coordinates up to the last row and column of the map
    (x = w - 0.5), a quarter of the joints unscored, and with `drop_roots` every third person without a root (the lift
    drops them and compacts the rest)."""
    rng = np.random.default_rng(seed)
    b = np.zeros((P, NJ, 4), np.float32)
    b[:, :, 0] = rng.uniform(0.5, W - 0.5, (P, NJ))
    b[:, :, 1] = rng.uniform(0.5, H - 0.5, (P, NJ))
    b[:, :, 0][rng.uniform(size=(P, NJ)) < 0.1] = W - 0.5
    b[:, :, 1][rng.uniform(size=(P, NJ)) < 0.1] = H - 0.5
    b[:, :, 3] = rng.uniform(0.2, 1, (P, NJ)) * (rng.uniform(size=(P, NJ)) > 0.25)
    b[:, 2, 3] = rng.uniform(0.2, 1, P)
    if drop_roots:
        b[1::3, 2, 3] = 0
    b[b[:, :, 3] == 0] = 0
    return b


def quantised_maps(seed):
    """det_d [14,H,W] with 7 values in 8x8 blocks (the 10 samples of a limb hold equal values, so the percentile clip
    compares equal values) and root_d [H,W]."""
    rng = np.random.default_rng(seed)
    dd = np.kron(rng.integers(-3, 4, (14, H // 8, W // 8)), np.ones((1, 8, 8))) * 7.5
    speck = rng.uniform(size=dd.shape) < 0.2
    dd[speck] = rng.integers(-3, 4, int(speck.sum())) * 7.5
    rd = rng.uniform(1, 9, (H, W))
    return dd.astype(np.float32), rd.astype(np.float32)


def capacity_lift_inputs():
    """The lift batch: one frame per LIFT_PERSONS entry, root-missing persons in the 64- and 126-person frames, every
    person kept in the others (18 and 19 kept persons straddle NP*NL = 256; 127 is the cap)."""
    B = len(LIFT_PERSONS)
    bodies = np.zeros((B, MAXP, NJ, 4), np.float32)
    dd = np.zeros((B, NL, H, W), np.float32)
    rd = np.zeros((B, H, W), np.float32)
    scs = []
    for i, P in enumerate(LIFT_PERSONS):
        bodies[i, :P] = capacity_bodies(P, 300 + i, drop_roots=P in (64, 126))
        dd[i], rd[i] = quantised_maps(400 + i)
        scs.append(lift_numpy.default_scale(*GEOMS[i % len(GEOMS)]))
    return bodies, np.array(LIFT_PERSONS, np.int32), dd, rd, scs


def passes(items):
    return -(-items // LIFT_THREADS)


def check_lift(p2, p3, rdp, co, b, o2, o3, ordp):
    m = len(o2)
    assert int(co[b]) == m
    assert np.array_equal(p2[b, :m], o2)
    assert np.array_equal(rdp[b, :m], ordp)
    np.testing.assert_allclose(p3[b, :m], o3, rtol=1e-12, atol=1e-12)
    assert not p2[b, m:].any() and not p3[b, m:].any() and not rdp[b, m:].any()


def run_lift(eng, bodies, counts, dd, rd, scs):
    from smap_b200.engine import scale_row

    out = eng.lift(dev(bodies), dev(counts), dev(dd), dev(rd), dev(np.stack([scale_row(s) for s in scs])))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def test_lift_at_capacity(eng):
    bodies, counts, dd, rd, scs = capacity_lift_inputs()
    p2, p3, rdp, co = run_lift(eng, bodies, counts, dd, rd, scs)
    print()
    nps = []
    for b, P in enumerate(LIFT_PERSONS):
        o2, o3, ordp = lift_numpy.lift(bodies[b, :P], dd[b], rd[b], scs[b])
        check_lift(p2, p3, rdp, co, b, o2, o3, ordp)
        NP = len(o2)
        nps.append(NP)
        print("lift frame %d: %3d persons, %3d kept, NP*NL = %4d (%d passes), NP*NJ = %4d (%d passes)"
              % (b, P, NP, NP * NL, passes(NP * NL), NP * NJ, passes(NP * NJ)))
    # what this test is for: second passes of both strided loops, compaction, and the clip on equal values
    assert max(nps) == MAXP and max(nps) * NL > LIFT_THREADS and max(nps) * NJ > LIFT_THREADS
    assert 18 in nps and 19 in nps  # 18*14 = 252 < 256 < 19*14
    assert any(n < P for n, P in zip(nps, LIFT_PERSONS))
    assert (bodies[:, :, :, 0] == W - 0.5).any() and (bodies[:, :, :, 1] == H - 0.5).any()


def crowded_frames():
    """Root channels saturated to the 127-peak cap (150 peaks on 5 depth values; the heap-sort and 3-value key sets)."""
    rng = np.random.default_rng(17)
    keys = [(0.5 + 0.25 * rng.permutation(np.arange(150) % 5)).astype(np.float32), sort_cases.heap_sort_keys(),
            sort_cases.key_sets()["few3_n127"]]
    frames = [tie_frame(k, 2, 500 + i) for i, k in enumerate(keys)]
    return np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])


def test_connect_then_lift_on_crowded_frames(eng):
    hms, rd = crowded_frames()
    B = len(hms)
    dd = np.stack([quantised_maps(600 + i)[0] for i in range(B)])
    scs = [lift_numpy.default_scale(*GEOMS[i % len(GEOMS)]) for i in range(B)]
    bodies, counts = eng.connect(dev(hms), dev(rd))
    from smap_b200.engine import scale_row

    out = eng.lift(bodies, counts, dev(dd), dev(rd), dev(np.stack([scale_row(s) for s in scs])))
    torch.cuda.synchronize()
    p2, p3, rdp, co = [t.cpu().numpy() for t in out]
    for b in range(B):
        ob = assoc.connect(hms[b], rd[b])
        assert int(counts[b]) == len(ob) == MAXP
        o2, o3, ordp = lift_numpy.lift(ob, dd[b], rd[b], scs[b])
        assert len(o2) == MAXP
        check_lift(p2, p3, rdp, co, b, o2, o3, ordp)


# ---- ground truth ----
def gt_frame(P, G, seed, dup_every=0, far_every=0):
    """Predictions whose roots sit on a 1.5 px heat-map grid (6 input px) and GT roots on the same grid, at grid midpoints
    and duplicated: most GT roots are within 30 px of many predictions, and many distances tie exactly.
    -> (bodies [P,15,4], GT roots float64 [G,2] in network-input pixels)."""
    rng = np.random.default_rng(seed)
    b = capacity_bodies(P, seed, drop_roots=True)
    if P:
        b[:, 2, 0] = 40 + 1.5 * (np.arange(P) % 16)
        b[:, 2, 1] = 30 + 1.5 * (np.arange(P) // 16)
    roots = np.zeros((G, 2), np.float64)
    for g in range(G):
        p = int(rng.integers(0, max(P, 1)))
        base = np.float64(b[p, 2, :2]) * 4 if P else np.array([200.0, 200.0])
        roots[g] = base + (rng.choice([0.0, 3.0, 6.0, -3.0]), rng.choice([0.0, 3.0]))
        if dup_every and g % dup_every == dup_every - 1:
            roots[g] = roots[rng.integers(0, g)]  # a duplicated GT root: equal distances to every prediction
        if far_every and g % far_every == 0:
            roots[g] = (800.0 - g, 500.0)  # no prediction within 30 px: unmatched
    return b, roots


GT_FRAMES = [(127, 127, 2, 0), (127, 127, 0, 9), (60, 127, 3, 0), (127, 40, 0, 0), (0, 5, 0, 0), (10, 0, 0, 0)]


def decisive_ties(bodies, roots, root_n=2):
    """Replays register_pred's greedy matching (ascending distance, then flat index) and returns the matches an exact
    distance tie decided: pairs (taken index, passed-over index) of equal distance where both entries were still
    available and shared a GT person or a prediction."""
    pd = (bodies[:, root_n, :2] * np.float32(4)).astype(np.float32)
    diff = roots[:, None, :] - pd[None, :, :]
    dist = np.sqrt(diff[:, :, 0] * diff[:, :, 0] + diff[:, :, 1] * diff[:, :, 1])
    G, P = dist.shape
    order = sorted((dist[g, p], g * P + p) for g in range(G) for p in range(P) if dist[g, p] < 30)
    gfree, pfree = np.ones(G, bool), np.ones(P, bool)
    out = []
    for i, (d, idx) in enumerate(order):
        g, p = divmod(idx, P)
        if not (gfree[g] and pfree[p]):
            continue
        j = i + 1
        while j < len(order) and order[j][0] == d:
            g2, p2 = divmod(order[j][1], P)
            if gfree[g2] and pfree[p2] and (g2 == g or p2 == p):
                out.append((idx, order[j][1]))
            j += 1
        gfree[g], pfree[p] = False, False
    return out, int((dist < 30).sum())


def test_lift_with_ground_truth_at_capacity(eng):
    from smap_b200.engine import scale_row

    B = len(GT_FRAMES)
    gmax = MAXP
    bodies = np.zeros((B, MAXP, NJ, 4), np.float32)
    counts = np.zeros(B, np.int32)
    gt_roots = np.zeros((B, gmax, 2), np.float64)
    gt_counts = np.zeros(B, np.int32)
    dd = np.zeros((B, NL, H, W), np.float32)
    rd = np.zeros((B, H, W), np.float32)
    scs, gts = [], []
    for i, (P, G, dup, far) in enumerate(GT_FRAMES):
        b, roots = gt_frame(P, G, 700 + i, dup, far)
        bodies[i, :P], counts[i] = b, P
        gt_roots[i, :G], gt_counts[i] = roots, G
        gt = np.zeros((G, NJ, 4), np.float64)
        gt[:, 2, :2] = roots
        gts.append(gt)
        dd[i], rd[i] = quantised_maps(800 + i)
        scs.append(lift_numpy.default_scale(*GEOMS[i % len(GEOMS)]))
    out = eng.lift_gt(dev(bodies), dev(counts), dev(dd), dev(rd), dev(np.stack([scale_row(s) for s in scs])),
                      dev(gt_roots), dev(gt_counts))
    torch.cuda.synchronize()
    p2, p3, rdp, co = [t.cpu().numpy() for t in out]
    print()
    all_ties, max_gp, max_under = [], 0, 0
    for i, (P, G, _, _) in enumerate(GT_FRAMES):
        if P == 0 or G == 0:  # no prediction: empty result; no GT person: the frame is skipped
            assert int(co[i]) == 0 and not p2[i].any() and not p3[i].any() and not rdp[i].any()
            continue
        o2, o3, ordp = lift_numpy.lift(bodies[i, :P], dd[i], rd[i], scs[i], gt_bodys=gts[i])
        check_lift(p2, p3, rdp, co, i, o2, o3, ordp)
        ties, under = decisive_ties(bodies[i, :P], gt_roots[i, :G])
        unmatched = int((~o2.any(axis=(1, 2))).sum())
        print("lift_gt frame %d: G = %3d, P = %3d, G*P = %5d (%2d passes), %5d distances < 30 px, %3d matches decided "
              "by an exact distance tie (%3d tied pairs), %3d GT persons unmatched"
              % (i, G, P, G * P, passes(G * P), under, len({a for a, _ in ties}), len(ties), unmatched))
        assert 0 < G - unmatched
        all_ties += ties
        max_gp, max_under = max(max_gp, G * P), max(max_under, under)
    # what this test is for: several distance entries per thread, candidates in many warps, ties across warps and strides
    assert max_gp > LIFT_THREADS and max_under > LIFT_THREADS
    assert len(all_ties) > 0
    assert any((a % LIFT_THREADS) // WARP != (c % LIFT_THREADS) // WARP and a // LIFT_THREADS != c // LIFT_THREADS
               for a, c in all_ties)


# ---------------------------------------------------------------------------------------------------------------------
# RefineNet at capacity
# ---------------------------------------------------------------------------------------------------------------------
# |y - r| <= tol * max|r|, r from the float64 network.  The device computes fp32 with one fmaf per step (K <= 256) on fp32
# folded weights; refine_mlp's outputs are the network's alone: REFINE_TOL.  In records mode the root (thousands of mm) is
# added and max|r| is the root's scale, about 100x the network's output; there the float32 rounding of the sum dominates
# (2^-24 relative) and the tighter RECORDS_TOL still leaves a wide margin while a wrong network moves outputs by ~1e-5.
REFINE_TOL = 1e-5
RECORDS_TOL = 1e-6
REFINE_COUNTS = (0, 1, 4, 5, 126, 127)  # empty frame, partial CTA, one full CTA, full + partial, partial last CTA, cap


def mlp64(sd, x, eps=1e-5, drop_out_bias=False, unshifted_layer=None):
    """model/refinenet.py in eval mode, in float64, with BatchNorm folded in float64 from the fp32 state dict.  The other
    arguments make the deliberately wrong references the bound must flag."""
    x = np.asarray(x, np.float64)
    for i in range(1, 5):
        p = "block.layer%d." % i
        w, b = sd[p + "0.weight"].astype(np.float64), sd[p + "0.bias"].astype(np.float64)
        g, beta = sd[p + "1.weight"].astype(np.float64), sd[p + "1.bias"].astype(np.float64)
        mu, var = sd[p + "1.running_mean"].astype(np.float64), sd[p + "1.running_var"].astype(np.float64)
        s = g / np.sqrt(var + eps)
        bias = b * s + beta if i == unshifted_layer else (b - mu) * s + beta
        x = np.maximum(x @ (w * s[:, None]).T + bias, 0.0)
    x = x @ sd["block.layer5.weight"].astype(np.float64).T
    if not drop_out_bias:
        x = x + sd["block.layer5.bias"].astype(np.float64)
    return x


def refine64(p2, p3, sd, root_n=2, **wrong):
    """lift_and_refine_3d_pose (test_util.py:102-131) around mlp64: the root added in float64, then rounded to float32."""
    n = len(p3)
    net = mlp64(sd, refine_torch.refine_inputs(p2, p3, root_n), **wrong).reshape(n, NJ, 3)
    out = np.zeros((n, NJ, 4), np.float64)
    out[:, :, :3] = (net + p3[:, root_n, None, :3]).astype(np.float32)
    out[:, root_n, :3] = p3[:, root_n, :3].astype(np.float32)
    out[:, :, 3] = (p3[:, root_n, 3] != 0)[:, None]
    return out


WRONG_REFS = {"bn_eps_1e-3": dict(eps=1e-3), "layer5_bias_dropped": dict(drop_out_bias=True),
              "layer2_bias_unshifted": dict(unshifted_layer=2)}


def rel_err(y, r):
    return float(np.abs(y - r).max() / np.abs(r).max())


@pytest.fixture(scope="module")
def refine_inputs_at_capacity():
    """Lift outputs (oracle; test_lift_at_capacity shows the device's are the same bits) of the 127-person frame, rows
    rotated per frame, cut to REFINE_COUNTS persons."""
    bodies, _, dd, rd, scs = capacity_lift_inputs()
    k = LIFT_PERSONS.index(MAXP)
    o2, o3, _ = lift_numpy.lift(bodies[k, :MAXP], dd[k], rd[k], scs[k])
    assert len(o2) == MAXP
    B = len(REFINE_COUNTS)
    p2 = np.zeros((B, MAXP, NJ, 4), np.float32)
    p3 = np.zeros((B, MAXP, NJ, 4), np.float64)
    for b, c in enumerate(REFINE_COUNTS):
        rows = (np.arange(c) + 17 * b) % MAXP
        p2[b, :c], p3[b, :c] = o2[rows], o3[rows]
    return p2, p3, np.array(REFINE_COUNTS, np.int32)


def test_refine_records_at_capacity(eng, refine_inputs_at_capacity):
    p2, p3, cnt = refine_inputs_at_capacity
    out = eng.refine(dev(p2), dev(p3), dev(cnt)).cpu().numpy()
    sd = refine_state_dict()
    print()
    worst = 0.0
    for b, c in enumerate(REFINE_COUNTS):
        assert not out[b, c:].any()
        if c == 0:
            continue
        got, r = out[b, :c], refine64(p2[b, :c], p3[b, :c], sd)
        assert np.array_equal(got[:, :, 3], r[:, :, 3])  # score column exact
        assert np.array_equal(got[:, 2, :3], r[:, 2, :3])  # root row = the lifted root, exact
        err = rel_err(got[:, :, :3], r[:, :, :3])
        worst = max(worst, err)
        print("refine frame %d: %3d persons, max|y - r| / max|r| = %.2e (bound %.0e)" % (b, c, err, RECORDS_TOL))
        assert err <= RECORDS_TOL
        if c >= 4:  # the bound discriminates: every wrong reference is flagged on the device output
            lim = RECORDS_TOL * np.abs(r[:, :, :3]).max()
            for name, wrong in WRONG_REFS.items():
                rw = refine64(p2[b, :c], p3[b, :c], sd, **wrong)
                outside = int((np.abs(got[:, :, :3] - rw[:, :, :3]) > lim).sum())
                old_ok = np.abs(got[:, :, :3] - rw[:, :, :3]).max() <= 1e-3 * np.abs(rw[:, :, :3]).max()
                print("    %-22s %5d elements outside the bound; passes the old 1e-3*max check: %s" % (name, outside, old_ok))
                assert outside > 0, name
    print("refine worst max|y - r| / max|r| = %.2e, bound %.0e" % (worst, RECORDS_TOL))


@pytest.mark.parametrize("n", [127, 300])
def test_refine_mlp_against_float64(eng, n):
    sd = refine_state_dict()
    x = (torch.randn(n, 75, generator=torch.Generator().manual_seed(30 + n)) * 50).float()
    got = eng.refine_mlp(x.cuda()).cpu().numpy().astype(np.float64)
    r = mlp64(sd, x.numpy())
    err = rel_err(got, r)
    print("\nrefine_mlp n = %d: max|y - r| / max|r| = %.2e (bound %.0e)" % (n, err, REFINE_TOL))
    assert err <= REFINE_TOL
    for name, wrong in WRONG_REFS.items():
        assert (np.abs(got - mlp64(sd, x.numpy(), **wrong)) > REFINE_TOL * np.abs(r).max()).any(), name
