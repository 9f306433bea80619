"""GPU: the association kernels and the CPU oracle against the UNMODIFIED reference extension, run live.

oracle/build_ref.py compiles the reference's association.cpp, gpu/nmsBase.cu and gpu/bodyPartConnectorBase.cu into
oracle/_ref/ during build(); this file loads that module and compares, bit for bit, on the adversarial frames of
tests/golden/assoc_adversary.py (threshold values, plateaus, borders, clipped and non-finite centroid windows, the
127-peak cap, sample counts, near and ratio thresholds, score ties, `used` competition, exact-zero penalties, root-depth
key sets) and on the breadth frames of the other association tests:
  * canary: the live reference still returns what tests/golden/assoc_ref.npz recorded;
  * Engine.extract equals dapalib.extract per frame (peak counts, peaks, the nA x nB score blocks), in batches of 8 and
    in one batch of 64;
  * Engine.connect equals dapalib.connect for root_idx 0 and 2, with and without the distance penalty;
  * oracle.assoc.extract / connect equal the live reference on the same frames.
Values are compared as uint32 bit patterns, so NaN payloads and the sign of zero count.  A failure names the frame,
the joint or limb and the index, with both values in hex.

The reference runs on the legacy default stream with synchronous copies and the engine on its own non-blocking stream:
every hand-over between them synchronises the device.  Frames with +-inf in a root plane are extract-only (the
reference's connect indexes the CPU depth map with the root peaks)."""
import time

import numpy as np
import pytest
import torch

import assoc_adversary as A
from oracle import assoc, build_ref

pytestmark = pytest.mark.gpu
COMBOS = [(r, d) for r in (0, 2) for d in (True, False)]
MAX_REPORT = 8


@pytest.fixture(scope="module")
def ref():
    r = build_ref.load_ref()
    if r is None:
        pytest.skip("oracle/_ref/dapalib_ref*.so is missing: build() builds it where the reference sources exist")
    return r


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=64, in_h=512, in_w=832)
    yield e
    e.close()


@pytest.fixture(scope="module")
def frames():
    return list(A.frames())


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def diff(got, want, what):
    """None when got and want are bit-identical, else a message with the first differing index and both values."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    if got.shape != want.shape:
        return "%s: shape %s, reference %s" % (what, got.shape, want.shape)
    g, w = bits(got), bits(want)
    if np.array_equal(g, w):
        return None
    i = tuple(int(k) for k in np.argwhere(g != w)[0])
    return "%s at %s: 0x%08x (%r), reference 0x%08x (%r)" % (what, i, g[i], float(got[i]), w[i], float(want[i]))


def report(errs, n_checked, what):
    assert n_checked > 0
    if errs:
        pytest.fail("%d of %d %s differ from the live reference:\n  %s" % (len(errs), n_checked, what,
                                                                             "\n  ".join(errs[:MAX_REPORT])))


def sync():
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# the live reference, once per frame
# ---------------------------------------------------------------------------------------------------------------------
def ref_extract_one(ref, hms):
    th = torch.from_numpy(hms).cuda().contiguous()  # exactly [43, 128, 208] float32: the reference copies that many
    assert tuple(th.shape) == (43, A.H, A.W) and th.dtype == torch.float32 and th.is_contiguous()
    sync()
    pk, sc = ref.extract(th)
    sync()
    return [p.numpy().copy() for p in pk], [s.numpy().copy() for s in sc]


def ref_connect_one(ref, hms, rd, root_idx, dist_flag):
    assert A.connectable(hms, root_idx)
    th = torch.from_numpy(hms).cuda().contiguous()
    sync()
    b = ref.connect(th, torch.from_numpy(rd).contiguous(), root_idx, dist_flag)  # depth map on the CPU
    sync()
    b = b.numpy().copy()
    return b if b.ndim == 3 else np.zeros((0, A.NJ, 4), np.float32)


@pytest.fixture(scope="module")
def ref_extract(ref, frames):
    t = time.time()
    out = [ref_extract_one(ref, hms) for _, hms, _, _ in frames]
    print("\nreference extract: %d frames in %.1f s" % (len(frames), time.time() - t))
    return out


_ref_connect = {}


def connected(name, hms, root_idx):
    """Frames connect runs on: every family frame, and a quarter of the random_heatmaps and make_scene seeds (the
    reference groups with one tensor .item() per pair score, about a second per 127-person frame; extract sees all)."""
    if not A.connectable(hms, root_idx):
        return False
    return not name.startswith(("random_", "scene_")) or int(name.split("_")[1]) % 4 == 0


def ref_connect(ref, frames, root_idx, dist_flag):
    key = (root_idx, dist_flag)
    if key not in _ref_connect:
        t = time.time()
        _ref_connect[key] = [ref_connect_one(ref, hms, rd, root_idx, dist_flag) if connected(name, hms, root_idx)
                             else None for name, hms, rd, _ in frames]
        print("\nreference connect(root_idx=%d, dist_flag=%s): %.1f s" % (root_idx, dist_flag, time.time() - t))
    return _ref_connect[key]


def compare_extract(name, peaks, scores, want):
    """peaks [15,128,3], scores [14,127,127] (engine or oracle layout) against the reference's lists."""
    wp, ws = want
    for j in range(A.NJ):
        n = len(wp[j])
        if int(peaks[j, 0, 0]) != n:
            return "%s joint %d: %d peaks, reference %d" % (name, j, int(peaks[j, 0, 0]), n)
        e = diff(peaks[j, 1:n + 1], wp[j], "%s joint %d peaks" % (name, j))
        if e:
            return e
    for l in range(A.NL):
        na, nb = ws[l].shape
        e = diff(scores[l, :na, :nb], ws[l], "%s limb %d scores" % (name, l))
        if e:
            return e
    return None


def compare_bodies(name, bodies, count, want):
    if count != len(want):
        return "%s: %d persons, reference %d" % (name, count, len(want))
    e = diff(bodies[:count], want, "%s bodies" % name)
    if e:
        return e
    if bodies[count:].any():
        return "%s: rows past the person count are not zero" % name
    return None


# ---------------------------------------------------------------------------------------------------------------------
def test_canary_live_reference_reproduces_the_recorded_one(ref):
    """If this fails, the reference built here is not the one the recorded digests came from: nothing below can be
    trusted until that is understood."""
    import os

    from test_assoc_gpu import _digest, reference_sets, scenes

    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "assoc_ref.npz"))
    for s, (hms, rd) in enumerate(reference_sets()):
        for b in range(hms.shape[0]):
            g = "s%d_b%d_" % (s, b)
            pk, sc = ref_extract_one(ref, np.ascontiguousarray(hms[b]))
            assert [tuple(p.shape) for p in pk] == [tuple(x) for x in gold[g + "peak_shapes"]], g
            assert [_digest(p) for p in pk] == list(gold[g + "peaks"]), g
            assert [_digest(x) for x in sc] == list(gold[g + "scores"]), g
            body = ref_connect_one(ref, np.ascontiguousarray(hms[b]), rd[b], 2, True)
            assert tuple(gold[g + "body_shape"]) == (body.shape if len(body) else (0,)), g
            if len(body):
                assert _digest(body) == gold[g + "bodies"], g
    hms, rd, _ = scenes(range(50, 53))
    for b in range(3):
        assert _digest(ref_connect_one(ref, hms[b], rd[b], 2, True)) == gold["o%d_bodies" % b]


def run_engine_extract(eng, hms):
    sync()
    p, s = eng.extract(torch.from_numpy(hms).cuda())
    sync()
    return p.cpu().numpy(), s.cpu().numpy()


def test_extract_matches_reference(eng, frames, ref_extract):
    errs = []
    for c in range(0, len(frames), 8):
        chunk = frames[c:c + 8]
        p, s = run_engine_extract(eng, np.stack([f[1] for f in chunk]))
        for b, (name, _, _, _) in enumerate(chunk):
            e = compare_extract(name, p[b], s[b], ref_extract[c + b])
            if e:
                errs.append(e)
    report(errs, len(frames), "frames (extract, batches of 8)")


def test_extract_batch64_matches_reference(eng, frames, ref_extract):
    chunk = frames[:64]
    p, s = run_engine_extract(eng, np.stack([f[1] for f in chunk]))
    errs = [e for e in (compare_extract(f[0], p[b], s[b], ref_extract[b]) for b, f in enumerate(chunk)) if e]
    report(errs, len(chunk), "frames (extract, one batch of 64)")


@pytest.mark.parametrize("root_idx,dist_flag", COMBOS)
def test_connect_matches_reference(ref, eng, frames, root_idx, dist_flag):
    want = ref_connect(ref, frames, root_idx, dist_flag)
    idx = [i for i, w in enumerate(want) if w is not None]
    errs = []
    for c in range(0, len(idx), 8):
        chunk = idx[c:c + 8]
        hms = np.stack([frames[i][1] for i in chunk])
        rd = np.stack([frames[i][2] for i in chunk])
        sync()
        bodies, counts = eng.connect(torch.from_numpy(hms).cuda(), torch.from_numpy(rd).cuda(), root_idx, dist_flag)
        sync()
        bodies, counts = bodies.cpu().numpy(), counts.cpu().numpy()
        for b, i in enumerate(chunk):
            e = compare_bodies(frames[i][0], bodies[b], int(counts[b]), want[i])
            if e:
                errs.append(e)
    report(errs, len(idx), "frames (connect root_idx=%d dist_flag=%s)" % (root_idx, dist_flag))


def test_oracle_extract_matches_reference(frames, ref_extract):
    errs = []
    for (name, hms, _, _), want in zip(frames, ref_extract):
        p, s = assoc.extract(hms)
        e = compare_extract("oracle " + name, p, s, want)
        if e:
            errs.append(e)
    report(errs, len(frames), "frames (oracle extract)")


@pytest.mark.parametrize("root_idx,dist_flag", COMBOS)
def test_oracle_connect_matches_reference(ref, frames, root_idx, dist_flag):
    want = ref_connect(ref, frames, root_idx, dist_flag)
    errs, n = [], 0
    for (name, hms, rd, _), w in zip(frames, want):
        if w is None:
            continue
        n += 1
        ob = assoc.connect(hms, rd, root_idx, dist_flag)
        e = compare_bodies("oracle " + name, np.concatenate([ob, np.zeros((1, A.NJ, 4), np.float32)]), len(ob), w)
        if e:
            errs.append(e)
    report(errs, n, "frames (oracle connect root_idx=%d dist_flag=%s)" % (root_idx, dist_flag))
