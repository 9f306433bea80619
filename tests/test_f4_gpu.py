"""GPU: SURVEY 8(f) f4 - (1) the GT-matching branch of register_pred + the float64 lift it implies (test_util.py:21-39),
against the golden outputs of the unmodified reference functions (tests/golden/lift_gt_cases.npz) and the oracle;
(2) association at a map size other than the reference's hard-coded 128x208 (extensions/association.cpp:21): 256x256 maps
(config 5, a 1024x1024 input: PAF gathers from global memory) and 64x96 (a small map: vectorised NMS, staged PAF),
bit-exact against the oracle, and the whole path at 1024x1024.  tests/test_assoc_sizes_gpu.py checks these instances and
the scalar NMS against the live reference and the oracle on the adversarial frames."""
import os

import numpy as np
import pytest
import torch

from cases import N_GT_CASES, lift_gt_case_inputs
from oracle import assoc, lift_numpy
from smap_b200 import schema
from smap_b200.synth import make_scene

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_lift_with_ground_truth_matches_reference_golden():
    from smap_b200.engine import MAXP, NJ, Engine, scale_row

    eng = Engine(0, max_batch=N_GT_CASES, in_h=512, in_w=832)
    gold = np.load(os.path.join(G, "lift_gt_cases.npz"))
    B = N_GT_CASES
    bodies = np.zeros((B, MAXP, NJ, 4), np.float32)
    counts = np.zeros(B, np.int32)
    dd = np.zeros((B, 14, 128, 208), np.float32)
    rd = np.zeros((B, 128, 208), np.float32)
    scales = np.zeros((B, 9), np.float64)
    gmax = 8
    gt_roots = np.zeros((B, gmax, 2), np.float64)
    gt_counts = np.zeros(B, np.int32)
    for ci in range(B):
        b, det_d, root_d, (iw, ih), gt = lift_gt_case_inputs(ci)
        bodies[ci, :len(b)] = b
        counts[ci] = len(b)
        dd[ci], rd[ci] = det_d, root_d
        sc = lift_numpy.default_scale(iw, ih)
        sc.update(f_x=gt[0, 0, 7], f_y=gt[0, 0, 8], cx=gt[0, 0, 9], cy=gt[0, 0, 10])  # test.py:91-95
        scales[ci] = scale_row(sc)
        gt_roots[ci, :len(gt)] = gt[:, 2, :2]
        gt_counts[ci] = len(gt)
    t = lambda a: torch.from_numpy(a).cuda()  # noqa: E731
    p2, p3, rdp, co = eng.lift_gt(t(bodies), t(counts), t(dd), t(rd), t(scales), t(gt_roots), t(gt_counts))
    torch.cuda.synchronize()
    p2, p3, rdp, co = p2.cpu().numpy(), p3.cpu().numpy(), rdp.cpu().numpy(), co.cpu().numpy()
    matched = 0
    for ci in range(B):
        g2, g3, gr = gold["c%d_pred2d" % ci], gold["c%d_pred3d" % ci], gold["c%d_rootdepth" % ci]
        n = len(g2)
        assert int(co[ci]) == n, ci
        assert np.array_equal(p2[ci, :n], g2), ci                     # float64 rows, bit for bit
        assert np.array_equal(rdp[ci, :n], gr), ci
        np.testing.assert_allclose(p3[ci, :n], g3, rtol=1e-12, atol=1e-12)
        assert not p2[ci, n:].any() and not p3[ci, n:].any()
        matched += int((g2[:, 2, 3] != 0).sum())
    assert matched >= 10
    eng.close()


@pytest.mark.parametrize("h,w,persons", [(256, 256, 12), (64, 96, 3), (128, 208, 15)])
def test_association_at_runtime_map_size_is_bit_exact(h, w, persons):
    """NMS (cluster of row bands), PAF scoring (gathers from global memory when the planes exceed shared memory) and
    grouping at (h, w) != 128x208."""
    from smap_b200.engine import Engine

    eng = Engine(0, max_batch=2, in_h=4 * h, in_w=4 * w)
    ss = [make_scene(300 + i, persons, h=h, w=w) for i in range(2)]
    hms = np.stack([s["hms"] for s in ss])
    rd = np.stack([s["root_d"] for s in ss])
    rng = np.random.default_rng(5)
    hms[1, :15] += rng.normal(0, 0.08, hms[1, :15].shape).astype(np.float32)  # plenty of spurious peaks in frame 1
    hd, rdd = torch.from_numpy(hms).cuda(), torch.from_numpy(rd).cuda()
    peaks, scores = eng.extract(hd)
    bodies, counts = eng.connect(hd, rdd)
    torch.cuda.synchronize()
    for i in range(2):
        rb, rp, rs = assoc.connect(hms[i], rd[i], return_all=True)
        _, rs_dense = assoc.extract(hms[i])
        assert np.array_equal(peaks[i].cpu().numpy(), rp), "peaks frame %d" % i
        assert np.array_equal(scores[i].cpu().numpy(), rs_dense), "pair scores frame %d" % i
        n = int(counts[i])
        assert n == len(rb)
        assert np.array_equal(bodies[i, :n].cpu().numpy(), rb)
    eng.close()


def test_whole_path_at_1024x1024_config5_end_to_end():
    """Config 5 beyond the backbone: smapb_infer_device on a 1024x1024 frame (256x256 maps) equals the oracle association +
    lift run on the backbone tensors the same handle produced."""
    from smap_b200.engine import Engine, records_to_numpy, scale_row
    from oracle import smap_torch

    eng = Engine(0, max_batch=1, in_h=1024, in_w=1024)
    eng.load_state_dict(schema.make_state_dict(0, "identity"))
    x = schema.make_input(1, 1024, 1024, seed=9).cuda()
    sc = lift_numpy.default_scale(2048, 2048, net_w=1024, net_h=1024)
    scales = torch.from_numpy(scale_row(sc)[None]).cuda()
    rec = records_to_numpy(eng.infer_device(x, scales))
    hm, dd, rd = eng.forward(x)
    torch.cuda.synchronize()
    hms = smap_torch.rescale_reference_cuda(hm.clone())
    bodies = assoc.connect(hms[0].cpu().numpy(), rd[0, 0].cpu().numpy())
    p2, p3, rdep = lift_numpy.lift(bodies, dd[0].cpu().numpy(), rd[0, 0].cpu().numpy(), sc)
    n = int(rec["count"][0])
    assert n == len(p2) and n > 0
    assert np.array_equal(rec["pred2d"][0, :n], p2)
    np.testing.assert_allclose(rec["pred3d"][0, :n], p3, rtol=1e-12, atol=1e-12)
    eng.close()
