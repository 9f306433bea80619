"""The reference of the whole-path tests (tests/test_path_state_gpu.py, tests/dist_worker.py): the records of one call,
computed stage by stage on a handle of their own, and calls whose content differs from every other call.

stagewise_records runs Engine.forward, forward(flip(x)) and merge_scale when flipping, connect, lift and refine when
refinement is on, and packs the results into RECORD_DTYPE.  None of those stage calls is captured into a graph or looked
up in a cache, and none writes records_dev, rec_buf, gather_dev or a slot, so a record that reached the caller through
the wrong graph or the wrong buffer cannot equal it by construction.  tests/test_pipeline_gpu.py,
tests/test_plan_geometry_gpu.py and tests/test_refine_gpu.py hold the stages themselves to the oracle chain; the
criterion here is byte equality, without tolerances.

Calls hands out the calls.  Every call has its own frames (schema.make_input of its own seed plus seeded 8x8 blocks of
Gaussian noise, which is what gives random weights people to find) and its own scale rows (img_width, f_x and cx vary
per frame, so pred3d differs even for equal frames).  It asserts that every frame it hands out has at least one person
and that no two references it handed out are equal: a test in which two calls expect the same bytes cannot tell them
apart.

Not a test module: it makes no CUDA call at import."""
import hashlib

import numpy as np
import torch

from smap_b200 import schema
from smap_b200.engine import RECORD_BYTES, RECORD_DTYPE, scale_row

H, W = 96, 160  # a few ms per forward; tests/test_plan_geometry_gpu.py pins the whole path at this size to the oracle


def make_call(seed, B, h=H, w=W):
    """-> (frames fp32 cpu [B,3,h,w], scale rows float64 cpu [B,9]) of call `seed`; no two seeds share a frame or a row."""
    g = torch.Generator().manual_seed(100000 + seed)
    blocks = torch.kron(torch.randn(B, 3, h // 8, w // 8, generator=g), torch.ones(8, 8))
    x = (schema.make_input(B, h, w, seed=seed) + blocks).contiguous()
    rows = []
    for b in range(B):
        k = seed * 8 + b
        img_w, img_h = 4 * w + 16 * (k % 13), 4 * h
        rows.append(scale_row(dict(scale=min(w / img_w, h / img_h), img_width=img_w, img_height=img_h, net_width=w,
                                   net_height=h, f_x=img_w * (1 + 0.003 * (k % 17)), f_y=float(img_w),
                                   cx=img_w / 2 + k % 11, cy=img_h / 2)))
    return x, torch.from_numpy(np.stack(rows))


def stagewise_records(ref, x, scales, do_flip=False, refine=False):
    """Records of one batch through the stage-wise API of `ref` (a handle no whole-path call is made on), on torch's
    current stream -> uint8 cpu [B, RECORD_BYTES]."""
    x, scales = x.to(ref.device), scales.to(ref.device)
    B = x.shape[0]
    hm, dd, rd = ref.forward(x)
    hm_f = ref.forward(torch.flip(x, [-1]).contiguous())[0] if do_flip else None
    ref.merge_scale(hm, hm_f, True)
    bodies, counts = ref.connect(hm, rd)
    p2, p3, rdep, cnt = ref.lift(bodies, counts, dd, rd, scales)
    if refine:
        p3 = ref.refine(p2, p3, cnt)
    rec = np.zeros(B, RECORD_DTYPE)  # pad_ stays 0, as the lift kernel stores it in a record
    rec["pred3d"], rec["root_depth"] = p3.cpu().numpy(), rdep.cpu().numpy()
    rec["pred2d"], rec["count"] = p2.cpu().numpy(), cnt.cpu().numpy()
    return torch.from_numpy(rec.view(np.uint8).reshape(B, RECORD_BYTES))


class Calls:
    """Distinct calls and their references.  ref: the stage-wise handle (weights loaded; RefineNet weights too when any
    call refines)."""

    def __init__(self, ref, h=H, w=W, first_seed=1):
        self.ref, self.h, self.w, self.seed = ref, h, w, first_seed
        self.seen = {}

    def _hand_out(self, want, what):
        digest = hashlib.sha256(want.numpy().tobytes()).digest()
        tag = "reference %d (%s)" % (len(self.seen), what)
        assert digest not in self.seen, "%s has the bytes of %s" % (tag, self.seen.get(digest))
        self.seen[digest] = tag
        return want

    def reference(self, x, scales, do_flip=False, refine=False):
        """stagewise_records of given content, checked: a person in every frame, and bytes no earlier reference had."""
        want = stagewise_records(self.ref, x, scales, do_flip, refine)
        persons = want.numpy().view(RECORD_DTYPE)["count"].reshape(-1)
        assert (persons > 0).all(), "a frame without a person makes an all-zero record: %s" % persons
        return self._hand_out(want, "B=%d flip=%d refine=%d" % (x.shape[0], do_flip, refine))

    def new(self, B, do_flip=False, refine=False):
        """-> (frames cpu, scale rows cpu, reference records cpu) of a call no other shares content with.  Seeds whose
        frames hold nobody are passed over: an empty frame's record is all zeros whatever path it took."""
        for _ in range(64):
            x, scales = make_call(self.seed, B, self.h, self.w)
            self.seed += 1
            want = stagewise_records(self.ref, x, scales, do_flip, refine)
            if (want.numpy().view(RECORD_DTYPE)["count"].reshape(-1) > 0).all():
                return x, scales, self._hand_out(want, "seed %d B=%d flip=%d refine=%d" % (self.seed - 1, B, do_flip, refine))
        raise AssertionError("no seed in 64 gave %d frames with a person each" % B)
