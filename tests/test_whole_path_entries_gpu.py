"""GPU: the whole-path entry points of smap_b200/csrc/engine.cu (smapb_infer_device[_gather[_async]], smapb_infer_host,
smapb_submit_host[_gather]) - the launch count of a graph replay, and calls the argument check refuses.

launch_count() is what bench.py reports as its launches per step.  A graph replay adds the launches counted while its
graph was captured, so every call of one kind adds the same number whether it runs eagerly, is captured or is replayed;
a count kept beside infer_body by hand would drift from the eager one with the next op added to the path.

A refused call returns before it changes anything: no launch, no handle state, so the calls after it return what they
return on a fresh handle."""
import ctypes
import os
import sys

import pytest
import torch

from smap_b200 import schema

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import path_check  # noqa: E402
from cases import refine_state_dict  # noqa: E402

pytestmark = pytest.mark.gpu
MB = 3


@pytest.fixture(scope="module")
def sd():
    return schema.make_state_dict(0, "identity")


def _engine(sd, refine=False):
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=MB, in_h=path_check.H, in_w=path_check.W)
    e.load_state_dict(sd)
    if refine:
        e.load_refine_state_dict(refine_state_dict())
        e.set_refine(True)
    return e


@pytest.mark.parametrize("refine", [False, True], ids=["plain", "refine"])
@pytest.mark.parametrize("form", ["infer_device", "submit_host"])
def test_a_replay_counts_the_launches_of_an_eager_call(sd, form, refine):
    """For B = 1 and 3, with and without do_flip: two eager calls, then captures and replays (submit_host: on both slots,
    whose buffers are two graph keys); the launch_count() delta of every call is the same."""
    from smap_b200.engine import RECORD_BYTES

    eng = _engine(sd, refine)
    try:
        seed = 1
        for B in (1, MB):
            for flip in (False, True):
                deltas = []
                for i in range(6):  # eager, eager, capture, capture or replay, replay, replay
                    x, s = path_check.make_call(seed, B)
                    seed += 1
                    before = eng.launch_count()
                    if form == "infer_device":
                        eng.infer_device(x.cuda(), s.cuda(), do_flip=flip)
                    else:
                        out = torch.zeros(B, RECORD_BYTES, dtype=torch.uint8).pin_memory()
                        eng.submit_host(i % 2, x.pin_memory(), s.pin_memory(), out, do_flip=flip)
                        eng.wait(i % 2)
                    deltas.append(eng.launch_count() - before)
                torch.cuda.synchronize()
                assert deltas[0] > 0 and deltas == [deltas[0]] * 6, (B, flip, deltas)
    finally:
        eng.close()


def test_refused_calls_change_nothing(sd):
    """B = 0, B = max_batch + 1, slot 2 and the gather forms without a communicator, on every entry that takes them: each
    returns its code and names the reason, launches nothing, and the valid calls that follow - infer_device, then
    submit_host on both slots - return the records a fresh handle returns."""
    from smap_b200.engine import RECORD_BYTES, RECORD_DTYPE

    eng, fresh = _engine(sd), _engine(sd)
    try:
        lib, h = eng.lib, eng._h
        x, s = path_check.make_call(1, MB)
        xd, sdev, xh, sh = x.cuda(), s.cuda(), x.pin_memory(), s.pin_memory()
        out_d = torch.zeros(MB + 1, RECORD_BYTES, dtype=torch.uint8, device="cuda")
        out_h = torch.zeros(MB + 1, RECORD_BYTES, dtype=torch.uint8).pin_memory()
        torch.cuda.synchronize()

        def p(t):
            return ctypes.c_void_p(t.data_ptr())

        def refused(rc, code, text, what):
            assert rc == code, (what, rc)
            assert text in lib.smapb_last_error(h).decode(), (what, lib.smapb_last_error(h))

        for B in (0, MB + 1):
            for fn in ("smapb_infer_device", "smapb_infer_host"):
                refused(getattr(lib, fn)(h, p(xd if fn == "smapb_infer_device" else xh),
                                         p(sdev if fn == "smapb_infer_device" else sh), B, 0,
                                         p(out_d if fn == "smapb_infer_device" else out_h), None),
                        -1, "B outside [1, max_batch]", (fn, B))
            for slot in (0, 1):
                refused(lib.smapb_submit_host(h, slot, p(xh), p(sh), B, 0, p(out_h)), -1, "B outside [1, max_batch]",
                        ("smapb_submit_host", slot, B))
        for slot in (-1, 2):
            for fn in ("smapb_submit_host", "smapb_submit_host_gather"):
                refused(getattr(lib, fn)(h, slot, p(xh), p(sh), MB, 0, p(out_h)), -1, "slot must be 0 or 1", (fn, slot))
        for fn in ("smapb_infer_device_gather", "smapb_infer_device_gather_async"):
            refused(getattr(lib, fn)(h, p(xd), p(sdev), MB, 0, p(out_d), None), -52, "no communicator", fn)
        refused(lib.smapb_submit_host_gather(h, 0, p(xh), p(sh), MB, 0, p(out_h)), -52, "no communicator",
                "smapb_submit_host_gather")
        assert eng.launch_count() == 0, "a refused call launched"
        assert lib.smapb_wait(h, 0) == -1 and lib.smapb_wait(h, 1) == -1, "a refused submission left a slot in use"

        got, want = eng.infer_device(xd, sdev).cpu(), fresh.infer_device(xd, sdev).cpu()
        assert got.numpy().view(RECORD_DTYPE)["count"].min() > 0, "every frame must have someone to compare"
        assert torch.equal(got, want), "infer_device after the refused calls"
        for slot in (0, 1):
            outs = [torch.zeros(MB, RECORD_BYTES, dtype=torch.uint8).pin_memory() for _ in range(2)]
            for e, o in zip((eng, fresh), outs):
                e.submit_host(slot, xh, sh, o)
                e.wait(slot)
            assert torch.equal(outs[0], outs[1]), "submit_host on slot %d after the refused calls" % slot
            assert torch.equal(outs[0], want), "submit_host on slot %d" % slot
    finally:
        eng.close()
        fresh.close()
