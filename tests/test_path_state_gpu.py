"""GPU: the host code that strings the kernels together - the graph cache, the handle-owned record buffers, the two-slot
host pipeline and the legacy-stream bridge of smap_b200/csrc/engine.cu - on one handle without a communicator.

A mistake in that code returns a correct record for the wrong input.  So every call here has its own frames and its own
scale rows (tests/path_check.py), and every result is compared byte for byte with the stage-wise reference of THAT call,
computed on a second handle that never runs the whole path.  The exchange half is in tests/dist_worker.py.

What these tests pin is which buffer and which graph a call uses, not timing.  A missing stream or event wait is not
reliably observable here (a copy takes microseconds, a forward milliseconds) and nothing below loops in the hope of a
race."""
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


def _engine(sd, precision="bf16x3", stream=None):
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=MB, in_h=path_check.H, in_w=path_check.W, stream=stream)
    e.load_state_dict(sd, precision)
    e.load_refine_state_dict(refine_state_dict())
    return e


@pytest.fixture(scope="module")
def sd():
    return schema.make_state_dict(0, "identity")


@pytest.fixture(scope="module")
def calls(sd):
    """The stage-wise handle and the calls it vouches for; one for the module, so that no two tests share content."""
    ref = _engine(sd)
    yield path_check.Calls(ref)
    ref.close()


@pytest.fixture()
def eng(sd):
    e = _engine(sd)
    yield e
    e.close()


def _warm(eng, calls, B, do_flip=False):
    """The two eager runs of (B, do_flip), checked like every other call; the next call of that kind is captured."""
    for _ in range(2):
        x, s, want = calls.new(B, do_flip)
        assert torch.equal(eng.infer_device(x.cuda(), s.cuda(), do_flip=do_flip).cpu(), want)


def test_every_field_of_the_graph_key_discriminates(eng, calls):
    """Graphs are keyed by (B, do_flip, gather, imgs, scales).  Calls that agree in all but one field are interleaved,
    each past its capture, and every one returns the records of its own content: a key that ignored the field would
    replay the other call's graph."""
    x1, s1, want11 = calls.new(MB)
    x2, s2, _ = calls.new(MB)
    x1, s1, x2, s2 = x1.cuda(), s1.cuda(), x2.cuda(), s2.cuda()
    variants = {  # name -> (imgs, scales, do_flip)
        # B = 1 is captured before B = 3 on the same pointers: the other way round, a key without B would replay three
        # frames for a call that wants the first of them, and be right
        "x1[:1] s1[:1]": (x1[:1], s1[:1], False), "x1 s1": (x1, s1, False), "x1 s2": (x1, s2, False), "x2 s1": (x2, s1, False),
        "x1 s1 flip": (x1, s1, True), "x1[:1] s1[:1] flip": (x1[:1], s1[:1], True),
    }
    assert x1[:1].data_ptr() == x1.data_ptr() and s1[:1].data_ptr() == s1.data_ptr()
    want = {k: want11 if k == "x1 s1" else calls.reference(x, s, f) for k, (x, s, f) in variants.items()}
    for B in (MB, 1):
        for flip in (False, True):
            _warm(eng, calls, B, flip)
    order = list(variants)
    for rnd in range(3):  # capture, replay, replay - in an order that changes, so each graph follows each other one
        for k in order:
            x, s, f = variants[k]
            assert torch.equal(eng.infer_device(x, s, do_flip=f).cpu(), want[k]), "round %d: %s" % (rnd, k)
        order = order[1::2] + order[0::2]


def test_replay_reads_the_tensors_as_they_are_now(eng, calls):
    """A graph holds pointers, not content: after copy_ into a captured imgs tensor, and into a captured scales tensor,
    the replay returns the records of what the tensors hold now."""
    _warm(eng, calls, MB)
    x, s, want = calls.new(MB)
    x, s = x.cuda(), s.cuda()
    for _ in range(2):  # capture, replay
        assert torch.equal(eng.infer_device(x, s).cpu(), want)
    x2, s2, want2 = calls.new(MB)
    x.copy_(x2)
    assert torch.equal(eng.infer_device(x, s).cpu(), calls.reference(x, s)), "imgs overwritten in place"
    s.copy_(s2)
    assert torch.equal(eng.infer_device(x, s).cpu(), want2), "scales overwritten in place"


def test_eviction_beyond_16_graphs_never_returns_another_entrys_records(eng, calls):
    """18 pointer pairs with distinct content through the 16-entry cache, each used three times, pair 0 once more before
    pairs 16 and 17 push entries out, then all of them again in other orders: a pair never gets the records of another
    pair's graph, or of one that was destroyed.  This does not pin WHICH entry is evicted.  The policy (least recently
    used) only decides what is captured again; no record depends on it and the ABI shows nothing else, so a cache that
    evicted the oldest entry instead would pass."""
    _warm(eng, calls, 1)
    pairs = []

    def use(i, times):
        x, s, want = pairs[i]
        for t in range(times):
            assert torch.equal(eng.infer_device(x, s).cpu(), want), "pair %d, use %d" % (i, t)

    for i in range(18):
        if i == 16:
            use(0, 1)
        x, s, want = calls.new(1)
        pairs.append((x.cuda(), s.cuda(), want))
        use(i, 3)
    for i in (0, 1, 2, 17, 16, 3, 0):
        use(i, 1)
    for i in reversed(range(18)):
        use(i, 1)


def test_set_refine_drops_the_graphs_captured_without_it(eng, calls):
    _warm(eng, calls, MB)
    x, s, plain = calls.new(MB)
    x, s = x.cuda(), s.cuda()
    refined = calls.reference(x, s, refine=True)
    for _ in range(2):
        assert torch.equal(eng.infer_device(x, s).cpu(), plain)
    eng.set_refine(True)
    for _ in range(2):
        assert torch.equal(eng.infer_device(x, s).cpu(), refined), "same pointers after set_refine(True)"
    eng.set_refine(False)
    for _ in range(2):
        assert torch.equal(eng.infer_device(x, s).cpu(), plain), "same pointers after set_refine(False)"


def test_new_weights_and_another_precision_replace_live_graphs(eng, calls):
    """load_state_dict a second and a third time on a handle with captured graphs - the same weights in another
    precision, then other weights: the same pointers give what a fresh handle with those weights gives, stage by
    stage.  The other weights are seed 0's with the depth heads of seed 1: a whole state dict of another seed, or one
    with random BatchNorm statistics, finds nobody in these frames, and an all-zero record proves little."""
    _warm(eng, calls, MB)
    x, s, want = calls.new(MB)
    x, s = x.cuda(), s.cuda()
    for _ in range(2):
        assert torch.equal(eng.infer_device(x, s).cpu(), want)
    seen = [want]
    sd0, sd1 = schema.make_state_dict(0, "identity"), schema.make_state_dict(1, "identity")
    heads = [k for k in sd0 if "res_d_conv2.conv" in k or "res_rd_conv2.conv" in k]
    assert len(heads) == 2 * 2 * 4 * 3  # weight and bias of both depth heads, four levels, three stages
    other = dict(sd0, **{k: sd1[k] for k in heads})
    for sd2, precision in ((sd0, "fp16"), (other, "bf16")):
        fresh = _engine(sd2, precision)
        try:
            want2 = path_check.Calls(fresh).reference(x, s)
        finally:
            fresh.close()
        assert not any(torch.equal(want2, w) for w in seen), "the new weights must show in the records"
        seen.append(want2)
        eng.load_state_dict(sd2, precision)
        for i in range(4):  # eager, eager, capture, replay
            assert torch.equal(eng.infer_device(x, s).cpu(), want2), "%s, call %d after the reload" % (precision, i)


def test_a_profiled_call_between_replays_changes_nothing(eng, calls):
    _warm(eng, calls, MB)
    xa, sa, wa = calls.new(MB)
    xb, sb, wb = calls.new(MB)
    xa, sa, xb, sb = xa.cuda(), sa.cuda(), xb.cuda(), sb.cuda()
    for _ in range(2):
        assert torch.equal(eng.infer_device(xa, sa).cpu(), wa)
    eng.profile_begin()
    got = eng.infer_device(xb, sb).cpu()  # eager, whatever the cache holds
    by_kind = eng.profile_end()
    assert torch.equal(got, wb)
    assert by_kind["conv"][1] > 0 and by_kind["lift"][1] == 1
    assert torch.equal(eng.infer_device(xa, sa).cpu(), wa), "replay after the profiled call"
    for _ in range(2):
        assert torch.equal(eng.infer_device(xb, sb).cpu(), wb), "capture and replay of the profiled call's pointers"


def test_host_pipeline_with_distinct_batches_both_sizes_and_the_other_entry_points_between(eng, calls):
    """submit_host on slots 0 and 1 alternately, every batch with its own content and B going 3, 3, 1, 1, 3, ... so that
    each slot sees both sizes, while infer_host and infer_device run on the same handle between submissions.  All of
    them share records_dev and the graph cache; a slot's buffers are keyed into that cache too, by pointer and by B."""
    from smap_b200.engine import RECORD_BYTES

    n = 10
    batches = []
    for i in range(n):
        x, s, want = calls.new(MB if (i // 2) % 2 == 0 else 1)
        out = torch.zeros(x.shape[0], RECORD_BYTES, dtype=torch.uint8).pin_memory()
        batches.append((x.pin_memory(), s.pin_memory(), out, want))
    xd, sdev, wd = calls.new(MB)
    xd, sdev = xd.cuda(), sdev.cuda()
    xh, sh, wh = calls.new(1)
    xh = xh.pin_memory()
    h = eng._h
    assert eng.lib.smapb_wait(h, 0) == -1 and eng.lib.smapb_wait(h, 1) == -1, "nothing submitted yet"
    assert b"nothing submitted" in eng.lib.smapb_last_error(h)
    for slot in (-1, 2):
        assert eng.lib.smapb_wait(h, slot) == -1
        assert eng.lib.smapb_submit_host(h, slot, ctypes.c_void_p(batches[0][0].data_ptr()),
                                         ctypes.c_void_p(batches[0][1].data_ptr()), MB, 0,
                                         ctypes.c_void_p(batches[0][2].data_ptr())) == -1
        assert b"slot must be 0 or 1" in eng.lib.smapb_last_error(h)
    for i, (x, s, out, _) in enumerate(batches):
        slot = i % 2
        if i >= 2:
            eng.wait(slot)  # the previous occupant of the slot; its records stay in its own `out`
        eng.submit_host(slot, x, s, out)
        if i % 3 == 1:  # batch i is in flight on the handle's stream
            assert torch.equal(eng.infer_device(xd, sdev).cpu(), wd), "infer_device after submission %d" % i
        if i % 3 == 2:
            assert eng.infer_host(xh, sh).tobytes() == wh.numpy().tobytes(), "infer_host after submission %d" % i
    eng.wait(0)
    eng.wait(1)
    for i, (_, _, out, want) in enumerate(batches):
        assert torch.equal(out, want), "batch %d (slot %d, B=%d)" % (i, i % 2, out.shape[0])


def test_default_stream_calls_equal_explicit_stream_calls_while_a_side_stream_is_busy(sd, eng, calls):
    """stream = NULL is torch's default stream: the library bridges it to the handle's own stream and back.  One round
    of eager, eager, capture, replay, with another stream kept busy, against a handle that issues on an explicit
    stream."""
    from smap_b200.engine import RECORD_BYTES

    st = torch.cuda.Stream()
    e2 = _engine(sd, stream=st)
    side = torch.cuda.Stream()
    big = torch.randn(32 * 1024 * 1024, device="cuda")
    torch.cuda.synchronize()
    try:
        with torch.cuda.stream(side):
            for _ in range(40):
                big * 1.0001 + 1.0
        for _ in range(4):
            x, s, want = calls.new(MB)
            x, s = x.cuda(), s.cuda()  # on the default stream, which the NULL-stream call is ordered after
            got = eng.infer_device(x, s)
            out = torch.zeros(MB, RECORD_BYTES, dtype=torch.uint8, device="cuda")
            st.wait_stream(torch.cuda.current_stream())
            e2.infer_device(x, s, out=out)
            st.synchronize()
            assert torch.equal(got.cpu(), want), "default stream"
            assert torch.equal(out.cpu(), want), "explicit stream"
    finally:
        torch.cuda.synchronize()
        e2.close()
