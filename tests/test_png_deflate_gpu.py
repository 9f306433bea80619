"""GPU: Engine.decode_png on DEFLATE streams zlib's deflate never writes (tests/golden/deflate_writer.py).  Every file it
must decode equals cv2 byte for byte, in one shuffled batch with the PNG corpus and one at a time; the files past its two
documented limits (block count, declared window) and the broken ones come back None; the inflate counters of each file
decoded alone equal the block oracle's prediction, so a change that sends blocks to the serial walk fails; a stream that
floods the block finder with candidates still decodes, alone and in a batch."""
import numpy as np
import pytest

from deflate_writer import blk_cap, cand_cap, cases
from png_corpus import corpus

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


@pytest.fixture(scope="module")
def eng():
    from smap_b200.engine import Engine

    e = Engine(0, max_batch=1)
    yield e
    e.close()


@pytest.fixture(scope="module")
def files():
    return cases()


def check(name, expect, b, g):
    if expect == "decode":
        assert g is not None, name
        g, ref = g.cpu().numpy(), cv2_read(b)
        assert g.shape == ref.shape and np.array_equal(g, ref), (name, int((g != ref).any(-1).sum()))
    else:
        assert g is None, (name, expect)


def test_adversarial_streams_equal_cv2_in_one_shuffled_batch_with_the_corpus_and_alone(eng, files):
    from smap_b200.engine import png_info

    batch = [(c.name, c.png, c.expect) for c in files] + [(n, b, "decode") for n, b in corpus()]
    order = np.random.default_rng(3).permutation(len(batch))
    batch = [batch[i] for i in order]
    got = eng.decode_png([b for _, b, _ in batch])
    for (name, b, expect), g in zip(batch, got):
        check(name, expect, b, g)
    for c in files:
        (g,) = eng.decode_png([c.png])
        check(c.name, c.expect, c.png, g)
        if c.expect == "device_refuses":
            assert png_info(c.png)[0] == 0, c.name  # the host walk accepts it: the refusal is the device's


def test_inflate_counters_equal_the_block_oracles_prediction(eng, files):
    from oracle import inflate_numpy as Z
    from oracle import png_numpy as P

    todo = [(c.name, c.png, c.expect) for c in files if c.name != "candidate_flood"]
    todo += [(n, b, "decode") for n, b in corpus() if len(P.parse(b)[1]["z"]) < 1 << 16]
    n_conf = n_serial = 0
    for name, b, expect in todo:
        if expect == "both_refuse":
            continue
        z = P.parse(b)[1]["z"]
        (g,) = eng.decode_png([b])
        st = eng.png_stats()
        if name == "cinfo0_distance_300":
            # count_kernel refuses the block (a distance past the window), so does the serial walk: nothing is chained
            want = dict(candidates=1, false_positives=0, confirmed=0, serial=0)
        else:
            want = Z.predicted_stats(z, max_blocks=blk_cap(len(z)) if expect == "device_refuses" else None)
        assert st == want, (name, st, want)
        n_conf += st["confirmed"]
        n_serial += st["serial"]
    assert n_conf > 1000 and n_serial > 1000, (n_conf, n_serial)


def test_candidate_flood_overflows_the_slots_and_equals_cv2(eng, files):
    from oracle import inflate_numpy as Z

    (c,) = [c for c in files if c.name == "candidate_flood"]
    (g,) = eng.decode_png([c.png])
    check(c.name, "decode", c.png, g)
    st = eng.png_stats()
    dyn = sum(k.type == 2 for k in Z.blocks(c.z)[1])
    # which candidates get a slot depends on the order of the finder's atomics: only bounds here
    assert st["candidates"] == len(Z.candidates(c.z)) > cand_cap([len(c.z)]), st
    assert st["confirmed"] < dyn and st["confirmed"] + st["serial"] == len(Z.blocks(c.z)[1]), st


def test_candidate_flood_leaves_the_other_files_of_its_batch_intact(eng, files):
    from oracle import png_numpy as P

    by = {c.name: c for c in files}
    batch = [by["candidate_flood"].png] + [c.png for c in files if c.name.startswith("sweep_")][:40]
    batch += [b for _, b in corpus()[:40]]
    got = eng.decode_png(batch)
    for i, (b, g) in enumerate(zip(batch, got)):
        check(i, "decode", b, g)
    assert eng.png_stats()["candidates"] > cand_cap([len(P.parse(b)[1]["z"]) for b in batch])
