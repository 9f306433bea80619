"""CPU: the files of tests/golden/jpeg_writer.py (baseline streams libjpeg never writes) have the outcome each is listed
with: cv2 reads every file the decoder must decode to the oracle's pixels, smapb_jpeg_info and the oracle give the
status of every refused file, and cv2 reads the files the decoder leaves to it.  The CPU model of the sync passes puts
the adversaries at their worst case and cv2's files within one group of passes."""
import numpy as np
import pytest

import jpeg_writer as W
from oracle import jpeg_numpy as J

cv2 = pytest.importorskip("cv2")
pytest.importorskip("PIL")

SMALL = 1 << 16  # files the oracle's Python entropy decoder also decodes (bytes)


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


@pytest.fixture(scope="module")
def fams():
    return W.families()


def test_families_cover_what_they_claim(fams):
    dense = sum(len(e["coef"]) for e in fams["dense"])
    assert dense >= 100000, dense
    assert {e["name"].split("_")[1] for e in fams["dense"]} == set(W.SAMPLINGS)
    pairs = set()
    for e in fams["colour"]:
        c = e["coef"]
        assert (c[:, 1:] == 0).all()
        pairs |= set(zip(c[1::3, 0].tolist(), c[2::3, 0].tolist()))
    assert len(pairs) == 1 << 16 and len(fams["colour"]) == 16  # every (Cb, Cr) at 16 luma levels: 2^20 blocks
    names = {e["name"] for f in fams.values() for e in f}
    assert len(names) == sum(len(f) for f in fams.values())
    for s in ("420", "422", "440"):
        assert {"up_%s_%dx%d" % (s, w, h) for w in range(1, 9) for h in range(1, 9)} <= names
    outcomes = {e["expect"] for f in fams.values() for e in f}
    assert outcomes == {W.DECODE, J.UNSUPPORTED, J.MALFORMED, J.CORRUPT}


def test_dense_blocks_fill_the_guard_and_saturate(fams):
    for e in fams["dense"]:
        hd = J.parse(e["data"])
        lay = np.tile(J.mcu_layout(hd), hd["nmcu"])
        c = e["coef"]
        assert (c != 0).all(), e["name"]
        top = []
        for k, q in enumerate(hd["qt"]):
            dq, p1 = W.pass1(c[lay == k], q)
            assert dq.max() <= J.GUARD and p1.max() <= J.GUARD, e["name"]
            top.append(np.median(p1))
        assert min(top) > 0.85 * J.GUARD, (e["name"], top)
        img = cv2_read(e["data"])
        assert img.min() == 0 and img.max() == 255, e["name"]


def test_stuffed_bytes_fall_at_every_word_offset(fams):
    """FF00 pairs at every byte offset within a 32-bit word and at every byte of a 64-byte (512-bit) subsequence, in
    the unstuffed data the device decodes."""
    offs = set()
    for e in fams["dense"]:
        d = e["data"]
        for a, b in J.parse(d)["segments"]:
            u = np.frombuffer(d[a:b].replace(b"\xff\x00", b"\xff"), np.uint8)
            offs |= set((np.flatnonzero(u == 0xFF) % 64).tolist())
    assert offs == set(range(64))


@pytest.mark.parametrize("family", ["dense", "guard", "colour", "upsampling", "huffman", "sync"])
def test_outcomes(fams, family):
    from smap_b200.engine import jpeg_info

    for e in fams[family]:
        name, b, expect = e["name"], e["data"], e["expect"]
        st, h, w, _ = jpeg_info(b)
        assert (st, h, w, _) == J.info(b), name
        ref = cv2_read(b)
        if expect == J.MALFORMED:  # a table libjpeg refuses: cv2 fails, the decoder refuses at the header
            assert st == J.MALFORMED and ref is None, name
            continue
        assert ref is not None, name  # everything else cv2 reads
        if expect == J.UNSUPPORTED and st != 0:  # refused at the header
            continue
        assert st == 0 and (h, w) == ref.shape[:2], (name, st)
        if expect == W.DECODE:
            if e["coef"] is not None:
                hd = J.parse(b)
                got = J.colour(J.idct_planes(np.asarray(e["coef"], np.int16), hd), hd)
                assert np.array_equal(got, ref), name
            if len(b) <= SMALL or e["coef"] is None:
                assert np.array_equal(J.decode(b), ref), name
        else:  # refused on the device: the guard, a run past coefficient 63
            with pytest.raises(J.NotDecoded) as x:
                J.decode(b)
            assert x.value.status == expect, (name, str(x.value))


def test_writer_codes_the_coefficients(fams):
    """The oracle's entropy decoder gives back the coefficients each small file was written from."""
    n = 0
    for f in fams.values():
        for e in f:
            if e["coef"] is None or len(e["data"]) > SMALL or J.info(e["data"])[0] != 0:
                continue
            hd = J.parse(e["data"])
            assert np.array_equal(J.entropy_decode(e["data"], hd), e["coef"]), e["name"]
            n += 1
    assert n > 250


def test_sync_adversaries_reach_the_worst_case(fams):
    for e in fams["sync"]:
        for sb in W.SUB_BITS:
            P = W.predicted_passes(e["data"], sb)
            assert P["first_quiet"] <= P["bound"] <= max(P["nsub_seg"]) + 1, (e["name"], sb, P)
            if sb == e["sub_bits"]:
                assert P["worst"], (e["name"], P)
    ns = {(e["sub_bits"], n) for e in fams["sync"] for n in W.predicted_passes(e["data"], e["sub_bits"])["nsub_seg"]}
    for sb in W.SUB_BITS:
        assert {1, 8, 9, 16} <= {n for s, n in ns if s == sb}, sb
    quiet = {W.predicted_passes(e["data"], e["sub_bits"])["first_quiet"] % 2 for e in fams["sync"] if e["sub_bits"] == 512}
    assert quiet == {0, 1}  # the final pass reads either state buffer


def test_cv2_files_schedule():
    """cv2's flat files converge in pass 1 or 2 at the default 512-bit subsequences.  Dense ones need not converge
    within one group of 8: at 61x37, noise and checkerboards at q50-q100 and optimised tables take 9 to 90 passes
    (61x37 q100 checkerboard in 4:4:4: 90 of a possible 92); GPU tests pin the exact counts."""
    from jpeg_corpus import corpus

    slow = 0
    for name, b in corpus():
        P = W.predicted_passes(b, 512)
        assert P["first_quiet"] <= P["bound"], name
        if "_flat_" in name:
            assert P["first_quiet"] <= 2, (name, P)
        slow += P["first_quiet"] >= W.PASS_GROUP
    assert 0 < slow < 40


def test_model_counts_the_host_loop():
    """Launches for a first quiet pass q and a longest segment of n subsequences: groups of 8, capped at n + 2."""
    e = W.sync_adversaries()
    for x in e:
        P = W.predicted_passes(x["data"], x["sub_bits"])
        n, q = max(P["nsub_seg"]), P["first_quiet"]
        assert P["passes"] == min(W.PASS_GROUP * (q // W.PASS_GROUP + 1), n + 2), x["name"]
        assert P["launches"] == P["passes"] + W.FIXED_LAUNCHES
