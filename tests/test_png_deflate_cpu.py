"""CPU: the DEFLATE writer (tests/golden/deflate_writer.py) and the block oracle (oracle/inflate_numpy.py) on streams zlib's
deflate never writes.  zlib inflates every file to the writer's scanlines, the oracle reports the block structure the
writer meant, cv2 reads each file to the pixels of the same scanlines compressed by zlib (or refuses it where it must),
the PNG oracle agrees with cv2, and the vectorised finder agrees with its one-offset rule."""
import zlib

import numpy as np
import pytest

from deflate_writer import COUNT_MAX_SYMBOLS, blk_cap, cand_cap, cases
from oracle import inflate_numpy as Z
from oracle import png_numpy as P

cv2 = pytest.importorskip("cv2")

PAST_WINDOW = {"cinfo0_distance_300"}  # the oracle, like the device, refuses a distance past the declared window


def cv2_read(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


@pytest.fixture(scope="module")
def files():
    return cases()


def test_the_set_holds_every_kind_of_file(files):
    names = {c.name for c in files}
    assert len(files) > 300 and len(names) == len(files)
    kinds = {e: sum(c.expect == e for c in files) for e in ("decode", "device_refuses", "both_refuse")}
    assert kinds["device_refuses"] == 3 and kinds["both_refuse"] == 4, kinds
    for c in files:
        assert c.expect in kinds, c.name


def test_zlib_inflates_every_stream_to_the_writers_scanlines(files):
    for c in files:
        if c.expect == "both_refuse":
            with pytest.raises(zlib.error):
                zlib.decompress(c.z)
        else:
            assert zlib.decompress(c.z) == c.raw, c.name


def test_block_oracle_reports_the_intended_structure(files):
    residues = {0: set(), 1: set(), 2: set()}
    pads = set()
    for c in files:
        if c.expect == "both_refuse" or c.name in PAST_WINDOW:
            with pytest.raises(ValueError):
                Z.blocks(c.z)
            continue
        data, blocks = Z.blocks(c.z)
        assert data == c.raw, c.name
        assert [(k.type, k.start, k.syms, k.final) for k in blocks] == [tuple(r) for r in c.blocks], c.name
        assert blocks[-1].final and not any(k.final for k in blocks[:-1]), c.name
        for k in blocks:
            residues[k.type].add(k.start % 32)
            if k.type == 0:
                pads.add((8 - (k.start + 3) % 8) % 8)
    assert residues[1] == residues[2] == set(range(32)), residues
    assert {0, 7} <= pads, pads
    by = {c.name: c for c in files}
    syms = [k.syms for k in Z.blocks(by["symbols_65536_then_65537"].z)[1]]
    assert syms[:2] == [COUNT_MAX_SYMBOLS, COUNT_MAX_SYMBOLS + 1]
    for name, extra in (("blocks_eq_blk_cap_plus_0", 0), ("blocks_eq_blk_cap_plus_1", 1)):
        assert len(Z.blocks(by[name].z)[1]) == blk_cap(len(by[name].z)) + extra
    flush = by["partial_flush_200_empty_blocks"].z
    assert len(Z.blocks(flush)[1]) == 201 and len(flush) == 281


def test_header_fields_and_code_shapes_zlib_never_writes(files):
    """HCLEN 5..19 with trailing zero code-length lengths, an EOB-only literal code, runs across the literal/distance
    boundary and 15-bit literal and distance codes are in the set."""
    by = {c.name: c for c in files}
    z = by["hclen_5_to_19_eob_only_literal_only"].z
    hclens = []
    for k in Z.blocks(z)[1]:
        b = Z.Bits(z)
        b.p = k.start + 13
        hclens.append(b.get(4) + 4)
    assert hclens[:15] == list(range(5, 20))
    assert not Z.finder_accepts(z, Z.blocks(z)[1][15].start)  # the EOB-only code is incomplete
    for name in ("cross_boundary_16", "cross_boundary_17", "cross_boundary_18", "codes_of_15_bits"):
        b = Z.Bits(by[name].z)
        b.p = 19
        lit, dist = Z.dyn_lengths(b)
        if name == "codes_of_15_bits":
            assert max(lit) == 15 and max(dist) == 15
        else:
            assert lit[-1] == dist[0], name  # the run that crosses repeats the same length


def test_cv2_reads_each_file_as_zlib_would_and_refuses_the_broken_ones(files):
    for c in files:
        got = cv2_read(c.png)
        if c.expect == "both_refuse":
            assert got is None, c.name
            continue
        ref = cv2_read(c.ref_png)
        assert ref is not None and got is not None and np.array_equal(got, ref), c.name


def test_png_oracle_agrees_with_cv2(files):
    for c in files:
        st, got = P.decode(c.png)
        ref = cv2_read(c.png)
        if ref is None:
            assert st != P.OK, c.name
        else:
            assert st == P.OK and np.array_equal(got, ref), c.name


def test_candidates_agree_with_the_one_offset_rule(files):
    rng = np.random.default_rng(4)
    by = {c.name: c for c in files}
    for c in [by["candidate_flood"], by["symbols_65536_then_65537"], by["codes_of_15_bits"]] + files[-40:]:
        z = c.z
        cand = Z.candidates(z)
        assert cand == sorted(cand)
        cs = set(cand)
        sample = set(rng.integers(16, 8 * len(z) - 16, 3000).tolist()) | set(cand[:200]) | {p + 1 for p in cand[:50]}
        for p in sample:
            assert (p in cs) == Z.finder_accepts(z, p), (c.name, p)
        if c.expect == "decode" and c.name not in PAST_WINDOW:
            for k in Z.blocks(z)[1]:
                if k.type == 2:
                    b = Z.Bits(z)
                    b.p = k.start + 3
                    lit = Z.dyn_lengths(b)[0]
                    complete = sum(1 << (15 - l) for l in lit if l) == 1 << 15
                    assert (k.start in cs) == complete, (c.name, k)
    flood = by["candidate_flood"]
    assert len(Z.candidates(flood.z)) > cand_cap([len(flood.z)])


def test_predicted_stats_count_every_chained_block(files):
    for c in files[:30]:
        if c.expect != "decode":
            continue
        st = Z.predicted_stats(c.z)
        blocks = Z.blocks(c.z)[1]
        assert st["confirmed"] + st["serial"] == len(blocks), c.name
        assert st["candidates"] - st["false_positives"] <= sum(k.type == 2 for k in blocks), c.name
    by = {c.name: c for c in files}
    assert Z.predicted_stats(by["symbols_65536_then_65537"].z) == dict(candidates=2, false_positives=0, confirmed=1,
                                                                       serial=2)
