"""CPU: the C-ABI library builds, loads and exports every symbol include/smap_b200.h declares.
No compute call is made (no GPU here)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "smap_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(smapb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from smap_b200 import _lib, build

    build.build()
    lib = _lib.load()
    syms = declared_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), "missing export: " + s
    assert set(_lib.EXPORTS) == set(syms)
    assert lib.smapb_version() >= 100


def test_debug_header_symbols_are_exported_too():
    from smap_b200 import _lib

    src = open(os.path.join(ROOT, "include", "smap_b200_debug.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    syms = sorted(set(re.findall(r"\b(smapb_debug_[a-z0-9_]+)\s*\(", src)))
    assert syms == ["smapb_debug_checksums", "smapb_debug_dump", "smapb_debug_resize_plan"]
    lib = _lib.load()
    for s in syms:
        assert hasattr(lib, s), "missing export: " + s


def test_record_layout_matches_header():
    from smap_b200 import _lib, engine

    assert engine.RECORD_DTYPE.itemsize == _lib.RECORD_BYTES == 127 * 15 * 4 * 8 + 127 * 8 + 127 * 15 * 4 * 4 + 8
    assert engine.RECORD_DTYPE.fields["root_depth"][1] == 127 * 15 * 4 * 8
    assert engine.RECORD_DTYPE.fields["pred2d"][1] == 127 * 15 * 4 * 8 + 127 * 8


def test_engine_fails_loudly_without_gpu():
    import torch

    from smap_b200 import engine

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(engine.SmapB200Error):
        engine.Engine()


def test_create_reports_error_without_device():
    import ctypes

    import torch

    from smap_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    h = ctypes.c_void_p()
    rc = lib.smapb_create(ctypes.byref(h), 0, 1, 512, 832)
    assert rc != 0 and not h.value
    assert len(lib.smapb_last_error(None)) > 0


def test_tile_table_roundtrip_is_process_wide():
    """smapb_set_tile_table / smapb_get_tile_table (no GPU): comments and malformed lines are skipped, entries overwrite."""
    from smap_b200 import _lib, engine

    lib = _lib.load()
    n = lib.smapb_set_tile_table(b"# comment\nGEOM_A k1\t128\t2\nbroken line\nGEOM_B\t64\t1\nGEOM_A k1\t256\t2\n")
    assert n == 3
    txt = engine.get_tile_table()
    rows = dict(l.split("\t", 1) for l in txt.strip().split("\n"))
    assert rows["GEOM_A k1"] == "256\t2" and rows["GEOM_B"] == "64\t1"


def test_committed_tile_table_covers_the_bench_and_smoke_batches():
    import os

    from smap_b200 import engine

    rows = [l for l in open(engine.TILE_TABLE_PATH).read().split("\n") if l and not l.startswith("#")]
    assert len(rows) > 100
    for l in rows:
        key, bn, cg = l.split("\t")
        assert int(bn) in (32, 64, 128) and int(cg) == 1  # the tile shapes conv_tc_kernel is built for
    assert any(" 8x128x208 " in l for l in rows) and any(" 1x128x208 " in l for l in rows)
