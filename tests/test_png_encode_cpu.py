"""CPU: the PNG encoder oracle (oracle/png_encode_numpy.py) byte for byte against cv2.imencode(".png") and Python's zlib,
the window model it shares with png_enc.cu against a step-by-step replay of zlib's loop, png_enc.cu's registers, and the
run_inference --vis_format flag."""
import os
import struct
import sys
import zlib

import cv2
import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from png_encode_corpus import EXACT_SIZE, corpus, exact_frame, stream_len  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from oracle import png_encode_numpy as P  # noqa: E402
from smap_b200 import run_inference as ri  # noqa: E402

CORPUS = corpus()


def idat(png):
    p, z = 8, b""
    while p < len(png):
        n, = struct.unpack(">I", png[p:p + 4])
        if png[p + 4:p + 8] == b"IDAT":
            z += png[p + 8:p + 8 + n]
        p += 12 + n
    return z


@pytest.mark.parametrize("name,f", CORPUS, ids=[c[0] for c in CORPUS])
def test_oracle_equals_cv2(name, f):
    assert P.encode(f) == cv2.imencode(".png", f)[1].tobytes()


@pytest.mark.parametrize("name,f", [c for c in CORPUS if c[1].size < 10 ** 6], ids=[c[0] for c in CORPUS if c[1].size < 10 ** 6])
def test_stream_equals_python_zlib(name, f):
    """zlib.compressobj(1, DEFLATED, wbits, 8, Z_RLE) over the filtered stream, with libpng's header rewrite."""
    s = P.filtered(f)
    co = zlib.compressobj(1, zlib.DEFLATED, P.window_bits(len(s)), 8, zlib.Z_RLE)
    z = co.compress(s.tobytes()) + co.flush()
    assert P.zlib_stream(s) == bytes(P.zlib_header(len(s))) + z[2:]
    assert idat(P.encode(f)) == P.zlib_stream(s)


def test_corpus_covers_the_rules():
    kinds = {0: set(), 1: set(), 2: set()}
    wbits = set()
    for name, f in CORPUS:
        s = P.filtered(f)
        if len(s) > 300000:
            continue
        _, plans = P.plans(s)
        for p in plans:
            kinds[p["type"]].add(P.window_bits(len(s)))
        wbits.add(P.window_bits(len(s)))
    assert wbits == set(range(9, 16))
    assert len(kinds[0]) >= 5, "stored blocks under reduced windows"
    assert kinds[1] and kinds[2]
    s = P.filtered(exact_frame())
    assert len(s) == stream_len(*EXACT_SIZE)
    syms, plans = P.plans(s)
    assert len(syms) == P.BLOCK_SYMS and len(plans) == 2 and plans[1]["sym0"] == plans[1]["sym1"], "an empty final block"
    assert P.encode(np.zeros((1, 1, 3), np.uint8))[33 + 8:33 + 10] == b"\x08\x1d"


def test_runs_cross_rows():
    s = P.filtered(np.zeros((2000, 1, 3), np.uint8))
    syms, _ = P.parse(s)
    assert (syms == 256 + 255).sum() == (len(s) - 1) // 258  # 258-long matches over the whole column


def _replay_offsets(lengths, n, wsize):
    """zlib's deflate_rle loop with the whole input available, step by step: the window offset at each symbol start and
    at the end."""
    off, filled, p, out = 0, min(n, 2 * wsize), 0, []
    for ln in lengths + [0]:
        if filled - p <= P.MAX_MATCH:  # fill_window
            if p - off >= 2 * wsize - P.MIN_LOOKAHEAD:
                off += wsize
            filled = min(n, off + 2 * wsize)
        out.append((p, off))
        p += ln
    return out


def test_window_offset_matches_zlib_loop():
    rng = np.random.default_rng(3)
    for wsize in (512, 1024, 32768):
        for _ in range(20):
            n = int(rng.integers(1, 9 * wsize))
            lengths, left = [], n
            while left:
                ln = int(min(left, rng.choice([1, 1, 1, 3, 17, 258])))
                lengths.append(ln)
                left -= ln
            for p, off in _replay_offsets(lengths, n, wsize):
                assert P.window_offset(p, n, wsize) == off, (n, wsize, p)


def test_encoder_kernels_do_not_spill():
    """nvcc -Xptxas -v on png_enc.cu: none of its kernels uses local memory for spills."""
    import shutil
    import subprocess
    import tempfile

    from smap_b200 import build

    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not found")
    with tempfile.TemporaryDirectory() as tmp:
        p = subprocess.run(["nvcc"] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "png_enc.cu"),
                            "-o", os.path.join(tmp, "e.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    spills = [line for line in p.stdout.splitlines() if "spill" in line]
    assert len(spills) >= 16 and all(" 0 bytes spill stores, 0 bytes spill loads" in s for s in spills), p.stdout


def test_vis_names_png():
    paths = ["/d/a.png", "/d/sub/b.jpeg", "/d/c.jpg"]
    assert ri.vis_names(paths, "/d", ".png") == ["a.png", "sub/b.png", "c.png"]
    with pytest.raises(ValueError, match="/d/a.png and /d/a.jpg would both be written to a.png"):
        ri.vis_names(["/d/a.png", "/d/a.jpg"], "/d", ".png")


def test_vis_format_argument(monkeypatch, tmp_path):
    seen = {}

    def fake_run(*a, **k):
        seen.clear()
        seen.update(k)
        return 0

    monkeypatch.setattr(ri, "run", fake_run)
    monkeypatch.setattr(ri, "_load_checkpoints", lambda a: ({}, None))
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    assert ri.main(["--output_dir", str(tmp_path), "--vis_dir", "V", "--vis_format", "png"]) == 0
    assert seen["vis_format"] == "png" and seen["vis_dir"] == "V"
    assert ri.main(["--output_dir", str(tmp_path), "--vis_dir", "V", "--vis_format", "jpg"]) == 0
    assert "vis_format" not in seen, "the default format calls run() as before"
    for bad in (["--vis_format", "png"], ["--vis_dir", "V", "--vis_format", "bmp"]):
        with pytest.raises(SystemExit):
            ri.main(["--output_dir", str(tmp_path)] + bad)


def test_write_vis_png(tmp_path):
    class Encoder:
        def encode_png(self, frames, records, scales, **kw):
            return [P.encode(f) for f in frames]

        def encode_jpeg(self, *a, **k):
            raise AssertionError("JPEG requested")

    f = np.random.default_rng(0).integers(0, 256, (9, 7, 3), np.uint8)
    ri.write_vis(Encoder(), str(tmp_path), 95, ["s/a.png"], [f], None, None, fmt="png")
    assert (cv2.imread(str(tmp_path / "s" / "a.png")) == f).all()


def test_png_collision_is_refused_before_any_work(tmp_path, monkeypatch):
    (tmp_path / "a.png").write_bytes(b"x")
    (tmp_path / "a.jpg").write_bytes(b"x")

    def no_engine(*a, **k):
        raise AssertionError("an engine was created")

    monkeypatch.setattr(ri, "Engine", no_engine)
    with pytest.raises(ValueError, match="a.png"):
        ri.run({}, str(tmp_path), str(tmp_path / "o.json"), vis_dir=str(tmp_path / "v"), vis_format="png")
