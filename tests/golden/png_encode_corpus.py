"""Seeded frames for the PNG encoder tests (tests/test_png_encode_cpu.py, tests/test_png_encode_gpu.py).

n = H * (1 + 3 W) is the length of the filtered stream.  The sizes straddle every n at which libpng changes zlib's window
(n <= 16384, then n + 262 <= 8192, 4096, ... 512) or rewrites CINFO (n <= 2^k), so each window size is met, with noise
(stored blocks) and flat content (long runs).  EXACT is the frame whose 16383 symbols fill one block exactly, so its
stream ends in an empty final block."""
import numpy as np
from jpeg_encode_corpus import frame as jpeg_frame

TINY = [(1, 1), (2, 1), (1, 2), (5, 1), (100, 1), (6000, 1), (3, 2), (7, 5)]
THRESHOLDS = [16384] + [h - 262 for h in (8192, 4096, 2048, 1024, 512)] + [1 << k for k in range(7, 15)]
EXACT_SEED, EXACT_SIZE = 7, (3, 1820)  # n = 16383, no run of 4 equal bytes in the filtered stream


def stream_len(h, w):
    return h * (1 + 3 * w)


def _sizes_at(t):
    """The sizes with the largest n <= t and the smallest n > t (H <= 64)."""
    below, above = None, None
    for h in range(1, 65):
        for w in range(1, 6000):
            n = stream_len(h, w)
            if n <= t and (below is None or n > stream_len(*below)):
                below = (h, w)
            if n > t:
                if above is None or n < stream_len(*above):
                    above = (h, w)
                break
    return [below, above]


def threshold_sizes():
    return sorted({s for t in THRESHOLDS for s in _sizes_at(t)})


def frame(kind, h, w, seed):
    """noise / flat / four-level / photo (the JPEG corpus's photo-like frame) / black (zero runs that cross rows)."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), np.uint8)
    if kind == "flat":
        return np.broadcast_to(rng.integers(0, 256, 3, np.uint8), (h, w, 3)).copy()
    if kind == "levels":
        return (rng.integers(0, 4, (h, w, 3)) * 60).astype(np.uint8)
    if kind == "black":
        return np.zeros((h, w, 3), np.uint8)
    if kind == "rows":  # one random row repeated: equal rows, short runs inside them
        return np.broadcast_to(rng.integers(0, 256, (1, w, 3), np.uint8), (h, w, 3)).copy()
    return jpeg_frame("photo", h, w, seed)


def exact_frame():
    return frame("noise", *EXACT_SIZE, EXACT_SEED)


def corpus():
    """-> list of (name, frame): every size of TINY and threshold_sizes() in several kinds, runs over 258 bytes that
    cross rows, EXACT, and photo-like 1080p and 4032 x 3024 frames."""
    out = []
    for i, (h, w) in enumerate(TINY + threshold_sizes()):
        for j, kind in enumerate(("noise", "flat", "levels")):
            out.append(("%s_%dx%d" % (kind, h, w), frame(kind, h, w, 1000 + 10 * i + j)))
    for h, w in [(2000, 1), (200, 300), (33, 17)]:
        out.append(("black_%dx%d" % (h, w), frame("black", h, w, 0)))
    out.append(("rows_64x600", frame("rows", 64, 600, 5)))
    out.append(("photo_480x640", frame("photo", 480, 640, 6)))
    out.append(("exact_3x1820", exact_frame()))
    out.append(("photo_1080x1920", frame("photo", 1080, 1920, 8)))
    out.append(("photo_3024x4032", frame("photo", 3024, 4032, 9)))
    return out
