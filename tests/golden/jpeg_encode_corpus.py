"""Seeded frames for the JPEG encoder tests (tests/test_jpeg_encode_cpu.py, tests/test_jpeg_encode_gpu.py): noise, flat
frames, gradients and photo-like mixes at the sizes that exercise partial blocks and libjpeg's dummy MCU blocks."""
import numpy as np

SIZES = [(1, 1), (5, 5), (9, 11), (17, 33), (16, 16), (8, 24), (31, 2), (1081, 1919), (1080, 1920)]
# a frame whose last entropy-coded byte, padded with 1-bits, is 0xFF and is stuffed (found with the CPU oracle)
EOS_SEED, EOS_SIZE, EOS_QUALITY = 1595, (13, 21), 75


def frame(kind, h, w, seed):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), np.uint8)
    if kind == "flat":
        return np.broadcast_to(rng.integers(0, 256, 3, np.uint8), (h, w, 3)).copy()
    y, x = np.mgrid[0:h, 0:w]
    if kind == "gradient":
        g = np.stack([x * 255 // max(1, w - 1), y * 255 // max(1, h - 1), (x + y) * 255 // max(1, w + h - 2)], -1)
        return g.astype(np.uint8)
    # photo-like: smooth shading, a few hard-edged shapes and sensor noise
    img = 128 + 60 * np.sin(x[..., None] / (7.0 + 3 * np.arange(3))) * np.cos(y[..., None] / 11.0)
    for _ in range(4):
        cx, cy, r = rng.integers(0, w), rng.integers(0, h), rng.integers(2, max(3, min(h, w) // 3))
        img[(x - cx) ** 2 + (y - cy) ** 2 < r * r] = rng.integers(0, 256, 3)
    img += rng.normal(0, 6, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def corpus():
    out = []
    for i, (h, w) in enumerate(SIZES):
        for j, kind in enumerate(("noise", "flat", "gradient", "photo")):
            if h * w > 10 ** 6 and kind in ("flat", "gradient"):
                continue
            out.append(frame(kind, h, w, 100 * i + j))
    return out


def eos_stuffing_frame():
    """-> (frame, quality) whose stream ends in a stuffed 0xFF padding byte."""
    return frame("noise", *EOS_SIZE, EOS_SEED), EOS_QUALITY
