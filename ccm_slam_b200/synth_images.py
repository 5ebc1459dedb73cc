"""Seeded synthetic test images, numpy only.

make_image: 752x480 by default (SURVEY.md §8(d) config 1), multi-octave value noise + random rectangles, FAST-rich.
make_noise: textured frames (gravel, foliage, carpet) that give the ORB extractor far more FAST candidates than its quota:
            white noise, optionally smoothed with a Gaussian and stretched back to 0..255."""
import numpy as np


def make_image(seed=0, w=752, h=480):
    rng = np.random.default_rng(seed)
    img = np.zeros((h, w), np.float64)
    for octave, amp in [(6, 60.0), (12, 40.0), (24, 30.0), (48, 20.0), (96, 12.0)]:
        gh, gw = h // octave + 2, w // octave + 2
        g = rng.random((gh, gw))
        ys = np.arange(h) / octave; xs = np.arange(w) / octave
        y0 = ys.astype(int); x0 = xs.astype(int); fy = (ys - y0)[:, None]; fx = (xs - x0)[None, :]
        v = (g[y0][:, x0] * (1 - fy) * (1 - fx) + g[y0][:, x0 + 1] * (1 - fy) * fx +
             g[y0 + 1][:, x0] * fy * (1 - fx) + g[y0 + 1][:, x0 + 1] * fy * fx)
        img += amp * v
    for _ in range(140):
        x, y = rng.integers(0, w - 8), rng.integers(0, h - 8)
        ww, hh = rng.integers(6, 90), rng.integers(6, 70)
        img[y:y + hh, x:x + ww] += rng.uniform(-70, 70)
    img += rng.normal(0, 2.0, size=img.shape)
    img = (img - img.min()) / (img.max() - img.min()) * 255.0
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def make_noise(seed=0, w=752, h=480, sigma=0.0):
    """uniform white noise; sigma > 0 smooths it with a separable Gaussian (radius ceil(3 sigma), mirrored border) and
    stretches the result back to the full 0..255 range"""
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, size=(h, w)).astype(np.float64)
    if sigma > 0:
        r = int(np.ceil(3 * sigma))
        k = np.exp(-0.5 * (np.arange(-r, r + 1) / sigma) ** 2)
        k /= k.sum()
        for axis in (0, 1):
            pad = [(0, 0), (0, 0)]; pad[axis] = (r, r)
            p = np.pad(img, pad, mode="reflect")
            n = img.shape[axis]
            img = sum(k[i] * np.take(p, np.arange(i, i + n), axis=axis) for i in range(2 * r + 1))
        img = (img - img.min()) / (img.max() - img.min()) * 255.0
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)
