"""Seeded inputs for the batch-scale tests: images, latents, eps, colour and frame targets and boxes (every fourth a fixed
17x12 box, a 1x1 box, the full width, or a random box of <= 17 pixels a side), cached per (n, seed)."""
import numpy as np

_CACHE = {}


def inputs(n, seed):
    if (n, seed) not in _CACHE:
        rng = np.random.default_rng(seed)
        boxes = np.empty((n, 4), np.int32)
        for k in range(n):
            if k % 4 == 0:
                boxes[k] = [3, 5, 20, 17]
            elif k % 4 == 1:
                boxes[k] = [40, 30, 41, 31]                  # one pixel
            elif k % 4 == 2:
                boxes[k] = [0, 47, 64, 64]                   # the full width
            else:
                c1, r1 = rng.integers(0, 48, 2)
                boxes[k] = [c1, r1, c1 + rng.integers(2, 17), r1 + rng.integers(2, 17)]
        _CACHE[(n, seed)] = {
            "x": rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32),
            "z": rng.standard_normal((n, 100)).astype(np.float32),
            "eps": rng.standard_normal((n, 100)).astype(np.float32),
            "rgb": rng.uniform(-1, 1, (n, 3)).astype(np.float32),
            "frame": rng.uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32),
            "boxes": boxes}
    return _CACHE[(n, seed)]
