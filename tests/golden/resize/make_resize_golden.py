"""Writes tests/golden/resize/cv2_resize.npz: OpenCV's 8-bit INTER_LINEAR resize (cv2.resize) on small seeded
images, so that the restatement (tests/resize_ref.py) is pinned to cv2's bytes on machines without cv2.  Large cases
(500x375 -> 227x227 and the like) are stored as a SHA-256 of the output; their source is np.random.RandomState(seed).

  python tests/golden/resize/make_resize_golden.py
"""
import hashlib
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# (H, W, C, h, w): every up/down combination, 1-pixel axes, exact 2x both ways, equal sizes
SMALL = [(1, 1, 3, 4, 5), (1, 9, 1, 6, 3), (9, 1, 4, 3, 7), (5, 7, 3, 1, 1), (8, 8, 3, 16, 16), (16, 16, 1, 8, 8),
         (12, 10, 3, 12, 10), (3, 40, 3, 20, 9), (40, 3, 1, 9, 20), (17, 23, 4, 31, 11), (31, 11, 3, 17, 23),
         (2, 2, 3, 37, 29), (37, 29, 3, 2, 2), (25, 25, 3, 24, 26), (13, 50, 1, 27, 27)]
LARGE = [(375, 500, 3, 227, 227), (500, 375, 3, 227, 227), (256, 256, 3, 227, 227), (64, 64, 3, 32, 32),
         (480, 640, 3, 256, 256), (333, 500, 3, 256, 256)]


def source(seed, H, W, C):
    img = np.random.RandomState(seed).randint(0, 256, (H, W, C)).astype(np.uint8)
    return img


def main():
    import cv2
    cv2.setNumThreads(1)
    arrays, large = {}, []
    for k, (H, W, C, h, w) in enumerate(SMALL):
        src = source(100 + k, H, W, C)
        out = cv2.resize(src, (w, h), interpolation=cv2.INTER_LINEAR).reshape(h, w, C)
        arrays[f"src{k}"], arrays[f"out{k}"] = src, out
    for k, (H, W, C, h, w) in enumerate(LARGE):
        out = cv2.resize(source(200 + k, H, W, C), (w, h), interpolation=cv2.INTER_LINEAR).reshape(h, w, C)
        large.append(dict(seed=200 + k, src=[H, W, C], dst=[h, w], sha256=hashlib.sha256(out.tobytes()).hexdigest()))
    np.savez_compressed(os.path.join(HERE, "cv2_resize.npz"), **arrays)
    with open(os.path.join(HERE, "cv2_resize_large.json"), "w") as f:
        json.dump(dict(opencv=cv2.__version__, cases=large), f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
