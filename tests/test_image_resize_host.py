"""Host-only checks of the ragged-image path (DESIGN.md, "Images of any size"): the numpy restatement of OpenCV's
8-bit INTER_LINEAR resize against cv2 itself and against the committed cv2 fixtures, directed cases, and the refusals
that need no device (cos_image_transform's argument checks, the Python list conversion, NULL nets)."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import ROOT
import resize_ref as R

GOLDEN = os.path.join(ROOT, "tests", "golden", "resize")


def _sweep_pairs(n, seed):
    """n (H, W, C, h, w) with all four up/down combinations per axis pair, sides from 1, C in {1, 3, 4}."""
    rng = np.random.RandomState(seed)
    out = []
    for k in range(n):
        up_h, up_w = k % 2 == 0, (k // 2) % 2 == 0
        side = lambda: int(rng.randint(1, 300 if k % 7 == 0 else 64))  # noqa: E731
        H, W = side(), side()
        h = H + int(rng.randint(0, 60)) if up_h else max(1, H - int(rng.randint(0, H)))
        w = W + int(rng.randint(0, 60)) if up_w else max(1, W - int(rng.randint(0, W)))
        out.append((H, W, (1, 3, 4)[k % 3], h, w))
    return out


def test_restatement_equals_cv2_on_a_seeded_sweep():
    cv2 = pytest.importorskip("cv2")
    cv2.setNumThreads(1)
    pairs = _sweep_pairs(600, 7)
    kinds = {(h >= H, w >= W) for H, W, _, h, w in pairs}
    assert kinds == {(True, True), (True, False), (False, True), (False, False)}
    assert min(min(p[0], p[1], p[3], p[4]) for p in pairs) == 1
    rng = np.random.RandomState(8)
    for H, W, C, h, w in pairs:
        img = rng.randint(0, 256, (H, W, C)).astype(np.uint8)
        want = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR).reshape(h, w, C)
        assert np.array_equal(R.resize(img, h, w), want), (H, W, C, h, w)


def _generator():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_resize_golden", os.path.join(GOLDEN, "make_resize_golden.py"))
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    return G


def test_restatement_equals_the_cv2_fixtures():
    G = _generator()
    z = np.load(os.path.join(GOLDEN, "cv2_resize.npz"))
    for k, (H, W, C, h, w) in enumerate(G.SMALL):
        src, out = z[f"src{k}"], z[f"out{k}"]
        assert src.shape == (H, W, C) and out.shape == (h, w, C)
        assert np.array_equal(R.resize(src, h, w), out), (H, W, C, h, w)
    large = json.load(open(os.path.join(GOLDEN, "cv2_resize_large.json")))["cases"]
    assert len(large) == len(G.LARGE)
    for c in large:
        src = G.source(c["seed"], *c["src"])
        got = R.resize(src, *c["dst"])
        assert hashlib.sha256(got.tobytes()).hexdigest() == c["sha256"], c["src"]


def test_directed_cases():
    rng = np.random.RandomState(3)
    img = rng.randint(0, 256, (23, 31, 3)).astype(np.uint8)
    assert np.array_equal(R.resize(img, 23, 31), img)  # equal size: a copy
    # exact 2x down: the 2x2 mean, rounded half up
    a = rng.randint(0, 256, (16, 12, 3)).astype(np.int64)
    want = (a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2] + 2) >> 2
    assert np.array_equal(R.resize(a.astype(np.uint8), 8, 6), want)
    # exact 2x up: every output lies between its taps, and the grid keeps its corner pixels
    up = R.resize(a.astype(np.uint8), 32, 24).astype(np.int64)
    assert up[0, 0].tolist() == a[0, 0].tolist() and up[-1, -1].tolist() == a[-1, -1].tolist()
    # 1-pixel axes.  One source column gives identical columns (the horizontal fraction is clamped to 0).  One source
    # row gives rows within 1 of each other, not identical: the vertical coefficients stay unclamped and each of the
    # two products is truncated on its own (cv2 gives the same bytes: the sweep and the fixtures cover 1-row sources)
    row = rng.randint(0, 256, (1, 40, 3)).astype(np.uint8)
    out = R.resize(row, 7, 13).astype(int)
    assert np.abs(out - R.resize(row, 1, 13).astype(int)).max() == 1
    assert np.array_equal(out[:, :, 0][:, 3], [194, 194, 193, 194, 193, 194, 194])  # as cv2 4.13 gives them
    col = rng.randint(0, 256, (40, 1, 1)).astype(np.uint8)
    out = R.resize(col, 9, 5)
    assert (out == out[:, :1]).all()
    assert np.array_equal(R.resize(np.full((1, 1, 4), 77, np.uint8), 3, 2), np.full((3, 2, 4), 77, np.uint8))
    # 500x375 -> 227x227 (an ImageNet JPEG at the reference's CaffeNet size) keeps a constant image constant
    flat = np.full((375, 500, 3), 201, np.uint8)
    assert (R.resize(flat, 227, 227) == 201).all()
    assert R.resize(np.zeros((5, 5), np.uint8), 3, 4).shape == (3, 4)


def test_vertical_coefficients_are_not_clamped():
    """Upscaled top rows blend with the (clamped) row 0 using unclamped coefficients: with a clamped fraction the
    rule would give exactly row 0, which is not what it gives."""
    img = np.array([[0], [255]], np.uint8).reshape(2, 1, 1)
    out = R.resize(img, 8, 1)[:, 0, 0]
    i, f = R.taps(2, 8)
    assert i[0] == -1 and 0 < f[0] < 1  # the first output row's taps sit above the image
    assert out[0] == 0 and out[-1] == 255 and (np.diff(out.astype(int)) >= 0).all()


def test_post_resize_size():
    assert R.post_resize_size((375, 500), None) == (375, 500)
    assert R.post_resize_size((375, 500), (0, 0)) == (375, 500)
    assert R.post_resize_size((375, 500), (227, 227)) == (227, 227)


# ------------------------------------------------------------------------------------------------ refusals
def test_image_transform_argument_checks(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    fake = ctypes.c_void_p(16)  # never dereferenced: every call below is refused before a launch
    geom = ctypes.cast(fake, ctypes.POINTER(_lib.cos_image_geometry))
    mean = ctypes.cast(fake, ctypes.POINTER(ctypes.c_float))
    mv = (ctypes.c_float * 4)(1, 2, 3, 4)
    # in, geometry, num, C, rh, rw, out, oh, ow, crop, mirror, mean, mh, mw, mean_values, nmean
    ok = [fake, geom, 2, 3, 0, 0, fake, 8, 8, 0, 0, None, 0, 0, None, 0]
    bad = [
        ({0: None}, "NULL"), ({1: None}, "NULL"), ({6: None}, "NULL"),
        ({2: 0}, "positive"), ({3: 0}, "positive"), ({7: 0}, "positive"),
        ({4: 16}, "give both sides"), ({5: 16}, "give both sides"), ({4: -1, 5: -1}, "give both sides"),
        ({9: -1}, "negative"), ({9: 5}, "must be crop x crop"),
        ({4: 4, 5: 4, 9: 8}, "img_height >= crop_size"),
        ({4: 10, 5: 8}, "img_height == height"),
        ({11: mean, 12: 8, 13: 8, 14: mv, 15: 3}, "Cannot specify mean_file and mean_value"),
        ({11: mean, 12: 0, 13: 8}, "mean_height and mean_width must be positive"),
        ({4: 8, 5: 8, 11: mean, 12: 9, 13: 8}, "data_mean_.height()"),
        ({15: 3}, "mean_values is NULL"), ({14: mv, 15: 2}, "Specify either 1 mean_value or as many as channels"),
        ({8: 7000}, "exceeds"),
    ]
    for change, msg in bad:
        a = list(ok)
        for k, v in change.items():
            a[k] = v
        rc = L.cos_image_transform(*a, 1.0, 0, None)
        assert rc == 0, change
        err = L.cos_last_error().decode()
        assert err.startswith("cos_image_transform: ") and msg in err, (change, err)


def test_python_image_list_conversion_and_refusals(cos):
    from caffeonspark_b200 import caffenet
    imgs = [np.zeros((5, 7, 3), np.uint8), np.zeros((9, 4, 3), np.uint8)]
    blobs, keep = caffenet._raw_blob_array([imgs, np.zeros(2, np.float32)], (6, 6))
    assert (blobs[0].format, blobs[0].num, blobs[0].channels, blobs[0].height, blobs[0].width) == (2, 2, 3, 6, 6)
    arr = ctypes.cast(blobs[0].data, ctypes.POINTER(caffenet.cos_raw_image))
    assert [(arr[k].height, arr[k].width) for k in range(2)] == [(5, 7), (9, 4)]
    assert arr[1].data == imgs[1].ctypes.data
    blobs, _ = caffenet._raw_blob_array([[np.zeros((4, 4), np.uint8)]])  # H x W: one channel, no resize
    assert (blobs[0].channels, blobs[0].height, blobs[0].width) == (1, 0, 0)
    for bad in ([np.zeros((4, 4, 3), np.uint8), np.zeros((4, 4, 1), np.uint8)],  # mixed channels
                [np.zeros((4, 4, 3), np.float32)], [np.zeros((2, 4, 4, 3), np.uint8)], ["x"]):
        with pytest.raises(cos.CosError):
            caffenet._raw_blob_array([bad])


def test_entry_points_survive_null_and_garbage_images(cos):
    from caffeonspark_b200 import _lib
    L = _lib.lib()
    blob = _lib.cos_raw_blob()
    blob.format, blob.num, blob.channels = 2, 1, 3
    assert L.cos_net_train_raw(None, 0, ctypes.byref(blob), 1) == 0 and b"NULL" in L.cos_last_error()
    assert L.cos_net_train_raw(None, -1, ctypes.byref(blob), 1) == 0
