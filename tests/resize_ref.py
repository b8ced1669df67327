"""numpy restatement of OpenCV's 8-bit INTER_LINEAR resize (cv::resize on a uint8 cv::Mat), the rule the library's
COS_RAW_U8_IMAGES path resizes by (DESIGN.md, "Images of any size").  Integer arithmetic after the coefficients:

  scale = double(src) / dst per axis;  f = float((d + 0.5) * scale - 0.5);  i = floor(f);  f -= i
  c0 = rint(float(1 - f) * 2048),  c1 = 2048 - c0
  horizontal: i < 0 -> i = 0, f = 0;  i >= W - 1 -> i = W - 1, f = 0 (coefficients from the clamped f)
              S[y][x] = src[y][i] * cx0 + src[y][min(i + 1, W - 1)] * cx1                      (int32)
  vertical:   f and its coefficients are not clamped, only the rows: r0 = clamp(i, 0, H - 1), r1 = clamp(i + 1, ...)
              out = ((((cy0 * (S[r0] >> 4)) >> 16) + ((cy1 * (S[r1] >> 4)) >> 16) + 2) >> 2), saturated to uint8

Clamping the vertical coefficients like the horizontal ones would put upscaled border rows up to 1 off.
"""
import numpy as np


def taps(src, dst):
    """-> (i, f): the unclamped source index (int64) and float32 fraction of each of the dst output indices."""
    scale = np.float64(src) / np.float64(dst)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    i = np.floor(f)
    return i.astype(np.int64), (f - i).astype(np.float32)


def c0(f):
    """First fixed-point coefficient rint(float(1 - f) * 2048); the second is 2048 - c0."""
    return np.rint((np.float32(1) - np.asarray(f, np.float32)).astype(np.float32) * np.float32(2048)).astype(np.int64)


def resize(img, height, width):
    """img: uint8 H x W x C (or H x W) -> uint8 height x width x C (or height x width)."""
    a = np.asarray(img, np.uint8)
    flat = a.ndim == 2
    if flat:
        a = a[:, :, None]
    H, W, _ = a.shape
    # horizontal: the index and the fraction are clamped together
    ix, fx = taps(W, width)
    edge = (ix < 0) | (ix >= W - 1)
    ix = np.clip(ix, 0, W - 1)
    cx0 = c0(np.where(edge, np.float32(0), fx))
    src = a.astype(np.int64)
    S = src[:, ix, :] * cx0[None, :, None] + src[:, np.minimum(ix + 1, W - 1), :] * (2048 - cx0)[None, :, None]
    # vertical: only the rows are clamped
    iy, fy = taps(H, height)
    cy0 = c0(fy)
    r0, r1 = np.clip(iy, 0, H - 1), np.clip(iy + 1, 0, H - 1)
    v = ((cy0[:, None, None] * (S[r0] >> 4)) >> 16) + (((2048 - cy0)[:, None, None] * (S[r1] >> 4)) >> 16)
    out = np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)
    return out[:, :, 0] if flat else out


def post_resize_size(img_hw, target):
    """(height, width) of an image after the optional resize: the target, or the image's own size without one."""
    return tuple(img_hw) if not target or tuple(target) == (0, 0) else tuple(target)
