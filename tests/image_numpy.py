"""Numpy restatement of csrc/image.cu's resampling (PIL 12 Resample.c for 8-bit images) over the tables
jepa_b200/image_transforms.py builds, and the synthetic test images shared with tests/golden/make_golden_image_transforms.py.
tests/test_image_transforms_cpu.py pins the restatement bit for bit to PIL's Image.resize."""
import numpy as np

from jepa_b200.image_transforms import PRECISION_BITS, axis_entries


def _pass(src, ent, axis):
    """One pass over `axis` (1: columns, 0: rows) of int64 pixels with the entries (first tap, count, weights)."""
    out = []
    for e in ent:
        first, cnt = int(e[0]), int(e[1])
        taps = np.take(src, np.arange(first, first + cnt), axis=axis)
        w = e[2:2 + cnt].astype(np.int64)
        acc = (1 << (PRECISION_BITS - 1)) + np.tensordot(taps, w, axes=([axis], [0]))
        out.append(np.clip(acc >> PRECISION_BITS, 0, 255))
    return np.stack(out, axis=axis)


def apply_tables(img, c0, xent, r0, nrows, yent):
    """uint8 [H, W, 3] -> the resampled window: horizontal pass over source rows [r0, r0 + nrows) into uint8, then the
    vertical pass."""
    rows = img[r0:r0 + nrows, c0:].astype(np.int64)
    tmp = _pass(rows, xent, 1)
    return _pass(tmp, yent, 0).astype(np.uint8)


def pil_resize(img, box, out_hw, bicubic):
    """What img.crop(box).resize((ow, oh), BILINEAR | BICUBIC) gives, computed from the tables (box = (i, j, h, w))."""
    i, j, h, w = box
    oh, ow = out_hw
    xent = axis_entries(w, ow, 0, ow, bicubic)
    yent = axis_entries(h, oh, 0, oh, bicubic)
    lo = int(yent[:, 0].min())
    hi = int((yent[:, 0] + yent[:, 1]).max())
    yent = yent.copy()
    yent[:, 0] -= lo
    return apply_tables(img, j, xent, i + lo, hi - lo, yent)


def synth_image(seed, H, W):
    """Decoder-like uint8 RGB image [H, W, 3]: smooth colour ramps plus noise (numpy's legacy RandomState: stable)."""
    rs = np.random.RandomState(5000 + seed)
    y, x = np.mgrid[:H, :W]
    base = np.stack([x * 255 // max(W - 1, 1), y * 255 // max(H - 1, 1), ((x + 2 * y) * 5) % 256], -1)
    return np.clip(base + rs.randint(-30, 31, size=(H, W, 3)), 0, 255).astype(np.uint8)
