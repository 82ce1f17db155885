"""Numpy restatement of the RandAugment ops of the frozen video evaluation (rand-m7-n4-mstd0.5-inc1, PIL 12) on one
uint8 RGB frame [H, W, 3], written as the integer / float32 / float64 expressions Pillow's C code evaluates.  The GPU
kernels (jepa_b200/csrc/augment.cu) implement the same expressions; tests/test_randaugment_cpu.py pins this file bit for
bit to PIL's own outputs (tests/golden/golden_randaugment.pt), so the GPU tests need no PIL.

`apply_op(frame, op)` takes an op record as jepa_b200.transforms.sample_randaugment produces it:
(code, fval, ival, matrix) with the op's float factor, integer argument and affine matrix."""
import hashlib

import numpy as np

from jepa_b200.transforms import RA_OPS

F32 = np.float32


def _lut(frame, lut):
    """lut: [256] or [3, 256] (values clipped to 0..255 as Image.point stores them)."""
    lut = np.clip(np.asarray(lut, dtype=np.int64), 0, 255).astype(np.uint8)
    if lut.ndim == 1:
        return lut[frame]
    return np.stack([lut[c][frame[..., c]] for c in range(3)], -1)


def histogram(frame):
    """Image.histogram() of an RGB frame: [3, 256] counts."""
    return np.stack([np.bincount(frame[..., c].ravel(), minlength=256) for c in range(3)])


def to_l(frame):
    """RGB -> L (Convert.c rgb2l): (R * 19595 + G * 38470 + B * 7471 + 0x8000) >> 16."""
    f = frame.astype(np.int64)
    return ((f[..., 0] * 19595 + f[..., 1] * 38470 + f[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def autocontrast_lut(h):
    """ImageOps.autocontrast (cutoff 0): per channel lo / hi = first / last non-empty bin, then
    int(i * (255.0 / (hi - lo)) + (-lo * scale)) in double, clipped; identity when hi <= lo."""
    lut = np.empty((3, 256), np.int64)
    for c in range(3):
        nz = np.nonzero(h[c])[0]
        lo, hi = int(nz[0]), int(nz[-1])
        if hi <= lo:
            lut[c] = np.arange(256)
            continue
        scale = 255.0 / (hi - lo)
        offset = -lo * scale
        lut[c] = np.clip(np.trunc(np.arange(256, dtype=np.float64) * scale + offset), 0, 255)
    return lut


def equalize_lut(h):
    """ImageOps.equalize: step = (sum - last non-empty count) // 255; lut[i] = (step // 2 + sum(h[:i])) // step;
    identity when at most one bin is non-empty or step == 0."""
    lut = np.empty((3, 256), np.int64)
    for c in range(3):
        nz = np.nonzero(h[c])[0]
        step = (int(h[c].sum()) - int(h[c][nz[-1]])) // 255 if len(nz) > 1 else 0
        if step == 0:
            lut[c] = np.arange(256)
            continue
        excl = np.concatenate([[0], np.cumsum(h[c])[:-1]])
        lut[c] = (step // 2 + excl) // step
    return lut


def blend(degenerate, frame, factor):
    """Image.blend(degenerate, image, factor) (Blend.c): float32 d + factor * (int(image) - int(d)), clipped to 0..255
    and truncated (the interpolating branch for 0 <= factor <= 1 computes the same value without clipping)."""
    a = F32(factor)
    d = degenerate.astype(np.int32)
    t = d.astype(F32) + a * (frame.astype(np.int32) - d).astype(F32)
    return np.where(t <= 0, 0, np.where(t >= 255, 255, np.trunc(t))).astype(np.uint8)


def smooth(frame):
    """ImageFilter.SMOOTH, kernel (1 1 1 / 1 5 1 / 1 1 1) / 13: PIL's uint8 result is the weighted sum s rounded to
    nearest, (s + 6) // 13 (s / 13 is never a tie); the one-pixel border is copied from the input."""
    f = frame.astype(np.int64)
    out = frame.copy()
    H, W = frame.shape[:2]
    if H < 3 or W < 3:
        return out
    s = sum(f[dy:H - 2 + dy, dx:W - 2 + dx] * (5 if (dy, dx) == (1, 1) else 1) for dy in range(3) for dx in range(3))
    out[1:-1, 1:-1] = (s + 6) // 13
    return out


def _cubic(v1, v2, v3, v4, d):
    """Geometry.c BICUBIC (a = -0.5 kernel as PIL writes it), double precision, left-to-right evaluation."""
    p1 = v2
    p2 = -v1 + v3
    p3 = 2 * (v1 - v2) + v3 - v4
    p4 = -v1 + v2 - v3 + v4
    return p1 + d * (p2 + d * (p3 + d * p4))


def affine(frame, m, fill=128):
    """Image.transform(size, AFFINE, m, BICUBIC, fillcolor=fill): output pixel (x, y) samples the input at
    (m0 (x + .5) + m1 (y + .5) + m2, m3 (x + .5) + m4 (y + .5) + m5) in double; outside [0, W) x [0, H) it keeps the
    fill.  Bicubic over the 4 x 4 neighbours at floor(pos - .5) - 1 .., indices clamped to the frame, result clipped to
    0..255 and truncated."""
    H, W = frame.shape[:2]
    f = frame.astype(np.float64)
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64) + 0.5, np.arange(W, dtype=np.float64) + 0.5, indexing='ij')
    xin = m[0] * xs + m[1] * ys + m[2]
    yin = m[3] * xs + m[4] * ys + m[5]
    inside = (xin >= 0) & (xin < W) & (yin >= 0) & (yin < H)
    xi, yi = xin - 0.5, yin - 0.5
    x0, y0 = np.floor(xi), np.floor(yi)
    dx, dy = xi - x0, yi - y0
    x0, y0 = x0.astype(np.int64) - 1, y0.astype(np.int64) - 1
    cols = [np.clip(x0 + k, 0, W - 1) for k in range(4)]
    rows = [np.clip(y0 + k, 0, H - 1) for k in range(4)]
    out = np.full(frame.shape, fill, np.uint8)
    for c in range(3):
        v = [_cubic(*[f[r, cx, c] for cx in cols], dx) for r in rows]
        val = _cubic(*v, dy)
        u = np.where(val <= 0, 0, np.where(val >= 255, 255, np.trunc(np.where(np.isfinite(val), val, 0))))
        out[..., c] = np.where(inside, u, fill).astype(np.uint8)
    return out


def apply_op(frame, op):
    code, fval, ival, m = op
    name = RA_OPS[code]
    if name == 'AutoContrast':
        return _lut(frame, autocontrast_lut(histogram(frame)))
    if name == 'Equalize':
        return _lut(frame, equalize_lut(histogram(frame)))
    if name == 'Invert':
        return _lut(frame, 255 - np.arange(256))
    if name == 'PosterizeIncreasing':
        return _lut(frame, np.arange(256) & (~((1 << (8 - ival)) - 1) & 255)) if ival < 8 else frame.copy()
    if name == 'SolarizeIncreasing':
        i = np.arange(256)
        return _lut(frame, np.where(i < ival, i, 255 - i))
    if name == 'SolarizeAdd':
        i = np.arange(256)
        return _lut(frame, np.where(i < 128, np.minimum(255, i + ival), i))
    if name == 'ColorIncreasing':
        return blend(np.repeat(to_l(frame)[..., None], 3, -1), frame, fval)
    if name == 'ContrastIncreasing':
        hl = np.bincount(to_l(frame).ravel(), minlength=256)
        mean = int(float((np.arange(256) * hl).sum()) / float(hl.sum()) + 0.5)
        return blend(np.full_like(frame, mean), frame, fval)
    if name == 'BrightnessIncreasing':
        return blend(np.zeros_like(frame), frame, fval)
    if name == 'SharpnessIncreasing':
        return blend(smooth(frame), frame, fval)
    if m is None:             # Rotate by 0 degrees: PIL returns a copy
        return frame.copy()
    return affine(frame, m)


def rng_digests():
    """sha256 digests of random.getstate() and np.random.get_state(): equal digests mean equal generator states."""
    import random
    st = np.random.get_state()
    py = hashlib.sha256(repr(random.getstate()).encode()).hexdigest()
    npd = hashlib.sha256(repr((st[0], st[2], st[3], st[4])).encode() + np.asarray(st[1], np.uint32).tobytes()).hexdigest()
    return py, npd


def op_cases(golden):
    """(case, input frame, PIL's output) for every per-op case of golden_randaugment.pt."""
    for c in golden["ops"]:
        x = golden["frames"][c["frame"]]
        n = x.numel()
        yield c, x, golden["y"][c["off"]:c["off"] + n].view(x.shape)
