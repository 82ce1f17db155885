"""numpy restatement of torch's CPU F.interpolate(scale_factor=..., align_corners=False) for the two modes
interpolate_pos_encoding uses - the specification vj_pos_interp (jepa_b200/csrc/posinterp.cu) implements.  Every
operation is an fp32 round-to-nearest; where torch's x86-64 build fuses a multiply and an add, fma32 rounds once."""
import math

import numpy as np

f32 = np.float32


def fma32(a, b, c):
    """fp32 fused multiply-add, correctly rounded: the product is exact in fp64; the sum goes through round-to-odd in
    fp64 (exact remainder by TwoSum), so the final rounding to fp32 is the only one."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    e = (p - bp) + (c - (s - bp))            # TwoSum: s + e == p + c exactly
    bits = s.view(np.int64)
    other = np.nextafter(s, s + np.where(e > 0, np.inf, -np.inf))
    s = np.where((e != 0) & ((bits & 1) == 0), other, s)
    return s.astype(np.float32)


def scaled_size(n, scale):
    return int(n * scale)


def src_coord(s, dst):
    return fma32(s, np.arange(dst, dtype=f32) + f32(0.5), f32(-0.5))


def linear_axis(n_in, n_out, scale):
    """(i0, i1, l0, l1) per output index of one axis."""
    if n_in == n_out:
        i = np.arange(n_out)
        return i, i, np.ones(n_out, f32), np.zeros(n_out, f32)
    r = src_coord(f32(1.0 / scale), n_out)
    r = np.where(r < 0, f32(0), r)
    i0 = np.minimum(np.floor(r).astype(np.int64), n_in - 1)
    l1 = np.clip(r - i0.astype(f32), f32(0), f32(1)).astype(f32)
    i1 = i0 + (i0 < n_in - 1)
    return i0, i1, (f32(1) - l1).astype(f32), l1


def trilinear(table, scales):
    """table fp32 [Nt, Nh, Nw, D] -> [floor(Nt st), floor(Nh sh), floor(Nw sw), D]."""
    Nt, Nh, Nw, _ = table.shape
    (t0, t1, a0, a1), (h0, h1, b0, b1), (w0, w1, e0, e1) = (
        linear_axis(n, scaled_size(n, s), s) for n, s in zip((Nt, Nh, Nw), scales))
    T, H, W = len(t0), len(h0), len(w0)

    def tap(ti, hi, wi):
        return table[ti[:, None, None], hi[None, :, None], wi[None, None, :]]

    def wt(a, b, e):
        return ((a[:, None, None] * b[None, :, None]).astype(f32) * e[None, None, :]).astype(f32)[..., None]

    corners = [(t0, h0, w0, a0, b0, e0), (t0, h0, w1, a0, b0, e1), (t0, h1, w0, a0, b1, e0), (t0, h1, w1, a0, b1, e1),
               (t1, h0, w0, a1, b0, e0), (t1, h0, w1, a1, b0, e1), (t1, h1, w0, a1, b1, e0), (t1, h1, w1, a1, b1, e1)]
    vals = [tap(ti, hi, wi) for ti, hi, wi, _, _, _ in corners]
    ws = [wt(a, b, e) for _, _, _, a, b, e in corners]
    # t0 w0 + (t1 w1 + (... + (t6 w6 + t7 w7))), every step fused
    acc = fma32(vals[7], ws[7], (vals[6] * ws[6]).astype(f32))
    for k in range(5, -1, -1):
        acc = fma32(vals[k], ws[k], acc)
    assert acc.shape[:3] == (T, H, W)
    return acc


def _cubic1(x):
    return ((fma32(f32(1.25), x, f32(-2.25)) * x).astype(f32) * x).astype(f32) + f32(1)


def _cubic2(x):
    return (fma32(fma32(f32(-0.75), x, f32(3.75)), x, f32(-6)) * x).astype(f32) - f32(-3)


def cubic_axis(n_in, n_out, scale):
    """tap indices [n_out, 4] and weights [n_out, 4] of one axis (A = -0.75)."""
    r = src_coord(f32(1.0 / scale), n_out)
    i0 = np.minimum(np.floor(r).astype(np.int64), n_in - 1)
    t = np.clip(r - i0.astype(f32), f32(0), f32(1)).astype(f32)
    x2 = (f32(1) - t).astype(f32)
    w = np.stack([_cubic2((t + f32(1)).astype(f32)), _cubic1(t), _cubic1(x2), _cubic2((x2 + f32(1)).astype(f32))], 1)
    idx = np.clip(i0[:, None] + np.arange(-1, 3)[None, :], 0, n_in - 1)
    return idx, w.astype(f32)


def _sum4(v, w):
    """v [..., 4, D], w [..., 4]: fma(v0, w0, v1 w1) -> fma(v2, w2, .) -> fma(v3, w3, .)."""
    w = w[..., None]
    acc = fma32(v[..., 0, :], w[..., 0, :], (v[..., 1, :] * w[..., 1, :]).astype(f32))
    acc = fma32(v[..., 2, :], w[..., 2, :], acc)
    return fma32(v[..., 3, :], w[..., 3, :], acc)


def bicubic(table, scale):
    """table fp32 [Nh, Nw, D] -> [floor(Nh s), floor(Nw s), D]: W taps first, then H taps."""
    Nh, Nw, _ = table.shape
    hi, hw = cubic_axis(Nh, scaled_size(Nh, scale), scale)
    wi, ww = cubic_axis(Nw, scaled_size(Nw, scale), scale)
    g = table[hi[:, None, :, None], wi[None, :, None, :]]                    # [H, W, 4 (h taps), 4 (w taps), D]
    rows = _sum4(g, np.broadcast_to(ww[None, :, None, :], g.shape[:4]))      # [H, W, 4, D]
    return _sum4(rows, np.broadcast_to(hw[:, None, :], rows.shape[:3]))


def video_scales(grid0, grid):
    return tuple(g / n for g, n in zip(grid, grid0))


def image_scale(n0, n):
    return math.sqrt((n * n) / (n0 * n0))
