"""GPU input pipeline, host side (SURVEY 8f-3): the reference's VideoTransform (app/vjepa/transforms.py:40-117) split
into (a) the RANDOM DECISIONS - crop box and flip, drawn here on the host in exactly the reference's RNG call order, so
a seeded run picks the same boxes - and (b) the PIXEL MATH, which runs in one CUDA kernel (csrc/preprocess.cu:
uint8 -> bilinear random-resized crop -> flip -> normalise -> [B,3,T,S,S]) after the uint8 frames have crossed PCIe.

    tf = make_transforms(crop_size=224, ...)          # same signature as the reference factory
    item = tf(buffer_uint8_THWC)                      # in the DataLoader worker: no pixel is touched, returns a ClipTicket
    clips = preprocess_batch([item, ...], device)     # on the training process: one H2D copy of uint8 frames + one kernel

auto_augment / motion_shift / random erasing are PIL / per-frame CPU augmentations outside this path; they raise.
"""
import math
import random

import numpy as np
import torch

from . import _lib
from . import kernels as K

DEFAULT_NORMALIZE = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


def get_param_spatial_crop(scale, ratio, height, width, num_repeat=10, log_scale=True, switch_hw=False):
    """Crop box (i, j, h, w) of a random-resized crop; RNG draws in the order of
    src/datasets/utils/video/transforms.py:503-542 (random.uniform x2, np.random.uniform, random.randint x2 per try)."""
    for _ in range(num_repeat):
        area = height * width
        target_area = random.uniform(*scale) * area
        if log_scale:
            log_ratio = (math.log(ratio[0]), math.log(ratio[1]))
            aspect_ratio = math.exp(random.uniform(*log_ratio))
        else:
            aspect_ratio = random.uniform(*ratio)
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if np.random.uniform() < 0.5 and switch_hw:
            w, h = h, w
        if 0 < w <= width and 0 < h <= height:
            i = random.randint(0, height - h)
            j = random.randint(0, width - w)
            return i, j, h, w
    in_ratio = float(width) / float(height)     # fall back to a central crop
    if in_ratio < min(ratio):
        w = width
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = height
        w = int(round(h * max(ratio)))
    else:
        w, h = width, height
    return (height - h) // 2, (width - w) // 2, h, w


class ClipTicket:
    """One clip on its way to the GPU: the untouched uint8 frames [T,H,W,3] plus the decisions the kernel will apply."""
    __slots__ = ("frames", "box", "flip")

    def __init__(self, frames, box, flip):
        self.frames, self.box, self.flip = frames, box, flip


class GpuVideoTransform(object):
    """Drop-in for the reference's VideoTransform on its non-auto-augment path: __call__(buffer) consumes the same RNG
    draws (crop box, then one np.random.uniform for the flip, app/vjepa/transforms.py:100-108) and returns a ClipTicket."""

    def __init__(self, random_horizontal_flip=True, random_resize_aspect_ratio=(3 / 4, 4 / 3), random_resize_scale=(0.3, 1.0),
                 reprob=0.0, auto_augment=False, motion_shift=False, crop_size=224, normalize=DEFAULT_NORMALIZE):
        if auto_augment or motion_shift or reprob > 0:
            raise NotImplementedError("auto_augment / motion_shift / random erasing are CPU (PIL, per-frame) augmentations "
                                      "outside the GPU input path; every shipped pre-training config has them off")
        self.random_horizontal_flip = random_horizontal_flip
        self.random_resize_aspect_ratio = tuple(random_resize_aspect_ratio)
        self.random_resize_scale = tuple(random_resize_scale)
        self.crop_size = crop_size
        self.mean, self.std = tuple(normalize[0]), tuple(normalize[1])

    def __call__(self, buffer):
        frames = torch.as_tensor(np.ascontiguousarray(buffer))
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3:
            raise ValueError("GpuVideoTransform expects decoded uint8 frames [T, H, W, 3]")
        box = get_param_spatial_crop(self.random_resize_scale, self.random_resize_aspect_ratio, frames.shape[1], frames.shape[2])
        flip = bool(np.random.uniform() < 0.5) if self.random_horizontal_flip else False
        return ClipTicket(frames, box, flip)


def make_transforms(random_horizontal_flip=True, random_resize_aspect_ratio=(3 / 4, 4 / 3), random_resize_scale=(0.3, 1.0),
                    reprob=0.0, auto_augment=False, motion_shift=False, crop_size=224, normalize=DEFAULT_NORMALIZE):
    """Same signature as app/vjepa/transforms.py:15-38."""
    return GpuVideoTransform(random_horizontal_flip=random_horizontal_flip, random_resize_aspect_ratio=random_resize_aspect_ratio,
                             random_resize_scale=random_resize_scale, reprob=reprob, auto_augment=auto_augment,
                             motion_shift=motion_shift, crop_size=crop_size, normalize=normalize)


def pack_tickets(tickets, pin=True):
    """Host staging of a batch: ONE contiguous (pinned) uint8 buffer with every clip's frames back to back and the
    [B, 10] int32 parameter table the kernel reads (byte offset lo/hi, H, W, i, j, h, w, flip, pad)."""
    sizes = [int(t.frames.numel()) for t in tickets]
    offs = np.concatenate([[0], np.cumsum([(s + 15) // 16 * 16 for s in sizes])]).astype(np.int64)
    buf = torch.empty(int(offs[-1]), dtype=torch.uint8, pin_memory=pin and torch.cuda.is_available())
    tab = np.zeros((len(tickets), 10), dtype=np.int32)
    for b, t in enumerate(tickets):
        buf[offs[b]:offs[b] + sizes[b]] = t.frames.reshape(-1)
        T, H, W, _ = t.frames.shape
        i, j, h, w = t.box
        tab[b, 0:2] = np.array([offs[b]], dtype=np.int64).view(np.int32)      # little-endian long long
        tab[b, 2:9] = (H, W, i, j, h, w, int(t.flip))
    table = torch.from_numpy(tab)
    if pin and torch.cuda.is_available():
        table = table.pin_memory()
    return buf, table


def preprocess_batch(tickets, device, crop_size, mean=DEFAULT_NORMALIZE[0], std=DEFAULT_NORMALIZE[1], dtype=torch.float32,
                     out=None):
    """uint8 tickets -> normalised clips [B, 3, T, S, S] on `device` (fp32 like the reference's loader, or bf16).  Host
    -> device traffic is the uint8 frames (T*H*W*3 bytes per clip) instead of fp32 crops (12*T*S*S bytes)."""
    import ctypes
    T = int(tickets[0].frames.shape[0])
    if any(int(t.frames.shape[0]) != T for t in tickets):
        raise ValueError("all clips of a batch must have the same number of frames")
    buf, table = pack_tickets(tickets)
    dbuf = buf.to(device, non_blocking=True)
    dtab = table.to(device, non_blocking=True)
    B, S = len(tickets), int(crop_size)
    if out is None:
        out = torch.empty(B, 3, T, S, S, dtype=dtype, device=device)
    m3 = (ctypes.c_float * 3)(*[float(x) for x in mean])
    s3 = (ctypes.c_float * 3)(*[float(x) for x in std])
    _lib.call("vj_clip_preprocess", dbuf.data_ptr(), dtab.data_ptr(), out.data_ptr(), 1 if out.dtype == torch.float32 else 0,
              B, T, S, ctypes.cast(m3, ctypes.c_void_p), ctypes.cast(s3, ctypes.c_void_p), K._s())
    return out     # dbuf / dtab go back to the caching allocator, which only reuses them in stream order


# -------------------------------------------------------------------------------------------------
# Deterministic evaluation views (evals/video_classification_frozen/utils.py:199-323 of the reference)
# -------------------------------------------------------------------------------------------------
def short_side_size(H, W, size):
    """Frame size after resize_clip(clip, size) (src/datasets/utils/video/functional.py:33-81): unchanged when the short
    side already equals `size`, else the short side becomes `size` and the long side int(size * long / short)."""
    if (W <= H and W == size) or (H <= W and H == size):
        return H, W
    if W < H:
        return int(size * H / W), size
    return size, int(size * W / H)


def view_geometry(H, W, crop_size, num_views):
    """(resized H, resized W, [(row, col) origin of each crop_size x crop_size view]) of a decoded H x W clip.
    num_views > 1: EvalVideoTransform - short side to crop_size, windows along the long side (rows when H > W) at
    spatial_step = (max(H, W) - crop_size) // (num_views - 1).  num_views == 1: VideoTransform(training=False) - short
    side to int(crop_size * 256 / 224), centre crop at int(round((h - crop_size) / 2.)) (Python's round)."""
    S = int(crop_size)
    if num_views > 1:
        rh, rw = short_side_size(H, W, S)
        step = (max(rh, rw) - S) // (num_views - 1)
        return rh, rw, [(i * step, 0) if rh > rw else (0, i * step) for i in range(num_views)]
    rh, rw = short_side_size(H, W, int(S * 256 / 224))
    return rh, rw, [(int(round((rh - S) / 2.)), int(round((rw - S) / 2.)))]


def resize_axis_coefs(src, dst, clamp_weights):
    """OpenCV's INTER_LINEAR fixed-point table for one axis (cv::resize, uint8): int32 [dst, 4] = (source index 0,
    source index 1, weight 0, weight 1), weights in units of 1/2048.  Source positions are computed as OpenCV does:
    fx = float((d + 0.5) * scale - 0.5) with scale = 1 / (dst / src) in double, sx = floor(fx), weights
    round((1 - frac) * 2048) and round(frac * 2048) in float32.  Columns (`clamp_weights`) clamp position and fraction at
    both borders; rows keep the fraction and clamp only the row indices.  src == dst gives the identity (2048, 0)."""
    if src == dst:
        idx = np.arange(dst, dtype=np.int64)
        return np.stack([idx, idx, np.full(dst, 2048), np.zeros(dst, np.int64)], 1).astype(np.int32)
    scale = 1.0 / (float(dst) / float(src))
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp_weights:
        lo, hi = s < 0, s >= src - 1
        f[lo], s[lo] = 0, 0
        f[hi], s[hi] = 0, src - 1
    w0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    w1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return np.stack([np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), w0, w1], 1).astype(np.int32)


def pack_views(clips, crop_size, num_views, n_segments=1):
    """Host staging for vj_clip_views.  clips: list (over segment-major (segment, clip) order) of uint8 frames
    [T, H, W, 3].  Returns (pinned uint8 buffer, int64 [n_jobs, 4] job table, int32 [n, 4] coefficient table); job
    (segment s, view v, clip b) writes block (s * num_views + v) * B + b of the [n_seg, n_views, B, 3, T, S, S] output."""
    S = int(crop_size)
    B = len(clips) // n_segments
    T = int(clips[0].shape[0])
    sizes = [int(c.numel()) for c in clips]
    offs = np.concatenate([[0], np.cumsum([(n + 15) // 16 * 16 for n in sizes])]).astype(np.int64)
    buf = torch.empty(int(offs[-1]), dtype=torch.uint8, pin_memory=torch.cuda.is_available())
    rows, tabs, n_tab = {}, [], 0

    def table(key, src, dst, clamp):
        nonlocal n_tab
        if key not in rows:
            t = resize_axis_coefs(src, dst, clamp)
            rows[key] = n_tab
            tabs.append(t)
            n_tab += len(t)
        return rows[key]

    jobs = np.zeros((n_segments * num_views * B, 4), dtype=np.int64)
    for k, c in enumerate(clips):
        buf[offs[k]:offs[k] + sizes[k]] = c.reshape(-1)
        s, b = divmod(k, B)
        H, W = int(c.shape[1]), int(c.shape[2])
        rh, rw, wins = view_geometry(H, W, S, num_views)
        ybase = table(("y", H, rh), H, rh, False)
        xbase = table(("x", W, rw), W, rw, True)
        for v, (oy, ox) in enumerate(wins):
            j = (s * num_views + v) * B + b
            jobs[j, 0] = offs[k]
            jobs[j, 1] = j * 3 * T * S * S
            jobs[j, 2] = H | (W << 32)                                       # int32 H, W (little-endian)
            jobs[j, 3] = (ybase + oy) | ((xbase + ox) << 32)                  # int32 ytab, xtab
    return buf, torch.from_numpy(jobs), torch.from_numpy(np.concatenate(tabs, 0))


def preprocess_views(segments, device, crop_size, num_views, mean=DEFAULT_NORMALIZE[0], std=DEFAULT_NORMALIZE[1],
                     dtype=torch.float32):
    """uint8 clips -> the reference's evaluation views on `device`, nested as its collated loader yields them:
    [[view [B, 3, T, S, S] for each view] for each segment].  segments: one entry per temporal segment, each a uint8
    [B, T, H, W, 3] tensor or a list of B uint8 [T, H, W, 3] clips (frame sizes may differ between clips).  One H2D copy
    of the uint8 frames and one vj_clip_views launch for all segments, views and clips."""
    import ctypes
    clips = [c for seg in segments for c in (seg.unbind(0) if torch.is_tensor(seg) else seg)]
    if any(c.dtype != torch.uint8 or c.dim() != 4 or c.shape[-1] != 3 for c in clips):
        raise ValueError("preprocess_views expects uint8 frames [T, H, W, 3]")
    T = int(clips[0].shape[0])
    if any(int(c.shape[0]) != T for c in clips):
        raise ValueError("all clips of a batch must have the same number of frames")
    n_seg, S = len(segments), int(crop_size)
    B = len(clips) // n_seg
    buf, jobs, tab = pack_views(clips, S, num_views, n_seg)
    dbuf = buf.to(device, non_blocking=True)
    djobs = jobs.to(device)
    dtab = tab.to(device)
    out = torch.empty(n_seg, num_views, B, 3, T, S, S, dtype=dtype, device=device)
    m3 = (ctypes.c_float * 3)(*[float(x) for x in mean])
    s3 = (ctypes.c_float * 3)(*[float(x) for x in std])
    _lib.call("vj_clip_views", dbuf.data_ptr(), djobs.data_ptr(), dtab.data_ptr(), out.data_ptr(),
              1 if dtype == torch.float32 else 0, int(jobs.shape[0]), T, S, ctypes.cast(m3, ctypes.c_void_p),
              ctypes.cast(s3, ctypes.c_void_p), K._s())
    return [[out[s, v] for v in range(num_views)] for s in range(n_seg)]


class GpuEvalVideoTransform(object):
    """Deterministic evaluation transform whose pixel work runs on the GPU: __call__(buffer) returns the uint8 frames
    [T, H, W, 3] untouched (so only uint8 is collated and crosses PCIe), and `views(segments, device)` turns a collated
    batch into the reference's views with vj_clip_views.  num_views_per_clip > 1 reproduces EvalVideoTransform, 1
    reproduces VideoTransform(training=False)."""

    def __init__(self, num_views_per_clip=1, crop_size=224, normalize=DEFAULT_NORMALIZE):
        self.num_views = int(num_views_per_clip)
        self.crop_size = int(crop_size)
        self.mean, self.std = tuple(normalize[0]), tuple(normalize[1])

    def __call__(self, buffer):
        frames = torch.as_tensor(np.ascontiguousarray(buffer))
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3:
            raise ValueError("GpuEvalVideoTransform expects decoded uint8 frames [T, H, W, 3]")
        return frames

    def views(self, segments, device, dtype=torch.float32):
        return preprocess_views(segments, device, self.crop_size, self.num_views, self.mean, self.std, dtype)


def make_eval_transforms(training=True, random_horizontal_flip=True, random_resize_aspect_ratio=(3 / 4, 4 / 3),
                         random_resize_scale=(0.3, 1.0), reprob=0.0, auto_augment=False, motion_shift=False, crop_size=224,
                         num_views_per_clip=1, normalize=DEFAULT_NORMALIZE):
    """Same signature as the evaluation's make_transforms (evals/video_classification_frozen/utils.py:162-196).  The
    training transform of the frozen evaluations uses RandAugment and random erasing (eval.py:460-470), which are PIL /
    per-frame CPU augmentations with no GPU counterpart here: they raise instead of being dropped."""
    if training:
        if auto_augment or reprob > 0:
            raise NotImplementedError("the evaluation's training transform with RandAugment (auto_augment) / random erasing "
                                      "(reprob > 0) has no GPU implementation; train the probe on pre-normalised clips "
                                      "(dataset_type: synthetic)")
        return GpuVideoTransform(random_horizontal_flip=random_horizontal_flip,
                                 random_resize_aspect_ratio=random_resize_aspect_ratio,
                                 random_resize_scale=random_resize_scale, reprob=reprob, auto_augment=auto_augment,
                                 motion_shift=motion_shift, crop_size=crop_size, normalize=normalize)
    return GpuEvalVideoTransform(num_views_per_clip=num_views_per_clip, crop_size=crop_size, normalize=normalize)
