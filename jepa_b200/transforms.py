"""GPU input pipeline, host side (SURVEY 8f-3): the reference's VideoTransform (app/vjepa/transforms.py:40-117) split
into (a) the RANDOM DECISIONS - crop box and flip, drawn here on the host in exactly the reference's RNG call order, so
a seeded run picks the same boxes - and (b) the PIXEL MATH, which runs in one CUDA kernel (csrc/preprocess.cu:
uint8 -> bilinear random-resized crop -> flip -> normalise -> [B,3,T,S,S]) after the uint8 frames have crossed PCIe.

    tf = make_transforms(crop_size=224, ...)          # same signature as the reference factory
    item = tf(buffer_uint8_THWC)                      # in the DataLoader worker: no pixel is touched, returns a ClipTicket
    clips = preprocess_batch([item, ...], device)     # on the training process: one H2D copy of uint8 frames + one kernel

With gpu_augment=True the transform also draws RandAugment and random-erasing decisions and returns an AugmentTicket;
augment_batch (csrc/augment.cu) then applies them on the GPU, bit-exact with PIL for the RandAugment ops.  Without it
auto_augment / random erasing raise; motion_shift always raises.
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


# -------------------------------------------------------------------------------------------------
# RandAugment (rand-m7-n4-mstd0.5-inc1) and random erasing (mode 'pixel', cube) decisions, drawn on the host
# (src/datasets/utils/video/randaugment.py, randerase.py of the reference); the pixel work is csrc/augment.cu
# -------------------------------------------------------------------------------------------------
RA_OPS = ("AutoContrast", "Equalize", "Invert", "Rotate", "PosterizeIncreasing", "SolarizeIncreasing", "SolarizeAdd",
          "ColorIncreasing", "ContrastIncreasing", "BrightnessIncreasing", "SharpnessIncreasing", "ShearX", "ShearY",
          "TranslateXRel", "TranslateYRel")            # _RAND_INCREASING_TRANSFORMS, in the reference's order
RA_MAGNITUDE, RA_MAGNITUDE_STD, RA_LAYERS = 7, 0.5, 4
ERASE_AREA, ERASE_LOG_ASPECT = (0.02, 1 / 3), (math.log(0.3), math.log(1 / 0.3))


def _negate(v):
    return -v if random.random() > 0.5 else v


def rotate_matrix(degrees, W, H):
    """Inverse affine matrix of Image.rotate(degrees) about the centre without expand (PIL 12 Image.py rotate), in the
    same double arithmetic; None when PIL returns a copy (angle % 360 == 0)."""
    angle = degrees % 360.0
    if angle == 0:
        return None
    if angle in (90, 180, 270):     # PIL transposes instead; |degrees| <= 30 never gets here
        raise NotImplementedError("rotation by a multiple of 90 degrees")
    cx, cy = W / 2, H / 2
    angle = -math.radians(angle)
    m = [round(math.cos(angle), 15), round(math.sin(angle), 15), 0.0,
         round(-math.sin(angle), 15), round(math.cos(angle), 15), 0.0]
    a, b, c, d, e, f = m
    m[2], m[5] = a * -cx + b * -cy + c, d * -cx + e * -cy + f
    m[2] += cx
    m[5] += cy
    return tuple(m)


def sample_randaugment(W, H):
    """RandAugment decisions for one clip of W x H frames, drawn in the reference's order: np.random.choice of 4 of
    the 15 ops (with replacement), then per op random.random() against prob 0.5, random.gauss(7, 0.5) clipped to
    [0, 10], and the level function (with its _randomly_negate draw).  Returns 4 entries, None for a skipped op, else
    (code, fval, ival, matrix): the op's index in RA_OPS, its blend factor, its integer argument, and for the geometric
    ops the inverse affine matrix PIL resamples with (Image.transform(AFFINE) data, or rotate's matrix)."""
    picks = np.random.choice(len(RA_OPS), RA_LAYERS, replace=True, p=None)
    out = []
    for code in picks:
        code = int(code)
        if random.random() > 0.5:
            out.append(None)
            continue
        level = min(10.0, max(0, random.gauss(RA_MAGNITUDE, RA_MAGNITUDE_STD))) / 10.0
        name, fval, ival, m = RA_OPS[code], 0.0, 0, None
        if name == "Rotate":
            m = rotate_matrix(_negate(level * 30.0), W, H)
        elif name == "PosterizeIncreasing":
            ival = 4 - int(level * 4)
        elif name == "SolarizeIncreasing":
            ival = 256 - int(level * 256)
        elif name == "SolarizeAdd":
            ival = int(level * 110)
        elif name.endswith("Increasing"):       # Color / Contrast / Brightness / Sharpness
            fval = 1.0 + _negate(level * 0.9)
        elif name == "ShearX":
            m = (1.0, _negate(level * 0.3), 0.0, 0.0, 1.0, 0.0)
        elif name == "ShearY":
            m = (1.0, 0.0, 0.0, _negate(level * 0.3), 1.0, 0.0)
        elif name == "TranslateXRel":
            m = (1.0, 0.0, _negate(level * 0.45) * W, 0.0, 1.0, 0.0)
        elif name == "TranslateYRel":
            m = (1.0, 0.0, 0.0, 0.0, 1.0, _negate(level * 0.45) * H)
        out.append((code, fval, ival, m))
    return out


def sample_erase(prob, S):
    """RandomErasing._erase_cube (mode 'pixel', max_count 1) on S x S outputs: None, or ((top, left, h, w), seed)
    with one box for every frame and the seed of its N(0, 1) noise, drawn from torch's default CPU generator (the
    generator the reference's per-frame normal_() uses)."""
    if random.random() > prob:
        return None
    for _ in range(100):
        target_area = random.uniform(*ERASE_AREA) * S * S
        aspect_ratio = math.exp(random.uniform(*ERASE_LOG_ASPECT))
        h = int(round(math.sqrt(target_area * aspect_ratio)))
        w = int(round(math.sqrt(target_area / aspect_ratio)))
        if w < S and h < S:
            top = random.randint(0, S - h)
            left = random.randint(0, S - w)
            return (top, left, h, w), int(torch.randint(0, 2 ** 62, (1,)).item())
    return None


class AugmentTicket(ClipTicket):
    """A ClipTicket plus the RandAugment ops (4 entries, None where skipped; or None without RandAugment) and the erase
    box and noise seed (erase None when not erasing)."""
    __slots__ = ("ops", "erase", "seed")

    def __init__(self, frames, box, flip, ops, erase, seed):
        super().__init__(frames, box, flip)
        self.ops, self.erase, self.seed = ops, erase, seed


class GpuVideoTransform(object):
    """Drop-in for the reference's VideoTransform: __call__(buffer) consumes the same RNG draws and returns a ticket.
    Without augmentation: the crop box, then one np.random.uniform for the flip (app/vjepa/transforms.py:100-108), and a
    ClipTicket.  With gpu_augment=True, auto_augment and reprob > 0 are accepted: the RandAugment decisions come first,
    then box and flip, then the erase decision (app/vjepa/transforms.py:86-115, evals/.../utils.py:251-283), and the
    ticket is an AugmentTicket for augment_batch."""

    def __init__(self, random_horizontal_flip=True, random_resize_aspect_ratio=(3 / 4, 4 / 3), random_resize_scale=(0.3, 1.0),
                 reprob=0.0, auto_augment=False, motion_shift=False, crop_size=224, normalize=DEFAULT_NORMALIZE,
                 gpu_augment=False):
        if motion_shift:
            raise NotImplementedError("motion_shift is a CPU per-frame augmentation outside the GPU input path")
        if (auto_augment or reprob > 0) and not gpu_augment:
            raise NotImplementedError("RandAugment (auto_augment) / random erasing (reprob > 0) run on the GPU only when "
                                      "enabled with gpu_augment: true (data_aug: in a pre-training config)")
        self.random_horizontal_flip = random_horizontal_flip
        self.random_resize_aspect_ratio = tuple(random_resize_aspect_ratio)
        self.random_resize_scale = tuple(random_resize_scale)
        self.crop_size = crop_size
        self.mean, self.std = tuple(normalize[0]), tuple(normalize[1])
        self.auto_augment, self.reprob = bool(auto_augment), float(reprob)

    def __call__(self, buffer):
        frames = torch.as_tensor(np.ascontiguousarray(buffer))
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3:
            raise ValueError("GpuVideoTransform expects decoded uint8 frames [T, H, W, 3]")
        H, W = int(frames.shape[1]), int(frames.shape[2])
        ops = sample_randaugment(W, H) if self.auto_augment else None
        box = get_param_spatial_crop(self.random_resize_scale, self.random_resize_aspect_ratio, H, W)
        flip = bool(np.random.uniform() < 0.5) if self.random_horizontal_flip else False
        if not (self.auto_augment or self.reprob > 0):
            return ClipTicket(frames, box, flip)
        erase = sample_erase(self.reprob, self.crop_size) if self.reprob > 0 else None
        return AugmentTicket(frames, box, flip, ops, erase[0] if erase else None, erase[1] if erase else 0)

    def batch(self, tickets, device, dtype=torch.float32):
        """Collated AugmentTickets -> [B, 3, T, S, S] on `device` (augment_batch with this transform's normalisation)."""
        return augment_batch(tickets, device, self.crop_size, self.mean, self.std, dtype)


def make_transforms(random_horizontal_flip=True, random_resize_aspect_ratio=(3 / 4, 4 / 3), random_resize_scale=(0.3, 1.0),
                    reprob=0.0, auto_augment=False, motion_shift=False, crop_size=224, normalize=DEFAULT_NORMALIZE,
                    gpu_augment=False):
    """Same signature as app/vjepa/transforms.py:15-38, plus gpu_augment (RandAugment / random erasing on the GPU)."""
    return GpuVideoTransform(random_horizontal_flip=random_horizontal_flip, random_resize_aspect_ratio=random_resize_aspect_ratio,
                             random_resize_scale=random_resize_scale, reprob=reprob, auto_augment=auto_augment,
                             motion_shift=motion_shift, crop_size=crop_size, normalize=normalize, gpu_augment=gpu_augment)


def collate_tickets(batch):
    """default_collate, except that tickets (ClipTicket / AugmentTicket: uint8 frames + decisions on their way to the
    GPU) are kept as per-clip lists when item[0] is a list of them: [[item[0][c] for item in batch] for each clip c]."""
    first = batch[0]
    if isinstance(first, (list, tuple)) and len(first) > 0 and isinstance(first[0], (list, tuple)) and \
            len(first[0]) > 0 and isinstance(first[0][0], ClipTicket):
        clips = [[item[0][c] for item in batch] for c in range(len(first[0]))]
        rest = torch.utils.data.default_collate([tuple(item[1:]) for item in batch])
        return [clips] + list(rest)
    return torch.utils.data.default_collate(batch)


def tickets_to_device(tickets, device, crop_size, mean=DEFAULT_NORMALIZE[0], std=DEFAULT_NORMALIZE[1],
                      dtype=torch.float32):
    """A collated list of tickets -> [B, 3, T, S, S]: augment_batch for AugmentTickets, preprocess_batch otherwise."""
    if isinstance(tickets[0], AugmentTicket):
        return augment_batch(tickets, device, crop_size, mean, std, dtype)
    return preprocess_batch(tickets, device, crop_size, mean, std, dtype)


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


AUG_CLIP = np.dtype([("off", "<i8"), ("H", "<i4"), ("W", "<i4"), ("i", "<i4"), ("j", "<i4"), ("h", "<i4"),
                     ("w", "<i4"), ("flip", "<i4"), ("final_buf", "<i4"), ("etop", "<i4"), ("eleft", "<i4"),
                     ("eh", "<i4"), ("ew", "<i4"), ("seed", "<u8")])            # struct AugClip (csrc/augment.cu)
AUG_OP = np.dtype([("m", "<f8", (6,)), ("code", "<i4"), ("fval", "<f4"), ("ival", "<i4"), ("in_buf", "<i4")])   # AugOp
HIST_OPS = (RA_OPS.index("AutoContrast"), RA_OPS.index("Equalize"), RA_OPS.index("ContrastIncreasing"))


def pack_augment(tickets):
    """Host staging of a batch of AugTickets: ONE pinned uint8 buffer holding every clip's frames back to back
    (16-byte aligned), then the AugClip table [B] and the AugOp table [n_layers, B] (64-byte aligned).  Returns
    (buffer, byte size of the frame region, n_layers, layer_flags).  The host follows which of the two work buffers
    holds each clip, so a skipped op (or a rotation by 0 degrees, which PIL returns as a copy) moves no pixel."""
    B = len(tickets)
    sizes = [int(t.frames.numel()) for t in tickets]
    offs = np.concatenate([[0], np.cumsum([(s + 15) // 16 * 16 for s in sizes])]).astype(np.int64)
    frame_bytes = int((offs[-1] + 63) // 64 * 64)
    L = max((len(t.ops) for t in tickets if t.ops is not None), default=0)
    clips = np.zeros(B, AUG_CLIP)
    ops = np.zeros((L, B), AUG_OP)
    flags = np.zeros(max(L, 1), np.int32)
    cur = np.zeros(B, np.int32)
    for l in range(L):
        for b, t in enumerate(tickets):
            op = t.ops[l] if t.ops is not None and l < len(t.ops) else None
            rec = ops[l, b]
            rec["in_buf"], rec["code"] = cur[b], -1
            if op is None or (RA_OPS[op[0]] in ("Rotate", "ShearX", "ShearY", "TranslateXRel", "TranslateYRel")
                              and op[3] is None):
                continue
            rec["code"], rec["fval"], rec["ival"] = op[0], op[1], op[2]
            if op[3] is not None:
                rec["m"] = op[3]
            cur[b] ^= 1
            flags[l] |= 1 | (2 if op[0] in HIST_OPS else 0)
    for b, t in enumerate(tickets):
        T, H, W, _ = t.frames.shape
        e = t.erase or (0, 0, 0, 0)
        clips[b] = (offs[b], H, W, *t.box, int(t.flip), cur[b], *e, t.seed)
    tables = np.concatenate([clips.view(np.uint8), ops.reshape(-1).view(np.uint8)])
    buf = torch.empty(frame_bytes + tables.size, dtype=torch.uint8, pin_memory=torch.cuda.is_available())
    for b, t in enumerate(tickets):
        buf[offs[b]:offs[b] + sizes[b]] = t.frames.reshape(-1)
    buf[frame_bytes:] = torch.from_numpy(tables)
    return buf, frame_bytes, L, flags


def augment_batch(tickets, device, crop_size, mean=DEFAULT_NORMALIZE[0], std=DEFAULT_NORMALIZE[1], dtype=torch.float32,
                  with_frames=False):
    """AugmentTickets -> [B, 3, T, S, S] on `device`: RandAugment, random-resized crop, flip, normalisation and erase
    (vj_clip_augment).  One H2D copy carries the uint8 frames and the decision tables; frame sizes may differ between
    clips.  The eval pipeline (normalise at full size, then crop) and the pre-training one (crop, then normalise in
    0..1 scale) differ only in fp32 rounding; both are computed as crop-then-normalise in 0..255 scale.
    with_frames=True also returns each clip's RandAugment output, uint8 [T, H, W, 3] on `device`."""
    import ctypes
    T = int(tickets[0].frames.shape[0])
    if any(int(t.frames.shape[0]) != T for t in tickets):
        raise ValueError("all clips of a batch must have the same number of frames")
    buf, frame_bytes, L, flags = pack_augment(tickets)
    dev = buf.to(device, non_blocking=True)
    work = torch.empty(frame_bytes, dtype=torch.uint8, device=device)
    B, S = len(tickets), int(crop_size)
    hist = torch.empty(max(L, 1) * B * T * 1024, dtype=torch.int32, device=device)
    out = torch.empty(B, 3, T, S, S, dtype=dtype, device=device)
    m3 = (ctypes.c_float * 3)(*[float(x) for x in mean])
    s3 = (ctypes.c_float * 3)(*[float(x) for x in std])
    fl = (ctypes.c_int * len(flags))(*[int(x) for x in flags])
    base = dev.data_ptr()
    _lib.call("vj_clip_augment", base, work.data_ptr(), base + frame_bytes, base + frame_bytes + 64 * B, hist.data_ptr(),
              ctypes.cast(fl, ctypes.c_void_p), L, out.data_ptr(), 1 if dtype == torch.float32 else 0, B, T, S,
              ctypes.cast(m3, ctypes.c_void_p), ctypes.cast(s3, ctypes.c_void_p), K._s())
    if not with_frames:
        return out
    clips = np.frombuffer(buf[frame_bytes:frame_bytes + 64 * B].numpy().tobytes(), AUG_CLIP)
    frames = [((work if c["final_buf"] else dev)[int(c["off"]):int(c["off"]) + t.frames.numel()]).view(t.frames.shape)
              for c, t in zip(clips, tickets)]
    return out, frames


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
                         num_views_per_clip=1, normalize=DEFAULT_NORMALIZE, gpu_augment=False):
    """Same signature as the evaluation's make_transforms (evals/video_classification_frozen/utils.py:162-196), plus
    gpu_augment.  The training transform of the frozen evaluations uses RandAugment and random erasing
    (eval.py:460-470); they run on the GPU (augment_batch) with gpu_augment=True and raise without it."""
    if training:
        if (auto_augment or reprob > 0) and not gpu_augment:
            raise NotImplementedError("the evaluation's training transform with RandAugment (auto_augment) / random erasing "
                                      "(reprob > 0) runs on the GPU only with gpu_augment: true under data:; or train "
                                      "the probe on pre-normalised clips (dataset_type: synthetic)")
        return GpuVideoTransform(random_horizontal_flip=random_horizontal_flip,
                                 random_resize_aspect_ratio=random_resize_aspect_ratio,
                                 random_resize_scale=random_resize_scale, reprob=reprob, auto_augment=auto_augment,
                                 motion_shift=motion_shift, crop_size=crop_size, normalize=normalize,
                                 gpu_augment=gpu_augment)
    return GpuEvalVideoTransform(num_views_per_clip=num_views_per_clip, crop_size=crop_size, normalize=normalize)
