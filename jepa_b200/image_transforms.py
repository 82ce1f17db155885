"""GPU input pipeline of the frozen image evaluation, host side: the reference's image transforms (evals/
image_classification_frozen/eval.py:392-409) split into the RANDOM DECISIONS, drawn here in the reference's RNG call
order, and the PIXEL MATH, which runs in csrc/image.cu after only the uint8 images have crossed PCIe.

    validation  Resize(int(S * 256 / 224)) -> CenterCrop(S) -> ToTensor -> Normalize          GpuImageEvalTransform
    training    timm create_transform(is_training=True, auto_augment='original', interpolation='bicubic',
                re_prob=0.25, re_mode='pixel', re_count=1): RandomResizedCropAndInterpolation -> RandomHorizontalFlip ->
                AutoAugment -> ToTensor -> Normalize -> RandomErasing                            GpuImageTransform

    tf = GpuImageTransform(crop_size=224)
    ticket = tf(pil_image)                        # in the DataLoader worker: decisions only, no pixel is touched
    imgs = tf.batch(tickets, device)              # [B, 3, S, S] on the device: one H2D copy, at most 7 launches

Every output is bit-exact with the reference on the CPU: the resampling reproduces PIL 12's Resample.c, the AutoAugment
ops are the RandAugment kernels' PIL arithmetic, normalisation is torchvision's fp32 arithmetic, and the erase noise is
drawn on the host with the reference's own torch.empty(3, h, w).normal_(), so torch's generator also stays in step.
"""
import ctypes
import math
import random

import numpy as np
import torch

from . import _lib
from . import kernels as K
from .transforms import (AUG_CLIP, AUG_OP, DEFAULT_NORMALIZE, ERASE_AREA, ERASE_LOG_ASPECT, RA_OPS, _negate,
                         rotate_matrix)

# -------------------------------------------------------------------------------------------------
# PIL's resampling coefficients (Resample.c precompute_coeffs + normalize_coeffs_8bpc), in double as PIL computes them
# -------------------------------------------------------------------------------------------------
PRECISION_BITS = 22


def _pil_filter(x, bicubic):
    x = np.abs(x)
    if bicubic:                 # Resample.c bicubic_filter, a = -0.5
        a = -0.5
        return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1,
                        np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * a, 0.0))
    return np.where(x < 1.0, 1.0 - x, 0.0)     # bilinear_filter


def pil_coefs(in_size, out_size, bicubic):
    """Resampling of one axis of in_size pixels to out_size (box (0, in_size)): (first tap int64 [out], tap count
    int64 [out], int32 weights [out, ksize]) exactly as PIL computes them for 8-bit images."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = (2.0 if bicubic else 1.0) * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(out_size) + 0.5) * scale
    ss = 1.0 / filterscale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)           # C (int) truncates toward zero
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size) - xmin
    x = np.arange(ksize)
    k = _pil_filter((x[None, :] + xmin[:, None] - center[:, None] + 0.5) * ss, bicubic)
    k = np.where(x[None, :] < xmax[:, None], k, 0.0)
    ww = np.zeros(out_size)
    for c in range(ksize):                      # left to right, as the C loop sums
        ww = ww + k[:, c]
    k = np.where(ww[:, None] != 0.0, k / np.where(ww == 0.0, 1.0, ww)[:, None], k)
    scaled = k * float(1 << PRECISION_BITS)
    kk = np.where(k < 0, np.trunc(-0.5 + scaled), np.trunc(0.5 + scaled)).astype(np.int32)
    return xmin, xmax, kk


def axis_entries(in_size, out_size, start, count, bicubic):
    """Coefficient entries of outputs [start, start + count) of one axis: int32 [count, 2 + taps] = (first tap, tap
    count, weights).  When out_size == in_size PIL skips the pass; the identity entry (x, 1, 1 << 22) reproduces it."""
    if out_size == in_size:
        e = np.zeros((count, 3), np.int32)
        e[:, 0] = np.arange(start, start + count)
        e[:, 1] = 1
        e[:, 2] = 1 << PRECISION_BITS
        return e
    xmin, cnt, kk = pil_coefs(in_size, out_size, bicubic)
    sl = slice(start, start + count)
    return np.concatenate([xmin[sl, None], cnt[sl, None], kk[sl]], 1).astype(np.int32)


def resample_spec(H, W, box, out_hw, window, S, bicubic):
    """Tables of one image for csrc/image.cu: region box = (i, j, h, w) of an H x W image, resized to out_hw = (oh, ow)
    (PIL's crop(box).resize), of which the S x S window at window = (top, left) is kept.  Returns
    (c0, xent [S, 2 + kx], r0, nrows, yent [S, 2 + ky]): horizontal taps count from source column c0, vertical taps from
    source row r0 (the first of the nrows rows the vertical pass reads)."""
    i, j, h, w = box
    oh, ow = out_hw
    top, left = window
    if not (0 <= top and top + S <= oh and 0 <= left and left + S <= ow):
        raise ValueError(f"window {window} of {S} x {S} outside the resized {oh} x {ow} image")
    if not (0 <= i and i + h <= H and 0 <= j and j + w <= W and h > 0 and w > 0):
        raise ValueError(f"box {box} outside the {H} x {W} image")
    xent = axis_entries(w, ow, left, S, bicubic)
    yent = axis_entries(h, oh, top, S, bicubic)
    lo = int(yent[:, 0].min())
    hi = int((yent[:, 0] + yent[:, 1]).max())
    yent = yent.copy()
    yent[:, 0] -= lo
    return j, xent, i + lo, hi - lo, yent


# -------------------------------------------------------------------------------------------------
# Validation geometry (torchvision Resize(int) / CenterCrop on a PIL image)
# -------------------------------------------------------------------------------------------------
def resized_size(H, W, size):
    """torchvision's _compute_resized_output_size for Resize(size: int): short side -> size, long side
    int(size * long / short).  Returns (h', w')."""
    short, long = (W, H) if W <= H else (H, W)
    new_short, new_long = size, int(size * long / short)
    return (new_long, new_short) if W <= H else (new_short, new_long)


def eval_geometry(H, W, S):
    """(h', w', top, left): the resize of Resize(int(S * 256 / 224)) and the origin of CenterCrop(S), which rounds
    (h' - S) / 2 with Python's round (half to even)."""
    rh, rw = resized_size(H, W, int(S * 256 / 224))
    return rh, rw, int(round((rh - S) / 2.0)), int(round((rw - S) / 2.0))


# -------------------------------------------------------------------------------------------------
# Training decisions
# -------------------------------------------------------------------------------------------------
# timm's auto_augment_policy_original: the AutoAugment paper's ImageNet policy (torchvision's AutoAugmentPolicy.IMAGENET,
# with Posterize as PosterizeOriginal); (op, probability, magnitude), magnitude None for the ops without a level
AA_POLICY = (
    (("PosterizeOriginal", 0.4, 8), ("Rotate", 0.6, 9)),
    (("Solarize", 0.6, 5), ("AutoContrast", 0.6, None)),
    (("Equalize", 0.8, None), ("Equalize", 0.6, None)),
    (("PosterizeOriginal", 0.6, 7), ("PosterizeOriginal", 0.6, 6)),
    (("Equalize", 0.4, None), ("Solarize", 0.2, 4)),
    (("Equalize", 0.4, None), ("Rotate", 0.8, 8)),
    (("Solarize", 0.6, 3), ("Equalize", 0.6, None)),
    (("PosterizeOriginal", 0.8, 5), ("Equalize", 1.0, None)),
    (("Rotate", 0.2, 3), ("Solarize", 0.6, 8)),
    (("Equalize", 0.6, None), ("PosterizeOriginal", 0.4, 6)),
    (("Rotate", 0.8, 8), ("Color", 0.4, 0)),
    (("Rotate", 0.4, 9), ("Equalize", 0.6, None)),
    (("Equalize", 0.0, None), ("Equalize", 0.8, None)),
    (("Invert", 0.6, None), ("Equalize", 1.0, None)),
    (("Color", 0.6, 4), ("Contrast", 1.0, 8)),
    (("Rotate", 0.8, 8), ("Color", 1.0, 2)),
    (("Color", 0.8, 8), ("Solarize", 0.8, 7)),
    (("Sharpness", 0.4, 7), ("Invert", 0.6, None)),
    (("ShearX", 0.6, 5), ("Equalize", 1.0, None)),
    (("Color", 0.4, 0), ("Equalize", 0.6, None)),
    (("Equalize", 0.4, None), ("Solarize", 0.2, 4)),
    (("Solarize", 0.6, 5), ("AutoContrast", 0.6, None)),
    (("Invert", 0.6, None), ("Equalize", 1.0, None)),
    (("Color", 0.6, 4), ("Contrast", 1.0, 8)),
    (("Equalize", 0.8, None), ("Equalize", 0.6, None)),
)
# AutoAugment op -> the RandAugment kernel op (csrc/augment.cu RaOp) that computes it
AA_KERNEL_OP = {"AutoContrast": "AutoContrast", "Equalize": "Equalize", "Invert": "Invert", "Rotate": "Rotate",
                "PosterizeOriginal": "PosterizeIncreasing", "Solarize": "SolarizeIncreasing", "Color": "ColorIncreasing",
                "Contrast": "ContrastIncreasing", "Sharpness": "SharpnessIncreasing", "ShearX": "ShearX"}
_POLICY_IDS = list(range(len(AA_POLICY)))     # random.choice over these draws as timm's random.choice(policy)
RRC_SCALE, RRC_RATIO = (0.08, 1.0), (3.0 / 4.0, 4.0 / 3.0)


def fill_color(mean):
    """timm's img_mean hparam: the geometric ops' fill, round(255 * mean) per channel ((124, 116, 104) for ImageNet)."""
    return tuple(min(255, round(255 * x)) for x in mean)


def rrc_params(H, W, scale=RRC_SCALE, ratio=RRC_RATIO):
    """RandomResizedCropAndInterpolation.get_params: (i, j, h, w), drawn with `random` (10 tries, then the central crop)."""
    area = W * H
    for _ in range(10):
        target_area = random.uniform(*scale) * area
        log_ratio = (math.log(ratio[0]), math.log(ratio[1]))
        aspect_ratio = math.exp(random.uniform(*log_ratio))
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if w <= W and h <= H:
            i = random.randint(0, H - h)
            j = random.randint(0, W - w)
            return i, j, h, w
    in_ratio = W / H
    if in_ratio < min(ratio):
        w = W
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = H
        w = int(round(h * max(ratio)))
    else:
        w, h = W, H
    return (H - h) // 2, (W - w) // 2, h, w


def sample_autoaugment(S):
    """AutoAugment 'original' on an S x S image, in timm's draw order: random.choice of the sub-policy, then per op
    random.random() > prob (only when prob < 1) and the level function (Rotate and ShearX draw a sign).  Returns
    (sub-policy index, [(name, level args) of each applied op], [kernel op record (code, fval, ival, matrix) or None
    per op])."""
    policy = random.choice(_POLICY_IDS)
    applied, ops = [], []
    for name, prob, mag in AA_POLICY[policy]:
        if prob < 1.0 and random.random() > prob:
            ops.append(None)
            continue
        level = min(10.0, max(0, mag)) if mag is not None else None
        code, fval, ival, m = RA_OPS.index(AA_KERNEL_OP[name]), 0.0, 0, None
        if name == "Rotate":
            args = (_negate((level / 10.0) * 30.0),)
            m = rotate_matrix(args[0], S, S)
        elif name == "ShearX":
            args = (_negate((level / 10.0) * 0.3),)
            m = (1.0, args[0], 0.0, 0.0, 1.0, 0.0)
        elif name == "PosterizeOriginal":
            args = (int((level / 10.0) * 4) + 4,)
            ival = args[0]
        elif name == "Solarize":
            args = (int((level / 10.0) * 256),)
            ival = args[0]
        elif name in ("Color", "Contrast", "Sharpness"):
            args = ((level / 10.0) * 1.8 + 0.1,)
            fval = args[0]
        else:
            args = ()
        applied.append((name, args))
        ops.append((code, fval, ival, m))
    return policy, applied, ops


def sample_erase(S, prob=0.25):
    """RandomErasing._erase (mode 'pixel', count 1) on a [3, S, S] image: None, or ((top, left, h, w), noise fp32
    [3, h, w]) with the noise drawn as the reference draws it, torch.empty(3, h, w).normal_() on the CPU."""
    if random.random() > prob:
        return None
    area = S * S
    for _ in range(10):
        target_area = random.uniform(*ERASE_AREA) * area
        aspect_ratio = math.exp(random.uniform(*ERASE_LOG_ASPECT))
        h = int(round(math.sqrt(target_area * aspect_ratio)))
        w = int(round(math.sqrt(target_area / aspect_ratio)))
        if w < S and h < S:
            top = random.randint(0, S - h)
            left = random.randint(0, S - w)
            return (top, left, h, w), torch.empty((3, h, w), dtype=torch.float32).normal_()
    return None


def as_uint8_image(img):
    """A PIL image (converted to RGB) or a uint8 [H, W, 3] array -> uint8 tensor [H, W, 3]."""
    if hasattr(img, "convert"):
        img = np.array(img.convert("RGB"))
    x = torch.as_tensor(np.ascontiguousarray(img))
    if x.dtype != torch.uint8 or x.dim() != 3 or x.shape[-1] != 3:
        raise ValueError("expected a PIL image or a uint8 [H, W, 3] array")
    return x


class ImageTicket:
    """One image on its way to the GPU: the untouched uint8 pixels [H, W, 3] (validation: nothing else)."""
    __slots__ = ("image",)

    def __init__(self, image):
        self.image = image


class ImageAugmentTicket(ImageTicket):
    """An image plus its training decisions: crop box (i, j, h, w), flip, AutoAugment sub-policy, applied ops
    [(name, args)] and kernel op records (2 entries, None where skipped), erase box (or None) and its noise [3, h, w]."""
    __slots__ = ("box", "flip", "policy", "applied", "ops", "erase", "noise")

    def __init__(self, image, box, flip, policy, applied, ops, erase, noise):
        super().__init__(image)
        self.box, self.flip, self.policy, self.applied, self.ops = box, flip, policy, applied, ops
        self.erase, self.noise = erase, noise


class GpuImageEvalTransform(object):
    """Validation transform of the frozen image evaluation: __call__(img) keeps only the uint8 pixels; batch() makes
    [B, 3, S, S] with vj_image_views, equal to Resize(int(S * 256 / 224)) / CenterCrop(S) / ToTensor / Normalize."""

    def __init__(self, crop_size=224, normalize=DEFAULT_NORMALIZE):
        self.crop_size = int(crop_size)
        self.mean, self.std = tuple(normalize[0]), tuple(normalize[1])

    def __call__(self, img):
        return ImageTicket(as_uint8_image(img))

    def batch(self, tickets, device, dtype=torch.float32):
        return image_views_batch(tickets, device, self.crop_size, self.mean, self.std, dtype)


class GpuImageTransform(GpuImageEvalTransform):
    """Training transform of the frozen image evaluation: __call__(img) draws the crop box (`random`), the flip
    (torch.rand(1) < 0.5), AutoAugment 'original' (`random`) and the erase box and noise (`random`, torch) in that order,
    as timm's composed transform draws them, and returns an ImageAugmentTicket; batch() applies them on the GPU
    (vj_image_augment)."""

    def __init__(self, crop_size=224, normalize=DEFAULT_NORMALIZE, re_prob=0.25):
        super().__init__(crop_size, normalize)
        self.re_prob = float(re_prob)

    def __call__(self, img):
        x = as_uint8_image(img)
        H, W = int(x.shape[0]), int(x.shape[1])
        box = rrc_params(H, W)
        if box[2] <= 0 or box[3] <= 0:
            raise ValueError(f"image of {W} x {H} pixels is too small for a random-resized crop")
        flip = bool(torch.rand(1) < 0.5)
        policy, applied, ops = sample_autoaugment(self.crop_size)
        er = sample_erase(self.crop_size, self.re_prob) if self.re_prob > 0 else None
        return ImageAugmentTicket(x, box, flip, policy, applied, ops, er[0] if er else None, er[1] if er else None)

    def batch(self, tickets, device, dtype=torch.float32):
        return image_augment_batch(tickets, device, self.crop_size, self.mean, self.std, dtype)


def collate_image_tickets(batch):
    """(ticket, label) items -> [list of tickets, label tensor]; anything else goes through default_collate."""
    if len(batch) > 0 and isinstance(batch[0], (list, tuple)) and isinstance(batch[0][0], ImageTicket):
        return [[item[0] for item in batch], torch.as_tensor([int(item[1]) for item in batch])]
    return torch.utils.data.default_collate(batch)


# -------------------------------------------------------------------------------------------------
# Packing: one pinned host buffer, one H2D copy
# -------------------------------------------------------------------------------------------------
IMG_JOB = np.dtype([("src_off", "<i8"), ("tmp_off", "<i8"), ("W", "<i4"), ("r0", "<i4"), ("nrows", "<i4"),
                    ("c0", "<i4"), ("xtab", "<i4"), ("ytab", "<i4"), ("xk", "<i4"), ("yk", "<i4"), ("flip", "<i4"),
                    ("pad", "<i4", (3,))])                                    # struct ImgJob (csrc/image.cu)
assert IMG_JOB.itemsize == 64 and AUG_CLIP.itemsize == 64 and AUG_OP.itemsize == 64


def _align(n, a=64):
    return (n + a - 1) // a * a


class _Packer:
    """Appends 64-byte aligned sections to one host byte buffer."""

    def __init__(self):
        self.parts, self.size = [], 0

    def add(self, arr):
        off = self.size
        b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
        self.parts.append((off, b))
        self.size = _align(off + b.size)
        return off


def pack_resample(images, specs, S):
    """images: uint8 [H, W, 3] tensors; specs: per image (box, out_hw, window, bicubic, flip).  Returns (packer with the
    images, job table and coefficient table appended, byte offsets of jobs and coefs, tmp bytes)."""
    pk = _Packer()
    offs = [pk.add(x.numpy()) for x in images]
    jobs = np.zeros(len(images), IMG_JOB)
    tabs, n_tab, tmp = [], 0, 0
    for b, (x, (box, out_hw, window, bicubic, flip)) in enumerate(zip(images, specs)):
        H, W = int(x.shape[0]), int(x.shape[1])
        c0, xent, r0, nrows, yent = resample_spec(H, W, box, out_hw, window, S, bicubic)
        jobs[b] = (offs[b], tmp, W, r0, nrows, c0, n_tab, n_tab + xent.size, xent.shape[1], yent.shape[1], int(flip),
                   (0, 0, 0))
        tabs += [xent.reshape(-1), yent.reshape(-1)]
        n_tab += xent.size + yent.size
        tmp += _align(nrows * S * 3, 16)
    jobs_off = pk.add(jobs)
    coefs_off = pk.add(np.concatenate(tabs).astype(np.int32))
    return pk, jobs_off, coefs_off, tmp


def to_device(pk, device):
    """The packer's sections in one pinned host buffer, copied to `device` in one H2D copy: (device, host) buffers."""
    buf = torch.zeros(max(pk.size, 64), dtype=torch.uint8, pin_memory=torch.cuda.is_available())
    host = buf.numpy()
    for off, b in pk.parts:
        host[off:off + b.size] = b
    return buf.to(device, non_blocking=True), buf


def _floats(v):
    return ctypes.cast((ctypes.c_float * 3)(*[float(x) for x in v]), ctypes.c_void_p)


def image_views_batch(tickets, device, crop_size, mean=DEFAULT_NORMALIZE[0], std=DEFAULT_NORMALIZE[1],
                      dtype=torch.float32):
    """Validation: ImageTickets (or uint8 [H, W, 3] tensors) -> [B, 3, S, S] on `device` (vj_image_views, 2 launches)."""
    S = int(crop_size)
    images = [t.image if isinstance(t, ImageTicket) else t for t in tickets]
    pk, jobs_off, coefs_off, tmp_bytes = pack_image_views(images, S)
    dev, _ = to_device(pk, device)
    tmp = torch.empty(max(tmp_bytes, 16), dtype=torch.uint8, device=device)
    out = torch.empty(len(images), 3, S, S, dtype=dtype, device=device)
    launch_image_views(dev, jobs_off, coefs_off, tmp, out, mean, std)
    return out


def pack_image_views(images, S):
    """Host staging of vj_image_views: each image's Resize(int(S * 256 / 224)) + CenterCrop(S) tables."""
    specs = []
    for x in images:
        H, W = int(x.shape[0]), int(x.shape[1])
        rh, rw, top, left = eval_geometry(H, W, S)
        specs.append(((0, 0, H, W), (rh, rw), (top, left), False, False))
    return pack_resample(images, specs, S)


def launch_image_views(dev, jobs_off, coefs_off, tmp, out, mean, std):
    """vj_image_views on a staged batch (`dev`: the packer's buffer on the device, only read)."""
    base = dev.data_ptr()
    B, S = int(out.shape[0]), int(out.shape[-1])
    _lib.call("vj_image_views", base, base + jobs_off, base + coefs_off, tmp.data_ptr(), out.data_ptr(),
              1 if out.dtype == torch.float32 else 0, B, S, _floats(mean), _floats(std), K._s())


def pack_image_augment(images, specs, S, ops_per_image, erases, noises):
    """Host staging of vj_image_augment: images resampled by `specs`, then the kernel op records (lists of
    (code, fval, ival, m) or None) and the erase boxes with their noise.  Returns a dict: `pk` (the packer: images, job,
    coefficient, clip, op tables and noise), the byte offsets of each table, tmp bytes, n_layers, layer flags and the
    work buffer that holds each image at the end.  The host follows which buffer holds each image, so a skipped op
    moves no pixel."""
    B = len(images)
    pk, jobs_off, coefs_off, tmp_bytes = pack_resample(images, specs, S)
    L = max((len(o) for o in ops_per_image), default=0)
    clips = np.zeros(B, AUG_CLIP)
    ops = np.zeros((max(L, 1), B), AUG_OP)
    flags = np.zeros(max(L, 1), np.int32)
    cur = np.zeros(B, np.int32)
    for l in range(L):
        for b in range(B):
            op = ops_per_image[b][l] if l < len(ops_per_image[b]) else None
            rec = ops[l, b]
            rec["in_buf"], rec["code"] = cur[b], -1
            if op is None or (op[3] is None and RA_OPS[op[0]] in ("Rotate", "ShearX")) or \
                    (RA_OPS[op[0]] == "PosterizeIncreasing" and op[2] >= 8):
                continue                    # skipped, a rotation PIL returns as a copy, or posterize keeping 8 bits
            rec["code"], rec["fval"], rec["ival"] = op[0], op[1], op[2]
            if op[3] is not None:
                rec["m"] = op[3]
            cur[b] ^= 1
            flags[l] |= 1 | (2 if RA_OPS[op[0]] in ("AutoContrast", "Equalize", "ContrastIncreasing") else 0)
    noise_parts, n_noise = [], 0
    for b in range(B):
        e, nz = erases[b], noises[b]
        if e is not None:
            clips[b] = (b * S * S * 3, S, S, 0, 0, S, S, 0, cur[b], *e, n_noise)
            noise_parts.append(nz.reshape(-1).numpy())
            n_noise += nz.numel()
        else:
            clips[b] = (b * S * S * 3, S, S, 0, 0, S, S, 0, cur[b], 0, 0, 0, 0, 0)
    clips_off = pk.add(clips)
    ops_off = pk.add(ops.reshape(-1))
    noise_off = pk.add(np.concatenate(noise_parts).astype(np.float32)) if noise_parts else None
    return dict(pk=pk, B=B, S=S, jobs_off=jobs_off, coefs_off=coefs_off, clips_off=clips_off, ops_off=ops_off,
                noise_off=noise_off, tmp_bytes=_align(max(tmp_bytes, 16), 256), img_bytes=_align(B * S * S * 3, 256),
                L=L, flags=flags, cur=cur)


def image_augment_scratch(packed, device):
    """Device scratch of one vj_image_augment launch: horizontal-pass rows, the two work buffers and the histograms."""
    return torch.empty(packed["tmp_bytes"] + 2 * packed["img_bytes"] + max(packed["L"], 1) * packed["B"] * 1024 * 4,
                       dtype=torch.uint8, device=device)


def launch_image_augment(dev, packed, scratch, out, mean, std, fill):
    """vj_image_augment on a staged batch: `dev` is the packer's buffer on the device (only read), `out` [B, 3, S, S]."""
    base, sp = dev.data_ptr(), scratch.data_ptr()
    tb, ib = packed["tmp_bytes"], packed["img_bytes"]
    fl = (ctypes.c_int * len(packed["flags"]))(*[int(x) for x in packed["flags"]])
    f3 = (ctypes.c_ubyte * 3)(*fill)
    noise_off = packed["noise_off"]
    _lib.call("vj_image_augment", base, base + packed["jobs_off"], base + packed["coefs_off"], sp, sp + tb,
              sp + tb + ib, base + packed["clips_off"], base + packed["ops_off"], sp + tb + 2 * ib,
              ctypes.cast(fl, ctypes.c_void_p), packed["L"], None if noise_off is None else base + noise_off,
              out.data_ptr(), 1 if out.dtype == torch.float32 else 0, packed["B"], packed["S"], _floats(mean),
              _floats(std), ctypes.cast(f3, ctypes.c_void_p), K._s())


def _run_augment(images, specs, S, ops_per_image, erases, noises, device, mean, std, fill, dtype):
    """pack_image_augment + one H2D copy + launch_image_augment.  Returns (out [B, 3, S, S], the two work buffers
    [B, S, S, 3], the buffer holding each image at the end)."""
    packed = pack_image_augment(images, specs, S, ops_per_image, erases, noises)
    dev, _ = to_device(packed["pk"], device)
    scratch = image_augment_scratch(packed, device)
    B, tb, ib = len(images), packed["tmp_bytes"], packed["img_bytes"]
    out = torch.empty(B, 3, S, S, dtype=dtype, device=device)
    launch_image_augment(dev, packed, scratch, out, mean, std, fill)
    b0 = scratch[tb:tb + B * S * S * 3].view(B, S, S, 3)
    b1 = scratch[tb + ib:tb + ib + B * S * S * 3].view(B, S, S, 3)
    return out, b0, b1, packed["cur"]


def image_augment_batch(tickets, device, crop_size, mean=DEFAULT_NORMALIZE[0], std=DEFAULT_NORMALIZE[1],
                        dtype=torch.float32, with_images=False):
    """Training: ImageAugmentTickets -> [B, 3, S, S] on `device` (vj_image_augment: bicubic crop-resize and flip,
    AutoAugment with fill round(255 * mean), ToTensor + Normalize, erase).  with_images=True also returns the uint8
    AutoAugment outputs [B, S, S, 3] on `device`."""
    S = int(crop_size)
    images = [t.image for t in tickets]
    specs = [(t.box, (S, S), (0, 0), True, t.flip) for t in tickets]
    out, b0, b1, cur = _run_augment(images, specs, S, [t.ops for t in tickets], [t.erase for t in tickets],
                                    [t.noise for t in tickets], device, mean, std, fill_color(mean), dtype)
    if not with_images:
        return out
    return out, torch.stack([(b1 if c else b0)[b] for b, c in enumerate(cur)])


def resample_images(images, specs, S, device, ops=None, fill=(128, 128, 128)):
    """uint8 S x S windows [B, S, S, 3] on `device` of images resampled by specs (box, out_hw, window, bicubic, flip),
    then the given kernel op records (one list per image), through vj_image_augment's passes."""
    ops = ops or [[] for _ in images]
    _, b0, b1, cur = _run_augment(images, specs, S, ops, [None] * len(images), [None] * len(images), device,
                                  DEFAULT_NORMALIZE[0], DEFAULT_NORMALIZE[1], fill, torch.float32)
    return torch.stack([(b1 if c else b0)[b] for b, c in enumerate(cur)])
