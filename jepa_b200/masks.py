"""Mask collators producing the int64 keep-index tensors that drive every gather on the hot path.

Behavioural mirror of src/masks/multiblock3d.py, src/masks/random_tube.py, src/masks/default.py.
These stay on the host (they run inside DataLoader workers in the reference); what matters is that
the index tensors are BIT-IDENTICAL to the reference's for the same torch / numpy RNG state, so the
order and kind of every RNG draw is preserved:
  * per call one `torch.Generator` seeded with the shared step counter draws three uniforms that
    fix the (t, h, w) block size for the whole batch (multiblock3d.py:106-136,162-170);
  * block positions come from the GLOBAL torch RNG, three `randint` draws per block in the order
    top, left, start (multiblock3d.py:138-142);
  * every row is truncated to the batch-minimum length, dropping the largest indices
    (multiblock3d.py:189-201).
"""
import math
from multiprocessing import Value

import numpy as np
import torch


class _StepCounter:
    """Process-shared iteration counter starting at -1 (multiblock3d.py:97-104)."""

    def __init__(self):
        self._v = Value('i', -1)

    def next(self):
        with self._v.get_lock():
            self._v.value += 1
            return self._v.value


class _MultiBlock3DGenerator(object):

    def __init__(self, crop_size=(224, 224), num_frames=16, spatial_patch_size=(16, 16), temporal_patch_size=2,
                 spatial_pred_mask_scale=(0.2, 0.8), temporal_pred_mask_scale=(1.0, 1.0), aspect_ratio=(0.3, 3.0),
                 npred=1, max_context_frames_ratio=1.0, max_keep=None):
        if not isinstance(crop_size, tuple):
            crop_size = (crop_size,) * 2
        self.crop_size = crop_size
        self.height = crop_size[0] // spatial_patch_size
        self.width = crop_size[1] // spatial_patch_size
        self.duration = num_frames // temporal_patch_size
        self.spatial_patch_size = spatial_patch_size
        self.temporal_patch_size = temporal_patch_size
        self.aspect_ratio = aspect_ratio
        self.spatial_pred_mask_scale = spatial_pred_mask_scale
        self.temporal_pred_mask_scale = temporal_pred_mask_scale
        self.npred = npred
        self.max_context_duration = max(1, int(self.duration * max_context_frames_ratio))
        self.max_keep = max_keep
        self._counter = _StepCounter()

    def step(self):
        return self._counter.next()

    def _block_size(self, gen):
        def draw(lo_hi):
            u = torch.rand(1, generator=gen).item()
            lo, hi = lo_hi
            return lo + u * (hi - lo)

        t = max(1, int(self.duration * draw(self.temporal_pred_mask_scale)))
        keep = int(self.height * self.width * draw(self.spatial_pred_mask_scale))
        ar = draw(self.aspect_ratio)
        h = min(int(round(math.sqrt(keep * ar))), self.height)
        w = min(int(round(math.sqrt(keep / ar))), self.width)
        return t, h, w

    def _context_after_one_block(self, size):
        """1 = token stays in the context, 0 = covered by this target block."""
        t, h, w = size
        top = torch.randint(0, self.height - h + 1, (1,))
        left = torch.randint(0, self.width - w + 1, (1,))
        start = torch.randint(0, self.duration - t + 1, (1,))
        keep = torch.ones((self.duration, self.height, self.width), dtype=torch.int32)
        keep[start:start + t, top:top + h, left:left + w] = 0
        if self.max_context_duration < self.duration:
            keep[self.max_context_duration:, :, :] = 0
        return keep

    def __call__(self, batch_size):
        gen = torch.Generator()
        gen.manual_seed(self.step())
        size = self._block_size(gen)

        enc_rows, pred_rows = [], []
        n_total = self.duration * self.height * self.width
        min_enc = min_pred = n_total
        while len(enc_rows) < batch_size:
            keep = torch.ones((self.duration, self.height, self.width), dtype=torch.int32)
            for _ in range(self.npred):
                keep *= self._context_after_one_block(size)
            keep = keep.flatten()
            pred_idx = torch.argwhere(keep == 0).squeeze()
            enc_idx = torch.nonzero(keep).squeeze()
            if len(enc_idx) == 0:  # degenerate draw: nothing left for the context - resample this sample
                continue
            min_pred = min(min_pred, len(pred_idx))
            min_enc = min(min_enc, len(enc_idx))
            pred_rows.append(pred_idx)
            enc_rows.append(enc_idx)
        if self.max_keep is not None:
            min_enc = min(min_enc, self.max_keep)
        masks_pred = torch.utils.data.default_collate([r[:min_pred] for r in pred_rows])
        masks_enc = torch.utils.data.default_collate([r[:min_enc] for r in enc_rows])
        return masks_enc, masks_pred


class _CollatorBase(object):
    mask_generators = ()

    def step(self):
        for g in self.mask_generators:
            g.step()

    @staticmethod
    def _collate(batch):
        """default_collate, except that ClipTickets (uint8 frames + crop/flip decisions on their way to the GPU input
        kernels, jepa_b200/transforms.py) are kept as per-clip lists: [[ticket_b for b in batch] for each clip]."""
        from .transforms import collate_tickets
        return collate_tickets(batch)

    def __call__(self, batch):
        collated = self._collate(batch)
        masks_enc, masks_pred = [], []
        for g in self.mask_generators:
            e, p = g(len(batch))
            masks_enc.append(e)
            masks_pred.append(p)
        return collated, masks_enc, masks_pred


class MultiBlock3DMaskCollator(_CollatorBase):
    """src.masks.multiblock3d.MaskCollator"""

    def __init__(self, cfgs_mask, crop_size=(224, 224), num_frames=16, patch_size=(16, 16), tubelet_size=2):
        self.mask_generators = [
            _MultiBlock3DGenerator(
                crop_size=crop_size, num_frames=num_frames, spatial_patch_size=patch_size,
                temporal_patch_size=tubelet_size, spatial_pred_mask_scale=m.get('spatial_scale'),
                temporal_pred_mask_scale=m.get('temporal_scale'), aspect_ratio=m.get('aspect_ratio'),
                npred=m.get('num_blocks'), max_context_frames_ratio=m.get('max_temporal_keep', 1.0),
                max_keep=m.get('max_keep', None)) for m in cfgs_mask]


class _RandomTubeGenerator(object):
    """Same random spatial keep-set repeated over time (random_tube.py:55-117); numpy global RNG."""

    def __init__(self, crop_size=(224, 224), num_frames=16, spatial_patch_size=(16, 16), temporal_patch_size=2,
                 ratio=0.9):
        if not isinstance(crop_size, tuple):
            crop_size = (crop_size,) * 2
        self.crop_size = crop_size
        self.height = crop_size[0] // spatial_patch_size
        self.width = crop_size[1] // spatial_patch_size
        self.duration = num_frames // temporal_patch_size
        self.spatial_patch_size = spatial_patch_size
        self.temporal_patch_size = temporal_patch_size
        self.num_patches_spatial = self.height * self.width
        self.ratio = ratio
        self.num_keep_spatial = int(self.num_patches_spatial * (1. - self.ratio))
        self.num_keep = self.num_keep_spatial * self.duration
        self._counter = _StepCounter()

    def step(self):
        return self._counter.next()

    def __call__(self, batch_size):
        enc_rows, pred_rows = [], []
        for _ in range(batch_size):
            frame = np.hstack([np.zeros(self.num_patches_spatial - self.num_keep_spatial),
                               np.ones(self.num_keep_spatial)])
            np.random.shuffle(frame)
            tube = torch.tensor(np.tile(frame, (self.duration, 1))).flatten()
            pred_rows.append(torch.argwhere(tube == 0).squeeze())
            enc_rows.append(torch.nonzero(tube).squeeze())
        return (torch.utils.data.default_collate(enc_rows), torch.utils.data.default_collate(pred_rows))


class RandomTubeMaskCollator(_CollatorBase):
    """src.masks.random_tube.MaskCollator"""

    def __init__(self, cfgs_mask, crop_size=(224, 224), num_frames=16, patch_size=(16, 16), tubelet_size=2):
        self.mask_generators = [
            _RandomTubeGenerator(crop_size=crop_size, num_frames=num_frames, spatial_patch_size=patch_size,
                                 temporal_patch_size=tubelet_size, ratio=m.get('ratio')) for m in cfgs_mask]


class DefaultCollator(object):
    """src.masks.default.DefaultCollator"""

    def __call__(self, batch):
        return torch.utils.data.default_collate(batch), None, None
