"""Data-loader factory with the reference's signature (src/datasets/data_manager.py:15-91).

Video decoding / augmentation (decord, PIL) is CPU dataloader work outside the accelerated hot path
(SURVEY.md section 2, rows 14-15).  What is provided here is the `synthetic` dataset the headline
metric is defined on (random N(0,1) clips, the distribution of normalised video) behind the same
`init_data(...) -> (loader, sampler)` contract, so `app.vjepa.train.main` runs end to end.
"""
import torch
from torch.utils.data import DataLoader, Dataset
from torch.utils.data.distributed import DistributedSampler


class SyntheticVideoDataset(Dataset):
    """Items shaped like VideoDataset's: ([clip_0, ..., clip_{num_clips-1}], label, clip_indices)."""

    def __init__(self, length, num_frames, crop_size, num_clips=1, seed=0):
        self.length, self.num_frames, self.crop_size, self.num_clips, self.seed = length, num_frames, crop_size, num_clips, seed

    def __len__(self):
        return self.length

    def __getitem__(self, index):
        g = torch.Generator().manual_seed(self.seed * 1000003 + index)
        clips = [torch.randn(3, self.num_frames, self.crop_size, self.crop_size, generator=g)
                 for _ in range(self.num_clips)]
        return clips, 0, [list(range(self.num_frames)) for _ in range(self.num_clips)]


class SyntheticUint8VideoDataset(Dataset):
    """Decoded-video stand-in: uint8 frames [T, H, W, 3] (H, W a bit larger than the crop, like decord output after the
    short-side resize) handed to `transform` exactly as VideoDataset hands its buffer to the reference transform
    (src/datasets/video_dataset.py:157-163).  With the GPU input pipeline the transform returns ClipTickets."""

    def __init__(self, length, num_frames, frame_hw, transform, num_clips=1, seed=0):
        self.length, self.num_frames, self.frame_hw, self.transform = length, num_frames, frame_hw, transform
        self.num_clips, self.seed = num_clips, seed

    def __len__(self):
        return self.length

    def __getitem__(self, index):
        g = torch.Generator().manual_seed(self.seed * 1000003 + index)
        H, W = self.frame_hw
        clips = []
        for _ in range(self.num_clips):
            buf = torch.randint(0, 256, (self.num_frames, H, W, 3), dtype=torch.uint8, generator=g).numpy()
            clips.append(self.transform(buf) if self.transform is not None else torch.from_numpy(buf))
        return clips, 0, [list(range(self.num_frames)) for _ in range(self.num_clips)]


def _class_pattern(label, shape, amplitude):
    """Fixed per-class pixel pattern (the same on every rank, split and item) that makes the labels learnable."""
    g = torch.Generator().manual_seed(7919 + int(label))
    return amplitude * torch.randn(*shape, generator=g)


class SyntheticEvalVideoDataset(Dataset):
    """Items shaped like the frozen video evaluation's VideoDataset + EvalVideoTransform output:
    ([[view_0, ..., view_{V-1}] per segment], label, [frame indices per segment]), each view a pre-normalised fp32
    [3, T, S, S] clip = class pattern + N(0, noise^2), labels index % num_classes.  After the default collate
    data[0][segment][view] is [B, 3, T, S, S] and data[2][segment] is [B, T]."""

    def __init__(self, length, num_frames, crop_size, num_classes, num_segments=1, num_views=1, seed=0, noise=0.25):
        self.length, self.num_frames, self.crop_size, self.num_classes = length, num_frames, crop_size, num_classes
        self.num_segments, self.num_views, self.seed, self.noise = num_segments, num_views, seed, noise
        self._patterns = {}

    def __len__(self):
        return self.length

    def _pattern(self, label):
        if label not in self._patterns:
            self._patterns[label] = _class_pattern(label, (3, self.num_frames, self.crop_size, self.crop_size), 1.0)
        return self._patterns[label]

    def __getitem__(self, index):
        g = torch.Generator().manual_seed(self.seed * 1000003 + index)
        label = index % self.num_classes
        base = self._pattern(label)
        clips = [[base + self.noise * torch.randn(base.shape, generator=g) for _ in range(self.num_views)]
                 for _ in range(self.num_segments)]
        idx = [torch.arange(self.num_frames) for _ in range(self.num_segments)]
        return clips, label, idx


class SyntheticUint8EvalVideoDataset(Dataset):
    """Decoded-video stand-in for the frozen video evaluation: per segment uint8 frames [T, H, W, 3] at a decoder-like,
    non-square size (class pattern + noise, clamped to 0..255), handed to `transform` as VideoDataset hands its buffer
    over.  With the GPU evaluation transform the frames stay uint8 through the collate and the views are made on the
    GPU (jepa_b200.transforms.preprocess_views)."""

    def __init__(self, length, num_frames, frame_hw, transform, num_classes, num_segments=1, seed=0):
        self.length, self.num_frames, self.frame_hw, self.transform = length, num_frames, frame_hw, transform
        self.num_classes, self.num_segments, self.seed = num_classes, num_segments, seed
        self._patterns = {}

    def __len__(self):
        return self.length

    def __getitem__(self, index):
        g = torch.Generator().manual_seed(self.seed * 1000003 + index)
        label = index % self.num_classes
        H, W = self.frame_hw
        if label not in self._patterns:
            self._patterns[label] = 128. + _class_pattern(label, (self.num_frames, H, W, 3), 48.)
        clips = []
        for _ in range(self.num_segments):
            buf = (self._patterns[label] + 16. * torch.randn(self._patterns[label].shape, generator=g))
            buf = buf.round_().clamp_(0, 255).to(torch.uint8).numpy()
            clips.append(self.transform(buf) if self.transform is not None else torch.from_numpy(buf))
        return clips, label, [torch.arange(self.num_frames) for _ in range(self.num_segments)]


class SyntheticImageDataset(Dataset):
    """Items shaped like the frozen image evaluation's ImageFolder output after its transform: (img [3, S, S] fp32,
    pre-normalised = class pattern + N(0, noise^2), label index % num_classes)."""

    def __init__(self, length, crop_size, num_classes, seed=0, noise=0.25):
        self.length, self.crop_size, self.num_classes, self.seed, self.noise = length, crop_size, num_classes, seed, noise
        self._patterns = {}

    def __len__(self):
        return self.length

    def __getitem__(self, index):
        g = torch.Generator().manual_seed(self.seed * 1000003 + index)
        label = index % self.num_classes
        if label not in self._patterns:
            self._patterns[label] = _class_pattern(label, (3, self.crop_size, self.crop_size), 1.0)
        return self._patterns[label] + self.noise * torch.randn(self._patterns[label].shape, generator=g), label


def _eval_dataset(kind, length, transform, clip_len, crop_size, num_clips, num_classes, num_views_per_clip, images,
                  training, seed):
    """The frozen evaluations' synthetic datasets (opt-in through num_classes)."""
    if images:
        if kind != 'synthetic':
            raise NotImplementedError(f"image evaluation dataset {kind!r}: only 'synthetic' (pre-normalised images) is "
                                      "provided; ImageFolder / ImageNet decoding is outside this package's scope")
        return SyntheticImageDataset(length, crop_size, num_classes, seed=seed)
    if kind == 'synthetic_uint8':
        from jepa_b200.transforms import GpuEvalVideoTransform
        if training or not isinstance(transform, GpuEvalVideoTransform):
            raise NotImplementedError(
                "dataset_type synthetic_uint8 in the frozen evaluation: the training transform uses RandAugment "
                "(auto_augment) and random erasing (reprob), which have no GPU implementation here; train on "
                "dataset_type synthetic (pre-normalised clips) - uint8 frames feed validation through vj_clip_views")
        hw = (int(crop_size * 8 / 7) // 2 * 2, int(crop_size * 4 / 3) // 2 * 2)
        return SyntheticUint8EvalVideoDataset(length, clip_len, hw, transform, num_classes, num_segments=num_clips,
                                              seed=seed)
    return SyntheticEvalVideoDataset(length, clip_len, crop_size, num_classes, num_segments=num_clips,
                                     num_views=num_views_per_clip or 1, seed=seed)


def init_data(batch_size, transform=None, shared_transform=None, data='ImageNet', collator=None, pin_mem=True,
              num_workers=8, world_size=1, rank=0, root_path=None, image_folder=None, training=True, copy_data=False,
              drop_last=True, tokenize_txt=True, subset_file=None, clip_len=8, frame_sample_rate=2, duration=None,
              num_clips=1, random_clip_sampling=True, allow_clip_overlap=False, filter_short_videos=False,
              filter_long_videos=int(1e9), decode_one_clip=True, datasets_weights=None, persistent_workers=False,
              repeat_wds=False, ipe=300, log_dir=None, crop_size=224, synthetic_length=None, num_classes=None,
              num_views_per_clip=None, images=False):
    """num_classes (opt-in): the frozen evaluations' labelled synthetic items (SyntheticEvalVideoDataset /
    SyntheticUint8EvalVideoDataset with num_views_per_clip views per segment, SyntheticImageDataset with images=True);
    left at None, the pre-training items are unchanged."""
    kind = str(data).lower()
    if num_classes is not None:
        length = synthetic_length or batch_size * world_size * ipe
        dataset = _eval_dataset(kind, length, transform, clip_len, crop_size, num_clips, num_classes, num_views_per_clip,
                                images, training, seed=rank + (0 if training else 7))
        sampler = DistributedSampler(dataset, num_replicas=world_size, rank=rank, shuffle=training)
        loader = DataLoader(dataset, collate_fn=collator, sampler=sampler, batch_size=batch_size, drop_last=drop_last,
                            pin_memory=pin_mem and kind == 'synthetic', num_workers=num_workers,
                            persistent_workers=num_workers > 0)
        return loader, sampler
    if kind == 'synthetic_uint8':
        # exercises the GPU input pipeline end to end: uint8 frames + host-side crop / flip decisions -> ClipTickets
        length = synthetic_length or batch_size * world_size * ipe
        hw = (int(crop_size * 8 / 7) // 2 * 2, int(crop_size * 4 / 3) // 2 * 2)
        dataset = SyntheticUint8VideoDataset(length, clip_len, hw, transform, num_clips=num_clips, seed=rank)
        sampler = DistributedSampler(dataset, num_replicas=world_size, rank=rank, shuffle=True)
        loader = DataLoader(dataset, collate_fn=collator, sampler=sampler, batch_size=batch_size, drop_last=drop_last,
                            pin_memory=False, num_workers=num_workers, persistent_workers=num_workers > 0)
        return loader, sampler
    if kind != 'synthetic':
        raise NotImplementedError(
            f"dataset_type={data!r}: video/image decoding pipelines (decord / PIL, src/datasets/video_dataset.py in the "
            "reference) are outside this package's scope; use dataset_type: synthetic or plug your own "
            "torch DataLoader whose collate_fn is the mask collator")
    length = synthetic_length or batch_size * world_size * ipe
    dataset = SyntheticVideoDataset(length, clip_len, crop_size, num_clips=num_clips, seed=rank)
    sampler = DistributedSampler(dataset, num_replicas=world_size, rank=rank, shuffle=True)
    loader = DataLoader(dataset, collate_fn=collator, sampler=sampler, batch_size=batch_size, drop_last=drop_last,
                        pin_memory=pin_mem, num_workers=num_workers, persistent_workers=num_workers > 0)
    return loader, sampler
