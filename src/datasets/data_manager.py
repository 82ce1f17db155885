"""Data-loader factory with the reference's signature (src/datasets/data_manager.py:15-91).

Video decoding / augmentation (decord, PIL) is CPU dataloader work outside the accelerated hot path
(SURVEY.md section 2, rows 14-15).  What is provided here is the `synthetic` dataset the headline
metric is defined on (random N(0,1) clips, the distribution of normalised video) behind the same
`init_data(...) -> (loader, sampler)` contract, so `app.vjepa.train.main` runs end to end.
"""
import os
from logging import getLogger

import torch
from torch.utils.data import DataLoader, Dataset
from torch.utils.data.distributed import DistributedSampler

logger = getLogger()


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


class SyntheticUint8ImageDataset(Dataset):
    """Decoded-image stand-in for the frozen image evaluation: (transform(uint8 [H, W, 3]), label) with a size that varies
    per item (landscape and portrait, like decoded photos), class pattern + noise clamped to 0..255, label
    index % num_classes.  The class pattern is a dark / bright texture whose orientation (label % 3: horizontal stripes,
    vertical stripes, checkerboard) and period (16 + 4 * (label // 3) pixels) survive what the training transform does
    to an image: crops down to 8 % of the area, flips, rotations up to 27 degrees, colour and histogram ops, inversion,
    erasing, and Solarize at any of its thresholds (dark 40 and bright 140 stay apart after 255 - v).  With the GPU image transforms the items are tickets and the pixel work runs on the GPU."""
    SIZES = ((3, 4), (4, 3), (9, 16), (1, 1), (5, 4), (3, 5))     # height : width

    def __init__(self, length, crop_size, num_classes, transform, seed=0):
        self.length, self.crop_size, self.num_classes, self.transform = length, crop_size, num_classes, transform
        self.seed = seed

    def __len__(self):
        return self.length

    def __getitem__(self, index):
        g = torch.Generator().manual_seed(self.seed * 1000003 + index)
        label = index % self.num_classes
        short = int(self.crop_size * (1.0 + 0.5 * torch.rand(1, generator=g).item()))
        a, b = self.SIZES[index % len(self.SIZES)]
        H, W = (short * a // min(a, b), short * b // min(a, b))
        half = 8 + 2 * (label // 3)
        y, x = torch.meshgrid(torch.arange(H) // half, torch.arange(W) // half, indexing='ij')
        bright = (y, x, y + x)[label % 3] % 2
        base = 40. + 100. * bright[..., None].float() + _class_pattern(label, (3,), 8.)
        img = (base + 8. * torch.randn(base.shape, generator=g)).round_().clamp_(0, 255).to(torch.uint8).numpy()
        return (self.transform(img) if self.transform is not None else torch.from_numpy(img)), label


IMAGE_FOLDERS = ('imagenet', 'inat21', 'places205')


def _image_folder_loader(transform, batch_size, collator, pin_mem, num_workers, world_size, rank, root_path,
                         image_folder, training, drop_last, persistent_workers):
    """src/datasets/image_dataset.py of the reference: torchvision ImageFolder at root_path/image_folder/{train,val}/
    (default PIL loader, RGB), DistributedSampler(dataset, world_size, rank) (shuffled on both splits)."""
    import torchvision
    from jepa_b200.image_transforms import GpuImageEvalTransform, collate_image_tickets
    data_path = os.path.join(root_path, image_folder, 'train/' if training else 'val/')
    logger.info(f'data-path {data_path}')
    dataset = torchvision.datasets.ImageFolder(root=data_path, transform=transform)
    sampler = DistributedSampler(dataset=dataset, num_replicas=world_size, rank=rank)
    tickets = isinstance(transform, GpuImageEvalTransform)
    if collator is None and tickets:
        collator = collate_image_tickets        # [tickets], labels: the pixels are made on the GPU
    loader = DataLoader(dataset, collate_fn=collator, sampler=sampler, batch_size=batch_size, drop_last=drop_last,
                        pin_memory=pin_mem and not tickets, num_workers=num_workers,
                        persistent_workers=persistent_workers and num_workers > 0)
    return loader, sampler


def _eval_dataset(kind, length, transform, clip_len, crop_size, num_clips, num_classes, num_views_per_clip, images,
                  training, seed):
    """The frozen evaluations' synthetic datasets (opt-in through num_classes)."""
    if images:
        if kind == 'synthetic_uint8':
            return SyntheticUint8ImageDataset(length, crop_size, num_classes, transform, seed=seed)
        if kind != 'synthetic':
            raise NotImplementedError(f"image evaluation dataset {kind!r}: 'synthetic', 'synthetic_uint8' and the "
                                      f"ImageFolder datasets {IMAGE_FOLDERS} are provided")
        return SyntheticImageDataset(length, crop_size, num_classes, seed=seed)
    if kind == 'synthetic_uint8':
        from jepa_b200.transforms import GpuEvalVideoTransform, GpuVideoTransform
        if not isinstance(transform, GpuVideoTransform if training else GpuEvalVideoTransform):
            raise NotImplementedError(
                "dataset_type synthetic_uint8 in the frozen evaluation: the training transform uses RandAugment "
                "(auto_augment) and random erasing (reprob), which run on the GPU only with gpu_augment: true under "
                "data:; or train on dataset_type synthetic (pre-normalised clips)")
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
    SyntheticUint8EvalVideoDataset with num_views_per_clip views per segment, SyntheticImageDataset /
    SyntheticUint8ImageDataset with images=True); left at None, the pre-training items are unchanged.  With images=True,
    data ImageNet / iNat21 / Places205 (any case) is an ImageFolder at root_path/image_folder/{train,val}/."""
    kind = str(data).lower()
    if images and kind in IMAGE_FOLDERS:
        if subset_file is not None or copy_data:
            raise NotImplementedError("ImageFolder datasets: subset_file and copy_data are not supported; point "
                                      "root_path / image_folder at the images to use")
        return _image_folder_loader(transform, batch_size, collator, pin_mem, num_workers, world_size, rank, root_path,
                                    image_folder, training, drop_last, persistent_workers)
    if num_classes is not None:
        length = synthetic_length or batch_size * world_size * ipe
        dataset = _eval_dataset(kind, length, transform, clip_len, crop_size, num_clips, num_classes, num_views_per_clip,
                                images, training, seed=rank + (0 if training else 7))
        sampler = DistributedSampler(dataset, num_replicas=world_size, rank=rank, shuffle=training)
        if collator is None and kind == 'synthetic_uint8' and images:
            from jepa_b200.image_transforms import collate_image_tickets
            collator = collate_image_tickets    # [tickets], labels
        elif collator is None and kind == 'synthetic_uint8' and training:
            from jepa_b200.transforms import collate_tickets
            collator = collate_tickets      # [[ticket for each clip] for each segment], labels, indices
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
