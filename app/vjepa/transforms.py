"""make_transforms with the reference's signature (app/vjepa/transforms.py:15).

The reference's VideoTransform does its pixel work on CPU dataloader workers.  Here the transform only takes the RANDOM
DECISIONS (crop box, flip - same RNG call order as the reference) in the worker and returns a ClipTicket with the
untouched uint8 frames; the pixels are produced on the GPU by one kernel per batch after the uint8 frames crossed PCIe
(jepa_b200/transforms.py, csrc/preprocess.cu).  auto_augment (RandAugment) and random erasing run on the GPU
(csrc/augment.cu) when data_aug.gpu_augment is true and are rejected otherwise; motion_shift is always rejected."""
from jepa_b200.transforms import make_transforms  # noqa: F401
