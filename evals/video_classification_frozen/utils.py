"""Import path of the reference (evals/video_classification_frozen/utils.py): the clip aggregation wrapper and the
evaluation transforms.  make_transforms(training=False) returns the GPU evaluation transform: the frames stay uint8
through the loader and vj_clip_views makes the EvalVideoTransform / VideoTransform(training=False) views on the device.
The training transform (RandAugment + random erasing in every shipped config) runs on the GPU with gpu_augment=True
and raises without it - see jepa_b200.transforms."""
import torch.nn as nn

from jepa_b200.pooler import ClipAggregation  # noqa: F401
from jepa_b200.transforms import make_eval_transforms as make_transforms  # noqa: F401


class FrameAggregation(nn.Module):
    """utils.py:23-83: an image encoder run frame by frame.  No V-JEPA configuration evaluates an image encoder
    (pretrain frames_per_clip == 1) on video; it is not implemented."""

    def __init__(self, model, max_frames=10000, use_pos_embed=False, attend_across_segments=False):
        raise NotImplementedError("FrameAggregation (pretrain frames_per_clip == 1: an image encoder evaluated on video) "
                                  "is not implemented; no V-JEPA configuration uses it")
