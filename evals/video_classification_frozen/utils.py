"""Import path of the reference (evals/video_classification_frozen/utils.py): the clip and frame aggregation wrappers and
the evaluation transforms.  make_transforms(training=False) returns the GPU evaluation transform: the frames stay uint8
through the loader and vj_clip_views makes the EvalVideoTransform / VideoTransform(training=False) views on the device.
The training transform (RandAugment + random erasing in every shipped config) runs on the GPU with gpu_augment=True
and raises without it - see jepa_b200.transforms."""
from jepa_b200.pooler import ClipAggregation, FrameAggregation  # noqa: F401
from jepa_b200.transforms import make_eval_transforms as make_transforms  # noqa: F401
