"""Frozen image evaluation: `evals.image_classification_frozen.eval.main(args_eval, resume_preempt=False)`.

Same config keys, log lines, CSV columns and checkpoint dictionary as the reference (evals/image_classification_frozen/
eval.py:63-521): a video encoder from pre-training sees each image repeated `frames_per_clip` times (a forward pre-hook,
reference :451-456), and the attentive probe trains on its tokens with one classifier call per step.  The optimizer,
checkpoint and encoder-loading helpers, the epoch loop (train_heads) and the batch loop (run_head_loop) are the video
evaluation's (the reference has identical copies of the helpers); run_one_epoch supplies the image batch and loss.

The reference autocasts the loop body to fp16 (eval.py:284, `autocast(dtype=torch.float16, enabled=use_bfloat16)`).
By default this loop opens no autocast region, so encoder and probe compute bf16 x bf16 -> fp32, and `use_bfloat16`
selects the GradScaler, as it does in the reference.  `optimization.fp16_autocast: true` opens that region where the
reference does and builds the classifier to follow it, exactly as in the video evaluation: fp16 encoder and probe with
`use_bfloat16: true`, bf16 throughout with `use_bfloat16: false`.  There is no fp32 path.

`optimization.multihead_kwargs` trains several probes on one encoder pass per batch, with the video evaluation's parser,
head construction, checkpoint and CSV layout (read_multihead_kwargs, build_heads, train_heads).
`optimization.probe_depth` (default 1) sets every head's AttentiveClassifier depth, as in the video evaluation.
"""
import os

try:
    # one visible device per process under SLURM
    os.environ['CUDA_VISIBLE_DEVICES'] = os.environ['SLURM_LOCALID']
except Exception:
    pass

import logging
import pprint

import numpy as np
import torch
import torch.multiprocessing as mp
import torch.nn.functional as F

import src.models.vision_transformer as vit
from evals.video_classification_frozen.eval import (  # noqa: F401  (the helpers both evaluations share)
    build_heads, init_opt, load_checkpoint, load_pretrained, loop_autocast, one_head, read_fp16_autocast,
    read_multihead_kwargs, read_probe_depth, require_cuda, run_head_loop, step_head, train_heads)
from src.datasets.data_manager import init_data
from src.models.attentive_pooler import AttentiveClassifier
from src.utils.distributed import init_distributed

logging.basicConfig()
logger = logging.getLogger()
logger.setLevel(logging.INFO)

_GLOBAL_SEED = 0
np.random.seed(_GLOBAL_SEED)
torch.manual_seed(_GLOBAL_SEED)

pp = pprint.PrettyPrinter(indent=4)


def main(args_eval, resume_preempt=False):
    # ------------------------------------------------------------------ config (same keys / defaults)
    args_pretrain = args_eval.get('pretrain')
    checkpoint_key = args_pretrain.get('checkpoint_key', 'target_encoder')
    model_name = args_pretrain.get('model_name', None)
    patch_size = args_pretrain.get('patch_size', None)
    pretrain_folder = args_pretrain.get('folder', None)
    ckp_fname = args_pretrain.get('checkpoint', None)
    tag = args_pretrain.get('write_tag', None)
    use_sdpa = args_pretrain.get('use_sdpa', True)
    use_SiLU = args_pretrain.get('use_silu', False)
    tight_SiLU = args_pretrain.get('tight_silu', True)
    uniform_power = args_pretrain.get('uniform_power', False)
    pretrained_path = os.path.join(pretrain_folder, ckp_fname)
    tubelet_size = args_pretrain.get('tubelet_size', 2)
    frames_per_clip = args_pretrain.get('frames_per_clip', 1)

    args_data = args_eval.get('data')
    dataset_name = args_data.get('dataset_name')
    num_classes = args_data.get('num_classes')
    root_path = args_data.get('root_path', None)
    image_folder = args_data.get('image_folder', None)
    resolution = args_data.get('resolution', 224)
    synthetic_length = args_data.get('synthetic_length', None)     # synthetic dataset only: items per split

    args_opt = args_eval.get('optimization')
    batch_size = args_opt.get('batch_size')
    num_epochs = args_opt.get('num_epochs')
    wd = args_opt.get('weight_decay')
    start_lr = args_opt.get('start_lr')
    lr = args_opt.get('lr')
    final_lr = args_opt.get('final_lr')
    warmup = args_opt.get('warmup')
    use_bfloat16 = args_opt.get('use_bfloat16')
    fp16_autocast = read_fp16_autocast(args_opt)
    multihead_kwargs = read_multihead_kwargs(args_opt)
    probe_depth = read_probe_depth(args_opt)

    resume_checkpoint = args_eval.get('resume_checkpoint', False) or resume_preempt
    eval_tag = args_eval.get('tag', None)

    # ------------------------------------------------------------------ setup
    try:
        mp.set_start_method('spawn')
    except Exception:
        pass

    device = require_cuda('evals.image_classification_frozen')
    world_size, rank = init_distributed()
    logger.info(f'Initialized (rank/world-size) {rank}/{world_size}')

    folder = os.path.join(pretrain_folder, 'image_classification_frozen/')
    if eval_tag is not None:
        folder = os.path.join(folder, eval_tag)
    if not os.path.exists(folder):
        os.makedirs(folder, exist_ok=True)
    log_file = os.path.join(folder, f'{tag}_r{rank}.csv')
    latest_path = os.path.join(folder, f'{tag}-latest.pth.tar')

    encoder = init_model(crop_size=resolution, device=device, pretrained=pretrained_path, model_name=model_name,
                         patch_size=patch_size, frames_per_clip=frames_per_clip, tubelet_size=tubelet_size,
                         uniform_power=uniform_power, checkpoint_key=checkpoint_key, use_SiLU=use_SiLU,
                         tight_SiLU=tight_SiLU, use_sdpa=use_sdpa)
    encoder.eval()
    for p in encoder.parameters():
        p.requires_grad = False

    settings = multihead_kwargs or [one_head(wd, start_lr, lr, final_lr, warmup)]
    classifiers = build_heads(lambda: AttentiveClassifier(embed_dim=encoder.embed_dim, num_heads=encoder.num_heads,
                                                          depth=probe_depth, num_classes=num_classes,
                                                          follow_autocast=fp16_autocast).to(device), len(settings))

    train_loader = make_dataloader(dataset_name=dataset_name, root_path=root_path, resolution=resolution,
                                   image_folder=image_folder, batch_size=batch_size, world_size=world_size, rank=rank,
                                   training=True, num_classes=num_classes, synthetic_length=synthetic_length)
    val_loader = make_dataloader(dataset_name=dataset_name, root_path=root_path, resolution=resolution,
                                 image_folder=image_folder, batch_size=batch_size, world_size=world_size, rank=rank,
                                 training=False, num_classes=num_classes, synthetic_length=synthetic_length)
    ipe = len(train_loader)
    logger.info(f'Dataloader created... iterations per epoch: {ipe}')

    def run_epoch(training, heads):
        return run_one_epoch(device=device, training=training, encoder=encoder,
                             data_loader=train_loader if training else val_loader, use_bfloat16=use_bfloat16,
                             fp16_autocast=fp16_autocast, **heads)
    train_heads(classifiers, settings, run_epoch, multihead=multihead_kwargs is not None, iterations_per_epoch=ipe,
                num_epochs=num_epochs, use_bfloat16=use_bfloat16, resume_checkpoint=resume_checkpoint,
                latest_path=latest_path, log_file=log_file, device=device, rank=rank, world_size=world_size,
                batch_size=batch_size)


def run_one_epoch(device, training, encoder, classifier, scaler, optimizer, scheduler, wd_scheduler, data_loader,
                  use_bfloat16, fp16_autocast=False):
    """eval.py:262-317: one classifier call per step, the cross-entropy of its logits as the loss and their argmax
    (not that of their softmax, whose rounding can tie) as the top-1.  The loop itself, also for per-head lists, is the
    video evaluation's run_head_loop."""
    def encode(data):
        if isinstance(data[0], list):       # uint8 image tickets: the transform's pixel work runs on the GPU
            imgs = data_loader.dataset.transform.batch(data[0], device)
        else:
            imgs = data[0].to(device)
        labels = data[1].to(device)
        return encoder(imgs), labels, len(imgs)

    def loss_and_scores(outputs, labels):
        return F.cross_entropy(outputs, labels), outputs

    return run_head_loop(training, classifier, scaler, optimizer, scheduler, wd_scheduler, data_loader, use_bfloat16,
                         fp16_autocast, encode, loss_and_scores)


def make_dataloader(dataset_name, root_path, image_folder, batch_size, world_size, rank, resolution=224, training=False,
                    subset_file=None, num_classes=None, synthetic_length=None):
    """eval.py:379-423.  ImageNet / iNat21 / Places205 (ImageFolder trees) and synthetic_uint8 images get the reference's
    transforms with the pixel work on the GPU (jepa_b200/image_transforms.py): timm's AutoAugment 'original' + random
    erasing for training, Resize + CenterCrop for validation, both bit-exact; the loader yields uint8 image tickets and
    run_one_epoch makes [B, 3, S, S] on the device.  The synthetic dataset yields pre-normalised images and needs none."""
    from jepa_b200.image_transforms import GpuImageEvalTransform, GpuImageTransform
    normalization = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
    kind = str(dataset_name).lower()
    transform, num_workers = None, 0
    if kind != 'synthetic':
        if training:
            logger.info('implementing auto-agument strategy')
            transform = GpuImageTransform(crop_size=resolution, normalize=normalization, re_prob=0.25)
        else:
            transform = GpuImageEvalTransform(crop_size=resolution, normalize=normalization)
        if kind != 'synthetic_uint8':
            num_workers = 8                 # PIL decoding in loader workers, as the reference's init_data default
    data_loader, _ = init_data(data=dataset_name, transform=transform, batch_size=batch_size, world_size=world_size,
                               rank=rank, root_path=root_path, image_folder=image_folder, training=training,
                               copy_data=False, drop_last=False, subset_file=subset_file, crop_size=resolution,
                               num_workers=num_workers, num_classes=num_classes, images=True,
                               synthetic_length=synthetic_length)
    return data_loader


def init_model(device, pretrained, model_name, patch_size=16, crop_size=224, frames_per_clip=16, tubelet_size=2,
               use_sdpa=False, use_SiLU=False, tight_SiLU=True, uniform_power=False, checkpoint_key='target_encoder'):
    """eval.py:426-461: a video encoder sees each image [B, C, H, W] as a clip of `frames_per_clip` equal frames."""
    if use_SiLU:
        raise NotImplementedError("use_silu: the encoder's MLP runs GELU in the GEMM epilogue; no V-JEPA config uses SiLU")
    encoder = vit.__dict__[model_name](img_size=crop_size, patch_size=patch_size, num_frames=frames_per_clip,
                                       tubelet_size=tubelet_size, uniform_power=uniform_power, use_sdpa=use_sdpa)
    if frames_per_clip > 1:
        def forward_prehook(module, input):
            input = input[0]  # [B, C, H, W]
            input = input.unsqueeze(2).repeat(1, 1, frames_per_clip, 1, 1)
            return (input)

        encoder.register_forward_pre_hook(forward_prehook)

    encoder.to(device)
    encoder = load_pretrained(encoder=encoder, pretrained=pretrained, checkpoint_key=checkpoint_key)
    return encoder
