"""Frozen video evaluation: `evals.video_classification_frozen.eval.main(args_eval, resume_preempt=False)`.

Same config keys, log lines, CSV columns and checkpoint dictionary as the reference (evals/video_classification_frozen/
eval.py:67-561), with every step on the sm_90a kernels of jepa_b200:
  frozen encoder, all clips and views in one batch -> ClipAggregation (jepa_b200.pooler)
  image encoder (pretrain frames_per_clip == 1)     -> FrameAggregation: every frame of the batch in one encoder call
  attentive probe forward / backward                -> AttentiveClassifier (vj_cross_attn_*, wgmma GEMMs, LayerNorm)
  AdamW / GradScaler                                -> FlatAdamW / FlatGradScaler over the probe's flat buffers
  DistributedDataParallel                           -> one averaging all-reduce of the probe's flat gradient per backward
  validation views (uint8 frames)                   -> vj_clip_views (EvalVideoTransform / VideoTransform eval path)

The reference autocasts the loop body to fp16 (eval.py:323, `autocast(dtype=torch.float16, enabled=use_bfloat16)`).
By default this loop opens no autocast region, so encoder and probe compute bf16 x bf16 -> fp32, and `use_bfloat16`
selects the GradScaler, as it does in the reference.  With `optimization.fp16_autocast: true` the loop body runs inside
that same region, where the reference opens it, and the classifier follows it (AttentiveClassifier(follow_autocast=True)):
with `use_bfloat16: true` the encoder, the probe's forward and its backward compute in fp16 as the reference's do, with
fp16 logits and GradScaler; with `use_bfloat16: false` the region is disabled, as in the reference, and everything
computes in bf16 as by default.  There is no fp32 path.

`optimization.multihead_kwargs` (a list of per-head lr / start_lr / final_lr / weight_decay / final_weight_decay /
warmup, read by read_multihead_kwargs) trains several probes ("heads") on one encoder pass per batch: every head starts
from the same weights and has its own optimizer, schedules, GradScaler and gradient exchange (train_heads).  Without the
key the driver trains one classifier with the reference's checkpoint, CSV and log lines.
"""
import collections.abc
import contextlib
import math
import os

try:
    # one visible device per process under SLURM (eval.py:10-18)
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
from evals.video_classification_frozen.utils import ClipAggregation, FrameAggregation, make_transforms
from jepa_b200.optim import FlatAdamW, FlatGradScaler
from jepa_b200.transforms import GpuEvalVideoTransform, GpuVideoTransform
from src.datasets.data_manager import init_data
from src.models.attentive_pooler import AttentiveClassifier
from src.utils.distributed import AllReduce, DistributedDataParallel, init_distributed
from src.utils.logging import AverageMeter, CSVLogger
from src.utils.schedulers import CosineWDSchedule, WarmupCosineSchedule

logging.basicConfig()
logger = logging.getLogger()
logger.setLevel(logging.INFO)

_GLOBAL_SEED = 0
np.random.seed(_GLOBAL_SEED)
torch.manual_seed(_GLOBAL_SEED)

pp = pprint.PrettyPrinter(indent=4)


def require_cuda(name):
    if not torch.cuda.is_available():
        raise RuntimeError(f"{name}: a CUDA (sm_90a) device is required - the frozen encoder and the probe have no CPU path")
    device = torch.device('cuda:0')
    torch.cuda.set_device(device)
    return device


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
    pretrain_frames_per_clip = args_pretrain.get('frames_per_clip', 1)

    args_data = args_eval.get('data')
    train_data_path = [args_data.get('dataset_train')]
    val_data_path = [args_data.get('dataset_val')]
    dataset_type = args_data.get('dataset_type', 'VideoDataset')
    num_classes = args_data.get('num_classes')
    eval_num_segments = args_data.get('num_segments', 1)
    eval_frames_per_clip = args_data.get('frames_per_clip', 16)
    eval_frame_step = args_pretrain.get('frame_step', 4)
    eval_duration = args_pretrain.get('clip_duration', None)
    eval_num_views_per_segment = args_data.get('num_views_per_segment', 1)
    synthetic_length = args_data.get('synthetic_length', None)     # synthetic datasets only: items per split
    gpu_augment = args_data.get('gpu_augment', False)     # training transform (RandAugment, erasing) on the GPU

    args_opt = args_eval.get('optimization')
    resolution = args_opt.get('resolution', 224)
    batch_size = args_opt.get('batch_size')
    attend_across_segments = args_opt.get('attend_across_segments', False)
    num_epochs = args_opt.get('num_epochs')
    wd = args_opt.get('weight_decay')
    start_lr = args_opt.get('start_lr')
    lr = args_opt.get('lr')
    final_lr = args_opt.get('final_lr')
    warmup = args_opt.get('warmup')
    use_bfloat16 = args_opt.get('use_bfloat16')
    fp16_autocast = read_fp16_autocast(args_opt)
    multihead_kwargs = read_multihead_kwargs(args_opt)

    resume_checkpoint = args_eval.get('resume_checkpoint', False) or resume_preempt
    eval_tag = args_eval.get('tag', None)

    # ------------------------------------------------------------------ setup
    try:
        mp.set_start_method('spawn')
    except Exception:
        pass

    device = require_cuda('evals.video_classification_frozen')
    world_size, rank = init_distributed()
    logger.info(f'Initialized (rank/world-size) {rank}/{world_size}')

    folder = os.path.join(pretrain_folder, 'video_classification_frozen/')
    if eval_tag is not None:
        folder = os.path.join(folder, eval_tag)
    if not os.path.exists(folder):
        os.makedirs(folder, exist_ok=True)
    log_file = os.path.join(folder, f'{tag}_r{rank}.csv')
    latest_path = os.path.join(folder, f'{tag}-latest.pth.tar')

    if rank == 0 and multihead_kwargs is None:
        csv_logger = CSVLogger(log_file, ('%d', 'epoch'), ('%.5f', 'loss'), ('%.5f', 'acc'))

    # -- pretrained encoder (frozen)
    encoder = init_model(crop_size=resolution, device=device, pretrained=pretrained_path, model_name=model_name,
                         patch_size=patch_size, tubelet_size=tubelet_size, frames_per_clip=pretrain_frames_per_clip,
                         uniform_power=uniform_power, checkpoint_key=checkpoint_key, use_SiLU=use_SiLU,
                         tight_SiLU=tight_SiLU, use_sdpa=use_sdpa)
    if pretrain_frames_per_clip == 1:
        if not attend_across_segments:
            # FrameAggregation returns one token sequence per view, which the per-segment loop below cannot take apart
            # (the reference leaves attend_across_segments=False as a TODO in FrameAggregation.forward)
            raise ValueError("an image encoder (pretrain frames_per_clip == 1) is evaluated with FrameAggregation, "
                             "which needs optimization.attend_across_segments: true")
        encoder = FrameAggregation(encoder).to(device)
    else:
        encoder = ClipAggregation(encoder, tubelet_size=tubelet_size,
                                  attend_across_segments=attend_across_segments).to(device)
    encoder.eval()
    for p in encoder.parameters():
        p.requires_grad = False

    classifiers = build_heads(lambda: AttentiveClassifier(embed_dim=encoder.embed_dim, num_heads=encoder.num_heads,
                                                          depth=1, num_classes=num_classes,
                                                          follow_autocast=fp16_autocast).to(device),
                              1 if multihead_kwargs is None else len(multihead_kwargs))

    train_loader = make_dataloader(dataset_type=dataset_type, root_path=train_data_path, resolution=resolution,
                                   frames_per_clip=eval_frames_per_clip, frame_step=eval_frame_step,
                                   eval_duration=eval_duration,
                                   num_segments=eval_num_segments if attend_across_segments else 1,
                                   num_views_per_segment=1, allow_segment_overlap=True, batch_size=batch_size,
                                   world_size=world_size, rank=rank, training=True, num_classes=num_classes,
                                   synthetic_length=synthetic_length, gpu_augment=gpu_augment)
    val_loader = make_dataloader(dataset_type=dataset_type, root_path=val_data_path, resolution=resolution,
                                 frames_per_clip=eval_frames_per_clip, frame_step=eval_frame_step,
                                 num_segments=eval_num_segments, eval_duration=eval_duration,
                                 num_views_per_segment=eval_num_views_per_segment, allow_segment_overlap=True,
                                 batch_size=batch_size, world_size=world_size, rank=rank, training=False,
                                 num_classes=num_classes, synthetic_length=synthetic_length)
    ipe = len(train_loader)
    logger.info(f'Dataloader created... iterations per epoch: {ipe}')

    if multihead_kwargs is not None:
        def run_epoch(training, heads):
            return run_one_epoch(device=device, training=training,
                                 num_temporal_views=eval_num_segments if (attend_across_segments or not training) else 1,
                                 attend_across_segments=attend_across_segments,
                                 num_spatial_views=1 if training else eval_num_views_per_segment, encoder=encoder,
                                 data_loader=train_loader if training else val_loader, use_bfloat16=use_bfloat16,
                                 fp16_autocast=fp16_autocast, **heads)
        train_heads(classifiers, multihead_kwargs, run_epoch, iterations_per_epoch=ipe, num_epochs=num_epochs,
                    use_bfloat16=use_bfloat16, resume_checkpoint=resume_checkpoint, latest_path=latest_path,
                    log_file=log_file, device=device, rank=rank, world_size=world_size, batch_size=batch_size)
        return

    classifier = classifiers[0]
    optimizer, scaler, scheduler, wd_scheduler = init_opt(
        classifier=classifier, wd=wd, start_lr=start_lr, ref_lr=lr, final_lr=final_lr, iterations_per_epoch=ipe,
        warmup=warmup, num_epochs=num_epochs, use_bfloat16=use_bfloat16)
    classifier = DistributedDataParallel(classifier, static_graph=True)

    start_epoch = 0
    if resume_checkpoint:
        classifier, optimizer, scaler, start_epoch = load_checkpoint(device=device, r_path=latest_path,
                                                                     classifier=classifier, opt=optimizer, scaler=scaler)
        for _ in range(start_epoch * ipe):
            scheduler.step()
            wd_scheduler.step()

    def save_checkpoint(epoch):
        save_dict = {
            'classifier': classifier.state_dict(),
            'opt': optimizer.state_dict(),
            'scaler': None if scaler is None else scaler.state_dict(),
            'epoch': epoch,
            'batch_size': batch_size,
            'world_size': world_size,
            'lr': lr,
        }
        if rank == 0:
            torch.save(save_dict, latest_path)

    for epoch in range(start_epoch, num_epochs):
        logger.info('Epoch %d' % (epoch + 1))
        train_acc = run_one_epoch(device=device, training=True,
                                  num_temporal_views=eval_num_segments if attend_across_segments else 1,
                                  attend_across_segments=attend_across_segments, num_spatial_views=1, encoder=encoder,
                                  classifier=classifier, scaler=scaler, optimizer=optimizer, scheduler=scheduler,
                                  wd_scheduler=wd_scheduler, data_loader=train_loader, use_bfloat16=use_bfloat16,
                                  fp16_autocast=fp16_autocast)
        val_acc = run_one_epoch(device=device, training=False, num_temporal_views=eval_num_segments,
                                attend_across_segments=attend_across_segments,
                                num_spatial_views=eval_num_views_per_segment, encoder=encoder, classifier=classifier,
                                scaler=scaler, optimizer=optimizer, scheduler=scheduler, wd_scheduler=wd_scheduler,
                                data_loader=val_loader, use_bfloat16=use_bfloat16, fp16_autocast=fp16_autocast)
        logger.info('[%5d] train: %.3f%% test: %.3f%%' % (epoch + 1, train_acc, val_acc))
        if rank == 0:
            csv_logger.log(epoch + 1, train_acc, val_acc)
        save_checkpoint(epoch + 1)


def read_fp16_autocast(args_opt):
    """`optimization.fp16_autocast` (default false): run the loop body inside the reference's
    autocast(dtype=torch.float16, enabled=use_bfloat16) region, with a classifier that follows it."""
    value = args_opt.get('fp16_autocast', False)
    if not isinstance(value, bool):
        raise ValueError(f"optimization.fp16_autocast must be true or false, got {value!r}")
    return value


def loop_autocast(fp16_autocast, use_bfloat16):
    """The autocast region of one loop body: the reference's (eval.py:323) when fp16_autocast is set - disabled unless
    use_bfloat16, as there - and none otherwise."""
    if not fp16_autocast:
        return contextlib.nullcontext()
    return torch.autocast('cuda', dtype=torch.float16, enabled=bool(use_bfloat16))


MULTIHEAD_FIELDS = ('lr', 'start_lr', 'final_lr', 'weight_decay', 'final_weight_decay', 'warmup')


def read_multihead_kwargs(args_opt):
    """`optimization.multihead_kwargs`: None when the key is absent (one classifier), else one resolved dict of
    MULTIHEAD_FIELDS per head, as floats.  A field a head leaves out takes the top-level `optimization` value;
    final_weight_decay defaults to 1e-6, the value init_opt uses for one classifier."""
    if 'multihead_kwargs' not in args_opt:
        return None
    value = args_opt['multihead_kwargs']
    if not isinstance(value, (list, tuple)) or len(value) == 0:
        raise ValueError(f"optimization.multihead_kwargs must be a non-empty list of mappings, got {value!r}")
    defaults = {'lr': args_opt.get('lr'), 'start_lr': args_opt.get('start_lr'), 'final_lr': args_opt.get('final_lr'),
                'weight_decay': args_opt.get('weight_decay'), 'final_weight_decay': 1e-6, 'warmup': args_opt.get('warmup')}
    heads = []
    for i, entry in enumerate(value):
        if not isinstance(entry, collections.abc.Mapping):
            raise ValueError(f"optimization.multihead_kwargs[{i}] must be a mapping, got {entry!r}")
        for key in entry:
            if key not in MULTIHEAD_FIELDS:
                raise ValueError(f"optimization.multihead_kwargs[{i}]: unknown key {key!r} "
                                 f"(allowed: {', '.join(MULTIHEAD_FIELDS)})")
        head = {}
        for key in MULTIHEAD_FIELDS:
            v = entry.get(key, defaults[key])
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
                where = '' if key in entry else f' (from optimization.{key})'
                raise ValueError(f"optimization.multihead_kwargs[{i}].{key} must be a finite number, got {v!r}{where}")
            if v < 0:
                raise ValueError(f"optimization.multihead_kwargs[{i}].{key} must not be negative, got {v!r}")
            head[key] = float(v)
        heads.append(head)
    return heads


def build_heads(make_classifier, num_heads):
    """num_heads classifiers with equal initial weights.  Head 0 draws from the global torch RNG exactly as one
    classifier does; the others are built with that RNG forked (the probe initialises on the host, so only the CPU
    generator is drawn from) and then take head 0's state.  The RNG is left where one classifier leaves it, so the data
    pipeline that draws from it next (erase seeds, samplers) sees the same stream for any number of heads."""
    heads = [make_classifier()]
    for _ in range(1, num_heads):
        with torch.random.fork_rng(devices=[]):
            clf = make_classifier()
        clf.load_state_dict(heads[0].state_dict())
        heads.append(clf)
    return heads


def train_heads(classifiers, multihead_kwargs, run_epoch, iterations_per_epoch, num_epochs, use_bfloat16,
                resume_checkpoint, latest_path, log_file, device, rank, world_size, batch_size):
    """The epoch loop of a multi-head run (both evaluation drivers): per head init_opt with its settings and its own
    DistributedDataParallel wrapper; resume through load_multihead_checkpoint; one CSV row (epoch, head, loss, acc) per
    head per epoch; checkpoint lists `classifiers` / `opts` / `scalers`.  run_epoch(training, heads) runs one epoch of
    every head (heads: run_one_epoch's per-head keyword lists) and returns the per-head accuracies."""
    ipe = iterations_per_epoch
    opts, scalers, schedulers, wd_schedulers, wrapped = [], [], [], [], []
    for clf, h in zip(classifiers, multihead_kwargs):
        optimizer, scaler, scheduler, wd_scheduler = init_opt(
            classifier=clf, wd=h['weight_decay'], final_wd=h['final_weight_decay'], start_lr=h['start_lr'],
            ref_lr=h['lr'], final_lr=h['final_lr'], iterations_per_epoch=ipe, warmup=h['warmup'],
            num_epochs=num_epochs, use_bfloat16=use_bfloat16)
        opts.append(optimizer)
        scalers.append(scaler)
        schedulers.append(scheduler)
        wd_schedulers.append(wd_scheduler)
        wrapped.append(DistributedDataParallel(clf, static_graph=True))
    logger.info(f'Training {len(wrapped)} attentive probes on one encoder pass per batch')

    start_epoch = 0
    if resume_checkpoint:
        start_epoch = load_multihead_checkpoint(device=device, r_path=latest_path, classifiers=wrapped, opts=opts,
                                                scalers=scalers, multihead_kwargs=multihead_kwargs)
        for scheduler, wd_scheduler in zip(schedulers, wd_schedulers):
            for _ in range(start_epoch * ipe):
                scheduler.step()
                wd_scheduler.step()

    if rank == 0:
        csv_logger = CSVLogger(log_file, ('%d', 'epoch'), ('%d', 'head'), ('%.5f', 'loss'), ('%.5f', 'acc'))
    heads = dict(classifier=wrapped, scaler=scalers, optimizer=opts, scheduler=schedulers, wd_scheduler=wd_schedulers)
    for epoch in range(start_epoch, num_epochs):
        logger.info('Epoch %d' % (epoch + 1))
        train_acc = run_epoch(True, heads)
        val_acc = run_epoch(False, heads)
        best = max(range(len(val_acc)), key=lambda k: val_acc[k])
        logger.info('[%5d] best of %d heads: head %d train: %.3f%% test: %.3f%%'
                    % (epoch + 1, len(val_acc), best, train_acc[best], val_acc[best]))
        if rank == 0:
            for k in range(len(wrapped)):
                csv_logger.log(epoch + 1, k, train_acc[k], val_acc[k])
            torch.save({
                'classifiers': [clf.state_dict() for clf in wrapped],
                'opts': [opt.state_dict() for opt in opts],
                'scalers': [None if s is None else s.state_dict() for s in scalers],
                'multihead_kwargs': multihead_kwargs,
                'epoch': epoch + 1,
                'batch_size': batch_size,
                'world_size': world_size,
            }, latest_path)


def load_multihead_checkpoint(device, r_path, classifiers, opts, scalers, multihead_kwargs):
    """Every head's classifier (module.-prefixed), optimizer and scaler state from a multi-head checkpoint; returns its
    epoch.  A checkpoint whose resolved head settings differ from `multihead_kwargs`, or any failure, restarts at
    epoch 0, as load_checkpoint does."""
    try:
        checkpoint = torch.load(r_path, map_location=torch.device('cpu'))
        if checkpoint.get('multihead_kwargs') != multihead_kwargs:
            raise ValueError(f"its heads {checkpoint.get('multihead_kwargs')} differ from the config's {multihead_kwargs}")
        epoch = checkpoint['epoch']
        for k, (clf, opt, scaler) in enumerate(zip(classifiers, opts, scalers)):
            msg = clf.load_state_dict(checkpoint['classifiers'][k])
            logger.info(f'loaded pretrained classifier {k} from epoch {epoch} with msg: {msg}')
            opt.load_state_dict(checkpoint['opts'][k])
            if scaler is not None:
                scaler.load_state_dict(checkpoint['scalers'][k])
        logger.info(f'loaded optimizers of {len(classifiers)} heads from epoch {epoch}')
        logger.info(f'read-path: {r_path}')
        del checkpoint
    except Exception as e:
        logger.info(f'Encountered exception when loading checkpoint {e}')
        epoch = 0
    return epoch


def load_clips(data, device, data_loader):
    """data[0] (segments of views, collated) -> device.  uint8 frames from a loader whose dataset carries the GPU
    evaluation transform become the reference's views through vj_clip_views; training tickets of every segment go
    through one augment_batch (RandAugment, crop, erase); pre-normalised views are copied."""
    transform = getattr(getattr(data_loader, 'dataset', None), 'transform', None)
    if isinstance(transform, GpuEvalVideoTransform):
        return transform.views(data[0], device)
    if isinstance(transform, GpuVideoTransform):
        B = len(data[0][0])
        out = transform.batch([t for seg in data[0] for t in seg], device)
        return [[out[s * B:(s + 1) * B]] for s in range(len(data[0]))]
    return [[dij.to(device, non_blocking=True) for dij in di] for di in data[0]]


def run_one_epoch(device, training, encoder, classifier, scaler, optimizer, scheduler, wd_scheduler, data_loader,
                  use_bfloat16, num_spatial_views, num_temporal_views, attend_across_segments, fp16_autocast=False):
    """eval.py:298-380.  Without attend_across_segments every (view, segment) token set goes through the classifier on
    its own; the probe's backward adds all of them into one flat gradient buffer, exchanged once across ranks.

    classifier, scaler, optimizer, scheduler and wd_scheduler may also be lists, one entry per head
    (optimization.multihead_kwargs): the encoder then runs once per batch, each head runs the loop body on its output in
    turn (forward, loss, accuracy, backward, its own scaler and optimizer step), and the per-head accuracies are
    returned.  One head computes what one classifier does."""
    multi = isinstance(classifier, (list, tuple))
    heads = list(zip(*[x if multi else [x] for x in (classifier, scaler, optimizer, scheduler, wd_scheduler)]))
    for clf, *_ in heads:
        clf.train(mode=training)
    criterion = torch.nn.CrossEntropyLoss()
    top1_meters = [AverageMeter() for _ in heads]
    for itr, data in enumerate(data_loader):

        if training:
            for *_, sched, wd_sched in heads:
                sched.step()
                wd_sched.step()

        # (without fp16_autocast no region: encoder and probe compute bf16 x bf16 -> fp32; see the module docstring)
        with loop_autocast(fp16_autocast, use_bfloat16):
            clips = load_clips(data, device, data_loader)
            clip_indices = [d.to(device, non_blocking=True) for d in data[2]]
            labels = data[1].to(device)
            batch_size = len(labels)

            with torch.no_grad():
                tokens = encoder(clips, clip_indices)

        for k, (clf, scaler, optimizer, _, _) in enumerate(heads):
            # the classifier calls run in the same region as the encoder; validation under no_grad
            with loop_autocast(fp16_autocast, use_bfloat16), torch.set_grad_enabled(training):
                if attend_across_segments:
                    outputs = [clf(o) for o in tokens]
                else:
                    outputs = [[clf(ost) for ost in os] for os in tokens]

            if attend_across_segments:
                loss = sum([criterion(o, labels) for o in outputs]) / len(outputs)
            else:
                loss = (sum([sum([criterion(ost, labels) for ost in os]) for os in outputs])
                        / len(outputs) / len(outputs[0]))
            with torch.no_grad():
                if attend_across_segments:
                    outputs = sum([F.softmax(o, dim=1) for o in outputs]) / len(outputs)
                else:
                    outputs = (sum([sum([F.softmax(ost, dim=1) for ost in os]) for os in outputs])
                               / len(outputs) / len(outputs[0]))
                top1_acc = 100. * outputs.max(dim=1).indices.eq(labels).sum() / batch_size
                top1_acc = float(AllReduce.apply(top1_acc))
                top1_meters[k].update(top1_acc)

            if training:
                step_head(clf, scaler, optimizer, loss, use_bfloat16)

            if itr % 20 == 0:
                logger.info(('[%5d] head %d: ' % (itr, k) if multi else '[%5d] ' % itr)
                            + '%.3f%% (loss: %.3f) [mem: %.2e]'
                            % (top1_meters[k].avg, loss, torch.cuda.max_memory_allocated() / 1024.**2))

    accs = [m.avg for m in top1_meters]
    return accs if multi else accs[0]


def step_head(classifier, scaler, optimizer, loss, use_bfloat16):
    """The reference's update (eval.py:358-370): GradScaler (use_bfloat16) or plain backward, clip to 1.0, AdamW step,
    zero_grad.  With several heads each has its own scaler: an overflowing head skips its step and halves its scale."""
    if use_bfloat16:
        scaler.scale(loss).backward()
        scaler.unscale_(optimizer)
        torch.nn.utils.clip_grad_norm_(classifier.parameters(), 1.0)
        scaler.step(optimizer)
        scaler.update()
    else:
        loss.backward()
        torch.nn.utils.clip_grad_norm_(classifier.parameters(), 1.0)
        optimizer.step()
    optimizer.zero_grad()


def load_checkpoint(device, r_path, classifier, opt, scaler):
    """eval.py:383-411: classifier (module.-prefixed), optimizer and scaler state; any failure restarts at epoch 0."""
    try:
        checkpoint = torch.load(r_path, map_location=torch.device('cpu'))
        epoch = checkpoint['epoch']
        pretrained_dict = checkpoint['classifier']
        msg = classifier.load_state_dict(pretrained_dict)
        logger.info(f'loaded pretrained classifier from epoch {epoch} with msg: {msg}')
        opt.load_state_dict(checkpoint['opt'])
        if scaler is not None:
            scaler.load_state_dict(checkpoint['scaler'])
        logger.info(f'loaded optimizers from epoch {epoch}')
        logger.info(f'read-path: {r_path}')
        del checkpoint
    except Exception as e:
        logger.info(f'Encountered exception when loading checkpoint {e}')
        epoch = 0
    return classifier, opt, scaler, epoch


def load_pretrained(encoder, pretrained, checkpoint_key='target_encoder'):
    """eval.py:414-439: the encoder entry of a pre-training checkpoint (`checkpoint_key`, else 'encoder'), with the
    'module.' / 'backbone.' prefixes stripped; entries of a different shape keep the model's own values."""
    logger.info(f'Loading pretrained model from {pretrained}')
    checkpoint = torch.load(pretrained, map_location='cpu')
    try:
        pretrained_dict = checkpoint[checkpoint_key]
    except Exception:
        pretrained_dict = checkpoint['encoder']

    pretrained_dict = {k.replace('module.', ''): v for k, v in pretrained_dict.items()}
    pretrained_dict = {k.replace('backbone.', ''): v for k, v in pretrained_dict.items()}
    for k, v in encoder.state_dict().items():
        if k not in pretrained_dict:
            logger.info(f'key "{k}" could not be found in loaded state dict')
        elif pretrained_dict[k].shape != v.shape:
            logger.info(f'key "{k}" is of different shape in model and loaded state dict')
            pretrained_dict[k] = v
    msg = encoder.load_state_dict(pretrained_dict, strict=False)
    logger.info(encoder)
    logger.info(f'loaded pretrained model with msg: {msg}')
    logger.info(f'loaded pretrained encoder from epoch: {checkpoint["epoch"]}\n path: {pretrained}')
    del checkpoint
    return encoder


def make_dataloader(root_path, batch_size, world_size, rank, dataset_type='VideoDataset', resolution=224,
                    frames_per_clip=16, frame_step=4, num_segments=8, eval_duration=None, num_views_per_segment=1,
                    allow_segment_overlap=True, training=False, num_workers=12, subset_file=None, num_classes=None,
                    synthetic_length=None, gpu_augment=False):
    """eval.py:442-488.  The training transform keeps the reference's arguments (RandAugment, random erasing): with
    gpu_augment it runs on the GPU, without it it raises for uint8 inputs; the synthetic dataset is pre-normalised and
    needs no transform.  num_classes /
    synthetic_length select the labelled synthetic evaluation items of src.datasets.data_manager."""
    kind = str(dataset_type).lower()
    transform = None
    if kind != 'synthetic':
        transform = make_transforms(training=training, num_views_per_clip=num_views_per_segment,
                                    random_horizontal_flip=False, random_resize_aspect_ratio=(0.75, 4 / 3),
                                    random_resize_scale=(0.08, 1.0), reprob=0.25, auto_augment=True, motion_shift=False,
                                    crop_size=resolution, gpu_augment=gpu_augment)
    if kind.startswith('synthetic'):
        num_workers = 0          # items are generated in-process
    data_loader, _ = init_data(data=dataset_type, root_path=root_path, transform=transform, batch_size=batch_size,
                               world_size=world_size, rank=rank, clip_len=frames_per_clip, frame_sample_rate=frame_step,
                               duration=eval_duration, num_clips=num_segments, allow_clip_overlap=allow_segment_overlap,
                               num_workers=num_workers, copy_data=False, drop_last=False, subset_file=subset_file,
                               training=training, crop_size=resolution, num_classes=num_classes,
                               num_views_per_clip=num_views_per_segment, synthetic_length=synthetic_length)
    return data_loader


def init_model(device, pretrained, model_name, patch_size=16, crop_size=224, frames_per_clip=16, tubelet_size=2,
               use_sdpa=False, use_SiLU=False, tight_SiLU=True, uniform_power=False, checkpoint_key='target_encoder'):
    """eval.py:491-519."""
    if use_SiLU:
        raise NotImplementedError("use_silu: the encoder's MLP runs GELU in the GEMM epilogue; no V-JEPA config uses SiLU")
    encoder = vit.__dict__[model_name](img_size=crop_size, patch_size=patch_size, num_frames=frames_per_clip,
                                       tubelet_size=tubelet_size, uniform_power=uniform_power, use_sdpa=use_sdpa)
    encoder.to(device)
    encoder = load_pretrained(encoder=encoder, pretrained=pretrained, checkpoint_key=checkpoint_key)
    return encoder


def init_opt(classifier, iterations_per_epoch, start_lr, ref_lr, warmup, num_epochs, wd=1e-6, final_wd=1e-6,
             final_lr=0.0, use_bfloat16=False):
    """eval.py:522-561: two AdamW groups (the second, biases and 1-D parameters, with WD_exclude), warm-up-cosine LR,
    cosine WD, GradScaler when use_bfloat16 - as one flat AdamW / flat unscale over the probe's store."""
    param_groups = [
        {'params': [p for n, p in classifier.named_parameters() if ('bias' not in n) and (len(p.shape) != 1)]},
        {'params': [p for n, p in classifier.named_parameters() if ('bias' in n) or (len(p.shape) == 1)],
         'WD_exclude': True, 'weight_decay': 0},
    ]
    logger.info('Using AdamW')
    optimizer = FlatAdamW(param_groups)
    scheduler = WarmupCosineSchedule(optimizer, warmup_steps=int(warmup * iterations_per_epoch), start_lr=start_lr,
                                     ref_lr=ref_lr, final_lr=final_lr, T_max=int(num_epochs * iterations_per_epoch))
    wd_scheduler = CosineWDSchedule(optimizer, ref_wd=wd, final_wd=final_wd, T_max=int(num_epochs * iterations_per_epoch))
    scaler = FlatGradScaler() if use_bfloat16 else None
    return optimizer, scaler, scheduler, wd_scheduler
