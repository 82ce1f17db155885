"""V-JEPA pre-training loop: `app.vjepa.train.main(args, resume_preempt=False)`.

Same config schema, schedules, CSV columns, log lines and checkpoint format as the reference
(app/vjepa/train.py), with the math of every step running on the sm_90a kernels of jepa_b200:
  target forward + LN + gather  -> jepa_b200.step.forward_target      (train.py:419-429)
  context encoder + predictor   -> fused multi-mask passes            (train.py:431-438)
  L1 latent loss / variance reg -> jepa_b200.step.jepa_loss/reg_loss  (train.py:440-459)
  AdamW                         -> jepa_b200.optim.FlatAdamW          (train.py:462-475)
  EMA                           -> jepa_b200.step.ema_update          (train.py:484-487)

`optimization.accum_iter: k` (default 1; the reference has no such key) accumulates k loader batches of
`data.batch_size` clips into each optimizer step, so a recipe's global batch is reachable on fewer GPUs: the first
k - 1 backwards run under DistributedDataParallel.no_sync() and add into the flat gradient buffers, the last one adds
and all-reduces.  `ipe` counts optimizer steps (an epoch reads ipe * k loader batches), so the LR / WD / EMA schedules
mean what they mean at k = 1; one CSV row per optimizer step, its losses the mean over the k micro-batches.
"""
import os

try:
    # one visible device per process under SLURM (app/vjepa/train.py:10-18)
    os.environ['CUDA_VISIBLE_DEVICES'] = os.environ['SLURM_LOCALID']
except Exception:
    pass

import contextlib
import copy
import time

import numpy as np
import torch
import torch.multiprocessing as mp
from src.utils.distributed import DistributedDataParallel   # flat-buffer gradient exchange, torch DDP surface

from app.vjepa.transforms import make_transforms
from app.vjepa.utils import init_opt, init_video_model, load_checkpoint
from jepa_b200 import step as vj
from jepa_b200.checkpoint import AsyncCheckpointer
from jepa_b200.transforms import tickets_to_device
from src.datasets.data_manager import init_data
from src.masks.multiblock3d import MaskCollator as MB3DMaskCollator
from src.masks.random_tube import MaskCollator as TubeMaskCollator
from src.utils.distributed import AllReduce, init_distributed
from src.utils.logging import AverageMeter, CSVLogger, adamw_logger, get_logger, gpu_timer, grad_logger
from src.utils.tensors import repeat_interleave_batch

log_timings = True
log_freq = 10
checkpoint_freq = 1

_GLOBAL_SEED = 0
np.random.seed(_GLOBAL_SEED)
torch.manual_seed(_GLOBAL_SEED)

logger = get_logger(__name__)


def main(args, resume_preempt=False):
    # ------------------------------------------------------------------ config (same keys/defaults)
    meta = args.get('meta')
    load_model = meta.get('load_checkpoint') or resume_preempt
    r_file = meta.get('read_checkpoint', None)
    seed = meta.get('seed', _GLOBAL_SEED)
    save_every_freq = meta.get('save_every_freq', -1)
    skip_batches = meta.get('skip_batches', -1)
    use_sdpa = meta.get('use_sdpa', False)
    which_dtype = meta.get('dtype')
    logger.info(f'{which_dtype=}')
    if which_dtype.lower() == 'bfloat16':
        dtype, mixed_precision = torch.bfloat16, True
    elif which_dtype.lower() == 'float16':
        raise NotImplementedError("dtype float16: the wgmma kernels compute bf16 x bf16 -> fp32 only")
    else:
        raise NotImplementedError("dtype float32: there is no fp32 tensor-core path; use dtype: bfloat16 "
                                  "(the configuration of every shipped pre-training config)")

    cfgs_mask = args.get('mask')

    model = args.get('model')
    model_name = model.get('model_name')
    pred_depth = model.get('pred_depth')
    pred_embed_dim = model.get('pred_embed_dim')
    uniform_power = model.get('uniform_power', True)
    use_mask_tokens = model.get('use_mask_tokens', True)
    zero_init_mask_tokens = model.get('zero_init_mask_tokens', True)

    data = args.get('data')
    dataset_type = data.get('dataset_type', 'videodataset')
    mask_type = data.get('mask_type', 'multiblock3d')
    dataset_paths = data.get('datasets', [])
    datasets_weights = data.get('datasets_weights', None)
    if datasets_weights is not None:
        assert len(datasets_weights) == len(dataset_paths), 'Must have one sampling weight specified for each dataset'
    batch_size = data.get('batch_size')
    num_clips = data.get('num_clips')
    num_frames = data.get('num_frames')
    tubelet_size = data.get('tubelet_size')
    sampling_rate = data.get('sampling_rate')
    duration = data.get('clip_duration', None)
    crop_size = data.get('crop_size', 224)
    patch_size = data.get('patch_size')
    pin_mem = data.get('pin_mem', False)
    num_workers = data.get('num_workers', 1)
    filter_short_videos = data.get('filter_short_videos', False)
    decode_one_clip = data.get('decode_one_clip', True)
    log_resource_util_data = data.get('log_resource_utilization', False)

    aug = args.get('data_aug')
    ar_range = aug.get('random_resize_aspect_ratio', [3 / 4, 4 / 3])
    rr_scale = aug.get('random_resize_scale', [0.3, 1.0])
    motion_shift = aug.get('motion_shift', False)
    reprob = aug.get('reprob', 0.)
    use_aa = aug.get('auto_augment', False)
    gpu_augment = aug.get('gpu_augment', False)     # RandAugment / random erasing on the GPU

    loss_cfg = args.get('loss')
    loss_exp = loss_cfg.get('loss_exp')
    reg_coeff = loss_cfg.get('reg_coeff')

    opt_cfg = args.get('optimization')
    ipe = opt_cfg.get('ipe', None)
    ipe_scale = opt_cfg.get('ipe_scale', 1.0)
    clip_grad = opt_cfg.get('clip_grad', None)
    wd = float(opt_cfg.get('weight_decay'))
    final_wd = float(opt_cfg.get('final_weight_decay'))
    num_epochs = opt_cfg.get('epochs')
    warmup = opt_cfg.get('warmup')
    start_lr = opt_cfg.get('start_lr')
    lr = opt_cfg.get('lr')
    final_lr = opt_cfg.get('final_lr')
    ema = opt_cfg.get('ema')
    betas = opt_cfg.get('betas', (0.9, 0.999))
    eps = opt_cfg.get('eps', 1.e-8)
    accum_iter = opt_cfg.get('accum_iter', 1)      # loader batches (micro-batches) per optimizer step
    if isinstance(accum_iter, bool) or not isinstance(accum_iter, int) or accum_iter < 1:
        raise ValueError(f"optimization.accum_iter must be an integer >= 1, got {accum_iter!r}")

    log_cfg = args.get('logging')
    folder = log_cfg.get('folder')
    tag = log_cfg.get('write_tag')

    # ------------------------------------------------------------------ setup
    np.random.seed(seed)
    torch.manual_seed(seed)
    try:
        mp.set_start_method('spawn')
    except Exception:
        pass

    world_size, rank = init_distributed()
    logger.info(f'Initialized (rank/world-size) {rank}/{world_size}')

    if not torch.cuda.is_available():
        raise RuntimeError("app.vjepa.train: a CUDA (sm_90a) device is required - the training step has no CPU path")
    device = torch.device('cuda:0')
    torch.cuda.set_device(device)

    log_file = os.path.join(folder, f'{tag}_r{rank}.csv')
    latest_path = os.path.join(folder, f'{tag}-latest.pth.tar')
    load_path = None
    if load_model:
        load_path = os.path.join(folder, r_file) if r_file is not None else latest_path
        if not os.path.exists(load_path):
            load_path = None
            load_model = False

    csv_logger = CSVLogger(log_file, ('%d', 'epoch'), ('%d', 'itr'), ('%.5f', 'loss'), ('%.5f', 'loss-jepa'),
                           ('%.5f', 'reg-loss'), ('%.5f', 'enc-grad-norm'), ('%.5f', 'pred-grad-norm'),
                           ('%d', 'gpu-time(ms)'), ('%d', 'wall-time(ms)'))

    encoder, predictor = init_video_model(
        uniform_power=uniform_power, use_mask_tokens=use_mask_tokens, num_mask_tokens=len(cfgs_mask),
        zero_init_mask_tokens=zero_init_mask_tokens, device=device, patch_size=patch_size, num_frames=num_frames,
        tubelet_size=tubelet_size, model_name=model_name, crop_size=crop_size, pred_depth=pred_depth,
        pred_embed_dim=pred_embed_dim, use_sdpa=use_sdpa)
    target_encoder = copy.deepcopy(encoder)

    collator_cls = MB3DMaskCollator if mask_type == 'multiblock3d' else TubeMaskCollator
    logger.info('Initializing basic multi-block mask' if mask_type == 'multiblock3d' else 'Initializing random tube mask')
    mask_collator = collator_cls(crop_size=crop_size, num_frames=num_frames, patch_size=patch_size,
                                 tubelet_size=tubelet_size, cfgs_mask=cfgs_mask)
    transform = make_transforms(random_horizontal_flip=True, random_resize_aspect_ratio=ar_range,
                                random_resize_scale=rr_scale, reprob=reprob, auto_augment=use_aa,
                                motion_shift=motion_shift, crop_size=crop_size, gpu_augment=gpu_augment)

    (unsupervised_loader, unsupervised_sampler) = init_data(
        data=dataset_type, root_path=dataset_paths, batch_size=batch_size, training=True, clip_len=num_frames,
        frame_sample_rate=sampling_rate, filter_short_videos=filter_short_videos, decode_one_clip=decode_one_clip,
        duration=duration, num_clips=num_clips, transform=transform, datasets_weights=datasets_weights,
        collator=mask_collator, num_workers=num_workers, world_size=world_size, pin_mem=pin_mem, rank=rank,
        log_dir=folder if log_resource_util_data else None, crop_size=crop_size, ipe=(ipe or 300) * accum_iter)
    try:
        _dlen = len(unsupervised_loader)
    except Exception:
        _dlen = unsupervised_loader.num_batches
    if ipe is None:
        ipe = _dlen // accum_iter
        if ipe < 1:
            raise ValueError(f"optimization.accum_iter={accum_iter} exceeds the {_dlen} batches of the loader")
    logger.info(f'iterations per epoch/dataest length: {ipe}/{_dlen}')

    optimizer, scaler, scheduler, wd_scheduler = init_opt(
        encoder=encoder, predictor=predictor, wd=wd, final_wd=final_wd, start_lr=start_lr, ref_lr=lr,
        final_lr=final_lr, iterations_per_epoch=ipe, warmup=warmup, num_epochs=num_epochs, ipe_scale=ipe_scale,
        mixed_precision=mixed_precision, betas=betas, eps=eps)
    encoder = DistributedDataParallel(encoder, static_graph=True)
    predictor = DistributedDataParallel(predictor, static_graph=True)
    target_encoder = DistributedDataParallel(target_encoder)
    for p in target_encoder.parameters():
        p.requires_grad = False

    total_steps = int(ipe * num_epochs * ipe_scale)
    momentum_scheduler = (ema[0] + i * (ema[1] - ema[0]) / (ipe * num_epochs * ipe_scale) for i in range(total_steps + 1))

    start_epoch = 0
    if load_model or os.path.exists(latest_path):
        (encoder, predictor, target_encoder, optimizer, scaler, start_epoch) = load_checkpoint(
            r_path=load_path, encoder=encoder, predictor=predictor, target_encoder=target_encoder, opt=optimizer,
            scaler=scaler)
        for _ in range(start_epoch * ipe):
            scheduler.step()
            wd_scheduler.step()
            next(momentum_scheduler)
            for _ in range(accum_iter):     # the collator drew masks for every loader batch of those steps
                mask_collator.step()

    checkpointer = AsyncCheckpointer()

    def save_checkpoint(epoch, path):
        if rank != 0:
            return
        save_dict = {
            'encoder': encoder.state_dict(), 'predictor': predictor.state_dict(), 'opt': optimizer.state_dict(),
            'scaler': None if scaler is None else scaler.state_dict(), 'target_encoder': target_encoder.state_dict(),
            'epoch': epoch, 'loss': loss_meter.avg, 'batch_size': batch_size, 'world_size': world_size, 'lr': lr,
        }
        if accum_iter > 1:      # batch_size stays the per-GPU micro-batch; the global batch is their product
            save_dict['accum_iter'] = accum_iter
        # asynchronous: device->host snapshot enqueued now, serialisation + disk write in a background thread
        checkpointer.save(save_dict, path)
        if checkpointer.error is not None:
            logger.info(f'Encountered exception when saving checkpoint: {checkpointer.error}')
            checkpointer.error = None

    logger.info('Initializing loader...')
    loader = iter(unsupervised_loader)

    if skip_batches > 0:
        logger.info(f'Skip {skip_batches} batches')
        unsupervised_sampler.set_epoch(start_epoch)
        for itr in range(skip_batches):
            if itr % 10 == 0:
                logger.info(f'Skip {itr}/{skip_batches} batches')
            try:
                next(loader)
            except Exception:
                loader = iter(unsupervised_loader)
                next(loader)

    # ------------------------------------------------------------------ training loop
    for epoch in range(start_epoch, num_epochs):
        logger.info('Epoch %d' % (epoch + 1))
        unsupervised_sampler.set_epoch(epoch)

        loss_meter = AverageMeter()
        input_var_meter = AverageMeter()
        input_var_min_meter = AverageMeter()
        jepa_loss_meter = AverageMeter()
        reg_loss_meter = AverageMeter()
        mask_meters = [AverageMeter() for _ in range(len(cfgs_mask))]
        gpu_time_meter = AverageMeter()
        wall_time_meter = AverageMeter()

        for itr in range(ipe):
            itr_start_time = time.time()
            micro = []      # (clips, masks_enc, masks_pred) of each of the accum_iter loader batches of this step
            for _ in range(accum_iter):
                try:
                    udata, masks_enc, masks_pred = next(loader)
                except Exception:
                    logger.info('Exhausted data loaders. Refreshing...')
                    loader = iter(unsupervised_loader)
                    udata, masks_enc, masks_pred = next(loader)
                assert len(masks_enc) == len(masks_pred), 'Currently require num encoder masks = num predictor masks'

                # host -> device; every clip of a sample reuses that sample's mask pair (train.py:391-409)
                def to_device(u):
                    if isinstance(u, (list, tuple)):   # tickets: uint8 frames cross PCIe, the kernels augment / crop / normalise
                        return tickets_to_device(list(u), device, crop_size)
                    return u.to(device, non_blocking=True)
                clips = torch.cat([to_device(u) for u in udata[0]], dim=0)
                masks_enc = [repeat_interleave_batch(m.to(device, non_blocking=True), batch_size, repeat=num_clips)
                             for m in masks_enc]
                masks_pred = [repeat_interleave_batch(m.to(device, non_blocking=True), batch_size, repeat=num_clips)
                              for m in masks_pred]
                for _i, m in enumerate(mask_meters):
                    m.update(masks_enc[_i][0].size(-1))
                micro.append((clips, masks_enc, masks_pred))

            def train_step():
                _new_lr = scheduler.step()
                _new_wd = wd_scheduler.step()

                losses = []
                for i, (clips, masks_enc, masks_pred) in enumerate(micro):
                    with contextlib.ExitStack() as no_sync:
                        if i < accum_iter - 1:      # add into the gradient buffers; the last backward exchanges the sum
                            no_sync.enter_context(encoder.no_sync())
                            no_sync.enter_context(predictor.no_sync())
                        # Step 1. forward (bf16 tensor-core math, fp32 accumulation - the reference's autocast region);
                        # every micro-batch of the step sees the same target weights
                        h = vj.forward_target(target_encoder, clips, masks_pred)
                        z = encoder(clips, masks_enc)
                        z = predictor(z, h, masks_enc, masks_pred)
                        loss_jepa = vj.jepa_loss(z, h, loss_exp)
                        loss_reg = vj.reg_loss(z, with_grad=(reg_coeff != 0.0))   # differentiable only when it is used
                        loss = loss_jepa + reg_coeff * loss_reg

                        # Step 2. backward (GradScaler kept: it is active for bf16 in the reference too); the
                        # accumulated gradient is the mean over the micro-batches, as over one batch of k times the size
                        scaler.scale(loss if accum_iter == 1 else loss / accum_iter).backward()
                    losses.append((loss, loss_jepa, loss_reg))

                # optimizer step, once per accum_iter micro-batches: an inf / NaN in any of them skips the whole step
                _enc_norm, _pred_norm = 0., 0.
                scaler.unscale_(optimizer)
                if (epoch > warmup) and (clip_grad is not None):
                    _enc_norm = vj.clip_grad_norm_(encoder, clip_grad)
                    _pred_norm = vj.clip_grad_norm_(predictor, clip_grad)
                scaler.step(optimizer)
                scaler.update()
                grad_stats = grad_logger(encoder.named_parameters())
                grad_stats.global_norm = float(_enc_norm)
                grad_stats_pred = grad_logger(predictor.named_parameters())
                grad_stats_pred.global_norm = float(_pred_norm)
                optimizer.zero_grad()
                optim_stats = adamw_logger(optimizer)

                # Step 3. momentum update of the target encoder
                vj.ema_update(encoder, target_encoder, next(momentum_scheduler))

                loss, loss_jepa, loss_reg = (sum(float(l[j]) for l in losses) / accum_iter for j in range(3))
                return loss, loss_jepa, loss_reg, _new_lr, _new_wd, grad_stats, grad_stats_pred, optim_stats

            (loss, loss_jepa, loss_reg, _new_lr, _new_wd, grad_stats, grad_stats_pred, optim_stats), gpu_etime_ms = \
                gpu_timer(train_step)
            iter_elapsed_time_ms = (time.time() - itr_start_time) * 1000.
            loss_meter.update(loss)
            for clips, _, _ in micro:
                flat_clips = clips.view(clips.shape[0], -1)
                input_var = float(AllReduce.apply(flat_clips.var(dim=1).mean(dim=0)))
                input_var_min = float(AllReduce.apply(torch.min(flat_clips.var(dim=1))))
                input_var_meter.update(input_var)
                input_var_min_meter.update(input_var_min)
            jepa_loss_meter.update(loss_jepa)
            reg_loss_meter.update(loss_reg)
            gpu_time_meter.update(gpu_etime_ms)
            wall_time_meter.update(iter_elapsed_time_ms)

            csv_logger.log(epoch + 1, itr, loss, loss_jepa, loss_reg, grad_stats.global_norm,
                           grad_stats_pred.global_norm, gpu_etime_ms, iter_elapsed_time_ms)
            if (itr % log_freq == 0) or np.isnan(loss) or np.isinf(loss):
                logger.info(
                    '[%d, %5d] loss: %.3f | p%.3f r%.3f | input_var: %.3f %.3f | masks: %s [wd: %.2e] [lr: %.2e] '
                    '[mem: %.2e] [gpu: %.1f ms][wall: %.1f ms]'
                    % (epoch + 1, itr, loss_meter.avg, jepa_loss_meter.avg, reg_loss_meter.avg, input_var_meter.avg,
                       input_var_min_meter.avg, '[' + ', '.join(['%.1f' % m.avg for m in mask_meters]) + ']', _new_wd,
                       _new_lr, torch.cuda.max_memory_allocated() / 1024.0 ** 2, gpu_time_meter.avg,
                       wall_time_meter.avg))
                if optim_stats is not None:
                    logger.info('[%d, %5d] first moment: %.2e [%.2e %.2e] second moment: %.2e [%.2e %.2e]'
                                % (epoch + 1, itr, optim_stats.get('exp_avg').avg, optim_stats.get('exp_avg').min,
                                   optim_stats.get('exp_avg').max, optim_stats.get('exp_avg_sq').avg,
                                   optim_stats.get('exp_avg_sq').min, optim_stats.get('exp_avg_sq').max))
                for name, gs in (('enc', grad_stats), ('pred', grad_stats_pred)):
                    if gs is not None:
                        logger.info('[%d, %5d] %s_grad_stats: f/l[%.2e %.2e] mn/mx(%.2e, %.2e) %.2e'
                                    % (epoch + 1, itr, name, gs.first_layer, gs.last_layer, gs.min, gs.max,
                                       gs.global_norm))
            assert not np.isnan(loss), 'loss is nan'

        logger.info('avg. loss %.3f' % loss_meter.avg)
        if epoch % checkpoint_freq == 0 or epoch == (num_epochs - 1):
            save_checkpoint(epoch + 1, latest_path)
            if save_every_freq > 0 and epoch % save_every_freq == 0:
                save_checkpoint(epoch + 1, os.path.join(folder, f'{tag}-e{epoch}.pth.tar'))
    checkpointer.wait()
    if checkpointer.error is not None:
        logger.info(f'Encountered exception when saving checkpoint: {checkpointer.error}')
