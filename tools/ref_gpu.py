#!/usr/bin/env python
"""Run the UNMODIFIED reference (facebookresearch/jepa, copied into oracle/_ref by
oracle/make_ref.sh) on cuda:0.  Measurement / test infrastructure only - the product never imports this.

  bench : the reference's own training entry app.vjepa.train.main(args) at a BASELINE config (bf16 autocast, eager
          PyTorch: cuBLASLt GEMMs, SDPA, cuDNN Conv3d, c10d DDP over a 1-rank NCCL group), synthetic clips, its own
          MaskCollator (seed 0, first call reused like bench.py), timed by its own gpu_timer -> the CSV column
          `gpu-time(ms)` (src/utils/logging.py:14-31, app/vjepa/train.py:499).  This is the GPU bar SURVEY 8d asks
          for: "the same reference code on the same GPU".  --loggers off stubs grad_logger / adamw_logger
          (the ~1000 host syncs per step, SURVEY 8d (A)); --loggers on is the as-shipped step (B).
  step  : one forward/backward of the reference modules on seeded weights / clips / masks (tests/golden/common.py)
          at a chosen width/depth, in bf16 autocast AND in fp32, dumped to a .pt file (sampled into the golden fixture of
          tests/test_gpu_reference.py by tests/golden/make_golden_reference.py).

The repo root holds drop-in `src/` and `app/` packages with the reference's names, so this script must run in its own
process with the repo root OFF sys.path.
"""
import argparse
import copy
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")
sys.path = [p for p in sys.path if os.path.abspath(p or os.getcwd()) != ROOT]
if not os.path.isdir(os.path.join(REF, "app")):
    print(json.dumps({"impl": "reference-gpu", "unavailable": "oracle/_ref missing: run oracle/make_ref.sh"}))
    sys.exit(0)
sys.path.insert(0, REF)
sys.path.insert(1, os.path.join(ROOT, "tests", "golden"))

import torch  # noqa: E402

VITL16_MASKS = [
    dict(aspect_ratio=[0.75, 1.5], num_blocks=8, spatial_scale=[0.15, 0.15], temporal_scale=[1.0, 1.0],
         max_temporal_keep=1.0, max_keep=None),
    dict(aspect_ratio=[0.75, 1.5], num_blocks=2, spatial_scale=[0.7, 0.7], temporal_scale=[1.0, 1.0],
         max_temporal_keep=1.0, max_keep=None),
]
CONFIGS = {   # name: (model_name, crop, frames, batch/GPU)  - BASELINE.json configs[1..4]
    "vitl16": ("vit_large", 224, 16, 32),
    "vith16": ("vit_huge", 224, 16, 24),
    "vith16_384": ("vit_huge", 384, 16, 10),
    "tiny": ("vit_tiny", 224, 8, 2),
}


def run_bench(a):
    import torch.distributed as dist
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29577")
    if a.backend == "nccl":
        torch.cuda.set_device(0)
    dist.init_process_group(a.backend, rank=0, world_size=1)   # init_distributed() then early-returns (distributed.py:20-21)
    if a.threads:
        torch.set_num_threads(a.threads)
    import app.vjepa.train as T
    model_name, crop, frames, B = CONFIGS[a.config]
    if a.batch:
        B = a.batch
    iters = a.warmup + a.steps
    clips = torch.randn(B, 3, frames, crop, crop, generator=torch.Generator().manual_seed(0))

    class Sampler:
        def set_epoch(self, e):
            pass

    class Loader:
        """What the reference's DataLoader yields: collator(list of (buffer=[clip], label, clip_indices))."""

        def __init__(self, collator):
            torch.manual_seed(0)
            self.fixed = collator([([clips[i]], 0, [0]) for i in range(B)])   # first collator call, reused (bench.py does the same)
            self.collator = collator

        def __len__(self):
            return iters

        def __iter__(self):
            for _ in range(iters):
                if a.dynamic_masks:
                    yield self.collator([([clips[i]], 0, [0]) for i in range(B)])
                else:
                    yield self.fixed

    def init_data(**kw):
        return Loader(kw["collator"]), Sampler()

    T.init_data = init_data
    T.make_transforms = lambda **kw: None
    if a.loggers == "off":
        class _Stats:
            first_layer = last_layer = 0.
            min = max = avg = 0.
            global_norm = 0.

        T.grad_logger = lambda named_params: _Stats()
        T.adamw_logger = lambda optimizer: None
    folder = tempfile.mkdtemp(prefix="ref_gpu_")
    args = {
        "meta": dict(load_checkpoint=False, read_checkpoint=None, seed=234, eval_freq=100, use_sdpa=True, dtype="bfloat16"),
        "mask": VITL16_MASKS,
        "model": dict(model_name=model_name, pred_depth=12, pred_embed_dim=384, uniform_power=True, use_mask_tokens=True,
                      zero_init_mask_tokens=True),
        "data": dict(dataset_type="VideoDataset", datasets=[], batch_size=B, num_clips=1, num_frames=frames, tubelet_size=2,
                     sampling_rate=4, crop_size=crop, patch_size=16, pin_mem=True, num_workers=0),
        "data_aug": dict(auto_augment=False, motion_shift=False, random_resize_aspect_ratio=[0.75, 1.35],
                         random_resize_scale=[0.3, 1.0], reprob=0.0),
        "loss": dict(loss_exp=1.0, reg_coeff=0.0),
        "optimization": dict(ipe=iters, ipe_scale=1.25, clip_grad=10.0, weight_decay=0.04, final_weight_decay=0.4,
                             epochs=1, warmup=40, start_lr=0.0002, lr=0.000625, final_lr=1e-6, ema=[0.998, 1.0]),
        "logging": dict(folder=folder, write_tag="jepa"),
    }
    real_save = torch.save
    torch.save = lambda *x, **k: None     # the 5 GB end-of-epoch checkpoint is not part of the step
    t0 = time.time()
    try:
        T.main(args)
    finally:
        torch.save = real_save
    wall = time.time() - t0
    gpu_ms, losses = [], []
    on_gpu = a.backend == "nccl"
    with open(os.path.join(folder, "jepa_r0.csv")) as f:
        header = f.readline().strip().split(",")
        # on the CPU the reference's gpu_timer returns -1 (logging.py:16): use its wall-time column (train.py:500)
        gi, li = header.index("gpu-time(ms)" if on_gpu else "wall-time(ms)"), header.index("loss")
        for line in f:
            c = line.strip().split(",")
            gpu_ms.append(float(c[gi]))
            losses.append(float(c[li]))
    timed = sorted(gpu_ms[a.warmup:])
    med = timed[len(timed) // 2]
    mean = sum(timed) / len(timed)
    out = {
        "impl": "reference-gpu" if on_gpu else "reference-cpu",
        "what": "unmodified facebookresearch/jepa app.vjepa.train.main, " + ("cuda:0, bf16 autocast, eager PyTorch" if on_gpu else
                f"CPU fp32 (torch.cuda.amp autocast / GradScaler disable themselves), {torch.get_num_threads()} threads"),
        "threads": torch.get_num_threads(),
        "config": a.config, "model": model_name, "batch": B, "frames": frames, "crop": crop, "loggers": a.loggers,
        "dynamic_masks": bool(a.dynamic_masks), "steps": a.steps, "warmup": a.warmup,
        "gpu_ms_per_step_median": med, "gpu_ms_per_step_mean": round(mean, 2), "gpu_ms_all": gpu_ms,
        "clips_per_s": round(B / (med * 1e-3), 4),
        "timer": "reference gpu_timer (CUDA events around train_step)" if on_gpu else "reference wall-time(ms) column",
        "losses": losses, "wall_s": round(wall, 1), "torch": torch.__version__,
        "max_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2) if torch.cuda.is_available() else None,
    }
    print(json.dumps(out), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f)
    dist.destroy_process_group()


def run_step(a):
    """One reference step on seeded inputs (weights / clips exactly as tests/parity_util.py builds them)."""
    from functools import partial
    import torch.nn as nn
    import torch.nn.functional as F
    from common import VITL16_MASKS as MASKS, synth_clips, synth_state
    import src.models.vision_transformer as ref_vit
    import src.models.predictor as ref_pred
    from src.masks.multiblock3d import MaskCollator
    from src.masks.utils import apply_masks
    from src.models.utils.multimask import MultiMaskWrapper, PredictorMultiMaskWrapper
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device(a.device)
    enc = ref_vit.VisionTransformer(img_size=a.crop, patch_size=16, num_frames=a.frames, tubelet_size=2, embed_dim=a.embed_dim,
                                    depth=a.depth, num_heads=a.heads, mlp_ratio=4, qkv_bias=True,
                                    norm_layer=partial(nn.LayerNorm, eps=1e-6), uniform_power=True, use_sdpa=True)
    pred = ref_pred.vit_predictor(img_size=a.crop, use_mask_tokens=True, patch_size=16, num_frames=a.frames, tubelet_size=2,
                                  embed_dim=a.embed_dim, predictor_embed_dim=384, depth=a.pred_depth, num_heads=a.heads,
                                  uniform_power=True, num_mask_tokens=2, zero_init_mask_tokens=True, use_sdpa=True)
    enc_shapes = {k: tuple(v.shape) for k, v in enc.state_dict().items()}
    pred_shapes = {k: tuple(v.shape) for k, v in pred.state_dict().items()}
    enc.load_state_dict(synth_state(enc_shapes, seed=11, keep=("pos_embed",)), strict=False)
    pred.load_state_dict(synth_state(pred_shapes, seed=12, keep=("pos_embed",)), strict=False)
    tgt = copy.deepcopy(enc)
    tgt.load_state_dict(synth_state(enc_shapes, seed=13, keep=("pos_embed",)), strict=False)
    enc, pred, tgt = MultiMaskWrapper(enc).to(dev), PredictorMultiMaskWrapper(pred).to(dev), MultiMaskWrapper(tgt).to(dev)
    for p in tgt.parameters():
        p.requires_grad = False
    clips = synth_clips(a.batch, a.frames, a.crop, a.crop, seed=0).to(dev)
    torch.manual_seed(0)
    coll = MaskCollator(cfgs_mask=MASKS, crop_size=a.crop, num_frames=a.frames, patch_size=16, tubelet_size=2)
    _, me, mp = coll([torch.zeros(1) for _ in range(a.mask_batch)])
    me, mp = [m[:a.batch].to(dev) for m in me], [m[:a.batch].to(dev) for m in mp]
    result = {"masks_enc": [m.cpu() for m in me], "masks_pred": [m.cpu() for m in mp]}
    for tag, dtype, mixed in (("bf16", torch.bfloat16, True), ("fp32", torch.float32, False)):
        for net in (enc, pred):
            for p in net.parameters():
                p.grad = None
        with torch.autocast(dev.type, dtype=dtype, enabled=mixed):     # train.py:453
            with torch.no_grad():
                h = tgt(clips)
                h = F.layer_norm(h, (h.size(-1),))
                h = apply_masks(h, mp, concat=False)
            z_enc = enc(clips, me)
            z = pred(z_enc, h, me, mp)
            loss = sum(torch.mean(torch.abs(zi - hi)) for zi, hi in zip(z, h)) / len(mp)
            pstd = sum(torch.sqrt(zi.var(dim=1) + 0.0001) for zi in z) / len(z)
            loss_reg = torch.mean(F.relu(1. - pstd))
        (loss * (65536.0 if mixed else 1.0)).backward()              # GradScaler's initial scale, unscaled below
        inv = 1.0 / 65536.0 if mixed else 1.0
        result[tag] = dict(
            loss_jepa=float(loss), loss_reg=float(loss_reg),
            h=[t.detach().float().cpu() for t in h], z=[t.detach().float().cpu() for t in z],
            z_enc=[t.detach().float().cpu() for t in z_enc],
            z_dtype=str(z[0].dtype), z_enc_dtype=str(z_enc[0].dtype), h_dtype=str(h[0].dtype),
            enc_grad={n: (p.grad.detach().float() * inv).cpu() for n, p in enc.backbone.named_parameters() if p.grad is not None},
            pred_grad={n: (p.grad.detach().float() * inv).cpu() for n, p in pred.backbone.named_parameters() if p.grad is not None})
    torch.save(result, a.out)
    print(json.dumps({"impl": "reference-gpu", "mode": "step", "out": a.out,
                      "loss_bf16": result["bf16"]["loss_jepa"], "loss_fp32": result["fp32"]["loss_jepa"]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="mode", required=True)
    b = sub.add_parser("bench")
    b.add_argument("--config", default="vitl16", choices=sorted(CONFIGS))
    b.add_argument("--steps", type=int, default=10)
    b.add_argument("--warmup", type=int, default=4)
    b.add_argument("--batch", type=int, default=0)
    b.add_argument("--loggers", default="off", choices=["off", "on"])
    b.add_argument("--dynamic-masks", action="store_true")
    b.add_argument("--out", default="")
    b.add_argument("--backend", default="nccl", help="nccl: cuda:0;  gloo: the reference's CPU path (fp32) on the host cores")
    b.add_argument("--threads", type=int, default=0)
    s = sub.add_parser("step")
    s.add_argument("--embed-dim", type=int, required=True)
    s.add_argument("--heads", type=int, required=True)
    s.add_argument("--depth", type=int, required=True)
    s.add_argument("--pred-depth", type=int, required=True)
    s.add_argument("--frames", type=int, default=16)
    s.add_argument("--crop", type=int, default=224)
    s.add_argument("--batch", type=int, default=1)
    s.add_argument("--mask-batch", type=int, default=32)
    s.add_argument("--out", required=True)
    s.add_argument("--device", default="cuda:0", help="cpu only for dry runs of this script")
    a = ap.parse_args()
    if not torch.cuda.is_available() and getattr(a, "device", "cuda:0") != "cpu" and getattr(a, "backend", "nccl") != "gloo":
        print(json.dumps({"impl": "reference-gpu", "unavailable": "no CUDA device"}))
        return
    (run_bench if a.mode == "bench" else run_step)(a)


if __name__ == "__main__":
    main()
