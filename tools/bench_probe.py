#!/usr/bin/env python
"""Frozen-evaluation probe training step (or validation step), clips/sec, at the ViT-L/16 K400 shape.

    python tools/bench_probe.py [--steps K] [--warmup W] [--batch B] [--mode train|val]

--mode val times the validation branch of the same loop (configs/evals/vitl16_k400_16x8x3.yaml: 8 segments x 3 spatial
views): B clips of uint8 frames [16, 256, 340, 3] per segment on the host -> vj_clip_views (EvalVideoTransform on the GPU,
one H2D copy of uint8) -> frozen encoder over all 24 views -> 3 classifier calls (attend_across_segments) -> softmax
average.  It also times vj_clip_views alone on device-resident frames and reports GB/s (uint8 read + output written,
from the shapes).

One step is the training branch of the reference's evaluation loop (evals/video_classification_frozen/eval.py:317-373
with configs/evals/vitl16_k400_16x8x3.yaml): B clips of 8 segments x 16 frames at 224^2 through the frozen encoder under
no_grad (ClipAggregation with attend_across_segments: 8 x 1568 = 12544 tokens per clip), then the attentive probe's
forward + backward (CrossEntropyLoss, 400 classes), GradScaler unscale, clip to 1.0, FlatAdamW step, zero_grad.
Synthetic inputs resident on the device.  Prints ONE JSON line: clips/s over the timed steps (wall clock), the median
encoder-forward and probe fwd + bwd + optimiser times (CUDA events), the card's name and power limit, and the SM clock
nvidia-smi sampled during the timed steps.  Writes nothing into the repository.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402


def run(args):
    from jepa_b200.models import vit_large
    from jepa_b200.optim import FlatAdamW, FlatGradScaler
    from jepa_b200.pooler import AttentiveClassifier, ClipAggregation
    from jepa_b200.step import clip_grad_norm_
    device = torch.device("cuda:0")
    torch.manual_seed(0)
    B = args.batch
    n_seg, frames, crop, n_cls = 8, 16, 224, 400
    enc = vit_large(img_size=crop, num_frames=frames, tubelet_size=2, uniform_power=True).to(device).eval()
    encoder = ClipAggregation(enc, tubelet_size=2, attend_across_segments=True)
    clf = AttentiveClassifier(embed_dim=enc.embed_dim, num_heads=enc.num_heads, depth=1, num_classes=n_cls).to(device)
    groups = [{"params": [p for n, p in clf.named_parameters() if ("bias" not in n) and (len(p.shape) != 1)]},
              {"params": [p for n, p in clf.named_parameters() if ("bias" in n) or (len(p.shape) == 1)],
               "WD_exclude": True, "weight_decay": 0}]
    opt = FlatAdamW(groups, lr=1e-3, weight_decay=0.01)
    scaler = FlatGradScaler()
    crit = torch.nn.CrossEntropyLoss()
    g = torch.Generator(device="cpu").manual_seed(0)
    clips = [[torch.randn(B, 3, frames, crop, crop, generator=g).to(device)] for _ in range(n_seg)]
    labels = torch.randint(0, n_cls, (B,), generator=g).to(device)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    enc_ms, probe_ms = [], []

    def step(timed):
        if timed:
            ev[0].record()
        with torch.no_grad():
            outputs = encoder(clips)
        if timed:
            ev[1].record()
        loss = sum([crit(clf(o), labels) for o in outputs]) / len(outputs)
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        clip_grad_norm_(clf, 1.0)
        scaler.step(opt)
        scaler.update()
        opt.zero_grad()
        if timed:
            ev[2].record()

    for _ in range(args.warmup):
        step(False)
    torch.cuda.synchronize()
    sampler = ClockSampler(0)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step(True)
        torch.cuda.synchronize()
        enc_ms.append(ev[0].elapsed_time(ev[1]))
        probe_ms.append(ev[1].elapsed_time(ev[2]))
    wall = time.perf_counter() - t0
    clocks = sampler.stop()
    try:
        card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    except Exception:
        card = []
    med = lambda v: sorted(v)[len(v) // 2]
    print(json.dumps({
        "metric": "clips/sec ViT-L/16 K400 frozen-evaluation probe training step (8x16x224^2 per clip, 400 classes)",
        "value": round(B * args.steps / wall, 2), "unit": "clips/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "higher_is_better": True, "dtype": "bf16", "data": "synthetic",
        "config": {"workload": f"batch {B}/GPU, {n_seg} segments x {frames} frames, attend_across_segments "
                               f"({n_seg * enc.num_patches} tokens per clip), AttentiveClassifier depth 1, "
                               "CrossEntropyLoss, FlatGradScaler + clip 1.0 + FlatAdamW"},
        "encoder_fwd_ms": round(med(enc_ms), 3),
        "probe_fwd_bwd_opt_ms": round(med(probe_ms), 3),
        "timing": "CUDA events per step, median over the timed steps; value = wall clock over the timed steps",
        "gpu": card[0] if card else None,
        "power_limit_w": float(card[1]) if len(card) > 1 else None,
        "clocks": clocks,
    }), flush=True)


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    except Exception:
        return []


def run_val(args):
    import ctypes
    import torch.nn.functional as F
    from jepa_b200 import _lib
    from jepa_b200 import kernels as K
    from jepa_b200.models import vit_large
    from jepa_b200.pooler import AttentiveClassifier, ClipAggregation
    from jepa_b200.transforms import DEFAULT_NORMALIZE, pack_views, preprocess_views
    device = torch.device("cuda:0")
    torch.manual_seed(0)
    B = args.batch
    n_seg, n_views, frames, crop, n_cls, H0, W0 = 8, 3, 16, 224, 400, 256, 340
    enc = vit_large(img_size=crop, num_frames=frames, tubelet_size=2, uniform_power=True).to(device).eval()
    for p in enc.parameters():          # frozen, as in the evaluation: the forward keeps no activations
        p.requires_grad = False
    encoder = ClipAggregation(enc, tubelet_size=2, attend_across_segments=True)
    clf = AttentiveClassifier(embed_dim=enc.embed_dim, num_heads=enc.num_heads, depth=1, num_classes=n_cls).to(device).eval()
    g = torch.Generator().manual_seed(0)
    segments = [torch.randint(0, 256, (B, frames, H0, W0, 3), dtype=torch.uint8, generator=g).pin_memory()
                for _ in range(n_seg)]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    view_ms, enc_ms = [], []

    def step(timed):
        if timed:
            ev[0].record()
        with torch.no_grad():
            clips = preprocess_views(segments, device, crop, n_views)
            if timed:
                ev[1].record()
            outputs = [clf(o) for o in encoder(clips)]
            probs = sum([F.softmax(o, dim=1) for o in outputs]) / len(outputs)
        if timed:
            ev[2].record()
        return probs

    for _ in range(args.warmup):
        step(False)
    torch.cuda.synchronize()
    sampler = ClockSampler(0)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step(True)
        torch.cuda.synchronize()
        view_ms.append(ev[0].elapsed_time(ev[1]))
        enc_ms.append(ev[1].elapsed_time(ev[2]))
    wall = time.perf_counter() - t0
    clocks = sampler.stop()

    # vj_clip_views alone, frames already on the device
    clips_u8 = [c for seg in segments for c in seg.unbind(0)]
    buf, jobs, tab = pack_views(clips_u8, crop, n_views, n_seg)
    dbuf, djobs, dtab = buf.to(device), jobs.to(device), tab.to(device)
    out = torch.empty(n_seg * n_views * B * 3 * frames * crop * crop, dtype=torch.float32, device=device)
    m3 = (ctypes.c_float * 3)(*DEFAULT_NORMALIZE[0])
    s3 = (ctypes.c_float * 3)(*DEFAULT_NORMALIZE[1])
    kern_ms = []
    for i in range(args.warmup + args.steps):
        ev[0].record()
        _lib.call("vj_clip_views", dbuf.data_ptr(), djobs.data_ptr(), dtab.data_ptr(), out.data_ptr(), 1,
                  int(jobs.shape[0]), frames, crop, ctypes.cast(m3, ctypes.c_void_p), ctypes.cast(s3, ctypes.c_void_p),
                  K._s())
        ev[1].record()
        torch.cuda.synchronize()
        if i >= args.warmup:
            kern_ms.append(ev[0].elapsed_time(ev[1]))
    moved = n_seg * B * frames * H0 * W0 * 3 + out.numel() * 4
    card = _card()
    med = lambda v: sorted(v)[len(v) // 2]
    print(json.dumps({
        "metric": "clips/sec ViT-L/16 K400 frozen-evaluation validation step (8 segments x 3 views x 16x224^2 per clip, "
                  "uint8 frames in)",
        "value": round(B * args.steps / wall, 2), "unit": "clips/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "higher_is_better": True, "dtype": "bf16", "data": "synthetic uint8",
        "config": {"workload": f"batch {B}/GPU, {n_seg} segments x {n_views} views of {frames} frames from uint8 "
                               f"{H0}x{W0} frames (EvalVideoTransform via vj_clip_views), attend_across_segments, "
                               f"{n_views} classifier calls, softmax average"},
        "views_ms": round(med(view_ms), 3),
        "encoder_probe_ms": round(med(enc_ms), 3),
        "clip_views_kernel_ms": round(med(kern_ms), 3),
        "clip_views_gbps": round(moved / (med(kern_ms) * 1e-3) / 1e9, 1),
        "clip_views_bytes": moved,
        "timing": "CUDA events per step, median over the timed steps; value = wall clock over the timed steps; "
                  "views_ms includes host packing and the uint8 H2D copy",
        "gpu": card[0] if card else None,
        "power_limit_w": float(card[1]) if len(card) > 1 else None,
        "clocks": clocks,
    }), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4, help="clips per step (K400 eval config: 4 per GPU)")
    ap.add_argument("--mode", choices=("train", "val"), default="train",
                    help="train: probe training step; val: validation step from uint8 frames")
    args = ap.parse_args()
    run(args) if args.mode == "train" else run_val(args)


if __name__ == "__main__":
    main()
