#!/usr/bin/env python
"""Frozen-evaluation probe training step, clips/sec, at the ViT-L/16 K400 shape.

    python tools/bench_probe.py [--steps K] [--warmup W] [--batch B]

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4, help="clips per step (K400 eval config: 4 per GPU)")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
