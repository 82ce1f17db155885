"""Encoder inputs at a size other than the configured one, on one GPU.

  1. vj_pos_interp alone, GB/s (bytes written + table bytes read, over CUDA-event kernel time):
     ViT-L 8x14x14 -> 16x20x20 (trilinear, D 1024) and ViT-H 8x24x24 -> 16x24x24 (trilinear, D 1280)
  2. the frozen ViT-L/16 encoder forward (built for 16x224^2) at batch 4, clips/s: 16x224^2 (configured: no
     interpolation), 16x320^2 and 32x224^2
  3. an image ViT-L/16 (224^2) under FrameAggregation, one 16-frame clip per item at batch 4, clips/s

Random weights, synthetic inputs resident on the device, no_grad.  Prints ONE JSON line with every number, the card's
name and power limit and the SM clock nvidia-smi sampled during the timed region.  Writes nothing into the repository.
    python tools/bench_offsize.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402


def _events(fn, steps, warmup):
    """Median ms of fn() over `steps` calls (CUDA events around each), after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return sorted(ms)[len(ms) // 2]


def _card():
    try:
        c = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return c[0], float(c[1])
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_offsize measures on a CUDA device"
    dev = torch.device("cuda:0")
    from jepa_b200 import kernels as K
    from jepa_b200.engine import pos_interp_scales
    from jepa_b200.models import vit_large
    from jepa_b200.pooler import FrameAggregation
    torch.manual_seed(0)
    out = {"metric": "off-size encoder inputs: vj_pos_interp GB/s, ViT-L/16 frozen forward clips/s", "n_gpus": 1,
           "steps": args.steps, "warmup": args.warmup, "dtype": "bf16 GEMM operands, fp32 tables"}
    sampler = ClockSampler(0)

    interp = {}
    for name, D, src, dst in (("vitl_8x14x14_to_16x20x20", 1024, (8, 14, 14), (16, 20, 20)),
                              ("vith_8x24x24_to_16x24x24", 1280, (8, 24, 24), (16, 24, 24))):
        table = torch.randn(*src, D, device=dev)
        res = torch.empty(*dst, D, device=dev)
        scales = pos_interp_scales(src, dst, True)
        reps = 50
        ms = _events(lambda: [K.pos_interp(table, res, scales, 3) for _ in range(reps)], args.steps, args.warmup) / reps
        nbytes = res.numel() * 4 + table.numel() * 4
        interp[name] = {"us": round(ms * 1e3, 2), "bytes": nbytes, "gbps": round(nbytes / (ms * 1e-3) / 1e9, 1)}
    out["pos_interp"] = interp

    B = 4
    enc = vit_large(img_size=224, num_frames=16, tubelet_size=2, uniform_power=True).to(dev).eval()
    fwd = {}
    for T, S in ((16, 224), (16, 320), (32, 224)):
        x = torch.randn(B, 3, T, S, S, device=dev)
        with torch.no_grad():
            ms = _events(lambda: enc(x), args.steps, args.warmup)
        fwd[f"{T}x{S}x{S}"] = {"ms": round(ms, 2), "clips_per_s": round(B / (ms * 1e-3), 2),
                               "tokens": (T // 2) * (S // 16) ** 2}
    out["vitl_encoder_fwd_b4"] = fwd
    del enc

    img = vit_large(img_size=224, num_frames=1, uniform_power=True).to(dev).eval()
    agg = FrameAggregation(img).eval()
    clips = [[torch.randn(B, 3, 16, 224, 224, device=dev)]]
    with torch.no_grad():
        ms = _events(lambda: agg(clips), args.steps, args.warmup)
    out["vitl_image_frameagg_16f_b4"] = {"ms": round(ms, 2), "clips_per_s": round(B / (ms * 1e-3), 2),
                                         "images_per_call": B * 16}
    out["clocks"] = sampler.stop()
    out["gpu"], out["power_limit_w"] = _card()
    out["timing"] = "CUDA events, median over the timed calls (pos_interp: 50 launches per timed call)"
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
