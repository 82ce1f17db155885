#!/usr/bin/env python
"""Gradient accumulation throughput: the V-JEPA pre-training step of bench.py (ViT-L/16, 16x224^2 synthetic clips,
fixed seeded masks) with k micro-batches of B clips per optimizer step, k in {1, 2, 4, 8}.

    python tools/bench_accum.py [--batch 32] [--accum 1 2 4 8] [--steps 4] [--warmup 2] [--config vitl16]
    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tools/bench_accum.py ...

One optimizer step = k x (target forward, context encoder + predictor forward, L1 loss, backward of loss / k; the
first k - 1 under DistributedDataParallel.no_sync()) + once: unscale, AdamW, GradScaler update, zero_grad, EMA, LR / WD
schedule.  Per k it prints clips/s per GPU, ms per optimizer step and library launches per optimizer step
(vj_launch_count, rank 0), then one JSON line with the table, the GPU name, its power limit and the median SM clock
sampled during the timed steps.  Writes nothing into the repository.
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import CONFIGS, ClockSampler, build_training_state, seeded_masks  # noqa: E402


def accum_step(st, clips, me, mp, k):
    from jepa_b200 import step as vj
    st["scheduler"].step()
    st["wd_scheduler"].step()
    scaler, opt = st["scaler"], st["optimizer"]
    enc, pred = st["encoder"], st["predictor"]
    for i in range(k):
        with contextlib.ExitStack() as no_sync:
            if i < k - 1 and hasattr(enc, "no_sync"):
                no_sync.enter_context(enc.no_sync())
                no_sync.enter_context(pred.no_sync())
            h = vj.forward_target(st["target"], clips, mp)
            z = pred(enc(clips, me), h, me, mp)
            loss = vj.jepa_loss(z, h)
            vj.reg_loss(z)
            scaler.scale(loss if k == 1 else loss / k).backward()
    scaler.unscale_(opt)
    scaler.step(opt)
    scaler.update()
    opt.zero_grad()
    vj.ema_update(enc, st["target"], next(st["momentum"]))


def gpu_info(index):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, power, sm_max = [c.strip() for c in out.strip().split(",")]
        return dict(gpu=name, power_limit_w=float(power), sm_max_mhz=float(sm_max))
    except Exception:
        return dict(gpu=torch.cuda.get_device_name(index), power_limit_w=None, sm_max_mhz=None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="vitl16", choices=sorted(CONFIGS))
    ap.add_argument("--batch", type=int, default=32, help="clips per micro-batch per GPU")
    ap.add_argument("--accum", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--steps", type=int, default=4, help="timed optimizer steps per k")
    ap.add_argument("--warmup", type=int, default=2, help="untimed optimizer steps per k")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_accum.py measures the GPU step: no CUDA device")

    import torch.distributed as dist
    from jepa_b200 import _lib
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
    lib = _lib.load()

    _, _, _, _, crop, frames, _ = CONFIGS[args.config]
    B = args.batch
    me, mp = seeded_masks(crop, frames, B, seed=0)
    clips = torch.randn(B, 3, frames, crop, crop, generator=torch.Generator().manual_seed(rank)).to(device)
    me, mp = [m.to(device) for m in me], [m.to(device) for m in mp]
    st = build_training_state(args.config, device, world, rank)

    def sync_all():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    rows = []
    for k in args.accum:
        for _ in range(args.warmup):
            accum_step(st, clips, me, mp, k)
        sync_all()
        sampler = ClockSampler(local_rank) if rank == 0 else None
        n0 = lib.vj_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            accum_step(st, clips, me, mp, k)
        e1.record()
        sync_all()
        ms = e0.elapsed_time(e1) / args.steps
        if world > 1:       # the slowest rank sets the step time
            t = torch.tensor([ms], device=device)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t)
        launches = (lib.vj_launch_count() - n0) / args.steps
        clk = sampler.stop() if sampler is not None else {}
        rows.append(dict(k=k, micro_batch=B, global_batch=B * k * world, ms_per_step=round(ms, 2),
                         clips_per_s_per_gpu=round(B * k / (ms / 1e3), 2), launches_per_step=launches,
                         sm_mhz_median=clk.get("sm_mhz"), throttle=clk.get("reasons")))

    if rank == 0:
        info = gpu_info(local_rank)
        print(f"{info['gpu']}, power limit {info['power_limit_w']} W, max SM clock {info['sm_max_mhz']} MHz, "
              f"{world} GPU(s), {args.config}, micro-batch {B} clips per GPU")
        print(f"{'k':>3} {'global batch':>12} {'ms/step':>9} {'clips/s/GPU':>12} {'launches/step':>14} {'SM MHz':>7}")
        for r in rows:
            print(f"{r['k']:>3} {r['global_batch']:>12} {r['ms_per_step']:>9.1f} {r['clips_per_s_per_gpu']:>12.1f} "
                  f"{r['launches_per_step']:>14.0f} {str(r['sm_mhz_median']):>7}")
        print(json.dumps(dict(config=args.config, world=world, steps=args.steps, warmup=args.warmup, rows=rows, **info)))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
