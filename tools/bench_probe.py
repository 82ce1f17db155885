#!/usr/bin/env python
"""Frozen-evaluation probe training step (or validation step), clips/sec, at the ViT-L/16 K400 shape.

    python tools/bench_probe.py [--steps K] [--warmup W] [--batch B] [--mode train|val|image|xattn]
                                [--dtype bfloat16|float16] [--heads 1,4,16] [--depth 1,2,4]

--heads (train, val, image) runs the evaluation loop with several probes on one encoder pass
(optimization.multihead_kwargs): per step the encoder runs once, then every probe its forward (+ backward, GradScaler,
clip and FlatAdamW step when training) in turn.  The listed probe counts alternate step by step in one session, and the
JSON line gains one row per count: encoder ms, probe ms per probe and clips/s (images/s).  The top-level figures are
those of the first count.

--dtype float16 runs each step's encoder and classifier calls inside the reference's autocast(dtype=torch.float16)
region (evals/video_classification_frozen/eval.py:323) with AttentiveClassifier(follow_autocast=True): fp16 encoder,
fp16 probe forward and backward, fp16 logits, GradScaler.  The default bfloat16 is the evaluation loop without autocast.

--depth 1,2,4 times the probe alone (AttentiveClassifier(depth=d), ViT-L width, K400 classes) on device-resident
encoder tokens [B, 12544, 1024]: forward + backward + GradScaler unscale, clip and FlatAdamW step per training step, the
listed depths alternating step by step.  It also times vj_query_attn_fwd / _bwd alone (CUDA events around a CUDA graph of
200 back-to-back launches) at that shape's one query token per clip, and at 16 query tokens (an AttentivePooler with
num_queries=16).

--mode xattn times vj_cross_attn_fwd_lse and vj_cross_attn_bwd alone, bf16 and fp16 alternating, at the K400 probe
shapes (B 4, S 12 544, one query; ViT-L H 16 x hd 64 and ViT-H H 16 x hd 80), and reports GB/s from the bytes each must
move (the kv read, the dkv write).

--uint8 (train mode) starts each step from B x 8 uint8 clips [16, 256, 340, 3] on the host: the evaluation's training
transform draws its decisions there (RandAugment, crop, erase), then augment_batch runs them on the GPU; it reports the
augmentation's time and bytes, and, when oracle/_ref holds the reference, the reference's CPU transform per clip.

--mode val times the validation branch of the same loop (configs/evals/vitl16_k400_16x8x3.yaml: 8 segments x 3 spatial
views): B clips of uint8 frames [16, 256, 340, 3] per segment on the host -> vj_clip_views (EvalVideoTransform on the GPU,
one H2D copy of uint8) -> frozen encoder over all 24 views -> 3 classifier calls (attend_across_segments) -> softmax
average.  It also times vj_clip_views alone on device-resident frames and reports GB/s (uint8 read + output written,
from the shapes).

--mode image times the frozen IMAGE evaluation's probe training step at the ViT-L/16 in1k shape
(configs/evals/vitl16_in1k.yaml: 16 frames, each image repeated over them as the evaluation's forward pre-hook does,
batch 16, 1000 classes).  With --uint8 each step starts from B uint8 500x375 images on the host: GpuImageTransform draws
the decisions (crop, flip, AutoAugment 'original', erasing) and vj_image_augment makes [B, 3, 224, 224] on the GPU;
without it the images are pre-normalised and device-resident.  It also reports vj_image_augment and vj_image_views alone
(CUDA events, staged buffers already on the device) and, when oracle/_ref holds the reference, the reference's CPU
training transform per image (timm's composition of its pieces, one thread).

One step is the training branch of the reference's evaluation loop (evals/video_classification_frozen/eval.py:317-373
with configs/evals/vitl16_k400_16x8x3.yaml): B clips of 8 segments x 16 frames at 224^2 through the frozen encoder under
no_grad (ClipAggregation with attend_across_segments: 8 x 1568 = 12544 tokens per clip), then the attentive probe's
forward + backward (CrossEntropyLoss, 400 classes), GradScaler unscale, clip to 1.0, FlatAdamW step, zero_grad.
Synthetic inputs resident on the device.  Prints ONE JSON line: clips/s over the timed steps (wall clock), the median
encoder-forward and probe fwd + bwd + optimiser times (CUDA events), the card's name and power limit, and the SM clock
nvidia-smi sampled during the timed steps.  Writes nothing into the repository.
"""
import argparse
import contextlib
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


def _region(args):
    """The reference's loop-body autocast region with --dtype float16, none with bfloat16."""
    if args.dtype == "float16":
        return torch.autocast("cuda", dtype=torch.float16)
    return contextlib.nullcontext()


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
    heads = []
    for _ in range(max(args.heads)):
        clf = AttentiveClassifier(embed_dim=enc.embed_dim, num_heads=enc.num_heads, depth=1, num_classes=n_cls,
                                  follow_autocast=args.dtype == "float16").to(device)
        groups = [{"params": [p for n, p in clf.named_parameters() if ("bias" not in n) and (len(p.shape) != 1)]},
                  {"params": [p for n, p in clf.named_parameters() if ("bias" in n) or (len(p.shape) == 1)],
                   "WD_exclude": True, "weight_decay": 0}]
        heads.append((clf, FlatAdamW(groups, lr=1e-3, weight_decay=0.01), FlatGradScaler()))
    crit = torch.nn.CrossEntropyLoss()
    g = torch.Generator(device="cpu").manual_seed(0)
    labels = torch.randint(0, n_cls, (B,), generator=g).to(device)
    clips = None
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    aug_ms, aug_bytes = [], []
    if args.uint8:          # the evaluation's training transform (RandAugment + erasing) on the GPU, from uint8 frames
        from jepa_b200.transforms import augment_batch, make_eval_transforms, pack_augment
        H0, W0 = 256, 340
        tf = make_eval_transforms(training=True, random_horizontal_flip=False, random_resize_aspect_ratio=(0.75, 4 / 3),
                                  random_resize_scale=(0.08, 1.0), reprob=0.25, auto_augment=True, crop_size=crop,
                                  gpu_augment=True)
        host = [torch.randint(0, 256, (frames, H0, W0, 3), dtype=torch.uint8, generator=g).numpy()
                for _ in range(n_seg * B)]
    else:
        clips = [[torch.randn(B, 3, frames, crop, crop, generator=g).to(device)] for _ in range(n_seg)]

    def step(timed, n_heads):
        nonlocal clips
        if args.uint8:
            tickets = [tf(x) for x in host]              # host decisions, segment-major
            ev[3].record()
            out = augment_batch(tickets, device, crop)
            clips = [[out[s * B:(s + 1) * B]] for s in range(n_seg)]
            if timed:
                aug_bytes.append(_augment_bytes(tickets, pack_augment, out))
        if timed:
            ev[0].record()
        with _region(args):
            with torch.no_grad():
                outputs = encoder(clips)
        if timed:
            ev[1].record()
        for clf, opt, scaler in heads[:n_heads]:        # the evaluation loop's per-head body on one encoder pass
            with _region(args):
                logits = [clf(o) for o in outputs]
            loss = sum([crit(o, labels) for o in logits]) / len(logits)
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
            clip_grad_norm_(clf, 1.0)
            scaler.step(opt)
            scaler.update()
            opt.zero_grad()
        if timed:
            ev[2].record()

    def measure():
        return {"enc": ev[0].elapsed_time(ev[1]), "probe": ev[1].elapsed_time(ev[2]),
                "aug": ev[3].elapsed_time(ev[0]) if args.uint8 else None}

    sampler = ClockSampler(0)
    res = _alternate(args, step, measure)
    clocks = sampler.stop()
    times, wall = res[args.heads[0]]
    enc_ms, probe_ms, aug_ms = ([t[k] for t in times] for k in ("enc", "probe", "aug"))
    extra = {}
    if args.uint8:
        ms = sorted(aug_ms)[len(aug_ms) // 2]
        nbytes = sorted(aug_bytes)[len(aug_bytes) // 2]
        extra = {"data": "synthetic uint8 16x256x340 frames, RandAugment rand-m7-n4-mstd0.5-inc1 + erasing 0.25 on the GPU",
                 "augment_ms": round(ms, 3), "augment_bytes": nbytes,
                 "augment_gbps": round(nbytes / (ms * 1e-3) / 1e9, 1),
                 "augment_timing": "CUDA events from before augment_batch (host packing, uint8 H2D copy, kernels) to "
                                   "the encoder; bytes from the decision tables (each applied op reads and writes its "
                                   "clip, a histogram pass reads it, the last pass reads the clip and writes the output)",
                 "reference_cpu_ms_per_clip": _reference_cpu_ms(host[0], crop)}
    try:
        card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                              capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    except Exception:
        card = []
    med = lambda v: sorted(v)[len(v) // 2]
    print(json.dumps({
        "metric": "clips/sec ViT-L/16 K400 frozen-evaluation probe training step (8x16x224^2 per clip, 400 classes)",
        "value": round(B * args.steps / wall, 2), "unit": "clips/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "higher_is_better": True, "dtype": args.dtype, "data": "synthetic",
        "config": {"workload": f"batch {B}/GPU, {n_seg} segments x {frames} frames, attend_across_segments "
                               f"({n_seg * enc.num_patches} tokens per clip), AttentiveClassifier depth 1, "
                               "CrossEntropyLoss, FlatGradScaler + clip 1.0 + FlatAdamW"},
        "encoder_fwd_ms": round(med(enc_ms), 3),
        "probe_fwd_bwd_opt_ms": round(med(probe_ms), 3),
        "timing": "CUDA events per step, median over the timed steps; value = wall clock over the timed steps",
        "gpu": card[0] if card else None,
        "power_limit_w": float(card[1]) if len(card) > 1 else None,
        "clocks": clocks,
        **extra,
        **_heads_rows(args, res, B, "enc", "probe", "clips/s"),
    }), flush=True)


def _alternate(args, step, measure):
    """Warm-up at every head count, then args.steps timed rounds, each running one step at every head count of
    args.heads in turn (so that clock and thermal drift spread over all of them).  step(timed, n_heads) runs one step;
    measure() reads its CUDA events after the synchronisation.  Returns {n_heads: (per-step measures, wall seconds)}."""
    for n in args.heads:
        for _ in range(args.warmup):
            step(False, n)
    torch.cuda.synchronize()
    res = {n: ([], 0.0) for n in args.heads}
    for _ in range(args.steps):
        for n in args.heads:
            t0 = time.perf_counter()
            step(True, n)
            torch.cuda.synchronize()
            times, wall = res[n]
            times.append(measure())
            res[n] = (times, wall + time.perf_counter() - t0)
    return res


def _heads_rows(args, res, batch, enc_key, probe_key, unit):
    """With --heads: one row per head count - encoder ms, probe ms per head (all heads' time / heads) and throughput."""
    if not args.multi:
        return {}
    med = lambda v: sorted(v)[len(v) // 2]
    rows = []
    for n, (times, wall) in res.items():
        rows.append({"heads": n, "encoder_fwd_ms": round(med([t[enc_key] for t in times]), 3),
                     "probe_ms_per_head": round(med([t[probe_key] for t in times]) / n, 3),
                     "probe_ms_all_heads": round(med([t[probe_key] for t in times]), 3),
                     "value": round(batch * len(times) / wall, 2), "unit": unit})
    return {"heads": rows, "heads_timing": "head counts alternate step by step in one session; per head = median time "
                                           "of all heads' probe work after the encoder / heads; value = wall clock"}


def _augment_bytes(tickets, pack_augment, out):
    import numpy as np
    from jepa_b200.transforms import AUG_OP
    buf, frame_bytes, L, flags = pack_augment(tickets)
    ops = np.frombuffer(buf[frame_bytes + 64 * len(tickets):].numpy().tobytes(), AUG_OP).reshape(L, len(tickets))
    size = np.array([t.frames.numel() for t in tickets])
    hist = np.isin(ops["code"], (0, 1, 8))
    return int((2 * size * (ops["code"] >= 0)).sum() + (size * hist).sum() + size.sum() + out.numel() * out.element_size())


def _reference_cpu_ms(clip, crop):
    """The reference's pre-training transform with RandAugment and erasing (app/vjepa/transforms.py, the same ops as the
    evaluation's) on one uint8 clip, on this host's CPU, one thread: median ms over 8 calls; None without oracle/_ref."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "app")):
        return None
    code = ("import sys, time, random, numpy as np, torch; sys.path.insert(0, %r); torch.set_num_threads(1)\n"
            "from app.vjepa.transforms import VideoTransform\n"
            "tf = VideoTransform(random_resize_scale=(0.08, 1.0), reprob=0.25, auto_augment=True, crop_size=%d)\n"
            "x = np.load(sys.argv[1]); random.seed(0); np.random.seed(0); torch.manual_seed(0); ts = []\n"
            "for _ in range(8):\n    t0 = time.perf_counter(); tf(x); ts.append(time.perf_counter() - t0)\n"
            "print(sorted(ts)[4] * 1e3)") % (ref, crop)
    import tempfile
    import numpy as np
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "clip.npy")
        np.save(path, clip)
        r = subprocess.run([sys.executable, "-c", code, path], capture_output=True, text=True, cwd=d, timeout=600)
    try:
        return round(float(r.stdout.strip().splitlines()[-1]), 1)
    except (ValueError, IndexError):
        return None


def run_depth(args):
    from jepa_b200 import kernels as Kn
    from jepa_b200.optim import FlatAdamW, FlatGradScaler
    from jepa_b200.pooler import AttentiveClassifier
    from jepa_b200.step import clip_grad_norm_
    device = torch.device("cuda:0")
    torch.manual_seed(0)
    B, S, D, H, n_cls = args.batch, 12544, 1024, 16, 400
    fp16 = args.dtype == "float16"
    probes = {}
    for d in args.depth:
        clf = AttentiveClassifier(embed_dim=D, num_heads=H, depth=d, num_classes=n_cls, follow_autocast=fp16).to(device)
        groups = [{"params": [p for n, p in clf.named_parameters() if ("bias" not in n) and (len(p.shape) != 1)]},
                  {"params": [p for n, p in clf.named_parameters() if ("bias" in n) or (len(p.shape) == 1)],
                   "WD_exclude": True, "weight_decay": 0}]
        probes[d] = (clf, FlatAdamW(groups, lr=1e-3, weight_decay=0.01), FlatGradScaler())
    crit = torch.nn.CrossEntropyLoss()
    tokens = torch.randn(B, S, D, device=device)
    labels = torch.randint(0, n_cls, (B,), device=device)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {d: [] for d in args.depth}
    for i in range(args.warmup + args.steps):
        for d in args.depth:            # alternate the depths step by step: clock drift spreads over all of them
            clf, opt, scaler = probes[d]
            ev0.record()
            with _region(args):
                loss = crit(clf(tokens), labels)
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
            clip_grad_norm_(clf, 1.0)
            scaler.step(opt)
            scaler.update()
            opt.zero_grad()
            ev1.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                times[d].append(ev0.elapsed_time(ev1))
    med = lambda xs: sorted(xs)[len(xs) // 2]
    dt = torch.float16 if fp16 else torch.bfloat16
    kern = []
    for nq in (1, 16):
        qkv = torch.randn(B * nq, 3 * D, device=device).to(dt)
        out = torch.empty(B * nq, D, dtype=dt, device=device)
        dout = torch.randn(B * nq, D, device=device).to(dt)
        lse = torch.empty(B * nq, H, device=device)
        dqkv = torch.empty_like(qkv)
        row = {"nq": nq}
        for name, fn in (("fwd_us", lambda: Kn.query_attn_fwd(qkv, out, lse, B, nq, H, D // H, (D // H) ** -0.5)),
                         ("bwd_us", lambda: Kn.query_attn_bwd(qkv, out, dout, lse, dqkv, B, nq, H, D // H,
                                                              (D // H) ** -0.5))):
            for _ in range(20):
                fn()
            torch.cuda.synchronize()
            # replayed from a CUDA graph: the launches run back to back on the device, so the events time the kernels
            # rather than the host's ctypes dispatch of each call
            reps, replays = 200, 5
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(reps):
                    fn()
            graph.replay()
            ev0.record()
            for _ in range(replays):
                graph.replay()
            ev1.record()
            torch.cuda.synchronize()
            row[name] = round(ev0.elapsed_time(ev1) * 1000 / (reps * replays), 2)
        kern.append(row)
    card = _card()
    print(json.dumps({"mode": "depth", "dtype": args.dtype, "batch": B, "tokens_per_clip": S, "width": D, "heads": H,
                      "probe_step_ms": {str(d): round(med(t), 3) for d, t in times.items()},
                      "query_attn_kernel": kern, "steps": args.steps, "warmup": args.warmup,
                      "gpu": card[0] if card else None, "power_limit_w": card[1] if len(card) > 1 else None}))


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
    clfs = [AttentiveClassifier(embed_dim=enc.embed_dim, num_heads=enc.num_heads, depth=1, num_classes=n_cls,
                                follow_autocast=args.dtype == "float16").to(device).eval() for _ in range(max(args.heads))]
    g = torch.Generator().manual_seed(0)
    segments = [torch.randint(0, 256, (B, frames, H0, W0, 3), dtype=torch.uint8, generator=g).pin_memory()
                for _ in range(n_seg)]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]

    def step(timed, n_heads):
        if timed:
            ev[0].record()
        with torch.no_grad():
            clips = preprocess_views(segments, device, crop, n_views)
            if timed:
                ev[1].record()
            with _region(args):
                tokens = encoder(clips)
            if timed:
                ev[3].record()
            for clf in clfs[:n_heads]:
                with _region(args):
                    outputs = [clf(o) for o in tokens]
                probs = sum([F.softmax(o, dim=1) for o in outputs]) / len(outputs)
        if timed:
            ev[2].record()
        return probs

    def measure():
        return {"views": ev[0].elapsed_time(ev[1]), "enc_probe": ev[1].elapsed_time(ev[2]),
                "enc": ev[1].elapsed_time(ev[3]), "probe": ev[3].elapsed_time(ev[2])}

    sampler = ClockSampler(0)
    res = _alternate(args, step, measure)
    clocks = sampler.stop()
    times, wall = res[args.heads[0]]
    view_ms, enc_ms = [t["views"] for t in times], [t["enc_probe"] for t in times]

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
        "warmup": args.warmup, "higher_is_better": True, "dtype": args.dtype, "data": "synthetic uint8",
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
        **_heads_rows(args, res, B, "enc", "probe", "clips/s"),
    }), flush=True)


def run_image(args):
    import numpy as np
    from jepa_b200 import image_transforms as it
    from jepa_b200.models import vit_large
    from jepa_b200.optim import FlatAdamW, FlatGradScaler
    from jepa_b200.pooler import AttentiveClassifier
    from jepa_b200.step import clip_grad_norm_
    device = torch.device("cuda:0")
    torch.manual_seed(0)
    B = args.batch or 16
    frames, crop, n_cls, H0, W0 = 16, 224, 1000, 375, 500
    enc = vit_large(img_size=crop, num_frames=frames, tubelet_size=2, uniform_power=True).to(device).eval()
    for p in enc.parameters():
        p.requires_grad = False
    heads = []
    for _ in range(max(args.heads)):
        clf = AttentiveClassifier(embed_dim=enc.embed_dim, num_heads=enc.num_heads, depth=1, num_classes=n_cls,
                                  follow_autocast=args.dtype == "float16").to(device)
        groups = [{"params": [p for n, p in clf.named_parameters() if ("bias" not in n) and (len(p.shape) != 1)]},
                  {"params": [p for n, p in clf.named_parameters() if ("bias" in n) or (len(p.shape) == 1)],
                   "WD_exclude": True, "weight_decay": 0}]
        heads.append((clf, FlatAdamW(groups, lr=1e-3, weight_decay=0.01), FlatGradScaler()))
    crit = torch.nn.CrossEntropyLoss()
    g = torch.Generator(device="cpu").manual_seed(0)
    labels = torch.randint(0, n_cls, (B,), generator=g).to(device)
    tf = it.GpuImageTransform(crop_size=crop)
    host = [torch.randint(0, 256, (H0, W0, 3), dtype=torch.uint8, generator=g).numpy() for _ in range(B)]
    imgs = None if args.uint8 else torch.randn(B, 3, crop, crop, generator=g).to(device)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    host_ms = []

    def step(timed, n_heads):
        nonlocal imgs
        if args.uint8:
            t0 = time.perf_counter()
            tickets = [tf(x) for x in host]            # host decisions (what the loader workers do)
            if timed:
                host_ms.append((time.perf_counter() - t0) * 1e3)
            ev[3].record()
            imgs = tf.batch(tickets, device)
        if timed:
            ev[0].record()
        with _region(args):
            with torch.no_grad():
                outputs = enc(imgs.unsqueeze(2).repeat(1, 1, frames, 1, 1))
        if timed:
            ev[1].record()
        for clf, opt, scaler in heads[:n_heads]:        # the evaluation loop's per-head body on one encoder pass
            with _region(args):
                logits = clf(outputs)
            loss = crit(logits, labels)
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
            clip_grad_norm_(clf, 1.0)
            scaler.step(opt)
            scaler.update()
            opt.zero_grad()
        if timed:
            ev[2].record()

    def measure():
        return {"enc": ev[0].elapsed_time(ev[1]), "probe": ev[1].elapsed_time(ev[2]),
                "tf": ev[3].elapsed_time(ev[0]) if args.uint8 else None}

    sampler = ClockSampler(0)
    res = _alternate(args, step, measure)
    clocks = sampler.stop()
    times, wall = res[args.heads[0]]
    enc_ms, probe_ms = [t["enc"] for t in times], [t["probe"] for t in times]
    tf_ms = [t["tf"] for t in times] if args.uint8 else []

    # the kernels alone, on staged batches already on the device
    images = [torch.from_numpy(x) for x in host]
    tickets = [tf(x) for x in host]
    packed = it.pack_image_augment(images, [(t.box, (crop, crop), (0, 0), True, t.flip) for t in tickets], crop,
                                   [t.ops for t in tickets], [t.erase for t in tickets], [t.noise for t in tickets])
    dev, _ = it.to_device(packed["pk"], device)
    scratch = it.image_augment_scratch(packed, device)
    out = torch.empty(B, 3, crop, crop, device=device)
    fill = it.fill_color(it.DEFAULT_NORMALIZE[0])
    vpk, jobs_off, coefs_off, tmp_bytes = it.pack_image_views(images, crop)
    vdev, _ = it.to_device(vpk, device)
    vtmp = torch.empty(max(tmp_bytes, 16), dtype=torch.uint8, device=device)
    aug_k, views_k = [], []
    for i in range(args.warmup + args.steps):
        ev[0].record()
        it.launch_image_augment(dev, packed, scratch, out, *it.DEFAULT_NORMALIZE, fill)
        ev[1].record()
        it.launch_image_views(vdev, jobs_off, coefs_off, vtmp, out, *it.DEFAULT_NORMALIZE)
        ev[2].record()
        torch.cuda.synchronize()
        if i >= args.warmup:
            aug_k.append(ev[0].elapsed_time(ev[1]))
            views_k.append(ev[1].elapsed_time(ev[2]))
    card = _card()
    med = lambda v: round(sorted(v)[len(v) // 2], 3) if v else None
    print(json.dumps({
        "metric": "images/sec ViT-L/16 in1k frozen-evaluation probe training step (16x224^2 per image, 1000 classes)",
        "value": round(B * args.steps / wall, 2), "unit": "images/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "higher_is_better": True, "dtype": args.dtype,
        "data": (f"uint8 {W0}x{H0} images on the host, timm AutoAugment 'original' + erasing 0.25 on the GPU"
                 if args.uint8 else "pre-normalised images resident on the device"),
        "config": {"workload": f"batch {B}/GPU, each image repeated over {frames} frames ({enc.num_patches} tokens), "
                               "AttentiveClassifier depth 1, CrossEntropyLoss, FlatGradScaler + clip 1.0 + FlatAdamW"},
        "encoder_fwd_ms": med(enc_ms),
        "probe_fwd_bwd_opt_ms": med(probe_ms),
        "transform_ms": med(tf_ms),
        "host_decisions_ms": med(host_ms),
        "image_augment_kernels_ms": med(aug_k),
        "image_views_kernels_ms": med(views_k),
        "timing": "CUDA events per step, median over the timed steps; value = wall clock over the timed steps; "
                  "transform_ms: from before the batch call (host packing, one uint8 H2D copy, kernels) to the encoder; "
                  "host_decisions_ms: the transform's __call__ for the whole batch on one thread; *_kernels_ms: "
                  f"one launch sequence for {B} images staged on the device",
        "reference_cpu_ms_per_image": _reference_image_cpu_ms(host[0], crop),
        "gpu": card[0] if card else None,
        "power_limit_w": float(card[1]) if len(card) > 1 else None,
        "clocks": clocks,
        **_heads_rows(args, res, B, "enc", "probe", "images/s"),
    }), flush=True)


def _reference_image_cpu_ms(img, crop):
    """The reference's image training transform (timm's create_transform composition of the reference's
    RandomResizedCropAndInterpolation, RandomHorizontalFlip, AutoAugment of its AugmentOp, ToTensor, Normalize and
    RandomErasing) on one uint8 image, on this host's CPU, one thread: median ms over 16 calls; None without oracle/_ref."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "src")):
        return None
    from jepa_b200.image_transforms import AA_POLICY, DEFAULT_NORMALIZE, fill_color
    code = ("import sys, time, random, numpy as np, torch; sys.path.insert(0, %r)\n"
            "torch.set_num_threads(1)\n"
            "from PIL import Image; from torchvision import transforms as T\n"
            "import src.datasets.utils.video.randaugment as ra, src.datasets.utils.video.randerase as rr\n"
            "from src.datasets.utils.video.transforms import RandomResizedCropAndInterpolation\n"
            "AA_POLICY, fill, N, S = %r, %r, %r, %d\n"
            "hp = dict(translate_const=int(S * 0.45), img_mean=fill, interpolation=Image.BICUBIC)\n"
            "pol = [[ra.AugmentOp(n, prob=p, magnitude=m or 0, hparams=hp) for n, p, m in sp] for sp in AA_POLICY]\n"
            "pre = T.Compose([RandomResizedCropAndInterpolation(S, interpolation='bicubic'), T.RandomHorizontalFlip()])\n"
            "post = T.Compose([T.ToTensor(), T.Normalize(*N)])\n"
            "er = rr.RandomErasing(0.25, mode='pixel', max_count=1, device='cpu')\n"
            "x = Image.fromarray(np.load(sys.argv[1])); random.seed(0); torch.manual_seed(0); ts = []\n"
            "for _ in range(16):\n"
            "    t0 = time.perf_counter(); y = pre(x)\n"
            "    for op in random.choice(pol): y = op(y)\n"
            "    er(post(y)); ts.append(time.perf_counter() - t0)\n"
            "print(sorted(ts)[8] * 1e3)") % (ref, AA_POLICY, fill_color(DEFAULT_NORMALIZE[0]), DEFAULT_NORMALIZE, crop)
    import tempfile
    import numpy as np
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "img.npy")
        np.save(path, img)
        r = subprocess.run([sys.executable, "-c", code, path], capture_output=True, text=True, cwd=d, timeout=600)
    try:
        return round(float(r.stdout.strip().splitlines()[-1]), 2)
    except (ValueError, IndexError):
        return None


def run_xattn(args):
    """vj_cross_attn_fwd_lse / vj_cross_attn_bwd (+ its dq reduce) alone, bf16 and fp16 alternating per repetition."""
    from jepa_b200 import kernels as K
    device = torch.device("cuda:0")
    B, S, H, nq = args.batch or 4, 12544, 16, 1
    g = torch.Generator(device="cpu").manual_seed(0)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    rows = []
    for hd in args.head_dims:
        D = H * hd
        ref = {"q": torch.randn(B * nq, D, generator=g), "kv": torch.randn(B * S, 2 * D, generator=g),
               "dout": torch.randn(B * nq, D, generator=g)}
        bufs = {}
        for dt in (torch.bfloat16, torch.float16):
            t = {k: v.to(device, dt) for k, v in ref.items()}
            t["out"] = torch.empty(B * nq, D, dtype=dt, device=device)
            t["dkv"] = torch.empty(B * S, 2 * D, dtype=dt, device=device)
            t["lse"] = torch.empty(B * nq, H, device=device)
            t["dq"] = torch.empty(B * nq, D, device=device)
            bufs[dt] = t
        times = {dt: ([], []) for dt in bufs}
        for i in range(args.warmup + args.steps):
            for dt, t in bufs.items():
                ev[0].record()
                K.cross_attn_fwd_lse(t["q"], t["kv"], t["out"], t["lse"], B, nq, S, H, hd, hd ** -0.5)
                ev[1].record()
                K.cross_attn_bwd(t["q"], t["kv"], t["out"], t["dout"], t["lse"], t["dq"], t["dkv"], B, nq, S, H, hd,
                                 hd ** -0.5)
                ev[2].record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[dt][0].append(ev[0].elapsed_time(ev[1]))
                    times[dt][1].append(ev[1].elapsed_time(ev[2]))
        kv_bytes = B * S * 2 * D * 2
        for dt, (f, b) in times.items():
            fm, bm = sorted(f)[len(f) // 2], sorted(b)[len(b) // 2]
            rows.append({"hd": hd, "dtype": str(dt).replace("torch.", ""), "fwd_ms": round(fm, 4),
                         "bwd_ms": round(bm, 4), "fwd_gbps": round(kv_bytes / (fm * 1e-3) / 1e9, 1),
                         "bwd_gbps": round(2 * kv_bytes / (bm * 1e-3) / 1e9, 1),
                         "fwd_ms_min_max": [round(min(f), 4), round(max(f), 4)],
                         "bwd_ms_min_max": [round(min(b), 4), round(max(b), 4)]})
    card = _card()
    print(json.dumps({
        "metric": "cross-attention forward (with lse) and backward, bf16 vs fp16, K400 probe shape",
        "config": {"workload": f"B {B}, S {S}, H {H}, nq {nq}, hd {', '.join(map(str, args.head_dims))} "
                               "(ViT-L 64, ViT-H 80, ViT-g 88, ViT-G 104)"},
        "rows": rows,
        "timing": "CUDA events around each launch (backward: both kernels), median over the timed repetitions, the two "
                  "dtypes alternating; GB/s from the kv read (forward) and the kv read + dkv write (backward)",
        "gpu": card[0] if card else None,
        "power_limit_w": float(card[1]) if len(card) > 1 else None,
    }), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=None,
                    help="clips (images) per step; default 4 (K400 eval config) or, in image mode, 16 (in1k config)")
    ap.add_argument("--mode", choices=("train", "val", "image", "xattn"), default="train",
                    help="train: probe training step; val: validation step from uint8 frames; image: image probe step; "
                         "xattn: the cross-attention kernels alone, bf16 against fp16")
    ap.add_argument("--dtype", choices=("bfloat16", "float16"), default="bfloat16",
                    help="float16: encoder and probe under the reference's autocast(float16) region")
    ap.add_argument("--uint8", action="store_true",
                    help="train / image mode: uint8 frames / images through the GPU training transform")
    ap.add_argument("--heads", default=None,
                    help="train / val / image mode: comma-separated probe counts trained (validated) on one encoder "
                         "pass, e.g. 1,4,16, alternated step by step; reports encoder ms, probe ms per head and "
                         "throughput for each")
    ap.add_argument("--depth", default=None,
                    help="comma-separated probe depths, e.g. 1,2,4: ms per probe training step on device-resident "
                         "tokens for each, and the query self-attention kernels alone")
    ap.add_argument("--head-dims", default="64,80",
                    help="xattn mode: comma-separated head dims timed, e.g. 80,88,104,128")
    args = ap.parse_args()
    args.head_dims = [int(h) for h in args.head_dims.split(",")]
    args.multi = args.heads is not None
    args.heads = [int(n) for n in args.heads.split(",")] if args.multi else [1]
    if any(n < 1 for n in args.heads) or len(set(args.heads)) != len(args.heads):
        ap.error("--heads: distinct positive head counts")
    if args.multi and args.mode == "xattn":
        ap.error("--heads applies to --mode train, val and image")
    if args.depth is not None:
        args.depth = [int(d) for d in args.depth.split(",")]
        if any(d < 1 for d in args.depth) or len(set(args.depth)) != len(args.depth):
            ap.error("--depth: distinct positive depths")
        args.batch = args.batch or 4
        run_depth(args)
        return
    if args.mode == "image":
        run_image(args)
        return
    if args.mode == "xattn":
        run_xattn(args)
        return
    args.batch = args.batch or 4
    run(args) if args.mode == "train" else run_val(args)


if __name__ == "__main__":
    main()
