"""Patch embedding of ViT-G/14 (P = 3*2*14*14 = 1176, rows padded to 1216) next to ViT-g/16 (P = 1536, no padding) on one
GPU, 16x224^2 clips at batch 4, bf16:

  forward : vj_im2col_tubelets + the zero-padded [D, P_pad] weight copy (ViT-G/14 only) + the patch-embedding GEMM
            (bias and positional embedding in its epilogue), as engine.encoder_forward runs them
  wgrad   : the weight-gradient GEMM into the fp32 buffer (ViT-G/14: N = 1216 into a zeroed scratch, then the first
            1176 columns added into the flat gradient), as engine.encoder_backward runs it; bias gradient included

Random weights and inputs resident on the device.  CUDA events around each stage, median over the timed repetitions.
Prints ONE JSON line with the card's name and power limit.  Writes nothing into the repository.
    python tools/bench_patch_embed.py [--steps 50] [--warmup 10]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402


def _median_ms(fn, steps, warmup):
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


def case(name, factory, patch, B, steps, warmup):
    from jepa_b200 import engine, kernels as K
    from jepa_b200.params import padded_patch_dim
    dev = torch.device("cuda:0")
    mod = factory(img_size=224, patch_size=patch, num_frames=16, tubelet_size=2, uniform_power=True).to(dev)
    store = mod._store.adopt(mod)
    store.refresh_shadow()
    D, P = mod.embed_dim, mod.patch_embed.proj.weight[0].numel()
    Pp = padded_patch_dim(P)
    N = mod.num_patches
    T = B * N
    clips = torch.randn(B, 3, 16, 224, 224, device=dev)
    patches = torch.empty(T, Pp, dtype=torch.bfloat16, device=dev)
    x = torch.empty(T, D, dtype=torch.bfloat16, device=dev)
    pos = store.f32("pos_embed").view(N, D)
    bias = store.f32("patch_embed.proj.bias")

    def fwd():
        K.im2col_tubelets(clips, patches, None, 2, patch)
        w = engine.patch_embed_weight(mod, store, torch.bfloat16)
        K.gemm(patches, w, x, bias=bias, epi=K.EPI_ADD, aux=pos, aux_period=N)

    dx = torch.randn(T, D, device=dev).to(torch.bfloat16)
    gw = torch.zeros(D, P, device=dev)
    gb = torch.zeros(D, device=dev)
    pg = torch.empty(D, Pp, device=dev)

    def wgrad():
        if Pp == P:
            engine._wgrad(dx, patches, gw, gb, T)
        else:
            pg.zero_()
            engine._wgrad(dx, patches, pg, gb, T)
            K.head_pad(pg, gw, D, 1, P, Pp, 1, unpad_add=True)

    fwd()
    fm, wm = _median_ms(fwd, steps, warmup), _median_ms(wgrad, steps, warmup)
    flops = 2.0 * T * D * Pp
    return {"model": name, "tokens": T, "D": D, "P": P, "P_pad": Pp, "fwd_ms": round(fm, 4), "wgrad_ms": round(wm, 4),
            "fwd_tflops": round(flops / (fm * 1e-3) / 1e12, 1), "wgrad_tflops": round(flops / (wm * 1e-3) / 1e12, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_patch_embed: needs a CUDA device")
    from functools import partial

    from jepa_b200.models import VisionTransformer
    from tools.bench_probe import _card
    # the patch embedding only: the factories' widths and patch sizes, no blocks
    vitg14 = partial(VisionTransformer, embed_dim=1664, depth=0, num_heads=16, mlp_ratio=4, qkv_bias=True,
                     norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))
    vitg16 = partial(VisionTransformer, embed_dim=1408, depth=0, num_heads=16, mlp_ratio=48 / 11, qkv_bias=True,
                     norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))
    rows = [case("ViT-G/14", vitg14, 14, args.batch, args.steps, args.warmup),
            case("ViT-g/16", vitg16, 16, args.batch, args.steps, args.warmup)]
    card = _card()
    print(json.dumps({
        "metric": "patch-embedding forward and weight gradient, 16x224^2 clips, bf16",
        "config": {"batch": args.batch, "steps": args.steps, "warmup": args.warmup},
        "rows": rows,
        "timing": "CUDA events around each stage, median; TFLOP/s from 2 * tokens * D * P_pad",
        "gpu": card[0] if card else None,
        "power_limit_w": float(card[1]) if len(card) > 1 else None,
    }), flush=True)


if __name__ == "__main__":
    main()
