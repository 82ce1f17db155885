"""Frozen encoder in float16: the fp16 kernels (vj_gemm_f16, vj_attn_fwd_f16, fp16 LayerNorm, im2col and shadow cast)
against fp64 references computed on the device from the same fp16 inputs, and VisionTransformer under
torch.autocast('cuda', dtype=torch.float16), as the reference's eval loops run their encoder.

Bounds are about 8x tighter than the bf16 ones (fp16 keeps 11 significand bits, bf16 8):
  fp16-stored outputs : |err| <= 2.5e-3 + 1e-3 |ref|
  lse2                : |err| <= 1e-3
Run with -s to print the worst err / bound per case at the end of the module.
"""
import math

import pytest
import torch
import torch.nn.functional as Fn

from attention_ref import POISON_LENS, Packed, plant_last_key, poison_rows, reference

pytestmark = pytest.mark.gpu
F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
ATOL, RTOL, LSE_ATOL = 2.5e-3, 1e-3, 1e-3
WORST = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    yield torch.device("cuda:0")
    for k in sorted(WORST):
        print(f"\nworst err/bound {k}: {WORST[k]:.3g}")


def within(name, got, ref, atol=ATOL, rtol=RTOL):
    got, ref = got.double(), ref.double()
    ratio = torch.nan_to_num((got - ref).abs() / (atol + rtol * ref.abs()), nan=math.inf)
    worst = float(ratio.max())
    WORST[name] = max(WORST.get(name, 0.0), worst)
    assert worst <= 1.0, f"{name}: worst err/bound {worst:.4g}"


def h(shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(F16)


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


# ------------------------------------------------------------------------------------------------------------- GEMM
GEMM_SHAPES = [(333, 192, 384), (1000, 320, 1024), (257, 512, 4096), (129, 256, 4096)]   # ragged M, N odd x 64, long K


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
@pytest.mark.parametrize("case", ["none", "none_f32", "gelu", "gelu_grad", "add_f16", "add_f32_rowmap",
                                  "add_f32_period_f32out"])
def test_gemm_forward_f16_vs_fp64(dev, M, N, K, case):
    from jepa_b200 import kernels as Kn
    g = torch.Generator().manual_seed(M * 7 + N + K)
    a, b = h((M, K), g).to(dev), h((N, K), g, K ** -0.5).to(dev)
    bias = (torch.randn(N, generator=g) * 0.5).to(dev)
    acc = a.double() @ b.double().t() + bias.double()
    out = torch.full((M, N), float("nan"), dtype=F32 if case.endswith("f32out") or case == "none_f32" else F16,
                     device=dev)
    if case in ("none", "none_f32"):
        Kn.gemm(a, b, out, bias=bias)
        within("gemm " + case, out, acc)
    elif case in ("gelu", "gelu_grad"):
        aux_out = torch.full((M, N), float("nan"), dtype=F16, device=dev)
        Kn.gemm(a, b, out, bias=bias, epi=Kn.EPI_GELU if case == "gelu" else Kn.EPI_GELU_GRAD, aux_out=aux_out)
        within("gemm " + case, out, gelu64(acc))
        within("gemm " + case + " aux_out", aux_out, acc if case == "gelu" else gelu_grad64(acc))
    elif case == "add_f16":
        res = h((M, N), g, 4.0).to(dev)
        Kn.gemm(a, b, out, bias=bias, epi=Kn.EPI_ADD, aux=res)
        within("gemm " + case, out, acc + res.double())
    elif case == "add_f32_rowmap":
        table = torch.randn(50, N, generator=g).to(dev)
        rowmap = torch.randint(0, 50, (M,), generator=g, dtype=torch.int32).to(dev)
        Kn.gemm(a, b, out, bias=bias, epi=Kn.EPI_ADD, aux=table, aux_rowmap=rowmap)
        within("gemm " + case, out, acc + table.double()[rowmap.long()])
    else:
        table = torch.randn(37, N, generator=g).to(dev)
        Kn.gemm(a, b, out, bias=bias, epi=Kn.EPI_ADD, aux=table, aux_period=37)
        within("gemm " + case, out, acc + table.double()[torch.arange(M, device=dev) % 37])


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES[:3])
def test_gemm_dgrad_wgrad_f16_vs_fp64(dev, M, N, K):
    """dgrad (B read MN-major) plain and with MUL, and the fp32 weight gradient (both operands MN-major), accumulating."""
    from jepa_b200 import kernels as Kn
    g = torch.Generator().manual_seed(M + N * 3 + K)
    dy, w = h((M, K), g).to(dev), h((K, N), g, K ** -0.5).to(dev)      # dx[M, N] = dy[M, K] @ w[K, N]
    ref = dy.double() @ w.double()
    dx = torch.full((M, N), float("nan"), dtype=F16, device=dev)
    Kn.gemm(dy, w, dx, b_mn=True)
    within("dgrad", dx, ref)
    gp = h((M, N), g).to(dev)
    Kn.gemm(dy, w, dx, b_mn=True, epi=Kn.EPI_MUL, aux=gp)
    within("dgrad mul", dx, ref * gp.double())
    Mw = (M + 7) // 8 * 8
    x = h((K, Mw), g, K ** -0.5).to(dev)     # wgrad: out[Mw, N] += x^T[Mw, K] @ w[K, N]
    start = torch.randn(Mw, N, generator=g).to(dev)
    out = start.clone()
    Kn.gemm(x, w, out, a_mn=True, b_mn=True, accumulate=True, split_k=2)
    within("wgrad", out, start.double() + x.double().t() @ w.double(), atol=1e-4, rtol=1e-5)


def test_gemm_f16_overflow_is_inf_like_torch(dev):
    """A row whose true result exceeds 65504 comes out +-inf (round to nearest, no clamping), as F.linear in fp16."""
    from jepa_b200 import kernels as Kn
    g = torch.Generator().manual_seed(5)
    M, N, K = 130, 128, 384
    a, b = h((M, K), g).to(dev), h((N, K), g, K ** -0.5).to(dev)
    a[7] = 300.0
    b[3] = 1.0
    b[4] = -1.0
    out = torch.empty(M, N, dtype=F16, device=dev)
    Kn.gemm(a, b, out)
    want = Fn.linear(a, b)
    assert float(out[7, 3]) == math.inf and float(out[7, 4]) == -math.inf
    assert torch.equal(torch.isinf(out), torch.isinf(want))
    fin = ~torch.isinf(want)
    within("gemm overflow rows", out[fin], (a.double() @ b.double().t())[fin])


# -------------------------------------------------------------------------------------------------------- attention
def _rows16(L, H, hd, g):
    return [torch.randn(L, H, hd, generator=g).to(F16).float() for _ in range(4)]


@pytest.mark.parametrize("hd", [24, 64, 80, 128])
def test_attention_forward_f16_residue_sweep(dev, hd):
    """L = 1 ... 385, every sequence between poison sequences (tests/attention_ref.py), all in one launch per head dim;
    O and lse2 of every checked sequence against fp64, padded lanes exactly zero."""
    from jepa_b200 import kernels as Kn
    from jepa_b200.params import padded_head_dim
    H, hdp = 2, padded_head_dim(hd)
    pk = Packed()
    for L in range(1, 386):
        g = torch.Generator().manual_seed(1000 * hd + L)
        rows = _rows16(L, H, hd, g)
        plant_last_key(rows[0], rows[1], g)
        pk.add(poison_rows(POISON_LENS[0], rows[0], rows[1], g), checked=False)
        pk.add(rows)
    q, k, v = (t.half().float() for t in pk.tensors()[:3])     # what the kernel reads (poison rows included)
    T = q.shape[0]
    qkv = torch.zeros(T, 3, H, hdp, dtype=F16, device=dev)
    for i, t in enumerate((q, k, v)):
        qkv[:, i, :, :hd] = t.to(dev)
    qkv = qkv.view(T, 3 * H * hdp)
    cu = torch.tensor(pk.cu_seqlens(), dtype=torch.int32, device=dev)
    out = torch.full((T, H * hdp), float("nan"), dtype=F16, device=dev)
    lse = torch.full((H, T), float("nan"), device=dev)
    Kn.attn_fwd(qkv, out, lse, cu, len(pk.lens), max(pk.lens), H, hdp, hd ** -0.5)
    out = out.view(T, H, hdp)
    assert torch.equal(out[..., hd:], torch.zeros_like(out[..., hd:]))
    qd, kd, vd = (t.to(dev) for t in (q, k, v))
    for r0, L in pk.checked:
        s = slice(r0, r0 + L)
        ref = reference(qd[s], kd[s], vd[s], scale=hd ** -0.5)
        within(f"attn O hd {hd}", out[s, :, :hd], ref["o"])
        within(f"attn lse2 hd {hd}", lse[:, s], ref["lse2"], atol=LSE_ATOL, rtol=0.0)


# ---------------------------------------------------------------------------------------------- row kernels, shadow
@pytest.mark.parametrize("D", [8, 192, 264, 768, 1032, 1280, 2048])
@pytest.mark.parametrize("io", ["f16-f16", "f16-f32", "f32-f16"])
def test_layernorm_f16_vs_fp64(dev, D, io):
    from jepa_b200 import kernels as Kn
    ti, to = (F16 if s == "f16" else F32 for s in io.split("-"))
    g = torch.Generator().manual_seed(D)
    T = 777
    x = (torch.randn(T, D, generator=g) * 2 + 3).to(ti).to(dev)
    gamma, beta = (torch.randn(D, generator=g).to(dev) for _ in range(2))
    y = torch.full((T, D), float("nan"), dtype=to, device=dev)
    mean, rstd = torch.empty(T, device=dev), torch.empty(T, device=dev)
    Kn.layernorm_fwd(x, y, gamma, beta, 1e-6, mean, rstd)
    ref = Fn.layer_norm(x.double(), (D,), gamma.double(), beta.double(), 1e-6)
    within(f"layernorm {io}", y, ref, atol=ATOL if to == F16 else 1e-4, rtol=RTOL if to == F16 else 1e-5)
    within(f"layernorm {io} mean", mean, x.double().mean(-1), atol=1e-5, rtol=1e-6)


def test_layernorm_rejects_unpaired_f16(dev):
    from jepa_b200 import _lib, kernels as Kn
    x = torch.zeros(4, 64, dtype=F16, device=dev)
    with pytest.raises(_lib.VJError):
        Kn.layernorm_fwd(x, torch.empty(4, 64, dtype=BF16, device=dev), torch.ones(64, device=dev),
                         torch.zeros(64, device=dev), 1e-6)


def test_im2col_cast_head_pad_f16_bit_exact(dev):
    """fp32 -> fp16 conversions of the patch gather, the shadow cast and the head-padded weights are torch's .half()."""
    from jepa_b200 import kernels as Kn
    g = torch.Generator().manual_seed(11)
    clips = (torch.randn(2, 3, 4, 32, 48, generator=g) * 3e4).to(dev)     # includes values past 65504
    for idx in (None, torch.tensor([[5, 0, 11], [2, 2, 7]], device=dev)):
        K = 12 if idx is None else 3
        patches = torch.empty(2 * K, 3 * 2 * 16 * 16, dtype=F16, device=dev)
        Kn.im2col_tubelets(clips, patches, idx, 2, 16)
        ref = clips.view(2, 3, 2, 2, 2, 16, 3, 16).permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(2, 12, -1)
        if idx is not None:
            ref = torch.stack([ref[b, idx[b]] for b in range(2)])
        assert torch.equal(patches, ref.reshape(2 * K, -1).half())
    src = torch.randn(4096 + 64, generator=g).to(dev) * 1e3
    dst = torch.empty_like(src, dtype=F16)
    Kn.cast_f32_f16(src, dst)
    assert torch.equal(dst, src.half())
    w = torch.randn(3 * 4 * 80, 64, generator=g).to(dev)
    wp = torch.empty(3 * 4 * 128, 64, dtype=F16, device=dev)
    Kn.head_pad(w, wp, 1, 12, 80, 128, 64)
    ref = torch.zeros(12, 128, 64, device=dev)
    ref[:, :80] = w.view(12, 80, 64)
    assert torch.equal(wp, ref.view_as(wp).half())


# ----------------------------------------------------------------------------------------------- VisionTransformer
def _encoder_fp64(mod, x):
    """VisionTransformer.forward (vision_transformer.py:159-195) in fp64 from the fp32 master weights."""
    sd = {k: v.double() for k, v in mod.state_dict().items()}
    conv = Fn.conv3d if mod.is_video else Fn.conv2d
    t = conv(x.double(), sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=mod.patch_embed.proj.stride)
    t = t.flatten(2).transpose(1, 2) + sd["pos_embed"]
    H, D = mod.num_heads, mod.embed_dim
    for i in range(len(mod.blocks)):
        p = f"blocks.{i}."
        y = Fn.layer_norm(t, (D,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
        qkv = Fn.linear(y, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])
        B, N, _ = qkv.shape
        q, k, v = qkv.view(B, N, 3, H, D // H).permute(2, 0, 3, 1, 4)
        a = torch.softmax(q @ k.transpose(-1, -2) * (D // H) ** -0.5, -1) @ v
        t = t + Fn.linear(a.transpose(1, 2).reshape(B, N, D), sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        y = Fn.layer_norm(t, (D,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-6)
        y = Fn.linear(gelu64(Fn.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])), sd[p + "mlp.fc2.weight"],
                      sd[p + "mlp.fc2.bias"])
        t = t + y
    return Fn.layer_norm(t, (D,), sd["norm.weight"], sd["norm.bias"], 1e-6)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("arch", ["tiny_video", "huge_slice_video", "large_image"])
def test_vit_under_f16_autocast(dev, arch):
    """fp16 autocast: fp32 outputs (LayerNorm is on autocast's fp32 list), closer to fp64 than bf16 is; no autocast and
    bf16 autocast are bitwise what they were; out_layers taps are fp32 too."""
    from functools import partial

    from jepa_b200.models import VisionTransformer, vit_tiny
    torch.manual_seed(0)
    vit = partial(VisionTransformer, depth=2, mlp_ratio=4, qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))
    if arch == "tiny_video":
        mod, x = vit_tiny(img_size=224, num_frames=8), torch.randn(2, 3, 8, 224, 224)
    elif arch == "huge_slice_video":   # ViT-H's width and heads (hd 80, padded to 128), 2 blocks
        mod, x = vit(img_size=160, num_frames=4, embed_dim=1280, num_heads=16), torch.randn(2, 3, 4, 160, 160)
    else:                              # ViT-L's width and heads, 2 blocks, image encoder
        mod, x = vit(img_size=224, num_frames=1, embed_dim=1024, num_heads=16), torch.randn(3, 3, 224, 224)
    mod, x = mod.to(dev).eval(), x.to(dev)
    with torch.no_grad():
        ref = _encoder_fp64(mod, x)
        plain = mod(x)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            bf = mod(x)
        with torch.autocast("cuda", dtype=torch.float16):
            half = mod(x)
        with torch.cuda.amp.autocast(dtype=torch.float16):
            half2 = mod(x)
        again = mod(x)
    assert plain.dtype == BF16 and bf.dtype == BF16 and half.dtype == F32
    assert torch.equal(plain, bf) and torch.equal(plain, again) and torch.equal(half, half2)
    e16, e_bf = _rel(half, ref), _rel(plain, ref)
    print(f"\n{arch}: rel-L2 vs fp64: fp16 {e16:.3g}, bf16 {e_bf:.3g}")
    assert e16 <= 4e-3 and e16 <= 0.5 * e_bf
    mod.out_layers = [0, 1]
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        taps = mod(x)
    assert [t.dtype for t in taps] == [F32, F32]


def test_f16_autocast_training_and_predictor_raise(dev):
    from jepa_b200.models import vit_predictor, vit_tiny
    torch.manual_seed(0)
    mod = vit_tiny(img_size=32, num_frames=2).to(dev)
    x = torch.randn(1, 3, 2, 32, 32, device=dev)
    with torch.autocast("cuda", dtype=torch.float16):
        with pytest.raises(NotImplementedError, match="no_grad"):
            mod(x)
        pred = vit_predictor(img_size=32, num_frames=2, embed_dim=192, predictor_embed_dim=96, depth=1, num_heads=4,
                             use_mask_tokens=True).to(dev)
        m = torch.arange(4, device=dev).view(1, 4)
        with pytest.raises(NotImplementedError, match="predictor"):
            pred(torch.zeros(1, 4, 192, device=dev), None, m, m)


def test_reference_eval_loop_body_runs_under_f16_autocast(dev):
    """The reference's loop body as written (evals/video_classification_frozen/eval.py:320-340): the frozen encoder under
    no_grad and the classifier both inside autocast(float16), then GradScaler.  The encoder runs in fp16 and hands the
    probe fp32 features; the probe computes as it does outside autocast (bitwise the same logits) and trains."""
    from jepa_b200.models import vit_tiny
    from jepa_b200.pooler import AttentiveClassifier
    torch.manual_seed(0)
    enc = vit_tiny(img_size=64, num_frames=4).to(dev).eval()
    clf = AttentiveClassifier(embed_dim=192, num_heads=3, depth=1, num_classes=4).to(dev)
    opt = torch.optim.AdamW(clf.parameters(), lr=1e-3)
    scaler = torch.cuda.amp.GradScaler()
    g = torch.Generator().manual_seed(1)
    labels = torch.arange(4, device=dev).repeat(2)
    clips = (torch.randn(8, 3, 4, 64, 64, generator=g).to(dev) + labels.view(-1, 1, 1, 1, 1).float())
    losses = []
    for _ in range(30):
        with torch.cuda.amp.autocast(dtype=torch.float16):
            with torch.no_grad():
                feats = enc(clips)
            out = clf(feats)
        assert feats.dtype == F32 and out.dtype == F32
        with torch.no_grad():
            assert torch.equal(out, clf(feats))
        loss = Fn.cross_entropy(out, labels)
        opt.zero_grad()
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        losses.append(float(loss))
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]


def test_no_grad_forward_keeps_nothing_and_matches(dev):
    """Under torch.no_grad() the encoder saves no activations whether or not its parameters require grad; the bf16
    outputs are bitwise the same either way, and the un-normalised output (final_norm=False) is available there."""
    from jepa_b200.models import vit_tiny
    torch.manual_seed(0)
    mod = vit_tiny(img_size=64, num_frames=4).to(dev)
    x = torch.randn(2, 3, 4, 64, 64, device=dev)
    masks = [torch.arange(0, 32, 2, device=dev).repeat(2, 1)]
    with torch.no_grad():
        a = mod(x)
        ma = mod.forward_multi(x, masks, final_norm=False)[0].clone()
        for p in mod.parameters():
            p.requires_grad_(False)
        b = mod(x)
        mb = mod.forward_multi(x, masks, final_norm=False)[0].clone()
    assert a.dtype == BF16 and torch.equal(a, b) and torch.equal(ma, mb)
    for p in mod.parameters():
        p.requires_grad_(True)
    c = mod(x)                      # with grad: the saving forward, same values
    assert torch.equal(a, c.detach())
