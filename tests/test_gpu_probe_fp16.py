"""The attentive probe in float16 (-m gpu): the fp16 kernels it trains on (vj_cross_attn_*_f16, vj_layernorm_bwd_f16,
vj_colsum_f16) against fp64 computed on the device from the same fp16 inputs; AttentivePooler / AttentiveClassifier
with follow_autocast=True under torch.autocast('cuda', dtype=torch.float16) against the fp64 oracle; GradScaler with the
reference's loop body; and the evaluation drivers with `optimization.fp16_autocast: true` end to end.

Bounds, about 8x tighter than bf16's (as in test_gpu_fp16.py), and where the fp16 rounding of the fp64 value overflows
the stored value must be that inf (tests/xattn16_ref.py; tests/test_probe_fp16_cpu.py shows what they reject):
  fp16-stored outputs      : |err| <= 2.5e-3 + 1e-3 |ref|
  lse2                     : |err| <= 1e-3
  gradients (dq, dk, dv)   : |err| <= 4e-3 + 2.5e-3 |ref|
Run with -s to print the worst err / bound per group at the end of the module.
"""
import math
import os

import pytest
import torch
import torch.nn.functional as Fn

import xattn16_ref as X
from parity_util import rel_l2

pytestmark = pytest.mark.gpu
F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
WORST = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    yield torch.device("cuda:0")
    for k in sorted(WORST):
        print(f"\nworst err/bound {k}: {WORST[k]:.3g}")


def within(name, got, ref, atol, rtol):
    got, ref = got.double(), ref.double()
    ratio = torch.nan_to_num((got - ref).abs() / (atol + rtol * ref.abs()), nan=math.inf)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), worst)
    assert worst <= 1.0, f"{name}: worst err/bound {worst:.4g}"


# ------------------------------------------------------------------------------------------------- cross-attention
def run_xattn(dev, c):
    """The fp16 kernels on case c (tests/xattn16_ref.py): (out, lse2, dq, dkv) of all three clips."""
    from jepa_b200 import kernels as Kn
    B, nq, S, H, hd, scale = (c[k] for k in ("B", "nq", "S", "H", "hd", "scale"))
    q, kv, dout = (c[k].to(F16).to(dev) for k in ("q", "kv", "dout"))
    out = torch.full((B * nq, H * hd), float("nan"), dtype=F16, device=dev)
    out2 = torch.full_like(out, float("nan"))
    lse = torch.full((B * nq, H), float("nan"), device=dev)
    Kn.cross_attn_fwd(q, kv, out, B, nq, S, H, hd, scale)
    Kn.cross_attn_fwd_lse(q, kv, out2, lse, B, nq, S, H, hd, scale)
    assert torch.equal(out, out2), "out of _fwd_f16 and _fwd_lse_f16 differ"
    dq = torch.full((B * nq, H * hd), float("nan"), device=dev)
    dkv = torch.full((B * S, 2 * H * hd), float("nan"), dtype=F16, device=dev)
    Kn.cross_attn_bwd(q, kv, out, dout, lse, dq, dkv, B, nq, S, H, hd, scale)
    dq2, dkv2 = torch.empty_like(dq), torch.empty_like(dkv)
    Kn.cross_attn_bwd(q, kv, out, dout, lse, dq2, dkv2, B, nq, S, H, hd, scale)
    assert torch.equal(dq, dq2) and torch.equal(dkv, dkv2), "backward is not bitwise reproducible"
    return q, kv, dout, out, lse, dq, dkv


def xattn_case(dev, hd, nq, S, seed):
    c = X.make_case(hd, nq, S, seed)
    q, kv, dout, out, lse, dq, dkv = run_xattn(dev, c)
    ck = lambda t, n: X.checked(c, t, n)
    res = X.check(c, ck(out, nq), ck(lse, nq), ck(dq, nq), ck(dkv, S), X.reference(c, q, kv, dout, ck(out, nq)))
    for k, v in res.items():
        WORST[f"xattn {k} hd {hd}"] = max(WORST.get(f"xattn {k} hd {hd}", 0.0), v)
        assert v <= 1.0, (k, hd, nq, S, v)
    # the poison clips' own results stay finite: nothing of clip 1 leaked into them either
    assert torch.isfinite(out).all() and torch.isfinite(dq).all()


@pytest.mark.parametrize("hd", [32, 64, 80, 128])
@pytest.mark.parametrize("nq", [1, 3])
def test_cross_attn_f16_vs_fp64_every_residue(dev, hd, nq):
    """S = 1 ... 300: every residue of the lane-group width (32 / LPK keys per warp) and of the backward's key chunk."""
    for S in range(1, 301):
        xattn_case(dev, hd, nq, S, seed=hd * 1000 + nq * 400 + S)


@pytest.mark.parametrize("hd", [32, 64, 80, 128])
@pytest.mark.parametrize("S", [1568, 4608, 12544])
def test_cross_attn_f16_vs_fp64_encoder_lengths(dev, hd, S):
    for nq in (1, 3):
        xattn_case(dev, hd, nq, S, seed=S + hd + nq)


def test_cross_attn_f16_rejects(dev):
    """fp16 and bf16 operands do not mix; the bf16 entry points keep their own dtype checks."""
    from jepa_b200 import _lib, kernels as Kn
    q = torch.zeros(1, 64, dtype=F16, device=dev)
    kv = torch.zeros(8, 128, dtype=BF16, device=dev)
    with pytest.raises(_lib.VJError):
        Kn.cross_attn_fwd(q, kv, torch.empty(1, 64, dtype=F16, device=dev), 1, 1, 8, 1, 64, 0.125)
    with pytest.raises(_lib.VJError):
        Kn.cross_attn_fwd(q.float(), kv.float(), torch.empty(1, 64, device=dev), 1, 1, 8, 1, 64, 0.125)


# ----------------------------------------------------------------------------------------------------- row kernels
@pytest.mark.parametrize("D", [8, 192, 264, 768, 1032, 1280, 2048])   # every NV the dispatch picks (1, 2, 4, 5, 8)
def test_layernorm_bwd_f16_dy_vs_fp64(dev, D):
    from jepa_b200 import kernels as Kn
    g = torch.Generator().manual_seed(D)
    T = 777
    x = (torch.randn(T, D, generator=g) * 2 + 3).to(dev)
    gamma = torch.randn(D, generator=g).to(dev)
    dy = torch.randn(T, D, generator=g).to(F16).to(dev)
    dres = torch.randn(T, D, generator=g).to(dev)
    xd = x.double()
    mu = xd.mean(-1)
    rs = 1.0 / torch.sqrt(((xd - mu[:, None]) ** 2).mean(-1) + 1e-6)
    xh = (xd - mu[:, None]) * rs[:, None]
    gy = dy.double() * gamma.double()
    ref_dx = rs[:, None] * (gy - gy.mean(-1, keepdim=True) - xh * (gy * xh).mean(-1, keepdim=True)) + dres.double()
    dg0, db0 = torch.randn(D, generator=g).to(dev), torch.randn(D, generator=g).to(dev)
    dgamma, dbeta = dg0.clone(), db0.clone()
    dx = torch.full((T, D), float("nan"), device=dev)
    Kn.layernorm_bwd(dy, x, gamma, mu.float(), rs.float(), dres, dx, dgamma, dbeta)
    within("layernorm bwd f16 dy: dx", dx, ref_dx, 1e-4, 1e-4)
    within("layernorm bwd f16 dy: dgamma", dgamma, dg0.double() + (dy.double() * xh).sum(0), 1e-3, 1e-5)
    within("layernorm bwd f16 dy: dbeta", dbeta, db0.double() + dy.double().sum(0), 1e-3, 1e-5)


def test_layernorm_bwd_f16_dy_needs_fp32_x(dev):
    from jepa_b200 import _lib, kernels as Kn
    x = torch.zeros(4, 64, dtype=BF16, device=dev)
    z = torch.zeros(64, device=dev)
    with pytest.raises(_lib.VJError):
        Kn.layernorm_bwd(torch.zeros(4, 64, dtype=F16, device=dev), x, z, z[:4], z[:4], None, torch.empty_like(x), z, z)


@pytest.mark.parametrize("T,N,period,lo,hi", [(1, 8, 0, 0, 0), (777, 2048, 0, 0, 0), (12544, 1024, 0, 0, 0),
                                              (5000, 264, 0, 0, 0), (3 * 401, 1280, 3, 1, 2), (64 * 7 + 5, 400, 7, 2, 6)])
def test_colsum_f16_vs_fp64(dev, T, N, period, lo, hi):
    from jepa_b200 import kernels as Kn
    g = torch.Generator().manual_seed(T + N)
    x = (torch.randn(T, N, generator=g) * 3).to(F16).to(dev)
    start = torch.randn(N, generator=g).to(dev)
    out = start.clone()
    Kn.colsum(x, out, period=period, lo=lo, hi=hi)
    rows = torch.arange(T, device=dev)
    keep = torch.ones(T, dtype=torch.bool, device=dev) if period <= 0 else ((rows % period >= lo) & (rows % period < hi))
    ref = start.double() + x.double()[keep].sum(0)
    within("colsum f16", out, ref, 1e-5 * x.double()[keep].abs().sum(0).max() + 1e-6, 0.0)


def test_f16_stores_overflow_to_inf(dev):
    """Past 65504 an fp16 store becomes +-inf (round to nearest, no satfinite clamp): GradScaler needs the inf.  One key
    and three queries with upstream gradients of 60000: dv = 180000 must store as +inf, dq stays fp32 and finite."""
    from jepa_b200 import kernels as Kn
    c = X.overflow_case()
    q, kv, dout, out, lse, dq, dkv = run_xattn(dev, c)
    hd = c["hd"]
    assert torch.isinf(dkv[:, hd:]).all() and (dkv[:, hd:] > 0).all()
    assert torch.isfinite(dq).all()
    res = X.check(c, X.checked(c, out, 3), X.checked(c, lse, 3), X.checked(c, dq, 3), X.checked(c, dkv, 1),
                  X.reference(c, q, kv, dout, X.checked(c, out, 3)))
    assert max(res.values()) <= 1.0, res
    x = torch.full((4, 64), 6e4, dtype=F16, device=dev)
    acc = torch.zeros(64, device=dev)
    Kn.colsum(x, acc)
    assert float(acc[0]) == 2.4e5                          # summed in fp32: no fp16 intermediate


# ------------------------------------------------------------------------------------------------ probe modules
def _sharpen(mod, seed, query=5.0, qk=3.0):
    torch.manual_seed(seed)
    pool = mod.pooler if hasattr(mod, "pooler") else mod
    blk = pool.cross_attention_block
    xa = blk.xattn if pool.complete_block else blk
    with torch.no_grad():
        for n, p in mod.named_parameters():
            if n.endswith("bias") or "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
        pool.query_tokens.mul_(query)
        xa.q.weight.mul_(qk)
        xa.kv.weight.mul_(qk)
    return mod


# Loss scales of the 16-bit runs, as GradScaler applies them in the reference's loop: without one, per-token gradients of
# about p_j dO ~ 1 / S fall into fp16's subnormal range.  The classifier starts at 2^15, the scale GradScaler settles at
# there (its initial 2^16 overflows the fp16 loss's own gradient, 65536 > 65504, and is halved on the first step); the
# pooler tests start at 2^12, which keeps the fp16 output's incoming gradient dy * scale finite for a randn dy.  As
# GradScaler does, a backward with a non-finite gradient is discarded and repeated at half the scale.
LOSS_SCALE = {True: 2.0 ** 15, False: 2.0 ** 12}


def _scaled_backward(run, head, grads):
    """run() -> the loss; grads() -> {name: gradient or None}.  Backward of loss * scale, halving the scale while a
    gradient is non-finite; returns the gradients divided back, in fp64."""
    scale = LOSS_SCALE[head]
    for _ in range(16):
        (run().float() * scale).backward()
        g = {n: None if v is None else v.double() / scale for n, v in grads().items()}
        if all(v is None or bool(torch.isfinite(v).all()) for v in g.values()):
            return g
        scale /= 2
    raise AssertionError("no finite gradients at any loss scale")


def _oracle_run(S_, x, H, cb, head, dy, labels, dtype=F64, autocast=False):
    """The oracle restatement by autograd: fp64 (unscaled), or (autocast) eagerly under CUDA fp16 autocast from fp32
    weights with the loss scaled by LOSS_SCALE and the gradients divided back.  There the oracle uses torch's F.linear,
    F.layer_norm and F.gelu, as the reference does; its cross-attention stays matmul / softmax / matmul under autocast
    (fp16 matmuls, softmax in fp32), not the reference's fp16 SDPA."""
    from oracle import vjepa_oracle as O
    S_ = {k: v.to(dtype).detach().clone().requires_grad_(True) for k, v in S_.items()}
    out = {}

    def run():
        for v in S_.values():
            v.grad = None
        fused = O.FUSED
        O.FUSED = autocast
        try:
            with torch.autocast("cuda", dtype=F16, enabled=autocast):
                if head:
                    y = O.attentive_classifier(S_, x.to(dtype), H, cb)
                else:
                    y = O.attentive_pooler(S_, x.to(dtype), H, cb, pre="")
        finally:
            O.FUSED = fused
        out["y"] = y.detach()
        if head:
            return Fn.cross_entropy(y.float() if autocast else y, labels)
        return (y.to(dtype) * dy.to(dtype)).sum()

    grads = lambda: {k: v.grad for k, v in S_.items()}
    if not autocast:                     # fp64: no scaling
        run().backward()
        return out["y"], {k: None if v is None else v.double() for k, v in grads().items()}
    g = _scaled_backward(run, head, grads)
    return out["y"], g


def _probe_run(mod, x, head, dy, labels, fp16):
    """The probe's forward and backward (fp16 under autocast, else bf16) with the loss scaled by LOSS_SCALE, as
    GradScaler does, and the gradients divided back in fp64."""
    out = {}

    def run():
        mod.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=F16, enabled=fp16):
            y = mod(x)
        out["y"] = y.detach()
        return Fn.cross_entropy(y, labels) if head else (y.float() * dy).sum()

    g = _scaled_backward(run, head, lambda: {n: p.grad for n, p in mod.named_parameters()})
    return out["y"], g


PROBE_CASES = [  # D, H, S, B, nq, complete_block, head
    (1024, 16, 1568, 4, 1, True, True),
    (1280, 16, 4608, 1, 1, True, True),
    (1024, 16, 12544, 2, 1, True, True),
    (1280, 16, 1568, 3, 1, False, True),
    (1024, 16, 12544, 2, 3, True, False),
    (1280, 16, 4608, 2, 3, False, False),
]


@pytest.mark.parametrize("D,H,S,B,nq,cb,head", PROBE_CASES)
def test_probe_follows_f16_autocast_vs_oracle(dev, D, H, S, B, nq, cb, head):
    """Output dtypes of the reference's modules under fp16 autocast; the logits / pooled tokens and every parameter
    gradient (backward of a GradScaler-scaled loss) within rel-L2 4e-3 of fp64, at most half the bf16 probe's distance,
    and at most 2x (+ 1e-4) the distance of the oracle run eagerly under fp16 autocast.  One exemption from the half-bf16
    rule: the classifier bias, whose gradient sums the fp16 logits' gradient where the bf16 probe has fp32 logits.  Run
    with -s for every distance."""
    from jepa_b200.pooler import AttentiveClassifier, AttentivePooler
    if head:
        mod = AttentiveClassifier(embed_dim=D, num_heads=H, depth=1, num_classes=400, complete_block=cb,
                                  follow_autocast=True)
    else:
        mod = AttentivePooler(num_queries=nq, embed_dim=D, num_heads=H, depth=1, complete_block=cb, follow_autocast=True)
    _sharpen(mod, D + S + nq)
    sd = {k: v.clone() for k, v in mod.state_dict().items()}
    assert "follow_autocast" not in str(list(sd))
    mod = mod.to(dev).train()
    g = torch.Generator().manual_seed(S + B)
    x = torch.randn(B, S, D, generator=g).to(dev)
    labels = torch.randint(0, 400, (B,), generator=g).to(dev)
    dy = torch.randn(B, nq, D, generator=g).to(dev)
    y16, g16 = _probe_run(mod, x, head, dy, labels, fp16=True)
    want = F16 if head or not cb else F32
    assert y16.dtype == want, (y16.dtype, want)
    y16 = y16.float()
    ybf, gbf = _probe_run(mod, x, head, dy, labels, fp16=False)
    assert ybf.dtype == F32
    S64 = {k: v.to(dev) for k, v in sd.items()}
    y64, g64 = _oracle_run(S64, x, H, cb, head, dy, labels)
    yac, gac = _oracle_run(S64, x, H, cb, head, dy, labels, dtype=F32, autocast=True)
    y64 = y64.view_as(y16)

    rows = {"output": (y16, ybf.view_as(y16), yac.float(), y64)}
    for n, ref in g64.items():
        if ref is None or ".proj." in n:
            assert g16[n] is None, n
            continue
        rows[n] = (g16[n], gbf[n], gac[n], ref)
    bad = []
    for n, (a16, abf, aac, a64) in rows.items():
        e16, ebf, eac = rel_l2(a16.double(), a64), rel_l2(abf.double(), a64), rel_l2(aac.double().view_as(a64), a64)
        assert all(math.isfinite(e) for e in (e16, ebf, eac)), (n, e16, ebf, eac)
        print(f"\nprobe {D} {S} nq {nq} cb {int(cb)} {n}: rel-L2 fp16 {e16:.3g} bf16 {ebf:.3g} eager-autocast {eac:.3g}")
        WORST["probe rel-L2 fp16 / eager-autocast"] = max(WORST.get("probe rel-L2 fp16 / eager-autocast", 0.0),
                                                          e16 / (eac + 1e-30))
        if e16 > 4e-3 or e16 > 2 * eac + 1e-4 or (n != "linear.bias" and e16 > 0.5 * ebf):
            bad.append((n, e16, ebf, eac))
    assert not bad, bad


def test_fp16_tokens_train_like_fp32_tokens(dev):
    """fp16 encoder tokens into a probe that trains under fp16 autocast: read as fp32 (exact), so the LayerNorm backward
    gets the fp32 x its fp16 dy pairs with; logits are bitwise those of the same values given in fp32, gradients equal up
    to the order of the atomic partial sums."""
    from jepa_b200.pooler import AttentiveClassifier
    torch.manual_seed(0)
    clf = AttentiveClassifier(embed_dim=192, num_heads=3, depth=1, num_classes=5, follow_autocast=True).to(dev)
    x16 = torch.randn(4, 300, 192, device=dev).to(F16)
    labels = torch.arange(4, device=dev)
    out = {}
    for name, x in (("f16", x16), ("f32", x16.float())):
        y, grads = _probe_run(clf, x, True, None, labels, fp16=True)
        out[name] = (y, grads)
    assert out["f16"][0].dtype == F16 and torch.equal(out["f16"][0], out["f32"][0])
    for n, g in out["f16"][1].items():      # bias / LayerNorm affine sums add partials atomically: fp32-rounding close
        assert (g is None and out["f32"][1][n] is None) or rel_l2(g, out["f32"][1][n]) <= 1e-6, n


def test_follow_autocast_off_and_bf16_autocast_unchanged(dev):
    """follow_autocast=False inside fp16 autocast, and follow_autocast=True outside autocast or under bf16 autocast,
    compute bitwise what the default probe computes."""
    from jepa_b200.pooler import AttentiveClassifier
    torch.manual_seed(0)
    a = AttentiveClassifier(embed_dim=192, num_heads=3, depth=1, num_classes=5).to(dev).eval()
    b = AttentiveClassifier(embed_dim=192, num_heads=3, depth=1, num_classes=5, follow_autocast=True).to(dev).eval()
    b.load_state_dict(a.state_dict())
    x = torch.randn(4, 300, 192, device=dev)
    with torch.no_grad():
        ref = a(x)
        with torch.autocast("cuda", dtype=F16):
            off = a(x)
        on_plain = b(x)
        with torch.autocast("cuda", dtype=BF16):
            on_bf = b(x)
        with torch.autocast("cuda", dtype=F16):
            on_half = b(x)
    assert ref.dtype == F32 and torch.equal(ref, off) and torch.equal(ref, on_plain) and torch.equal(ref, on_bf)
    assert on_half.dtype == F16 and not torch.equal(on_half.float(), ref)


# ------------------------------------------------------------------------------------------- GradScaler, loop body
def _loop_setup(dev):
    from jepa_b200.models import vit_tiny
    from jepa_b200.pooler import AttentiveClassifier
    torch.manual_seed(0)
    enc = vit_tiny(img_size=64, num_frames=4).to(dev).eval()
    clf = AttentiveClassifier(embed_dim=192, num_heads=3, depth=1, num_classes=4, follow_autocast=True).to(dev)
    g = torch.Generator().manual_seed(1)
    labels = torch.arange(4, device=dev).repeat(2)
    clips = torch.randn(8, 3, 4, 64, 64, generator=g).to(dev) + labels.view(-1, 1, 1, 1, 1).float()
    return enc, clf, clips, labels


def _loop_step(enc, clf, clips, labels, opt, scaler):
    """The reference's loop body (evals/video_classification_frozen/eval.py:323-372)."""
    with torch.cuda.amp.autocast(dtype=torch.float16):
        with torch.no_grad():
            feats = enc(clips)
        out = clf(feats)
    out.retain_grad()
    loss = Fn.cross_entropy(out, labels)
    opt.zero_grad()
    scaler.scale(loss).backward()
    scaler.step(opt)
    scaler.update()
    return out, loss


def test_grad_scaler_trains_the_fp16_probe(dev):
    enc, clf, clips, labels = _loop_setup(dev)
    opt = torch.optim.AdamW(clf.parameters(), lr=1e-3)
    scaler = torch.cuda.amp.GradScaler()
    losses = []
    for _ in range(30):
        out, loss = _loop_step(enc, clf, clips, labels, opt, scaler)
        assert out.dtype == F16 and loss.dtype == F16
        losses.append(float(loss))
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0]
    assert all(torch.isfinite(p).all() for p in clf.parameters())


def test_grad_scaler_skips_a_step_whose_fp16_activation_gradient_overflows(dev):
    """Large classifier weights turn a finite fp16 logit gradient into an fp16 pooled-token gradient past 65504 (+-inf in
    the fp16 copy the MLP backward reads): the fp32 weight gradients become non-finite, GradScaler skips the step -
    parameters and Adam moments bitwise unchanged - and halves the scale."""
    enc, clf, clips, labels = _loop_setup(dev)
    opt = torch.optim.AdamW(clf.parameters(), lr=1e-3)
    scaler = torch.cuda.amp.GradScaler(init_scale=1.0)
    for _ in range(3):
        _loop_step(enc, clf, clips, labels, opt, scaler)
    with torch.no_grad():
        clf.linear.weight.mul_(0.0).add_(torch.randn_like(clf.linear.weight) * 64.0)
    scaler.update(new_scale=2.0 ** 15)         # 2^16 would already overflow the fp16 loss's own gradient
    params = [p.detach().clone() for p in clf.parameters()]
    moments = {id(p): {k: v.clone() for k, v in opt.state[p].items()} for p in clf.parameters() if p in opt.state}
    out, _ = _loop_step(enc, clf, clips, labels, opt, scaler)
    assert torch.isfinite(out).all() and torch.isfinite(out.grad).all(), "the logits' own gradient must stay finite"
    assert float(out.grad.abs().max()) > 1000.0
    assert scaler.get_scale() == 2.0 ** 14
    for p, before in zip(clf.parameters(), params):
        assert torch.equal(p.detach(), before)
    for p in clf.parameters():
        if id(p) in moments:
            for k, v in moments[id(p)].items():
                assert torch.equal(opt.state[p][k], v), k


# ------------------------------------------------------------------------------------------------------ end to end
N_ITEMS = 320


@pytest.fixture(scope="module")
def pretrained(dev, tmp_path_factory):
    from app.scaffold import main as app_main
    from test_gpu_train_entry import _cfg as pretrain_cfg
    folder = tmp_path_factory.mktemp("pretrain16")
    app_main("vjepa", pretrain_cfg(folder, epochs=1, load=False))
    return folder


def _eval_cfg(folder, tag, attend, epochs=2):
    from test_eval_cpu import _video_cfg
    cfg = _video_cfg(folder, "synthetic")
    cfg["tag"] = tag
    cfg["data"].update(num_classes=3, synthetic_length=N_ITEMS)
    cfg["optimization"].update(batch_size=8, num_epochs=epochs, attend_across_segments=attend, lr=5e-3, start_lr=5e-3,
                               final_lr=1e-3, warmup=0., fp16_autocast=True, use_bfloat16=True)
    return cfg


def _rows(folder, eval_name, tag, epochs):
    import csv
    out = os.path.join(folder, eval_name, tag)
    with open(os.path.join(out, "jepa_r0.csv")) as f:
        rows = [r for r in csv.reader(f)]
    assert rows[0] == ["epoch", "loss", "acc"]
    ck = torch.load(os.path.join(out, "jepa-latest.pth.tar"), map_location="cpu")
    assert set(ck) == {"classifier", "opt", "scaler", "epoch", "batch_size", "world_size", "lr"}
    assert ck["epoch"] == epochs and ck["scaler"] is not None
    assert all(k.startswith("module.") for k in ck["classifier"]) and "module.linear.weight" in ck["classifier"]
    return [r for r in rows[1:] if r and r[0] != "epoch"]      # a resumed run writes the header again


class _LogitDtypes:
    """Records the dtype of every AttentiveClassifier output while installed."""

    def __enter__(self):
        from jepa_b200.pooler import AttentiveClassifier
        self.seen, self._orig = set(), AttentiveClassifier.forward
        rec = self

        def fwd(mod, x):
            y = rec._orig(mod, x)
            rec.seen.add(y.dtype)
            return y
        AttentiveClassifier.forward = fwd
        return self

    def __exit__(self, *exc):
        from jepa_b200.pooler import AttentiveClassifier
        AttentiveClassifier.forward = self._orig


@pytest.mark.parametrize("attend", [False, True])
def test_video_eval_fp16_autocast_end_to_end(pretrained, attend):
    from evals.scaffold import main as eval_main
    tag = f"fp16_attend{int(attend)}"
    with _LogitDtypes() as rec:
        eval_main("video_classification_frozen", _eval_cfg(pretrained, tag, attend))
    assert rec.seen == {F16}
    body = _rows(pretrained, "video_classification_frozen", tag, 2)
    assert [r[0] for r in body] == ["1", "2"] and float(body[-1][1]) == 100.0, body
    if attend:
        return
    cfg = _eval_cfg(pretrained, tag, attend, epochs=3)
    cfg["resume_checkpoint"] = True
    eval_main("video_classification_frozen", cfg)
    body = _rows(pretrained, "video_classification_frozen", tag, 3)
    assert [r[0] for r in body] == ["1", "2", "3"]


def test_image_eval_fp16_autocast_end_to_end(pretrained):
    from evals.scaffold import main as eval_main
    cfg = _eval_cfg(pretrained, "fp16_img", False)
    cfg["eval_name"] = "image_classification_frozen"
    cfg["data"] = dict(dataset_name="synthetic", num_classes=3, resolution=224, synthetic_length=N_ITEMS)
    with _LogitDtypes() as rec:
        eval_main("image_classification_frozen", cfg)
    assert rec.seen == {F16}
    body = _rows(pretrained, "image_classification_frozen", "fp16_img", 2)
    assert float(body[-1][1]) == 100.0, body
