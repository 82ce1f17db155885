"""The attentive probe at ViT-g / ViT-G head dims (-m gpu): vj_cross_attn_fwd / _fwd_lse / _bwd at hd 88 and 104 (11 and
13 lanes per key) in bf16 and fp16 against fp64, and AttentiveClassifier at D 1408 / 1664 (16 heads) trained for a few
steps next to an eager fp32 restatement of the reference's modules."""
import pytest
import torch
import torch.nn.functional as Fn

import xattn16_ref as X
from parity_util import TOL_ACT, TOL_GRAD, TOL_LOSS, rel_l2

pytestmark = pytest.mark.gpu
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
# the bf16 kernels' bounds (tests/native/test_xattn.cu, every head dim): (atol, rtol) of out, lse2, dq and dkv
BF16_TOL = {"out": (1e-2, 5e-3), "lse2": (1e-4, 1e-5), "dq": (1e-2, 5e-3), "dkv": (1e-2, 5e-3)}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


def _run(dev, c, dt):
    """The dt kernels on case c of xattn16_ref: (q, kv, dout, out, lse2, dq, dkv) of all three clips."""
    from jepa_b200 import kernels as Kn
    B, nq, S, H, hd, scale = (c[k] for k in ("B", "nq", "S", "H", "hd", "scale"))
    q, kv, dout = (c[k].to(dt).to(dev) for k in ("q", "kv", "dout"))
    out = torch.full((B * nq, H * hd), float("nan"), dtype=dt, device=dev)
    out2 = torch.full_like(out, float("nan"))
    lse = torch.full((B * nq, H), float("nan"), device=dev)
    Kn.cross_attn_fwd(q, kv, out, B, nq, S, H, hd, scale)
    Kn.cross_attn_fwd_lse(q, kv, out2, lse, B, nq, S, H, hd, scale)
    assert torch.equal(out, out2)
    dq = torch.full((B * nq, H * hd), float("nan"), device=dev)
    dkv = torch.full((B * S, 2 * H * hd), float("nan"), dtype=dt, device=dev)
    Kn.cross_attn_bwd(q, kv, out, dout, lse, dq, dkv, B, nq, S, H, hd, scale)
    dq2, dkv2 = torch.empty_like(dq), torch.empty_like(dkv)
    Kn.cross_attn_bwd(q, kv, out, dout, lse, dq2, dkv2, B, nq, S, H, hd, scale)
    assert torch.equal(dq, dq2) and torch.equal(dkv, dkv2), "backward is not bitwise reproducible"
    return q, kv, dout, out, lse, dq, dkv


def _case(dev, hd, nq, S, dt):
    c = X.make_case(hd, nq, S, seed=hd * 100 + nq * 10000 + S)
    q, kv, dout, out, lse, dq, dkv = _run(dev, c, dt)
    ck = lambda t, n: X.checked(c, t, n)
    got = (ck(out, nq), ck(lse, nq), ck(dq, nq), ck(dkv, S))
    ref = X.reference(c, q, kv, dout, got[0])
    if dt == F16:
        res = X.check(c, *got, ref)
    else:
        res = {k: X.worst(g, r, *BF16_TOL[k]) for k, g, r in zip(("out", "lse2", "dq", "dkv"), got, ref)}
    for k, v in res.items():
        assert v <= 1.0, (k, hd, nq, S, dt, v)
    assert torch.isfinite(out).all() and torch.isfinite(dq).all()


@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("hd", [88, 104])
def test_cross_attn_new_head_dims_vs_fp64(dev, hd, dt):
    """S = 1 ... 3 backward key chunks (every residue of the 2 keys per warp and of the 32-key chunk), and the encoders'
    token counts (ViT-g/16: 1568, ViT-G/14: 2048 per 16-frame clip, 8 x 1568 for K400's 8 segments)."""
    chunk = X.key_chunk(hd)
    assert chunk == 32
    for nq in (1, 3):
        for S in list(range(1, 3 * chunk + 2)) + [1568, 2048, 12544]:
            _case(dev, hd, nq, S, dt)


def test_cross_attn_rejects_other_head_dims(dev):
    from jepa_b200 import _lib, kernels as Kn
    for hd in (72, 96, 112):
        q = torch.zeros(1, hd, dtype=BF16, device=dev)
        with pytest.raises(_lib.VJError, match="88 / 104"):
            Kn.cross_attn_fwd(q, torch.zeros(4, 2 * hd, dtype=BF16, device=dev), torch.empty_like(q), 1, 1, 4, 1, hd, 0.1)
    from jepa_b200.pooler import AttentivePooler
    with pytest.raises(NotImplementedError, match="88 / 104"):
        AttentivePooler(embed_dim=16 * 96, num_heads=16)


def _eager_logits(S, x, H):
    from oracle import vjepa_oracle as O
    return O.attentive_classifier(S, x, H)


@pytest.mark.parametrize("fp16", [False, True], ids=["bf16", "fp16"])
@pytest.mark.parametrize("D,S", [(1408, 1568), (1664, 2048)], ids=["vitg16", "vitG14"])
def test_classifier_trains_next_to_eager_fp32(dev, D, S, fp16):
    """Three SGD steps of AttentiveClassifier (16 heads of 88 / 104, 400 classes) on the kernels - bf16, or fp16 under
    autocast with follow_autocast=True and a GradScaler-style loss scale - and of the eager fp32 restatement from the
    same weights on the same batches: the loss, logits and every gradient at every step within the bf16 parity bounds
    (TOL_LOSS relative / TOL_ACT / TOL_GRAD), and the total update of every trained parameter within TOL_GRAD."""
    from jepa_b200.pooler import AttentiveClassifier
    from test_gpu_probe_fp16 import _scaled_backward, _sharpen
    H, B, C, lr = 16, 2, 400, 2e-3
    clf = _sharpen(AttentiveClassifier(embed_dim=D, num_heads=H, depth=1, num_classes=C, follow_autocast=fp16), D + S)
    S32 = {k: v.clone().to(dev).requires_grad_(True) for k, v in clf.state_dict().items()}
    start = {k: v.detach().clone() for k, v in S32.items()}
    clf = clf.to(dev).train()
    params = dict(clf.named_parameters())
    assert set(params) == set(S32)
    g = torch.Generator().manual_seed(S)
    for step in range(3):
        x = torch.randn(B, S, D, generator=g).to(torch.bfloat16).float().to(dev)
        labels = torch.randint(0, C, (B,), generator=g).to(dev)
        out = {}

        def run():
            clf.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=F16, enabled=fp16):
                out["y"] = clf(x)
            return Fn.cross_entropy(out["y"].float(), labels)
        grads = _scaled_backward(run, True, lambda: {n: p.grad for n, p in params.items()})
        loss = float(Fn.cross_entropy(out["y"].detach().float(), labels))
        assert out["y"].dtype == (F16 if fp16 else F32)

        y_ref = _eager_logits(S32, x, H)
        loss_ref = Fn.cross_entropy(y_ref, labels)
        ref = torch.autograd.grad(loss_ref, list(S32.values()), allow_unused=True)
        # TOL_LOSS is stated for losses near 1; a 400-class loss of sharpened logits is about 5
        assert abs(loss - float(loss_ref)) < TOL_LOSS * max(1.0, float(loss_ref)), (step, loss, float(loss_ref))
        assert rel_l2(out["y"].detach().float(), y_ref.detach()) < TOL_ACT, step
        with torch.no_grad():
            for (n, p), r in zip(S32.items(), ref):
                if r is None:       # attn.proj: CrossAttention.forward never applies it
                    assert grads[n] is None and ".proj." in n, n
                    continue
                assert rel_l2(grads[n].float(), r) < TOL_GRAD, (step, n, rel_l2(grads[n].float(), r))
                p.sub_(lr * r)
                params[n].sub_(lr * grads[n].float())
    for n, p in S32.items():
        if ".proj." in n:
            continue
        e = rel_l2(params[n].detach() - start[n], p.detach() - start[n])
        print(f"\nD {D} fp16 {fp16} {n}: update rel-L2 {e:.3g}")
        assert e < TOL_GRAD, (n, e)
