"""GPU parity tests (-m gpu): the CUDA product path, called through the C ABI, against the CPU oracle on
identical seeded inputs; against the committed reference-generated golden fixtures; and, at full
BASELINE sizes, through size-independent properties.

Stated tolerances (bf16 operands / fp32 accumulation vs the fp32 oracle):
  single kernel outputs stored as bf16 : |err| <= 2e-2 + 1e-2 |ref|      (one bf16 rounding + accumulation order)
  fp32-output kernels (LN stats, loss, wgrad, EMA, AdamW) : rel 1e-4 .. bit-exact where stated
  whole-network activations rel-L2 <= 3e-2, per-parameter gradients rel-L2 <= 6e-2, loss abs 5e-3
  index / gather paths: bit-exact (torch.equal)
"""
import os
import subprocess

import pytest
import torch

from common import synth_clips
from parity_util import (TOL_ACT, VITG_2B, VITH_2B, VITL_2B, c1_masks, compare_step, rel_l2, run_c1_step_cuda, run_c1_step_oracle)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()  # fail loudly if the extension is missing - there is no fallback
    return torch.device("cuda:0")


def bf(t):
    return t.to(torch.bfloat16).float()


def close_bf16(got, ref, atol=2e-2, rtol=1e-2):
    err = (got.float().cpu() - ref.float()).abs()
    bound = atol + rtol * ref.float().abs()
    assert bool((err <= bound).all()), f"max err {float(err.max()):.4g}, worst excess {float((err - bound).max()):.4g}"


# --------------------------------------------------------------------------------------------- native
@pytest.mark.parametrize("binary", ["test_gemm", "test_attn"])
def test_native_bringup_binaries(dev, binary):
    exe = os.path.join(ROOT, "tests", "native", binary)
    assert os.path.exists(exe), "run __graft_entry__.build() first"
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "ALL PASSED" in out.stdout, out.stdout[-3000:] + out.stderr[-1000:]


# --------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K", [(200, 192, 192), (333, 384, 1536), (1000, 1024, 256)])
def test_linear_forward_epilogues(dev, M, N, K):
    from jepa_b200 import kernels as Kn
    from oracle import vjepa_oracle as O
    g = torch.Generator().manual_seed(M + N)
    x, w = bf(torch.randn(M, K, generator=g)), bf(torch.randn(N, K, generator=g) * 0.05)
    b = torch.randn(N, generator=g) * 0.1
    res = bf(torch.randn(M, N, generator=g))
    xd, wd, bd, resd = x.to(dev, torch.bfloat16), w.to(dev, torch.bfloat16), b.to(dev), res.to(dev, torch.bfloat16)
    ref = O.linear(x, w, b)
    out = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
    close_bf16(Kn.gemm(xd, wd, out, bias=bd), ref)
    pre = torch.empty_like(out)
    close_bf16(Kn.gemm(xd, wd, out, bias=bd, epi=Kn.EPI_GELU, aux_out=pre), O.gelu(ref))
    close_bf16(pre, ref)
    close_bf16(Kn.gemm(xd, wd, out, bias=bd, epi=Kn.EPI_ADD, aux=resd), ref + res)
    out32 = torch.empty(M, N, dtype=torch.float32, device=dev)
    Kn.gemm(xd, wd, out32, bias=bd, epi=Kn.EPI_ADD, aux=res.to(dev))
    assert rel_l2(out32.cpu(), ref + res) < 1e-5


def test_linear_backward_gemms(dev):
    """dgrad (MN-major B), fused dGELU, wgrad (both operands MN-major, split-K reduce-add) vs fp64 autograd."""
    from jepa_b200 import kernels as Kn
    from oracle import vjepa_oracle as O
    T, Din, Dout = 520, 192, 768
    g = torch.Generator().manual_seed(5)
    x, w = bf(torch.randn(T, Din, generator=g)), bf(torch.randn(Dout, Din, generator=g) * 0.05)
    dy, hpre = bf(torch.randn(T, Dout, generator=g)), bf(torch.randn(T, Dout, generator=g))
    xd, wd, dyd, hd_ = (t.to(dev, torch.bfloat16) for t in (x, w, dy, hpre))
    dx = torch.empty(T, Din, dtype=torch.bfloat16, device=dev)
    close_bf16(Kn.gemm(dyd, wd, dx, b_mn=True), dy @ w, atol=5e-2)
    # dGELU epilogue: (dz @ W2) * gelu'(h) where W2 [Din, Dout] maps hidden(Dout) -> Din
    w2 = bf(torch.randn(Din, Dout, generator=g) * 0.05)
    dz = bf(torch.randn(T, Din, generator=g))
    hh = hpre.double().requires_grad_(True)
    O.gelu(hh).backward((dz @ w2).double())
    dh = torch.empty(T, Dout, dtype=torch.bfloat16, device=dev)
    close_bf16(Kn.gemm(dz.to(dev, torch.bfloat16), w2.to(dev, torch.bfloat16), dh, b_mn=True, epi=Kn.EPI_DGELU, aux=hd_),
               hh.grad.float(), atol=3e-2)
    # wgrad accumulates into fp32
    dw0 = torch.randn(Dout, Din, generator=g)
    dw = dw0.clone().to(dev)
    Kn.gemm(dyd, xd, dw, a_mn=True, b_mn=True, accumulate=True, split_k=3)
    assert rel_l2(dw.cpu(), dw0 + dy.t() @ x) < 1e-5
    db = torch.zeros(Dout, device=dev)
    Kn.colsum(dyd, db)
    assert rel_l2(db.cpu(), dy.sum(0)) < 1e-5


# --------------------------------------------------------------------------------------------- rows
@pytest.mark.parametrize("D", [192, 384, 768, 1024, 1280, 1408, 2048])
def test_layernorm_fwd_bwd(dev, D):
    from jepa_b200 import kernels as Kn
    from oracle import vjepa_oracle as O
    T = 777
    g = torch.Generator().manual_seed(D)
    x = bf(torch.randn(T, D, generator=g) * 2 + 0.5)
    w, b = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    dy, dres = bf(torch.randn(T, D, generator=g)), bf(torch.randn(T, D, generator=g))
    xr = x.double().requires_grad_(True)
    wr, br = w.double().requires_grad_(True), b.double().requires_grad_(True)
    y = O.layer_norm(xr, wr, br, 1e-6)
    y.backward(dy.double())
    xd = x.to(dev, torch.bfloat16)
    yd = torch.empty_like(xd)
    mean, rstd = torch.empty(T, device=dev), torch.empty(T, device=dev)
    Kn.layernorm_fwd(xd, yd, w.to(dev), b.to(dev), 1e-6, mean, rstd)
    close_bf16(yd, y.detach().float())
    assert rel_l2(mean.cpu(), x.mean(-1)) < 1e-5
    dx = torch.empty_like(xd)
    dg, db = torch.zeros(D, device=dev), torch.zeros(D, device=dev)
    Kn.layernorm_bwd(dy.to(dev, torch.bfloat16), xd, w.to(dev), mean, rstd, dres.to(dev, torch.bfloat16), dx, dg, db)
    close_bf16(dx, (xr.grad + dres.double()).float(), atol=3e-2)
    assert rel_l2(dg.cpu(), wr.grad.float()) < 1e-4 and rel_l2(db.cpu(), br.grad.float()) < 1e-4
    # fp32 in / fp32 out variant
    y32 = torch.empty(T, D, device=dev)
    Kn.layernorm_fwd(x.to(dev), y32, w.to(dev), b.to(dev), 1e-6)
    assert rel_l2(y32.cpu(), y.detach().float()) < 1e-5


def test_gather_paths_bit_exact(dev):
    from jepa_b200 import kernels as Kn
    from src.masks.utils import apply_masks
    from oracle import vjepa_oracle as O
    B, N, D = 3, 784, 192
    me, mp = c1_masks(2)
    idx = torch.cat([me[0], me[0][:1].flip(1)], 0)  # also a descending row
    for dt in (torch.float32, torch.bfloat16):
        x = torch.randn(B, N, D).to(dt)
        ref = O.apply_masks(x, [idx])
        got = Kn.gather_rows(x.to(dev), idx.to(dev))
        assert torch.equal(got.cpu(), ref)
        assert torch.equal(apply_masks(x.to(dev), [idx.to(dev)]).cpu(), ref)
    # empty / ragged: K = 0 rows is a no-op that returns an empty tensor
    assert Kn.gather_rows(x.to(dev), torch.zeros(B, 0, dtype=torch.int64, device=dev)).shape == (B, 0, D)
    # scatter-add is the exact adjoint on unique indices
    dy = torch.randn(B, idx.shape[1], D)
    dx = torch.zeros(B, N, D, device=dev)
    Kn.scatter_rows_add(dy.to(dev), dx, idx.to(dev))
    ref = torch.zeros(B, N, D)
    ref.scatter_add_(1, idx.unsqueeze(-1).expand(-1, -1, D), dy)
    assert torch.equal(dx.cpu(), ref)


def test_patch_embed_matches_oracle(dev):
    from jepa_b200 import kernels as Kn
    from oracle import vjepa_oracle as O
    B, T, H = 2, 8, 224
    D, P = 192, 1536
    g = torch.Generator().manual_seed(1)
    clips = synth_clips(B, T, H, H, seed=3)
    w = bf(torch.randn(D, 3, 2, 16, 16, generator=g) * 0.03)
    b = torch.randn(D, generator=g) * 0.02
    pos = torch.randn(784, D, generator=g)
    me, _ = c1_masks(B)
    ref_all = O.patch_embed_3d(bf(clips), w, b) + pos
    patches = torch.empty(B * 784, P, dtype=torch.bfloat16, device=dev)
    Kn.im2col_tubelets(clips.to(dev), patches, None, 2, 16)
    out = torch.empty(B * 784, D, dtype=torch.bfloat16, device=dev)
    Kn.gemm(patches, w.reshape(D, P).to(dev, torch.bfloat16), out, bias=b.to(dev), epi=Kn.EPI_ADD, aux=pos.to(dev), aux_period=784)
    close_bf16(out.view(B, 784, D), ref_all, atol=3e-2)
    # gather-first context path: identical rows to embedding everything and gathering afterwards
    m = me[0].to(dev)
    Kk = m.shape[1]
    pk = torch.empty(B * Kk, P, dtype=torch.bfloat16, device=dev)
    Kn.im2col_tubelets(clips.to(dev), pk, m, 2, 16)
    assert torch.equal(pk.view(B, Kk, P), Kn.gather_rows(patches.view(B, 784, P), m))
    outk = torch.empty(B * Kk, D, dtype=torch.bfloat16, device=dev)
    Kn.gemm(pk, w.reshape(D, P).to(dev, torch.bfloat16), outk, bias=b.to(dev), epi=Kn.EPI_ADD, aux=pos.to(dev),
            aux_rowmap=m.reshape(-1).to(torch.int32))
    assert torch.equal(outk.view(B, Kk, D), Kn.gather_rows(out.view(B, 784, D), m))


def _attention_case(dev, H, hd, lens, late_max=False, backward=True, seed=None):
    """Attention (modules.py:61-78 core) vs an fp64 softmax on the host, incl. the zero-padded heads (predictor hd=24 ->
    32, ViT-H hd=80 -> 128) and ragged sequence tails.  late_max: a few keys far into the sequence (past KV tile 8) score
    ~2^6..2^12 times above everything before them for some query rows, so the running max of those rows, and with it
    the rescale of the forward's accumulator, moves late and more than once."""
    from attention_ref import plant_late_keys
    from jepa_b200 import kernels as Kn
    from jepa_b200.params import padded_head_dim
    hdp = padded_head_dim(hd)
    T = sum(lens)
    g = torch.Generator().manual_seed(hd if seed is None else seed)
    q, k, v, do = (bf(torch.randn(T, H, hd, generator=g)) for _ in range(4))
    if late_max:
        off = 0
        for L in lens:
            plant_late_keys(q[off:off + L], k[off:off + L])
            off += L
    qkv = torch.zeros(T, 3, H, hdp)
    qkv[:, 0, :, :hd], qkv[:, 1, :, :hd], qkv[:, 2, :, :hd] = q, k, v
    dop = torch.zeros(T, H, hdp)
    dop[..., :hd] = do
    cu = torch.tensor([0] + [sum(lens[:i + 1]) for i in range(len(lens))], dtype=torch.int32, device=dev)
    qkv_d = qkv.reshape(T, 3 * H * hdp).to(dev, torch.bfloat16)
    out = torch.empty(T, H * hdp, dtype=torch.bfloat16, device=dev)
    lse = torch.empty(H, T, device=dev)
    scale = hd ** -0.5
    Kn.attn_fwd(qkv_d, out, lse, cu, len(lens), max(lens), H, hdp, scale)
    out_c = out.float().cpu().view(T, H, hdp)
    dq_c = None
    if backward:
        dqkv, dq2 = torch.empty_like(qkv_d), torch.empty_like(qkv_d)
        for dst in (dqkv, dq2):   # deterministic: no atomics, so a second run is bitwise the same
            Kn.attn_bwd(qkv_d, out, dop.reshape(T, H * hdp).to(dev, torch.bfloat16), lse, torch.empty(H * T, device=dev),
                        dst, cu, len(lens), max(lens), H, hdp, scale)
        assert torch.equal(dqkv, dq2), "attention backward is not bitwise reproducible"
        dq_c = dqkv.float().cpu().view(T, 3, H, hdp)
    if hdp > hd:  # padded lanes stay exactly zero end to end
        assert float(out_c[..., hd:].abs().max()) == 0
        assert dq_c is None or float(dq_c[..., hd:].abs().max()) == 0
    lse_c = lse.cpu()
    off = 0
    for L in lens:
        qq, kk, vv = (t[off:off + L].double().transpose(0, 1).requires_grad_(backward) for t in (q, k, v))  # [H, L, hd]
        sc = (qq @ kk.transpose(-2, -1)) * scale
        att = torch.softmax(sc, dim=-1)
        o = att @ vv
        close_bf16(out_c[off:off + L, :, :hd], o.detach().transpose(0, 1).float())
        # log2-domain LSE saved for the backward
        ref_lse2 = torch.logsumexp(sc.detach(), dim=-1) * 1.4426950408889634
        assert float((lse_c[:, off:off + L].double() - ref_lse2).abs().max()) < 2e-2
        if backward:
            o.backward(do[off:off + L].double().transpose(0, 1))
            for i, t in enumerate((qq, kk, vv)):
                ref_g = t.grad.transpose(0, 1).float()
                # late_max plants keys whose probability is ~1 for ~L/7 query rows: their dK / dV rows are sums of
                # hundreds of O(1) terms, each carrying the bf16 rounding of P and dS (2^-9 relative), so the absolute
                # error scales with the largest gradient of the tensor rather than with the element itself
                atol = 3e-2 + (2e-2 * float(ref_g.abs().max()) if late_max else 0.0)
                close_bf16(dq_c[off:off + L, i, :, :hd], ref_g, atol=atol, rtol=2e-2)
                assert rel_l2(dq_c[off:off + L, i, :, :hd], ref_g) < (2e-2 if late_max else 1e-2)   # stated gradient tolerance: 3e-2
        off += L


@pytest.mark.parametrize("H,hd,lens", [(3, 64, [208, 160]), (16, 24, [296, 40, 128]), (3, 128, [200, 72]),
                                       (4, 80, [300, 100])])
def test_attention_fwd_bwd_vs_oracle(dev, H, hd, lens):
    _attention_case(dev, H, hd, lens)


# BASELINE sequence lengths (SURVEY appendix B): target 1568 = 12x128+32 (13 KV tiles), predictor 1184 / 1192 (hd 24 ->
# 32), context 360 / 48, ViT-H hd 80 -> 128, C5 context 1512 / 288 and predictor 3680 / 3600.
@pytest.mark.parametrize("H,hd,lens,late", [
    (2, 64, [1568], False), (2, 64, [1568], True), (2, 64, [360, 48, 360], False),
    (2, 24, [1184, 1192], False), (2, 24, [1192, 1184], True),
    (2, 80, [1568], False), (1, 80, [1568, 360, 48], True), (1, 80, [1512, 288], False), (1, 24, [3680, 3600], False),
])
def test_attention_baseline_shapes_vs_fp64(dev, H, hd, lens, late):
    _attention_case(dev, H, hd, lens, late_max=late, seed=hd + len(lens) + int(late))


@pytest.mark.parametrize("late", [False, True])
def test_attention_c5_long_sequence_forward(dev, late):
    """C5 target pass: S = 4608 (36 KV tiles), hd 80 -> 128, forward only (the target encoder has no backward)."""
    _attention_case(dev, 1, 80, [4608], late_max=late, backward=False, seed=7)


def test_target_ln_gather_and_loss(dev):
    from jepa_b200 import kernels as Kn
    from jepa_b200 import step as vj
    from jepa_b200.models import _token_views
    from oracle import vjepa_oracle as O
    B, N, D = 2, 784, 192
    g = torch.Generator().manual_seed(9)
    x = bf(torch.randn(B, N, D, generator=g) * 3)
    w, b = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    _, mp = c1_masks(B)
    ref = O.apply_masks(O.layer_norm(O.layer_norm(x, w, b, 1e-6), None, None, 1e-5), mp, concat=False)
    for m, r in zip(mp, ref):
        got = Kn.target_ln_gather(x.to(dev, torch.bfloat16), m.to(dev), w.to(dev), b.to(dev), 1e-6, 1e-5)
        assert rel_l2(got.cpu(), r) < 1e-5
    # L1 loss forward/backward vs autograd
    sizes = [int(m.shape[1]) for m in mp]
    z = [bf(torch.randn(B, k, D, generator=g)) for k in sizes]
    zc = torch.cat([t.reshape(-1, D) for t in z]).to(dev, torch.bfloat16).requires_grad_(True)
    hc = torch.cat([t.reshape(-1, D) for t in ref]).to(dev)
    loss = vj.jepa_loss(_token_views(zc, B, sizes), _token_views(hc, B, sizes))
    (loss * 65536.0).backward()
    zr = [t.clone().requires_grad_(True) for t in z]
    lref = O.loss_fn(zr, ref)
    (lref * 65536.0).backward()
    assert abs(float(loss) - float(lref)) < 1e-5
    close_bf16(zc.grad, torch.cat([t.grad.reshape(-1, D) for t in zr]), atol=1e-6, rtol=1e-2)
    assert abs(float(vj.reg_loss([t.to(dev, torch.bfloat16) for t in z])) - float(O.reg_fn(z))) < 1e-4


@pytest.mark.parametrize("loss_exp,reg_coeff", [(2.0, 0.0), (1.5, 0.0), (1.0, 0.7), (2.0, 0.3)])
def test_loss_exponent_and_variance_regulariser_gradients(dev, loss_exp, reg_coeff):
    """loss_fn with loss_exp != 1 and the reg_fn term with reg_coeff != 0 (app/vjepa/train.py:440-449,456-459): value and
    d loss / d z of the hand-written kernels vs autograd over the oracle's restatement."""
    from jepa_b200 import step as vj
    from jepa_b200.models import _token_views
    from oracle import vjepa_oracle as O
    B, D, sizes = 3, 192, [40, 24]
    g = torch.Generator().manual_seed(int(loss_exp * 10 + reg_coeff * 100))
    # token spread below AND above 1 so that relu(1 - pstd) is active for some (b, d) columns and inactive for others
    z = [bf(torch.randn(B, k, D, generator=g) * torch.linspace(0.3, 1.8, D)) for k in sizes]
    h = [torch.randn(B, k, D, generator=g) for k in sizes]
    zc = torch.cat([t.reshape(-1, D) for t in z]).to(dev, torch.bfloat16).requires_grad_(True)
    hc = torch.cat([t.reshape(-1, D) for t in h]).to(dev)
    zv, hv = _token_views(zc, B, sizes), _token_views(hc, B, sizes)
    loss_jepa = vj.jepa_loss(zv, hv, loss_exp)
    loss_reg = vj.reg_loss(zv, with_grad=reg_coeff != 0.0)
    loss = loss_jepa + reg_coeff * loss_reg
    (loss * 1024.0).backward()
    zr = [t.clone().requires_grad_(True) for t in z]
    lj, lr_ = O.loss_fn(zr, h, loss_exp), O.reg_fn(zr)
    ((lj + reg_coeff * lr_) * 1024.0).backward()
    assert abs(float(loss_jepa) - float(lj)) < 2e-5 * max(1.0, abs(float(lj)))
    assert abs(float(loss_reg) - float(lr_)) < 2e-5
    ref = torch.cat([t.grad.reshape(-1, D) for t in zr])
    assert float(ref.abs().max()) > 0
    assert rel_l2(zc.grad.float().cpu(), ref) < 6e-3          # dz is stored in bf16 (2^-9 per element)
    # the no-grad (logging-only) form returns the same value and leaves no graph
    with torch.no_grad():
        assert abs(float(vj.reg_loss(zv)) - float(lr_)) < 2e-5


def test_ema_bit_exact_and_adamw(dev):
    from jepa_b200 import kernels as Kn
    from jepa_b200.optim import FlatAdamW
    g = torch.Generator().manual_seed(4)
    n = 4096 * 3 + 64
    k, q = torch.randn(n, generator=g), torch.randn(n, generator=g)
    for m in (0.998, 0.99925, 1.0):
        kd = k.clone().to(dev)
        Kn.ema_update(kd, q.to(dev), m)
        ref = k.clone()
        ref.mul_(m).add_((1. - m) * q)       # the reference's op sequence, train.py:486-487
        assert torch.equal(kd.cpu(), ref), m
    # AdamW vs torch.optim.AdamW (fp32 CPU) over several steps, incl. weight decay and a skipped step
    p0, grads = torch.randn(256, 64, generator=g), [torch.randn(256, 64, generator=g) for _ in range(4)]
    pr = torch.nn.Parameter(p0.clone())
    ref_opt = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.05)
    pc = torch.nn.Parameter(p0.clone().to(dev))
    opt = FlatAdamW([pc], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.05)
    for gr in grads:
        pr.grad = gr.clone(); ref_opt.step()
        pc.grad = gr.clone().to(dev); opt.step()
    assert rel_l2(pc.detach().cpu(), pr.detach()) < 1e-6
    before = pc.detach().clone()
    opt.found_inf = torch.ones((), device=dev)
    pc.grad = grads[0].to(dev); opt.step()
    del opt.found_inf
    assert torch.equal(pc.detach(), before)


def test_cast_and_head_pad_round_trip(dev):
    from jepa_b200 import kernels as Kn
    w = torch.randn(3 * 16 * 24, 384)
    wd = w.to(dev)
    sh = torch.empty(w.numel(), dtype=torch.bfloat16, device=dev)
    Kn.cast_f32_bf16(wd.view(-1), sh)
    assert torch.equal(sh.cpu(), w.view(-1).to(torch.bfloat16))
    pad = torch.empty(3 * 16 * 32, 384, dtype=torch.bfloat16, device=dev)
    Kn.head_pad(wd, pad, 1, 48, 24, 32, 384)
    pv = pad.cpu().view(48, 32, 384)
    assert torch.equal(pv[:, :24], w.to(torch.bfloat16).view(48, 24, 384)) and float(pv[:, 24:].abs().max()) == 0
    gpad = torch.randn(3 * 16 * 32, 384)
    acc = torch.ones(3 * 16 * 24, 384, device=dev)
    Kn.head_pad(gpad.to(dev), acc, 1, 48, 24, 32, 384, unpad_add=True)
    assert torch.equal(acc.cpu(), 1 + gpad.view(48, 32, 384)[:, :24].reshape(-1, 384))
    # proj-style padding along columns
    wp = torch.randn(384, 16 * 24)
    pp = torch.empty(384, 16 * 32, dtype=torch.bfloat16, device=dev)
    Kn.head_pad(wp.to(dev), pp, 384, 16, 24, 32, 1)
    assert torch.equal(pp.cpu().view(384, 16, 32)[:, :, :24], wp.to(torch.bfloat16).view(384, 16, 24))


# --------------------------------------------------------------------------------------------- networks
def test_c1_step_shallow_vs_oracle(dev):
    """2+2 layer ViT-Tiny step: isolates wiring errors from depth-accumulated rounding."""
    got = run_c1_step_cuda(dev, batch=2, depth_limit=2)
    ref = run_c1_step_oracle(batch=2, depth_limit=2)
    compare_step(got, ref, verbose=True, tol_act=1.5e-2, tol_grad=3e-2)


def test_c1_step_full_vs_oracle_and_golden(dev, golden_dir):
    """BASELINE config[0]: ViT-Tiny/16, 2 clips, 8x224x224, multiblock3d masks, one full train step."""
    got = run_c1_step_cuda(dev)
    ref = run_c1_step_oracle()
    compare_step(got, ref, verbose=True)
    gold = torch.load(os.path.join(golden_dir, "golden_step_c1.pt"))
    assert abs(got["loss_jepa"] - gold["loss_jepa"]) < 5e-3
    for key, gkey in (("h", "h"), ("z", "z"), ("z_enc", "zenc")):
        for i, t in enumerate(got[key]):
            assert rel_l2(t[:, :4, :16], gold[f"{gkey}_slices"][i]) < 2 * TOL_ACT
            assert abs(float(t.norm()) - gold[f"{gkey}_norm"][i]) / gold[f"{gkey}_norm"][i] < TOL_ACT
    for key in ("enc", "pred"):
        for n, refn in gold[f"{key}_grad_norm"].items():
            assert abs(float(got[f"{key}_grad"][n].norm()) - refn) <= 6e-2 * refn + 1e-9, n
    for n, ref_slice in gold["ema_slices"].items():
        assert torch.equal(got["ema"][n].reshape(-1)[:32], ref_slice), n


@pytest.mark.parametrize("cfg", [VITL_2B, VITH_2B, VITG_2B], ids=["vitl16_2blocks", "vith16_2blocks", "vitg16_2blocks"])
def test_baseline_width_step_vs_oracle(dev, cfg):
    """SURVEY 8c(ii): a 2+2-block slice of the BASELINE networks at FULL width / heads / sequence lengths (ViT-L: D=1024,
    16 heads of 64; ViT-H: D=1280, 16 heads of 80 -> 128; ViT-g: D=1408, 16 heads of 88 -> 128, MLP 6144; predictor 384 / 16 heads of 24 -> 32; N=1568 target tokens,
    C2's seeded masks Ke=[360,48] Kp=[824,1144]), one clip, against the fp32 CPU oracle: target / context / predictor
    outputs, loss, every parameter gradient (BN=256 GEMM tiles, split-K wgrads at these K), EMA bit-exact."""
    got = run_c1_step_cuda(dev, cfg=cfg)
    ref = run_c1_step_oracle(cfg=cfg)
    assert [tuple(t.shape[1:]) for t in got["z"]] == [(824, cfg["embed_dim"]), (1144, cfg["embed_dim"])]
    compare_step(got, ref, verbose=True)


@pytest.mark.parametrize("T,n_out,k_in", [(13056, 4096, 1024), (76032, 1536, 384), (76032, 384, 1536), (50176 + 24, 1024, 1024)])
def test_wgrad_split_k_full_token_counts(dev, T, n_out, k_in):
    """wgrad GEMMs at the C2 token counts (context 13 056, predictor 76 032 rows; one count that is not a multiple of 64)
    with the engine's own split-K choice, fp32 reduce-add into a non-zero buffer, vs fp64 on a 256 x 256 output slice."""
    from jepa_b200 import kernels as Kn
    from jepa_b200.engine import _split_k_for
    g = torch.Generator().manual_seed(T % 997)
    dy = bf(torch.randn(T, n_out, generator=g))
    x = bf(torch.randn(T, k_in, generator=g) * 0.5)
    base = torch.randn(n_out, k_in, generator=g)
    dw = base.clone().to(dev)
    sk = _split_k_for(n_out, k_in, T)
    Kn.gemm(dy.to(dev, torch.bfloat16), x.to(dev, torch.bfloat16), dw, a_mn=True, b_mn=True, accumulate=True, split_k=sk)
    r0, c0 = n_out - 256, max(0, k_in - 256 - 64)
    ref = base[r0:r0 + 256, c0:c0 + 256].double() + dy[:, r0:r0 + 256].double().t() @ x[:, c0:c0 + 256].double()
    got = dw[r0:r0 + 256, c0:c0 + 256].cpu()
    e = rel_l2(got, ref)
    print(f"wgrad T={T} {n_out}x{k_in} split_k={sk}: rel-L2 vs fp64 {e:.3e}")
    # fp32 tensor-core accumulation over up to 76 032 products per output: summation-order noise ~ sqrt(K) * 2^-24 = 1.6e-5
    assert e < 5e-5, (sk, e)
    # stream-K decomposition of the same GEMM (split_k = -1): identical result up to summation order
    dw2 = base.clone().to(dev)
    Kn.gemm(dy.to(dev, torch.bfloat16), x.to(dev, torch.bfloat16), dw2, a_mn=True, b_mn=True, accumulate=True, split_k=-1)
    assert rel_l2(dw2[r0:r0 + 256, c0:c0 + 256].cpu(), ref) < 2e-5
    db = torch.zeros(n_out, device=dev)
    Kn.colsum(dy.to(dev, torch.bfloat16), db)
    e2 = rel_l2(db.cpu(), dy.double().sum(0))
    assert e2 < 1e-4, e2


def test_step_with_token_counts_not_multiple_of_8(dev):
    """Image-like / odd-batch settings give B*sum(K_i) % 8 != 0 (ADVICE r1): the wgrad GEMMs reduce over the token count, which
    only has to be positive.  One ViT-Tiny encoder fwd+bwd over masks keeping 21 and 13 tokens of 3 clips vs the oracle."""
    from jepa_b200.models import vit_tiny
    from oracle import vjepa_oracle as O
    torch.manual_seed(0)
    enc = vit_tiny(img_size=224, patch_size=16, num_frames=8, tubelet_size=2, uniform_power=True).to(dev)
    clips = synth_clips(3, 8, 224, 224, seed=5)
    g = torch.Generator().manual_seed(2)
    masks = [torch.stack([torch.randperm(784, generator=g)[:k].sort().values for _ in range(3)]) for k in (21, 13)]
    outs = enc.forward_multi(clips.to(dev), [m.to(dev) for m in masks])
    w = [torch.randn(o.shape, generator=g) for o in outs]
    sum((o.float() * wi.to(dev)).sum() for o, wi in zip(outs, w)).backward()
    S = {k: v.detach().float().cpu().clone() for k, v in enc.state_dict().items()}
    for k, v in S.items():
        if k != "pos_embed":
            v.requires_grad_(True)
    ref = [O.encoder(S, clips, [m], 12, 3) for m in masks]
    sum((o * wi).sum() for o, wi in zip(ref, w)).backward()
    for o, r in zip(outs, ref):
        assert rel_l2(o.detach().float().cpu(), r.detach()) < TOL_ACT
    for n, p in enc.named_parameters():
        if p.grad is not None:
            assert rel_l2(p.grad.float().cpu(), S[n].grad) < 3e-2, n


def test_multimask_fused_equals_per_mask_calls(dev):
    """MultiMaskWrapper semantics (multimask.py:17-26): the fused var-len pass == one backbone call per mask."""
    from jepa_b200.models import vit_tiny
    torch.manual_seed(0)
    enc = vit_tiny(img_size=224, patch_size=16, num_frames=8, tubelet_size=2, uniform_power=True).to(dev)
    clips = synth_clips(2, 8, 224, 224, seed=1).to(dev)
    me, _ = c1_masks(2)
    me = [m.to(dev) for m in me]
    with torch.no_grad():
        fused = enc.forward_multi(clips, me)
        single = [enc(clips, masks=m) for m in me]
        full = enc(clips)
    for a, b in zip(fused, single):
        assert torch.equal(a, b)
    assert full.shape == (2, 784, 192)
    cat = enc(clips, masks=[me[0], me[0]])
    assert cat.shape == (4, me[0].shape[1], 192) and torch.equal(cat[:2], cat[2:])


# --------------------------------------------------------------------------------------------- full size
def test_full_size_properties_vitl(dev):
    """BASELINE config[1] shapes (ViT-L/16, B=32, 16x224^2): properties that do not need a CPU oracle pass."""
    from jepa_b200 import kernels as Kn
    T, D, Hd = 32 * 1568, 1024, 4096
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(T, D, device=dev, generator=g).to(torch.bfloat16)
    w = (torch.randn(Hd, D, device=dev, generator=g) * 0.03).to(torch.bfloat16)
    y1 = torch.empty(T, Hd, dtype=torch.bfloat16, device=dev)
    y2 = torch.empty_like(y1)
    Kn.gemm(x, w, y1)
    Kn.gemm(x, w, y2, alpha=2.0)                      # linearity: exact in bf16 (power-of-two scale)
    assert torch.equal((y1.float() * 2).to(torch.bfloat16), y2)
    rows = torch.tensor([0, 1, 127, 128, 25087, 50175], device=dev)
    ref = x[rows].double() @ w.double().t()           # sampled rows in fp64
    close_bf16(y1[rows], ref.float().cpu(), atol=3e-2)
    # LayerNorm output rows are standardised
    yn = torch.empty_like(x)
    Kn.layernorm_fwd(x, yn, torch.ones(D, device=dev), torch.zeros(D, device=dev), 1e-6)
    s = yn[::997].float()
    assert float(s.mean(-1).abs().max()) < 1e-2 and float((s.var(-1, unbiased=False) - 1).abs().max()) < 3e-2
    # attention over full-length sequences: softmax rows are convex combinations -> |O| <= max|V|, and constant V is a fixed point
    H, hd, S, B = 16, 64, 1568, 4
    qkv = torch.randn(B * S, 3 * H * hd, device=dev, generator=g).to(torch.bfloat16)
    qkv[:, 2 * H * hd:] = 0.5
    out = torch.empty(B * S, H * hd, dtype=torch.bfloat16, device=dev)
    lse = torch.empty(H, B * S, device=dev)
    cu = torch.arange(0, (B + 1) * S, S, dtype=torch.int32, device=dev)
    Kn.attn_fwd(qkv, out, lse, cu, B, S, H, hd, hd ** -0.5)
    assert float((out.float() - 0.5).abs().max()) < 4e-3
    # gather / scatter-add round trip at full size is the identity on kept rows
    N, Kk = 1568, 360
    idx = torch.stack([torch.randperm(N, device=dev, generator=g)[:Kk].sort().values for _ in range(32)])
    xx = torch.randn(32, N, D, device=dev, generator=g)
    gat = Kn.gather_rows(xx, idx)
    back = torch.zeros_like(xx)
    Kn.scatter_rows_add(gat, back, idx)
    assert torch.equal(Kn.gather_rows(back, idx), gat)
    assert float(back.abs().sum(-1).ne(0).sum()) == 32 * Kk


def test_flat_adamw_single_launch_matches_torch(dev):
    """One vj_adamw_flat launch per backbone (group table per 64 elements) == torch.optim.AdamW with the
    reference's four parameter groups (app/vjepa/utils.py:173-194); frozen pos_embed untouched."""
    from app.vjepa.utils import init_opt, init_video_model
    from jepa_b200 import _lib
    torch.manual_seed(1)
    enc, pred = init_video_model(device=dev, patch_size=16, num_frames=8, tubelet_size=2, model_name="vit_tiny",
                                 crop_size=224, pred_depth=1, pred_embed_dim=384, uniform_power=True,
                                 use_mask_tokens=True, num_mask_tokens=2, use_sdpa=True)
    for net in (enc, pred):
        net.backbone._store.adopt(net.backbone)
    opt, _, sch, wds = init_opt(enc, pred, iterations_per_epoch=10, start_lr=1e-3, ref_lr=2e-3, warmup=1, num_epochs=2,
                                wd=0.04, final_wd=0.4)
    ref_params = {}
    ref_groups = []
    for g in opt.param_groups:
        clones = [torch.nn.Parameter(p.detach().clone()) for p in g["params"]]
        for p, c in zip(g["params"], clones):
            ref_params[p] = c
        ref_groups.append({"params": clones, "weight_decay": g["weight_decay"]})
    ref = torch.optim.AdamW(ref_groups, betas=(0.9, 0.999), eps=1e-8)
    pos0 = enc.backbone.pos_embed.detach().clone()
    gen = torch.Generator(device=dev).manual_seed(0)
    for it in range(3):
        lr, wd = sch.step(), wds.step()
        for rg, g in zip(ref.param_groups, opt.param_groups):
            rg["lr"], rg["weight_decay"] = g["lr"], g["weight_decay"]
        for net in (enc, pred):
            st = net.backbone._store
            gflat = st.new_grad_buffer()
            for n, p in net.backbone.named_parameters():
                if p.requires_grad:
                    view = st.grad_view(gflat, n)
                    view.copy_(torch.randn(view.shape, device=dev, generator=gen) * 0.01)
                    p.grad = view
                    ref_params[p].grad = view.clone()
        before = _lib.load().vj_launch_count()
        opt.step()
        assert _lib.load().vj_launch_count() - before == 4      # per backbone: one AdamW launch + the 1-thread step-counter advance
        ref.step()
    for p, c in ref_params.items():
        assert rel_l2(p.detach().cpu(), c.detach().cpu()) < 2e-6
    assert torch.equal(enc.backbone.pos_embed.detach(), pos0)
    sd = opt.state_dict()
    # entry for entry what torch.optim.AdamW keeps: no state for the frozen pos_embed tensors (they never get a gradient)
    assert len(sd["state"]) == len(ref.state_dict()["state"]) == len(ref_params) - 2
    assert float(next(iter(sd["state"].values()))["step"]) == 3.0


def test_flat_grad_statistics_scaler_clip_and_loggers(dev):
    """f1 / f2 (SURVEY 8f): the segmented single-pass kernels behind scaler.unscale_, grad_logger, adamw_logger and
    clip_grad_norm_ against the reference's own formulas (src/utils/logging.py:91-118, app/vjepa/train.py:462-471) and
    torch's implementations, on a ViT-Tiny encoder + predictor with synthetic flat gradients."""
    from app.vjepa.utils import init_opt, init_video_model
    from jepa_b200 import step as vj
    from jepa_b200.optim import FlatGradScaler
    from src.utils.logging import adamw_logger, grad_logger
    torch.manual_seed(3)
    enc, pred = init_video_model(device=dev, patch_size=16, num_frames=8, tubelet_size=2, model_name="vit_tiny",
                                 crop_size=224, pred_depth=2, pred_embed_dim=384, uniform_power=True,
                                 use_mask_tokens=True, num_mask_tokens=2, use_sdpa=True)
    for net in (enc, pred):
        net.backbone._store.adopt(net.backbone).refresh_shadow()   # what every forward does first: the bf16 operands exist
    opt, scaler, sch, wds = init_opt(enc, pred, iterations_per_epoch=10, start_lr=1e-3, ref_lr=2e-3, warmup=1, num_epochs=2,
                                     wd=0.04, final_wd=0.4, mixed_precision=True)
    assert isinstance(scaler, FlatGradScaler)
    gen = torch.Generator(device=dev).manual_seed(0)

    def fake_backward(scale, poison=False):
        for net in (enc, pred):
            st = net.backbone._store
            gflat = st.new_grad_buffer()
            for n, p in net.backbone.named_parameters():
                if p.requires_grad:
                    view = st.grad_view(gflat, n)
                    view.copy_(torch.randn(view.shape, device=dev, generator=gen) * 0.01 * scale)
                    p.grad = view
        if poison:
            enc.backbone.blocks[3].mlp.fc1.weight.grad[5, 7] = float("inf")

    # ---- unscale + per-tensor norms + loggers
    sch.step(); wds.step()
    fake_backward(65536.0)
    ref_norm = {n: float(p.grad.double().norm() / 65536.0) for n, p in enc.named_parameters() if p.grad is not None}
    scaler._lazy_init_scale_growth_tracker(dev)
    scaler.unscale_(opt)
    for n, p in enc.named_parameters():
        if p.grad is not None:
            assert abs(float(p.grad.double().norm()) - ref_norm[n]) <= 1e-5 * ref_norm[n] + 1e-12, n
    gs = grad_logger(enc.named_parameters())
    w = [v for n, v in ref_norm.items() if not (n.endswith(".bias") or enc.get_parameter(n).dim() == 1)]
    assert abs(gs.avg - sum(w) / len(w)) < 1e-5 * gs.avg and abs(gs.max - max(w)) < 1e-5 * gs.max and abs(gs.min - min(w)) < 1e-5 * gs.max
    qkv = [v for n, v in ref_norm.items() if "qkv" in n and n.endswith("weight")]
    assert abs(gs.first_layer - qkv[0]) < 1e-5 * qkv[0] and abs(gs.last_layer - qkv[-1]) < 1e-5 * qkv[-1]
    # ---- clip_grad_norm_ on the device == torch's
    ref_grads = [p.grad.clone() for p in pred.parameters() if p.grad is not None]
    refp = [torch.nn.Parameter(torch.zeros_like(g)) for g in ref_grads]
    for q, g in zip(refp, ref_grads):
        q.grad = g.clone()
    total_ref = torch.nn.utils.clip_grad_norm_(refp, 1e9)   # norm only: nothing is clipped at this bound
    max_norm = float(total_ref) * 0.5
    torch.nn.utils.clip_grad_norm_(refp, max_norm)
    total = vj.clip_grad_norm_(pred, max_norm)
    assert abs(float(total) - float(total_ref)) < 1e-5 * float(total_ref)
    for q, p in zip(refp, [p for p in pred.parameters() if p.grad is not None]):
        assert rel_l2(p.grad.cpu(), q.grad.cpu()) < 1e-6
    before = [p.grad.clone() for p in enc.parameters() if p.grad is not None]
    vj.clip_grad_norm_(enc, 1e9)                              # no clipping needed: gradients untouched
    assert all(torch.equal(a, p.grad) for a, p in zip(before, [p for p in enc.parameters() if p.grad is not None]))
    # ---- optimizer step: device-side step counter, bf16 shadow emitted with the update
    scaler.step(opt); scaler.update()
    st0 = opt.state[enc.backbone.blocks[0].attn.qkv.weight]
    assert st0["step"].is_cuda and float(st0["step"]) == 1.0
    store = enc.backbone._store
    assert store._shadow_fresh and torch.equal(store.shadow, store.flat.to(torch.bfloat16))
    am = adamw_logger(opt)
    ref1 = [float(s["exp_avg"].abs().mean()) for s in opt.state_dict()["state"].values()]
    ref2 = [float(s["exp_avg_sq"].abs().mean()) for s in opt.state_dict()["state"].values()]
    assert abs(am["exp_avg"].avg - sum(ref1) / len(ref1)) < 1e-5 * am["exp_avg"].avg
    assert abs(am["exp_avg_sq"].max - max(ref2)) < 1e-5 * am["exp_avg_sq"].max and am["exp_avg"].count == len(ref1)
    opt.zero_grad()
    # ---- an overflowing step is skipped: parameters, moments AND the step count stay put; the scale backs off
    p_before = store.flat.clone()
    sch.step(); wds.step()
    fake_backward(65536.0, poison=True)
    scaler.unscale_(opt)
    scaler.step(opt); scaler.update()
    assert torch.equal(store.flat, p_before) and float(st0["step"]) == 1.0 and float(scaler.get_scale()) == 32768.0
    opt.zero_grad()
    # ---- EMA emits the target's bf16 operands in the same pass, bit-exact with the reference op sequence
    import copy
    tgt = copy.deepcopy(enc)
    k0 = tgt.backbone._store.adopt(tgt.backbone).flat.clone()
    vj.ema_update(enc, tgt, 0.998)
    ref = k0.clone(); ref.mul_(0.998).add_((1. - 0.998) * store.flat)
    ks = tgt.backbone._store
    assert torch.equal(ks.flat, ref) and ks._shadow_fresh and torch.equal(ks.shadow, ref.to(torch.bfloat16))


def test_attentive_probe_vs_reference_fixture(dev):
    """SURVEY 8 f4: jepa_b200.pooler.AttentiveClassifier (vj_cross_attn_fwd + LayerNorm + wgmma GEMMs) vs the outputs the
    UNMODIFIED reference modules produced for the same seeded weights and inputs (tests/golden/make_golden_pooler.py);
    head dims 64 / 32 / 80 / 128, complete_block on and off, class counts that are not multiples of 64."""
    from test_oracle_cpu import _build_probe, _pooler_fixture
    for case in _pooler_fixture()["cases"]:
        clf = _build_probe(case).to(dev)
        x = case["x"].to(dev, torch.bfloat16)
        with torch.no_grad():
            pooled = clf.pooler(x).float().cpu()
            logits = clf(x).float().cpu()
        assert pooled.shape == case["pooled"].shape and logits.shape == case["logits"].shape
        assert rel_l2(pooled, case["pooled"]) < TOL_ACT and rel_l2(logits, case["logits"]) < TOL_ACT, case["cfg"]
        with pytest.raises(NotImplementedError):      # inference-only: the probe is trained by the reference's eval loop
            clf.pooler(x.float().requires_grad_(True))


@pytest.mark.parametrize("D,H,S,B", [(1024, 16, 1568, 4), (1280, 16, 392, 3), (1280, 16, 4608, 1)])
def test_attentive_probe_encoder_sizes_vs_oracle(dev, D, H, S, B):
    """The probe at the encoders' real widths (ViT-L hd 64, ViT-H hd 80) and token counts (1568; C5's 4608) vs the oracle."""
    from jepa_b200.pooler import AttentiveClassifier
    from oracle import vjepa_oracle as O
    torch.manual_seed(D + S)
    clf = AttentiveClassifier(embed_dim=D, num_heads=H, depth=1, num_classes=400).eval()
    with torch.no_grad():
        for n, p in clf.named_parameters():
            if n.endswith("bias") or "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
        # sharpen the attention a little (the init scale 0.02 gives an almost uniform softmax over S keys)
        clf.pooler.query_tokens.mul_(20.0)
        clf.pooler.cross_attention_block.xattn.q.weight.mul_(6.0)
        clf.pooler.cross_attention_block.xattn.kv.weight.mul_(6.0)
    x = bf(torch.randn(B, S, D, generator=torch.Generator().manual_seed(S)))
    S_ = {k: v.double() for k, v in clf.state_dict().items()}
    ref = O.attentive_classifier(S_, x.double(), H).float()
    with torch.no_grad():
        got = clf.to(dev)(x.to(dev, torch.bfloat16)).float().cpu()
    assert rel_l2(got, ref) < TOL_ACT


def test_out_layers_feature_taps_vs_oracle(dev):
    """f4 (frozen-encoder inference for the evals): VisionTransformer(out_layers=[...]) returns norm(x) after the chosen
    blocks (vision_transformer.py:183-190), here against the oracle."""
    from jepa_b200.models import vit_tiny
    from oracle import vjepa_oracle as O
    torch.manual_seed(0)
    enc = vit_tiny(img_size=224, patch_size=16, num_frames=8, tubelet_size=2, uniform_power=True, out_layers=[5, 8, 11]).to(dev)
    clips = synth_clips(2, 8, 224, 224, seed=4)
    with torch.no_grad():
        outs = enc(clips.to(dev))
    S = {k: v.detach().float().cpu() for k, v in enc.state_dict().items()}
    ref = O.encoder(S, clips, None, 12, 3, out_layers=[5, 8, 11])
    assert len(outs) == 3 and all(o.shape == (2, 784, 192) for o in outs)
    for o, r in zip(outs, ref):
        assert rel_l2(o.float().cpu(), r) < TOL_ACT
    # the last tap is the ordinary encoder output
    enc.out_layers = None
    with torch.no_grad():
        assert torch.equal(enc(clips.to(dev)), outs[-1])


def test_clip_preprocess_kernel_vs_reference_fixtures(dev, golden_dir):
    """f3: uint8 frames -> crop box / flip (host sampler, reference RNG order) -> ONE kernel (bilinear resize, flip,
    normalise) == the unmodified reference VideoTransform (tests/golden/golden_transforms.pt) and the oracle, per case
    and batched with different frame sizes per clip; bf16 output = rounded fp32 output."""
    import random
    import numpy as np
    from jepa_b200.transforms import make_transforms, preprocess_batch
    from oracle import vjepa_oracle as O
    cases = torch.load(os.path.join(golden_dir, "golden_transforms.pt"))
    tickets_by_crop = {}
    for c in cases:
        T, H, W = c["shape"]
        buf = np.random.RandomState(1000 + c["seed"]).randint(0, 256, size=(T, H, W, 3), dtype=np.uint8)
        tf = make_transforms(random_horizontal_flip=True, random_resize_aspect_ratio=c["ratio"],
                             random_resize_scale=c["scale"], crop_size=c["crop"])
        random.seed(c["seed"]); np.random.seed(c["seed"])
        tk = tf(buf)
        assert tuple(tk.box) == tuple(c["box"]) and tk.flip == c["flip"]
        y = preprocess_batch([tk], dev, c["crop"])
        assert y.shape == (1,) + tuple(c["out"].shape) and y.dtype == torch.float32
        assert float((y[0].cpu() - c["out"]).abs().max()) < 5e-5, c["seed"]
        assert float((y[0].cpu() - O.video_transform(buf, tk.box, tk.flip, c["crop"])).abs().max()) < 5e-5
        yb = preprocess_batch([tk], dev, c["crop"], dtype=torch.bfloat16)
        assert float((yb[0].float().cpu() - c["out"].to(torch.bfloat16).float()).abs().max()) < 2e-2
        tickets_by_crop.setdefault((c["crop"], T), []).append((tk, c))
    # a batch of clips with different decoded sizes goes through one launch
    T = 4
    mixed = []
    for seed, (H, W) in enumerate([(48, 64), (36, 100), (70, 50)]):
        buf = np.random.RandomState(77 + seed).randint(0, 256, size=(T, H, W, 3), dtype=np.uint8)
        tf = make_transforms(crop_size=32, random_resize_aspect_ratio=(0.75, 1.35), random_resize_scale=(0.3, 1.0))
        random.seed(seed); np.random.seed(seed)
        mixed.append((tf(buf), buf))
    yb = preprocess_batch([t for t, _ in mixed], dev, 32)
    for b, (tk, buf) in enumerate(mixed):
        assert float((yb[b].cpu() - O.video_transform(buf, tk.box, tk.flip, 32)).abs().max()) < 5e-5
