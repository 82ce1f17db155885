"""Row, reduction and flat-buffer kernels (layernorm.cu, rowops.cu, optim.cu, gradstats.cu) against plain float64
references, one kernel at a time, at every dispatch branch: each LayerNorm width instance (NV = ceil(D / 256) rounded
up to 1, 2, 4, 5 or 8) with full, partly empty and one-lane last chunks, every dtype pair, row-count tails and grids
whose grid-stride loops run more than once; the column-sum row filter and row stride; the predictor assembly and
sequence slices; the regulariser's token variance on channels with a large offset; the flat AdamW group table, the
non-finite flag and the clipping pass.

References are computed in float64 on the device from exactly the values the kernel reads, with the textbook formula
(mean / var / autograd), never by restating the kernel.  Tolerances:
  copies, single adds, casts                     : bit-exact
  bf16 outputs                                   : |err| <= 2^-8 |ref| + 1e-5 max|ref of the row|   (one bf16 ulp)
  fp32 elementwise outputs                       : |err| <= 1e-5 |ref| + 1e-5 max|ref of the row|
  fp32 reductions over rows (dgamma, colsum ...) : rel-L2 1e-4 of the accumulated increment
LayerNorm outputs also allow the fp32 rounding of the row mean, amplified by rstd: 2^-20 max|x| rstd |gamma| (a few
ulps of the mean; at a constant row, where rstd = eps^-1/2, this is the whole output error).  A wrong branch gives
O(1) errors, far outside every bound.  Indices are always in range: the gather / scatter kernels do not bounds-check.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
LN_EPS = 1e-6
# every NV instance: full last chunk (256, 1024, 2048), one-lane last chunk (264, 520, 1032, 1288), NV = 4 from nv = 3 (768)
LN_D = [8, 192, 256, 264, 384, 520, 768, 1024, 1032, 1280, 1288, 1408, 1664, 2048]
LN_T = [1, 2, 3, 17, 777]
# On 132 SMs the widest sweep of any LayerNorm grid-stride loop is ln_fwd2 at NV <= 2 (132 * 3 blocks * 8 warps * 2 rows
# = 6336 rows) and the backward's block count is capped at 4 * 132: 20011 rows make every loop run at least three times.
T_SWEEP = 20011
LN_SWEEP_D = (264, 1032, 2048)
LN_PAIRS = {"bf16-bf16": (BF16, BF16), "f32-f32": (F32, F32), "f32-bf16": (F32, BF16), "bf16-f32": (BF16, F32)}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _check(got, ref, rtol, slack=None, what=""):
    """|got - ref| <= rtol |ref| + 1e-5 max|ref| per row (last dim) + slack; got must be finite."""
    got, ref = got.double(), ref.double()
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output"
    rowmax = ref.abs().amax(-1, keepdim=True) if ref.dim() else ref.abs()
    bound = rtol * ref.abs() + 1e-5 * rowmax
    if slack is not None:
        bound = bound + slack
    excess = (got - ref).abs() - bound
    worst = float(excess.max())
    if worst > 0:
        at = tuple(int(i) for i in torch.nonzero(excess == worst)[0])
        raise AssertionError(f"{what}: max err {float((got - ref).abs().max()):.3e}, worst excess {worst:.3e} at {at}")


def _bf16(got, ref, slack=None, what=""):
    _check(got, ref, 2.0 ** -8, slack, what)


def _f32(got, ref, slack=None, what=""):
    _check(got, ref, 1e-5, slack, what)


def _rel_l2(got, ref):
    return float((got.double() - ref.double()).norm() / (ref.double().norm() + 1e-300))


def _ln_rows(dev, T, D, seed):
    """fp32 rows of three kinds, cycling by row index: ordinary N(0.5, 2), offset 64 + N(0, 0.25) and constant (one
    bf16-representable value per row, so that var = 0 exactly in either input dtype)."""
    g = _gen(dev, seed)
    x = torch.randn(T, D, device=dev, generator=g) * 2 + 0.5
    kind = (torch.arange(T, device=dev) % 3)[:, None]
    x = torch.where(kind == 1, 64 + 0.25 * torch.randn(T, D, device=dev, generator=g), x)
    return torch.where(kind == 2, x[:, :1].to(BF16).float(), x)


def _ln_affine(dev, D, seed):
    g = _gen(dev, seed + 7)
    return 1 + 0.3 * torch.randn(D, device=dev, generator=g), 0.3 * torch.randn(D, device=dev, generator=g)


def _ln_ref_stats(x):
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + LN_EPS)
    # fp32 rounding of the row mean, amplified by rstd (see the module docstring)
    amp = 2.0 ** -20 * xd.abs().amax(-1, keepdim=True) * rstd
    return xd, mean, rstd, amp


# ---------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("pair", list(LN_PAIRS))
@pytest.mark.parametrize("D", LN_D)
def test_layernorm_forward_vs_fp64(dev, D, pair):
    """vj_layernorm_fwd at every NV instance and dtype pair (bf16 -> bf16 is ln_fwd2_kernel, the others ln_fwd_kernel),
    row-count tails and a grid-stride sweep, with and without the mean / rstd outputs."""
    from jepa_b200 import kernels as Kn
    xt, yt = LN_PAIRS[pair]
    gamma, beta = _ln_affine(dev, D, D)
    for T in LN_T + ([T_SWEEP] if D in LN_SWEEP_D else []):
        x = _ln_rows(dev, T, D, seed=T * 7 + D).to(xt)
        xd, mean, rstd, amp = _ln_ref_stats(x)
        ref = (xd - mean) * rstd * gamma.double() + beta.double()
        y = torch.empty(T, D, dtype=yt, device=dev)
        mo, ro = torch.full((T,), float("nan"), device=dev), torch.full((T,), float("nan"), device=dev)
        Kn.layernorm_fwd(x, y, gamma, beta, LN_EPS, mo, ro)
        what = f"D={D} {pair} T={T}"
        slack = amp * gamma.double().abs()
        (_bf16 if yt == BF16 else _f32)(y, ref, slack, what + " y")
        _check(mo[:, None], mean, 1e-5, 2.0 ** -20 * xd.abs().amax(-1, keepdim=True), what + " mean")
        _f32(ro[:, None], rstd, what=what + " rstd")
        # without the statistics outputs the same kernel runs and writes the same rows
        y2 = torch.empty_like(y)
        Kn.layernorm_fwd(x, y2, gamma, beta, LN_EPS)
        assert torch.equal(y2, y), what + ": output differs when mean / rstd are not requested"


@pytest.mark.parametrize("xt", [BF16, F32], ids=["bf16", "f32"])
@pytest.mark.parametrize("D", LN_D)
def test_layernorm_backward_vs_fp64(dev, D, xt):
    """vj_layernorm_bwd: bf16 x runs ln_bwd2_kernel for NV <= 5 and ln_bwd_kernel<8, false> for D > 1280; fp32 x runs
    ln_bwd_kernel<NV, true> with fp32 dres / dx (the attentive probe's residual).  dres given and None, dgamma / dbeta
    accumulating into non-zero buffers, row tails, and a row count past the cap of ln_bwd_grid."""
    from jepa_b200 import kernels as Kn
    gamma, beta = _ln_affine(dev, D, D + 1)
    for i, T in enumerate(LN_T + ([T_SWEEP] if D in LN_SWEEP_D else [])):
        g = _gen(dev, T * 13 + D)
        x = _ln_rows(dev, T, D, seed=T * 11 + D).to(xt)
        dy = torch.randn(T, D, device=dev, generator=g).to(BF16)
        dres = torch.randn(T, D, device=dev, generator=g).to(xt) if i % 2 == 0 else None
        xr = x.double().requires_grad_(True)
        gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        xd, mean, rstd, amp = _ln_ref_stats(xr.detach())
        y = (xr - xr.mean(-1, keepdim=True)) / torch.sqrt(xr.var(-1, unbiased=False, keepdim=True) + LN_EPS) * gr + br
        y.backward(dy.double())
        ref_dx = xr.grad + (dres.double() if dres is not None else 0.0)
        dg0 = torch.randn(D, device=dev, generator=g)
        db0 = torch.randn(D, device=dev, generator=g)
        dg, db = dg0.clone(), db0.clone()
        dx = torch.empty_like(x)
        Kn.layernorm_bwd(dy, x, gamma, mean.float().view(T), rstd.float().view(T), dres, dx, dg, db)
        what = f"D={D} x={xt} T={T} dres={'yes' if dres is not None else 'None'}"
        # dx depends on the row mean through xhat * mean(g dy xhat): the same fp32-mean slack, times rstd |s2| <= rstd |g dy|
        slack = amp * rstd * (gamma.double() * dy.double()).abs().amax(-1, keepdim=True)
        (_bf16 if xt == BF16 else _f32)(dx, ref_dx, slack, what + " dx")
        e_g, e_b = _rel_l2(dg.double() - dg0.double(), gr.grad), _rel_l2(db.double() - db0.double(), br.grad)
        assert e_g < 1e-4 and e_b < 1e-4, f"{what}: dgamma rel-L2 {e_g:.2e}, dbeta rel-L2 {e_b:.2e}"


@pytest.mark.parametrize("D", [192, 384, 768, 1024, 1280, 1408, 2048])
def test_target_ln_gather_vs_fp64(dev, D):
    """vj_target_ln_gather: LN(affine, eps 1e-6) -> LN(no affine, eps 1e-5) of gathered rows, unsorted indices, rows
    with a large offset among ordinary ones."""
    from jepa_b200 import kernels as Kn
    B, N, K = 3, 1568, 824
    x = _ln_rows(dev, B * N, D, seed=D)
    spread = 0.25 * torch.randn(x.shape, device=dev, generator=_gen(dev, D + 1))
    x = torch.where((torch.arange(B * N, device=dev) % 3 == 2)[:, None], x + spread, x)    # no constant rows
    x = x.to(BF16).view(B, N, D)
    gamma, beta = _ln_affine(dev, D, D + 2)
    g = _gen(dev, D + 3)
    idx = torch.stack([torch.randperm(N, device=dev, generator=g)[:K] for _ in range(B)])
    got = Kn.target_ln_gather(x, idx, gamma, beta, LN_EPS, 1e-5)
    rows = torch.gather(x, 1, idx[..., None].expand(B, K, D))
    xd, mean, rstd, amp = _ln_ref_stats(rows)
    v = (xd - mean) * rstd * gamma.double() + beta.double()
    sv = torch.sqrt(v.var(-1, unbiased=False, keepdim=True) + 1e-5)
    ref = (v - v.mean(-1, keepdim=True)) / sv
    _f32(got, ref, amp * gamma.double().abs().max() / sv, f"D={D}")


# ---------------------------------------------------------------------------------------------------- column sums
@pytest.mark.parametrize("dt", [BF16, F32], ids=["bf16", "f32"])
@pytest.mark.parametrize("N", [8, 64, 264, 1024, 1032])
def test_colsum_windows_and_stride_vs_fp64(dev, N, dt):
    """vj_colsum: out[c] += sum of rows r with lo <= r % period < hi (period 0: every row), also over a column slice
    of a wider matrix (row stride ld > N); the output starts non-zero."""
    from jepa_b200 import _lib
    from jepa_b200 import kernels as Kn
    windows = [(0, 0, 0), (7, 2, 3), (5, 0, 5), (13, 4, 9), (64, 63, 64)]
    for T in (1, 63, 64, 65, 100003):
        g = _gen(dev, T + N)
        wide = (torch.randn(T, N + 24, device=dev, generator=g) + 0.5).to(dt)
        r = torch.arange(T, device=dev)
        for period, lo, hi in windows:
            sel = torch.ones(T, dtype=torch.bool, device=dev) if period == 0 else (r % period >= lo) & (r % period < hi)
            for strided in (False, True):
                x = wide[:, 8:8 + N] if strided else wide[:, :N].contiguous()
                ref = x[sel].double().sum(0)
                out0 = torch.randn(N, device=dev, generator=g)
                out = out0.clone()
                if strided:
                    _lib.call("vj_colsum", x.data_ptr(), int(dt == F32), out.data_ptr(), T, N, x.stride(0), period, lo, hi,
                              Kn._s())
                else:
                    Kn.colsum(x, out, period, lo, hi)
                what = f"T={T} N={N} {dt} window={period, lo, hi} ld={x.stride(0)}"
                if int(sel.sum()) == 0:
                    assert torch.equal(out, out0), what + ": no row selected, output must be untouched"
                else:
                    e = _rel_l2(out.double() - out0.double(), ref)
                    assert e < 1e-4, f"{what}: rel-L2 {e:.2e}"


# ---------------------------------------------------------------------------------------------------- predictor rows
PRED_SHAPES = [(3, 1568, 360, 824, 384), (1, 11, 3, 5, 8)]   # (B, N, Ke, Kp, Dp): C2 mask sizes, and a small odd case


@pytest.mark.parametrize("B,N,Ke,Kp,Dp", PRED_SHAPES)
def test_pred_assemble_and_seq_slice(dev, B, N, Ke, Kp, Dp):
    """vj_pred_assemble_fwd / _bwd and vj_seq_slice (gather, scatter, zero_ctx) in both residual dtypes."""
    from jepa_b200 import kernels as Kn
    g = _gen(dev, N + Dp)
    perm = torch.stack([torch.randperm(N, device=dev, generator=g)[:Ke + Kp] for _ in range(B)])
    idx_ctx, idx_tgt = perm[:, :Ke].contiguous(), perm[:, Ke:].contiguous()
    emb = torch.randn(B * Ke, Dp, device=dev, generator=g).to(BF16)
    pos = torch.randn(N, Dp, device=dev, generator=g)
    tok = torch.randn(Dp, device=dev, generator=g)
    S = Ke + Kp
    for dt in (BF16, F32):
        x = torch.empty(B, S, Dp, dtype=dt, device=dev)
        Kn.pred_assemble_fwd(emb, pos, tok, idx_ctx, idx_tgt, x, B, Ke, Kp, Dp)
        assert torch.equal(x[:, :Ke], (emb.float().view(B, Ke, Dp) + pos[idx_ctx]).to(dt)), dt
        assert torch.equal(x[:, Ke:], (tok + pos[idx_tgt]).to(dt)), dt
        # backward: context rows cast to bf16, mask-token gradient = column sum over the target rows of every sequence
        dx = torch.randn(B, S, Dp, device=dev, generator=g).to(dt)
        demb = torch.empty(B * Ke, Dp, dtype=BF16, device=dev)
        dtok0 = torch.randn(Dp, device=dev, generator=g)
        dtok = dtok0.clone()
        Kn.pred_assemble_bwd(dx, demb, dtok, B, Ke, Kp, Dp)
        assert torch.equal(demb, dx[:, :Ke].reshape(B * Ke, Dp).to(BF16)), dt
        e = _rel_l2(dtok.double() - dtok0.double(), dx[:, Ke:].double().sum((0, 1)))
        assert e < 1e-4, f"{dt}: dmask_token rel-L2 {e:.2e}"
        # seq_slice: target rows out, and back in (context rows untouched or zeroed)
        tgt = torch.empty(B * Kp, Dp, dtype=dt, device=dev)
        Kn.seq_slice(x, tgt, B, Ke, Kp, Dp)
        assert torch.equal(tgt, x[:, Ke:].reshape(B * Kp, Dp)), dt
        src = torch.randn(B * Kp, Dp, device=dev, generator=g).to(dt)
        for zero_ctx in (False, True):
            dst = torch.full((B, S, Dp), 7.0, dtype=dt, device=dev)
            Kn.seq_slice(src, dst, B, Ke, Kp, Dp, scatter=True, zero_ctx=zero_ctx)
            assert torch.equal(dst[:, Ke:], src.view(B, Kp, Dp)), (dt, zero_ctx)
            assert torch.equal(dst[:, :Ke], torch.full_like(dst[:, :Ke], 0.0 if zero_ctx else 7.0)), (dt, zero_ctx)


@pytest.mark.parametrize("dt", [BF16, F32], ids=["bf16", "f32"])
def test_scatter_rows_add_bit_exact(dev, dt):
    """vj_scatter_rows_add into non-zero rows, indices unique per row but unsorted: one fp32 add per element."""
    from jepa_b200 import kernels as Kn
    for B, N, K, D in ((3, 1568, 824, 384), (2, 13, 5, 8), (1, 784, 784, 1408)):
        g = _gen(dev, N + D)
        idx = torch.stack([torch.randperm(N, device=dev, generator=g)[:K] for _ in range(B)])
        dy = torch.randn(B, K, D, device=dev, generator=g).to(dt)
        dx0 = torch.randn(B, N, D, device=dev, generator=g).to(dt)
        dx = dx0.clone()
        Kn.scatter_rows_add(dy, dx, idx)
        ref = dx0.float().scatter_add(1, idx[..., None].expand(B, K, D), dy.float()).to(dt)
        assert torch.equal(dx, ref), (B, N, K, D)


# ---------------------------------------------------------------------------------------------------- regulariser
TSTD_CHANNELS = [(0.0, 1.0), (3.0, 0.3), (8.0, 0.1), (30.0, 0.5), (-60.0, 1.0)]   # (mean, std) of channel d % 5


@pytest.mark.parametrize("K1,K2", [(2, 3), (3, 2), (1144, 3600), (3600, 1144)])
def test_token_std_offset_channels_vs_fp64(dev, K1, K2):
    """vj_token_std_accum / vj_token_std_bwd over two masks (weight 1/2 each) on channels whose mean is far from zero
    compared with their spread across tokens: exactly the channels where relu(1 - pstd) is active.  pstd vs fp64
    sqrt(var_unbiased + 1e-4); dz vs fp64 autograd of mean(relu(1 - pstd_total)) times the device grad scale."""
    from jepa_b200 import kernels as Kn
    B, D = 3, 200   # D is not a multiple of the 128-thread block
    mu = torch.tensor([TSTD_CHANNELS[d % 5][0] for d in range(D)], device=dev, dtype=F64)
    sd = torch.tensor([TSTD_CHANNELS[d % 5][1] for d in range(D)], device=dev, dtype=F64)
    g = _gen(dev, K1 * 7 + K2)
    zs = [(torch.randn(B, k, D, device=dev, generator=g, dtype=F64) * sd + mu).to(BF16) for k in (K1, K2)]
    pstd = torch.zeros(B, D, device=dev)
    for z in zs:
        Kn.token_std_accum(z, pstd, 0.5)
    zr = [z.double().requires_grad_(True) for z in zs]
    ref = sum(0.5 * torch.sqrt(z.var(dim=1, unbiased=True) + 1e-4) for z in zr)
    rel = ((pstd.double() - ref.detach()).abs() / ref.detach())
    by_channel = ", ".join(f"{TSTD_CHANNELS[c]}: {float(rel[:, c::5].max()):.1e}" for c in range(5))
    assert float(rel.max()) <= 1e-5, f"K={K1},{K2}: pstd rel error by channel (mean, std) {by_channel}"
    torch.relu(1.0 - ref).mean().backward()
    gscale, scale = torch.tensor([1024.0], device=dev), 0.5
    # columns within 1e-4 of the relu kink may fall on either side in fp32; they are left out of the gradient check
    keep = ((ref.detach() - 1.0).abs() > 1e-4)[:, None, :]
    for z, r in zip(zs, zr):
        dz = torch.full_like(z, float("nan"))
        Kn.token_std_bwd(z, pstd, gscale, scale, dz, 0.5)
        ref_dz = r.grad * (1024.0 * scale)
        assert float(ref_dz.abs().max()) > 0
        _bf16(torch.where(keep, dz.double(), 0.0), torch.where(keep, ref_dz, 0.0), what=f"K={z.shape[1]} dz")


# ---------------------------------------------------------------------------------------------------- flat buffers
def _f32r(v):
    """v rounded to fp32, as the kernel receives it."""
    return float(torch.tensor(v, dtype=F32))


def test_adamw_flat_group_table_vs_fp64(dev):
    """vj_adamw_flat: a group table mixing ids 0-3 and 255 (frozen / padding), with and without the device step
    counter, found_inf, inv_scale and the bf16 shadow.  Id-255 blocks stay bit-identical in p, m, v and shadow; updated
    blocks match an fp64 restatement of torch.optim.AdamW, and the shadow is their bf16 cast."""
    from jepa_b200 import _lib
    from jepa_b200 import kernels as Kn
    nblk = 1237
    n = 64 * nblk
    g = _gen(dev, 3)
    gid = torch.tensor([0, 1, 2, 3, 255], dtype=torch.uint8, device=dev)[torch.randint(0, 5, (nblk,), device=dev, generator=g)]
    lr, wd = [1e-2, 3e-3, 5e-4, 2e-2], [0.05, 0.0, 0.4, 0.01]
    lr4, wd4 = (ctypes.c_float * 4)(*lr), (ctypes.c_float * 4)(*wd)    # host tables
    lr, wd = [_f32r(a) for a in lr], [_f32r(a) for a in wd]
    beta1, beta2, eps = _f32r(0.9), _f32r(0.999), _f32r(1e-8)
    frozen = (gid == 255).repeat_interleave(64)
    lr_e = torch.tensor(lr + [0.0], device=dev, dtype=F64)[torch.where(gid == 255, 4, gid.long())].repeat_interleave(64)
    wd_e = torch.tensor(wd + [0.0], device=dev, dtype=F64)[torch.where(gid == 255, 4, gid.long())].repeat_interleave(64)
    cases = [dict(step=1), dict(step=7, inv_scale=1.0 / 1024), dict(step_dev=4.0, shadow=True),
             dict(step_dev=2.0, inv_scale=1.0 / 65536, found_inf=0.0, shadow=True), dict(step_dev=5.0, found_inf=1.0, shadow=True)]
    for c in cases:
        p0 = torch.randn(n, device=dev, generator=g)
        m0 = 0.01 * torch.randn(n, device=dev, generator=g)
        v0 = 1e-4 * torch.rand(n, device=dev, generator=g)
        inv = c.get("inv_scale")
        grad = torch.randn(n, device=dev, generator=g) * 0.01 / (inv or 1.0)
        p, m, v = p0.clone(), m0.clone(), v0.clone()
        sh0 = torch.randn(n, device=dev, generator=g).to(BF16)
        sh = sh0.clone() if c.get("shadow") else None
        step_dev = torch.tensor([c["step_dev"]], device=dev) if "step_dev" in c else None
        inv_t = torch.tensor([inv], device=dev) if inv is not None else None
        fi = torch.tensor([c["found_inf"]], device=dev) if "found_inf" in c else None
        _lib.call("vj_adamw_flat", p.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), gid.data_ptr(), n,
                  ctypes.cast(lr4, ctypes.c_void_p), ctypes.cast(wd4, ctypes.c_void_p), beta1, beta2, eps,
                  c.get("step", 0), Kn._p(inv_t), Kn._p(fi), Kn._p(step_dev), Kn._p(sh), Kn._s())
        if c.get("found_inf"):
            assert torch.equal(p, p0) and torch.equal(m, m0) and torch.equal(v, v0) and torch.equal(sh, sh0), c
            assert float(step_dev) == c["step_dev"], "a skipped step must not advance the step counter"
            continue
        t = c["step_dev"] + 1 if step_dev is not None else c["step"]
        if step_dev is not None:
            assert float(step_dev) == t
        gr = grad.double() * (inv if inv is not None else 1.0)
        rm = beta1 * m0.double() + (1 - beta1) * gr
        rv = beta2 * v0.double() + (1 - beta2) * gr * gr
        denom = torch.sqrt(rv) / (1 - beta2 ** t) ** 0.5 + eps
        rp = p0.double() * (1 - lr_e * wd_e) - lr_e / (1 - beta1 ** t) * rm / denom
        live = ~frozen
        for name, got, ref, start in (("p", p, rp, p0), ("m", m, rm, m0), ("v", v, rv, v0)):
            assert torch.equal(got[frozen], start[frozen]), f"{c}: {name} changed in id-255 blocks"
            _f32(got[live].view(-1, 64), ref[live].view(-1, 64), what=f"{c} {name}")
        if sh is not None:
            assert torch.equal(sh[frozen], sh0[frozen]), f"{c}: shadow changed in id-255 blocks"
            assert torch.equal(sh[live], p[live].to(BF16)), f"{c}: shadow is not the bf16 cast of the update"


def _segment_table(dev, nblk, seed):
    """uint16 block -> segment id: lengths from one block to hundreds (spanning many warps' block ranges), with
    0xFFFF gaps; returns (table as int64, number of segments)."""
    gen = torch.Generator().manual_seed(seed)
    lens = torch.tensor([1, 1, 2, 3, 7, 30, 200])
    ids, s, b = [], 0, 0
    while b < nblk:
        if int(torch.randint(0, 3, (1,), generator=gen)) == 0:
            gap = min(int(torch.randint(1, 4, (1,), generator=gen)), nblk - b)
            ids += [0xFFFF] * gap
            b += gap
            continue
        L = min(int(lens[torch.randint(0, len(lens), (1,), generator=gen)]), nblk - b)
        ids += [s] * L
        s += 1
        b += L
    return torch.tensor(ids, dtype=torch.int64, device=dev), s


def _seg_sums(x, seg64, n_seg):
    """fp64 per-segment sums of x (fp64, one value per element)."""
    blk = x.view(-1, 64).sum(1)
    live = seg64 != 0xFFFF
    return torch.zeros(n_seg, dtype=F64, device=x.device).index_add_(0, seg64[live], blk[live])


def _rel_each(got, ref, what):
    """Sums of non-negative terms: elementwise relative error 1e-5."""
    rel = (got.double() - ref).abs() / ref
    assert float(rel.max()) <= 1e-5, f"{what}: max rel err {float(rel.max()):.2e}"


def test_grad_unscale_stats_nonfinite_and_write_back(dev):
    """vj_grad_unscale_stats: per-segment sums of squares of the unscaled gradient, written back or not, the
    non-finite flag raised by NaN and by -inf and left alone on a clean buffer; 0xFFFF blocks are never touched.
    vj_seg_abs_sum over the same table."""
    from jepa_b200 import kernels as Kn
    nblk = 20011
    seg64, n_seg = _segment_table(dev, nblk, seed=1)
    seg = seg64.cpu().to(torch.int32).to(torch.uint16).to(dev)
    skip = (seg64 == 0xFFFF).repeat_interleave(64)
    g = _gen(dev, 5)
    g0 = torch.randn(64 * nblk, device=dev, generator=g) * 300.0
    inv = torch.tensor([1.0 / 1024], device=dev)
    ref = _seg_sums((g0 * inv).double() ** 2, seg64, n_seg)     # the kernel squares the fp32 unscaled value
    for write_back in (True, False):
        buf = g0.clone()
        fi = torch.zeros(1, device=dev)
        out0 = torch.rand(n_seg, device=dev, generator=g)
        out = out0.clone()
        Kn.grad_unscale_stats(buf, seg, out, inv_scale=inv, found_inf=fi, write_back=write_back)
        assert float(fi) == 0.0, "found_inf raised on a finite buffer"
        _rel_each(out.double() - out0.double(), ref, f"sumsq write_back={write_back}")
        if write_back:
            assert torch.equal(buf[~skip], g0[~skip] * inv) and torch.equal(buf[skip], g0[skip])
        else:
            assert torch.equal(buf.view(torch.int32), g0.view(torch.int32)), "write_back=0 modified the buffer"
    # without inv_scale (the grad_logger call): plain sums of squares
    out = torch.zeros(n_seg, device=dev)
    Kn.grad_unscale_stats(g0.clone(), seg, out, write_back=False)
    _rel_each(out, _seg_sums(g0.double() ** 2, seg64, n_seg), "sumsq without inv_scale")
    # NaN / -inf inside a live block (one in the last live block of the buffer)
    live_pos = torch.nonzero(~skip).view(-1)
    for bad, pos in ((float("nan"), int(live_pos[-1])), (float("-inf"), int(live_pos[len(live_pos) // 3]))):
        buf = g0.clone()
        buf[pos] = bad
        fi = torch.zeros(1, device=dev)
        Kn.grad_unscale_stats(buf, seg, torch.zeros(n_seg, device=dev), inv_scale=inv, found_inf=fi, write_back=False)
        assert float(fi) == 1.0, f"found_inf not raised by {bad}"
    out = torch.zeros(n_seg, device=dev)
    Kn.seg_abs_sum(g0, seg, out)
    _rel_each(out, _seg_sums(g0.double().abs(), seg64, n_seg), "seg_abs_sum")


@pytest.mark.parametrize("n_seg", [1, 33, 300])
def test_clip_coef_and_scale_flat(dev, n_seg):
    """vj_clip_coef over 1, 33 and 300 segments (the strided loop), and vj_scale_flat on both sides of coef = 1."""
    from jepa_b200 import kernels as Kn
    g = _gen(dev, n_seg)
    sumsq = torch.rand(n_seg, device=dev, generator=g) * 10
    total = float(sumsq.double().sum().sqrt())
    for max_norm, coef_ref in ((0.37 * total, 0.37 * total / (total + 1e-6)), (2.0 * total, 1.0)):
        out = torch.empty(2, device=dev)
        Kn.clip_coef(sumsq, max_norm, out[0:1], out[1:2])
        assert abs(float(out[0]) - total) <= 1e-5 * total, (n_seg, float(out[0]), total)
        assert abs(float(out[1]) - coef_ref) <= 1e-5 * coef_ref, (n_seg, float(out[1]), coef_ref)
    x0 = torch.randn(64 * 1001, device=dev, generator=g)
    for c in (1.0, 3.0):
        x = x0.clone()
        Kn.scale_flat(x, torch.tensor([c], device=dev))
        assert torch.equal(x.view(torch.int32), x0.view(torch.int32)), f"coef {c} >= 1 must leave the buffer alone"
    coef = torch.tensor([0.37], device=dev)
    x = x0.clone()
    Kn.scale_flat(x, coef)
    assert torch.equal(x, x0 * coef)


def test_ema_update_shadow_bit_exact(dev):
    """vj_ema_update_shadow == k.mul_(m).add_((1 - m) * q) op for op, and its shadow == the bf16 cast."""
    from jepa_b200 import kernels as Kn
    g = torch.Generator().manual_seed(6)
    n = 4096 * 3 + 64
    k, q = torch.randn(n, generator=g), torch.randn(n, generator=g)
    for m in (0.998, 0.99925, 1.0):
        kd = k.clone().to(dev)
        sh = torch.empty(n, dtype=BF16, device=dev)
        Kn.ema_update_shadow(kd, q.to(dev), m, sh)
        ref = k.clone()
        ref.mul_(m).add_((1. - m) * q)
        assert torch.equal(kd.cpu(), ref), m
        assert torch.equal(sh.cpu(), ref.to(BF16)), m
