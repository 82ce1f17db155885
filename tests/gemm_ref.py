"""GEMM test inputs, an fp64 reference and the comparator, shared by tests/test_gpu_gemm.py (vj_gemm / vj_gemm_f16 on the
GPU) and tests/test_gemm_sensitivity_cpu.py (the same comparator against emulations of kernels with known faults, on the
same inputs).  Everything here runs on the device of the tensors it is given.

The reference is the operation, not the kernel: D = epi(alpha * A B^T + bias) in float64 from exactly the 16-bit values
the kernel reads, the GELU by its textbook formula.  Nothing below knows a tile size.

Bound, elementwise, for an output stored with unit roundoff `ulp` (2^-8 bf16, 2^-11 fp16, 0 fp32: the most one
round-to-nearest can cost relative to the value):

    |got - ref| <= ulp |ref| + floor + gain * C_ACC * absdot + extra

  floor    half the spacing of the stored type's subnormals (2^-25 fp16: below 2^-14 its values are 2^-24 apart).

  absdot   |alpha| (|A| |B|^T) + |bias| (+ |aux| for ADD, + |d0| when accumulating): the sum of the magnitudes of
           everything the kernel adds in fp32.  It is the scale of the accumulation error and does not shrink under
           cancellation.  A wrong k-block, K tail, bias or aux row errs by about absdot / sqrt(K), thousands of times
           C_ACC * absdot.
  gain     what the epilogue multiplies the accumulator's error by: 1; |aux| for MUL; |gelu'(aux)| for DGELU;
           GELU_GAIN = 1.13 for GELU / GELU_GRAD (max |gelu'| = 1.129 at x = sqrt 2).
  extra    the epilogue's own approximations.  erf_as (Abramowitz-Stegun 7.1.26) is within 1.5e-7 of erf, so Phi is within
           7.5e-8 and, with the fp32 roundings of the polynomial and of __expf, within PHI_ABS = 2.5e-7: the activation
           gets PHI_ABS |x|.  gelu'(x) = Phi + x phi(x) adds __expf's error in phi: GRAD_ABS = 1e-6 absolute on the
           GELU_GRAD aux_out, GRAD_ABS |v| on a DGELU output.

C_ACC is measured.  On an H100 (80 GB HBM3, 700 W limit) the largest |err| / absdot of any fp32-stored output of
tests/test_gpu_gemm.py is ACC_MEASURED = 7.1e-7 (the plain-epilogue sweep in fp16; 6.1e-7 in bf16, 6.0e-7 over the
epilogues, 5.6e-7 over split-K / stream-K, 3.6e-7 at the probe's call sites, 3.6e-8 for the weight gradients at step
shapes, whose accumulation is promoted every 256 products).  C_ACC = 2e-6 is 2.8 times that, so the worst err / bound
of an fp32 output is 0.35.  For 16-bit outputs the rounding term dominates and the worst err / bound sits just under 1
(measured 0.94 .. 0.995 per family: an element at the bottom of its binade whose fp32 value lies next to a tie); a
store that truncates instead of rounding errs by up to 2 ulp |ref| and fails.  Run the GPU file with -s to print the
worst err / bound per case family.
"""
import math
import zlib
from dataclasses import dataclass
from types import SimpleNamespace

import torch

EPI_NONE, EPI_GELU, EPI_ADD, EPI_DGELU, EPI_MUL, EPI_GELU_GRAD = 0, 1, 2, 3, 4, 5
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
ULP = {BF16: 2.0 ** -8, F16: 2.0 ** -11, F32: 0.0}
FLOOR = {BF16: 2.0 ** -134, F16: 2.0 ** -25, F32: 0.0}
ACC_MEASURED = 7.1e-7
C_ACC = 2e-6
GELU_GAIN = 1.13
PHI_ABS = 2.5e-7
GRAD_ABS = 1e-6
WORST = {}              # case family -> largest err / bound seen; the GPU file prints it at teardown
WORST_ACC = {}          # case family -> largest |err| / absdot of an fp32-stored output


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def aux_rows(M, aux_rowmap, aux_period, device):
    if aux_rowmap is not None:
        return aux_rowmap.long()
    r = torch.arange(M, device=device)
    return r % aux_period if aux_period > 0 else r


def reference(a, b, *, a_mn=False, b_mn=False, bias=None, alpha=1.0, epi=EPI_NONE, aux=None, aux_rowmap=None,
              aux_period=0, d0=None):
    """fp64 D [M, N], aux_out (GELU: the pre-activation, GELU_GRAD: gelu' of it, else None) and absdot (module
    docstring).  a is [M, K] ([K, M] if a_mn), b is [N, K] ([K, N] if b_mn), as the kernel takes them."""
    A = a.double().t() if a_mn else a.double()
    B = b.double() if b_mn else b.double().t()       # [K, N]
    v = alpha * (A @ B)
    absdot = abs(alpha) * (A.abs() @ B.abs())
    if bias is not None:
        v = v + bias.double()
        absdot = absdot + bias.double().abs()
    x = None
    if epi in (EPI_ADD, EPI_MUL, EPI_DGELU):
        x = aux.double()[aux_rows(v.shape[0], aux_rowmap, aux_period, v.device)]
    aux_out = None
    if epi == EPI_GELU:
        d, aux_out = gelu64(v), v
    elif epi == EPI_GELU_GRAD:
        d, aux_out = gelu64(v), gelu_grad64(v)
    elif epi == EPI_ADD:
        d, absdot = v + x, absdot + x.abs()
    elif epi == EPI_MUL:
        d = v * x
    elif epi == EPI_DGELU:
        d = v * gelu_grad64(x)
    else:
        d = v
    if d0 is not None:
        d, absdot = d + d0.double(), absdot + d0.double().abs()
    return d, aux_out, absdot


def compare(name, got, ref, absdot, ulp, gain=1.0, extra=0.0, bad=None, floor=0.0):
    """Appends to `bad` (and returns it) a line if got leaves the bound of the module docstring anywhere or is not finite
    where ref is; keeps the worst err / bound of family `name` in WORST."""
    bad = [] if bad is None else bad
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    bound = ulp * ref.abs() + floor + gain * C_ACC * absdot + extra
    ratio = torch.nan_to_num(err / bound, nan=math.inf)       # NaN: got is NaN, or 0 / 0
    ratio[err == 0] = 0.0
    worst = float(ratio.max())
    WORST[name] = max(WORST.get(name, 0.0), worst)
    if ulp == 0.0:
        acc = torch.nan_to_num(err / (gain * absdot), nan=math.inf)
        acc[err == 0] = 0.0
        WORST_ACC[name] = max(WORST_ACC.get(name, 0.0), float(acc.max()))
    if not worst <= 1.0:
        at = tuple(int(i) for i in torch.nonzero(ratio == worst)[0])
        bad.append(f"{name}: worst err/bound {worst:.4g} at {at} (got {float(got[at]):.9g}, ref {float(ref[at]):.9g}, "
                   f"bound {float(bound[at]):.3g})")
    return bad


# ---------------------------------------------------------------------------------------------------------- cases
@dataclass(frozen=True)
class Case:
    family: str
    dt: torch.dtype
    M: int
    N: int
    K: int
    a_mn: bool = False
    b_mn: bool = False
    d_f32: bool = False
    epi: int = EPI_NONE
    aux: str = ""            # "16": 16-bit [M, N]; "f32": fp32 [M, N]; "rowmap": fp32 table + row map; "period": fp32 table
    bias: bool = False
    alpha: float = 1.0
    aux_out: bool = False
    accumulate: bool = False
    split_k: int = 1

    @property
    def id(self):
        s = f"{self.M}x{self.N}x{self.K}-{int(self.a_mn)}{int(self.b_mn)}-{'f32' if self.d_f32 else '16'}-e{self.epi}{self.aux}"
        s += f"-a{self.alpha:g}" + ("-bias" if self.bias else "") + ("-auxout" if self.aux_out else "")
        return s + ("-acc" if self.accumulate else "") + (f"-s{self.split_k}" if self.split_k != 1 else "")

    @property
    def out_dtype(self):
        return F32 if self.d_f32 else self.dt


ROWMAP_ROWS, PERIOD = 50, 37      # the table of a row map is shorter than M: rows repeat, out of order; 37 does not divide 128


def make_inputs(c):
    """Seeded CPU tensors of case c, in the layout the kernel takes them: a, b, bias, aux, rowmap, period, d0 (None where
    the case has none).  N(0, 1) activations, N(0, 1/K) weights, so accumulators are O(1)."""
    g = torch.Generator().manual_seed(zlib.crc32(f"{c.family} {c.id} {c.dt}".encode()))
    rn = lambda *s: torch.randn(*s, generator=g)
    a = rn(c.M, c.K).to(c.dt)
    b = (rn(c.N, c.K) * c.K ** -0.5).to(c.dt)
    tr = lambda x: torch.empty(x.shape[1], x.shape[0], dtype=x.dtype).copy_(x.t())   # dense strides even for one row
    t = SimpleNamespace(a=tr(a) if c.a_mn else a, b=tr(b) if c.b_mn else b, bias=None, aux=None, rowmap=None, period=0,
                        d0=None)
    if c.bias:
        t.bias = rn(c.N) * 0.5
    if c.aux == "16":
        t.aux = (rn(c.M, c.N) * 2).to(c.dt)
    elif c.aux == "f32":
        t.aux = rn(c.M, c.N) * 2
    elif c.aux == "rowmap":
        t.aux = rn(ROWMAP_ROWS, c.N) * 2
        t.rowmap = torch.randint(0, ROWMAP_ROWS, (c.M,), generator=g, dtype=torch.int32)
    elif c.aux == "period":
        t.aux, t.period = rn(PERIOD, c.N) * 2, PERIOD
    if c.accumulate:
        t.d0 = rn(c.M, c.N)
    return t


def to_device(t, dev):
    return SimpleNamespace(**{k: v.to(dev) if torch.is_tensor(v) else v for k, v in vars(t).items()})


def expected(c, t):
    """reference() of case c on inputs t, with the gains and extras of the module docstring: dict d, aux_out, absdot, gain,
    extra, aux_extra."""
    d, aux_out, absdot = reference(t.a, t.b, a_mn=c.a_mn, b_mn=c.b_mn, bias=t.bias, alpha=c.alpha, epi=c.epi, aux=t.aux,
                                   aux_rowmap=t.rowmap, aux_period=t.period, d0=t.d0)
    gain, extra, aux_extra = 1.0, 0.0, 0.0
    if c.epi in (EPI_GELU, EPI_GELU_GRAD, EPI_DGELU):
        pre = reference(t.a, t.b, a_mn=c.a_mn, b_mn=c.b_mn, bias=t.bias, alpha=c.alpha)[0]     # v = alpha acc + bias
    if c.epi in (EPI_GELU, EPI_GELU_GRAD):
        gain, extra = GELU_GAIN, PHI_ABS * pre.abs()
        aux_extra = GRAD_ABS if c.epi == EPI_GELU_GRAD else 0.0
    elif c.epi in (EPI_MUL, EPI_DGELU):
        x = t.aux.double()[aux_rows(c.M, t.rowmap, t.period, d.device)]
        gain = x.abs() if c.epi == EPI_MUL else gelu_grad64(x).abs()
        extra = GRAD_ABS * pre.abs() if c.epi == EPI_DGELU else 0.0
    return dict(d=d, aux_out=aux_out, absdot=absdot, gain=gain, extra=extra, aux_extra=aux_extra)


def check(c, t, got_d, got_aux_out=None, exp=None):
    """Violations (empty: pass) of the kernel outputs of case c against the fp64 reference of inputs t."""
    e = expected(c, t) if exp is None else exp
    fam = f"{c.family} {'bf16' if c.dt == BF16 else 'fp16'}{' f32 D' if c.d_f32 else ''}"
    bad = compare(fam, got_d, e["d"], e["absdot"], ULP[c.out_dtype], e["gain"], e["extra"], floor=FLOOR[c.out_dtype])
    if got_aux_out is not None:
        # aux_out is the accumulator (GELU) or gelu' of it (GELU_GRAD, |gelu''| <= 0.5 at 0) rounded once to 16 bits
        compare(fam + " aux_out", got_aux_out, e["aux_out"], e["absdot"], ULP[c.dt], 1.0, e["aux_extra"], bad, FLOOR[c.dt])
    return [f"{c.id}: {b}" for b in bad]


M_KMAJOR = (1, 8, 63, 64, 65, 127, 128, 129, 200, 1050)
M_MNMAJOR = (8, 64, 72, 120, 128, 136, 200, 1048)
# reduction lengths.  K-major operands need 16-byte rows (K % 8 == 0 when dense): tails of 8 and 56, one block, one block
# and a tail, many blocks and a tail, and 47 / 48 k-blocks (3008, 3016 .. 3072): either side of the cooperative
# 128 x 256 schedule's threshold.  Where K is the outer dimension of both operands (weight gradients) any count goes.
K_KMAJOR = (8, 56, 64, 72, 1000, 3008, 3016, 3072)
K_OUTER = (1, 7, 13, 64, 174, 333, 1000, 4099)
SWEEP_N = (64, 192, 128, 384, 256, 512)
LAYOUTS = ((False, False), (False, True), (True, True))


def sweep_cases(dt, a_mn, b_mn, N):
    """Plain epilogue: every M with one K each (rotating with N so that every (tile width, K) pair occurs), both output
    types; at N % 256 == 0 also the cooperative schedule at ragged M (at M = 1050 the second warpgroup's half of the last
    tile lies wholly past M) and just below its threshold."""
    Ms, Ks = (M_MNMAJOR, K_OUTER) if a_mn else (M_KMAJOR, K_KMAJOR)
    shift = SWEEP_N.index(N)
    mk = [(M, Ks[(i + shift) % len(Ks)]) for i, M in enumerate(Ms)]
    if not a_mn and N % 256 == 0:
        mk += [(1050, 3016), (1050, 3072), (129, 3008), (65, 3016), (1, 3072), (127, 3072)]
    if a_mn:
        mk += [(8, 1), (64, 174), (1048, 4099)]
    out = []
    for M, K in dict.fromkeys(mk):
        for d_f32 in (False, True):
            if a_mn and not d_f32 and dt != BF16:
                continue            # fp16 weight gradients are instantiated with fp32 D only
            out.append(Case("sweep", dt, M, N, K, a_mn, b_mn, d_f32))
    return out


EPI_SHAPES = ((300, 192, 328), (333, 384, 200), (257, 512, 3080))     # 64-wide, 128-wide, cooperative 256-wide; ragged M


def epilogue_cases(dt):
    """Every instantiated epilogue on each tile width.  Bias and alpha rotate through (1, 0.5, -2) and no bias."""
    out = []
    for i, (M, N, K) in enumerate(EPI_SHAPES):
        alphas = [(1.0, 0.5, -2.0)[(i + j) % 3] for j in range(16)]
        mk = lambda j, **kw: Case("epilogue", dt, M, N, K, alpha=alphas[j], **kw)
        out += [
            mk(0, bias=True), mk(1), mk(2, bias=True, d_f32=True),
            mk(3, epi=EPI_GELU, bias=True), mk(4, epi=EPI_GELU, bias=True, aux_out=True), mk(5, epi=EPI_GELU),
            mk(6, epi=EPI_GELU_GRAD, bias=True, aux_out=True), mk(7, epi=EPI_GELU_GRAD, bias=True),
            mk(8, epi=EPI_ADD, aux="16", bias=True), mk(9, epi=EPI_ADD, aux="16"),
            mk(10, epi=EPI_ADD, aux="f32", bias=True), mk(11, epi=EPI_ADD, aux="f32", d_f32=True),
            mk(12, epi=EPI_ADD, aux="rowmap", bias=True), mk(13, epi=EPI_ADD, aux="rowmap", bias=True, d_f32=True),
            mk(14, epi=EPI_ADD, aux="period", bias=True), mk(15, epi=EPI_ADD, aux="period", d_f32=True),
            mk(0, epi=EPI_MUL, aux="16", b_mn=True), mk(1, epi=EPI_MUL, aux="16", b_mn=True, bias=True),
            mk(2, b_mn=True, bias=True), mk(3, b_mn=True, d_f32=True, bias=True),
        ]
        if dt == BF16:
            out += [mk(4, epi=EPI_DGELU, aux="16"), mk(5, epi=EPI_DGELU, aux="16", b_mn=True, bias=True)]
    return out


# split_k values: clamped when above the k-block count; 10 k-blocks / 4 -> 3 per split, 4 splits (the last holds one);
# 9 k-blocks / 4 -> 3 per split, 3 splits.  -1 is stream-K (accumulating only).
def split_cases(dt):
    out = []
    for a_mn, b_mn in LAYOUTS:
        M = 264 if a_mn else 261
        for N, K, splits in ((192, 640, (1, 2, 3, 4, 7, 16, 100, -1)), (384, 576, (2, 4, 9, -1)), (256, 3096, (3, 16, -1))):
            for s in splits:
                for acc in ((True,) if s < 0 else (False, True)):
                    out.append(Case("split", dt, M, N, K, a_mn, b_mn, True, bias=True, alpha=(0.5 if acc else -2.0),
                                    accumulate=acc, split_k=s))
    # stream-K with tiles * k-blocks below, at and above an H100's 132 SMs: 2 x 1 tiles x 3 k-blocks = 6; 3 x 2 x 22 = 132;
    # 5 x 3 x 30 = 450
    for M, N, K in ((256, 128, 192), (384, 256, 1408), (640, 384, 1904)):
        out.append(Case("split", dt, M, N, K, True, True, True, bias=True, alpha=0.5, accumulate=True, split_k=-1))
        out.append(Case("split", dt, M - 3, N, K, False, True, True, bias=True, alpha=0.5, accumulate=True, split_k=-1))
    return out


def probe_cases(dt):
    """The attentive probe's GEMMs at their real sizes (pooler.py): logits^T = W pooled^T + bias through an fp32 aux; the
    head's weight gradient and the query-token gradient as dgrad-layout GEMMs accumulating into fp32; dpooled through the
    weight-gradient kernel with a plain fp32 store and K = class count; the split_k = 1 accumulating weight gradient."""
    out = []
    for C, D in ((174, 1024), (400, 1280), (1000, 1024)):
        out.append(Case("probe", dt, C, 64, D, d_f32=True, epi=EPI_ADD, aux="f32"))                      # logits^T
        out.append(Case("probe", dt, C, D, 64, b_mn=True, d_f32=True, accumulate=True))                  # dW += dlogits^T pooled
        out.append(Case("probe", dt, 64, D, C, True, True, True))                                        # dpooled = dlogits W
    for nq in (1, 3):
        out.append(Case("probe", dt, nq, 1024, 1024, b_mn=True, d_f32=True, accumulate=True))            # query tokens
        out.append(Case("probe", dt, nq, 1280, 1280, b_mn=True, d_f32=True, accumulate=True))
    for D, rows in ((1024, 8), (1280, 1568)):
        out.append(Case("probe", dt, D, D, rows, True, True, True, accumulate=True))                     # _wgrad(split_k=1)
    return out


def patch_embed_case(dt):
    """engine.py's patch embedding: row-mapped fp32 positional table into 16-bit D at K = 3 * 2 * 16 * 16."""
    return Case("patch embed", dt, 1003, 384, 1536, epi=EPI_ADD, aux="rowmap", bias=True)


def stride_cases(dt):
    """Run with every operand a column window of a wider tensor (row stride larger than the width)."""
    return [Case("strided", dt, 200, 192, 328, epi=EPI_GELU, bias=True, aux_out=True),
            Case("strided", dt, 200, 384, 328, epi=EPI_ADD, aux="16", bias=True),
            Case("strided", dt, 200, 256, 328, b_mn=True, epi=EPI_MUL, aux="16"),
            Case("strided", dt, 200, 128, 333, True, True, True, accumulate=True)]


# Controlled pre-activations: B = I (64 x 64), alpha = 1, no bias, so the accumulator is A exactly and absdot = |A|.
def controlled_values(dt):
    """x on a dense grid over [-12, 12], +-0, every 16-bit value of [-0.77, -0.73] (the GELU's minimum is at -0.7518),
    every bf16 / every 8th fp16 value of 5 <= |x| <= 9 (where 1 - erf underflows the polynomial) and large finite values."""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dt).float()
    bits = bits[torch.isfinite(bits)]
    near_min = bits[(bits >= -0.77) & (bits <= -0.73)]
    tails = bits[(bits.abs() >= 5) & (bits.abs() <= 9)][::8 if dt == F16 else 1]
    big = [3e4, -3e4, 6e4, -6e4] if dt == F16 else [1e30, -1e30, 3e38, -3e38, 1e5, -1e5]
    x = torch.cat([torch.linspace(-12, 12, 6001), torch.tensor([0.0, -0.0, 1e-30, -1e-30] + big), near_min, tails]).to(dt)
    pad = (-x.numel()) % 64
    return torch.cat([x, x[:pad]]).view(-1, 64)


def controlled_case(dt, epi, b_mn=False):
    return Case("controlled", dt, controlled_values(dt).shape[0], 64, 64, b_mn=b_mn, epi=epi,
                aux="16" if epi == EPI_DGELU else "", aux_out=epi in (EPI_GELU, EPI_GELU_GRAD))


def controlled_inputs(c):
    """GELU / GELU_GRAD: A holds the values; DGELU: aux holds them and A is +-1, +-2."""
    x = controlled_values(c.dt)
    eye = torch.eye(64).to(c.dt)
    t = SimpleNamespace(a=x, b=eye, bias=None, aux=None, rowmap=None, period=0, d0=None)
    if c.epi == EPI_DGELU:
        t.aux = x
        t.a = ((torch.arange(x.numel()) % 4).float() - 1.5).mul(4 / 3).round().view_as(x).to(c.dt)   # -2, -1, 1, 2
    return t

