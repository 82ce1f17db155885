"""Power of the GEMM comparator, on the CPU.  tests/test_gpu_gemm.py checks vj_gemm / vj_gemm_f16 with gemm_ref.check
against an fp64 reference.  Here the same comparator, on the same inputs, must pass an emulation that rounds where the
kernels round (fp32 product of the 16-bit operands, fp32 epilogue with torch's erf, one round-to-nearest to the stored
type) and must reject that emulation with one known fault at every case where the fault changes the result:
  k_tail_dropped       K rounded down to a multiple of 64 (the TMA zero-fill of the last k-block lost)
  k_block_dropped      one 64-wide k-block never multiplied
  k_block_twice        one k-block multiplied twice (a ring stage read again)
  bias_per_split       the bias added by every split-K piece instead of the one holding the first k-block
  bias_omitted
  alpha_after_bias     alpha (acc + bias) instead of alpha acc + bias
  aux_row_off_by_one   aux row m + 1 for output row m
  rowmap_ignored       aux row m instead of rowmap[m]
  period_128           aux row m % 128 (the tile height) instead of m % period
  tanh_gelu            the tanh approximation instead of erf
  grad_without_xphi    gelu'(x) = Phi(x), its x phi(x) term lost (GELU_GRAD's aux_out, DGELU)
  truncated_store      the 16-bit store truncates instead of rounding to nearest
  aux_out_activation   GELU's aux_out holds the activation instead of the pre-activation
  d0_overwritten       an accumulating GEMM stores instead of adding
  mn_blocks_swapped    the first two 64-wide blocks of an MN-major operand tile exchanged
The full-step weight-gradient shapes of the GPU file (up to 76 032 x 1536 x 384) are too large for a CPU suite; they use
the same comparator on the same kind of inputs as the sweep's weight-gradient cases here.
"""
import math

import pytest
import torch

import gemm_ref as R
from gemm_ref import BF16, EPI_ADD, EPI_DGELU, EPI_GELU, EPI_GELU_GRAD, EPI_MUL, F16, F32

DTS = (BF16, F16)
DT_IDS = ("bf16", "fp16")


def truncate(x, dt):
    """fp32 -> dt towards zero: where round-to-nearest went away from zero, one step back (sign-magnitude bits)"""
    h = x.to(dt)
    away = h.float().abs() > x.abs()
    return (h.view(torch.int16) - away.to(torch.int16)).view(dt)


def pieces(c):
    """split-K pieces per output tile as vj_gemm's header describes them (stream-K: at least two for some tile)"""
    kb = (c.K + 63) // 64
    if c.split_k < 0:
        return 2
    per = -(-kb // min(max(c.split_k, 1), kb))
    return -(-kb // per)


def emulate(c, t, fault=None):
    """(D, aux_out) of case c on inputs t as a kernel that rounds where ours do would store them, with `fault`."""
    A = (t.a.t() if c.a_mn else t.a).float()            # [M, K]
    B = (t.b if c.b_mn else t.b.t()).float()            # [K, N]
    w = torch.ones(c.K)
    blk = ((c.K + 63) // 64) // 2 * 64                  # a k-block in the middle (the only one if K <= 64)
    if fault == "k_tail_dropped":
        w[c.K // 64 * 64:] = 0
    elif fault == "k_block_dropped":
        w[blk:blk + 64] = 0
    elif fault == "k_block_twice":
        w[blk:blk + 64] = 2
    if fault == "mn_blocks_swapped":
        swap = torch.cat([torch.arange(64, 128), torch.arange(0, 64)])
        if c.b_mn and c.N >= 128:
            B = B.clone()
            B[:, :128] = B[:, swap]
        else:
            A = A.clone()
            A[:128] = A[swap]
    acc = (A * w) @ B
    bias = 0.0 if t.bias is None or fault == "bias_omitted" else t.bias * (pieces(c) if fault == "bias_per_split" else 1)
    v = (acc + bias) * c.alpha if fault == "alpha_after_bias" else acc * c.alpha + bias
    x = None
    if t.aux is not None:
        rows = R.aux_rows(c.M, t.rowmap, t.period, v.device)
        if fault == "rowmap_ignored":
            rows = torch.arange(c.M) % t.aux.shape[0]
        elif fault == "period_128":
            rows = torch.arange(c.M) % 128 % t.aux.shape[0]
        if fault == "aux_row_off_by_one":
            rows = (rows + 1) % t.aux.shape[0]
        x = t.aux.float()[rows]
    phi = lambda z: torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    cdf = lambda z: 0.5 * (1 + torch.erf(z / math.sqrt(2)))
    grad = (lambda z: cdf(z)) if fault == "grad_without_xphi" else (lambda z: cdf(z) + z * phi(z))
    gelu = lambda z: z * cdf(z)
    if fault == "tanh_gelu":
        gelu = lambda z: 0.5 * z * (1 + torch.tanh(math.sqrt(2 / math.pi) * (z + 0.044715 * z ** 3)))
    aux_out = None
    if c.epi == EPI_GELU:
        d, aux_out = gelu(v), (gelu(v) if fault == "aux_out_activation" else v)
    elif c.epi == EPI_GELU_GRAD:
        d, aux_out = gelu(v), grad(v)
    elif c.epi == EPI_ADD:
        d = v + x
    elif c.epi == EPI_MUL:
        d = v * x
    elif c.epi == EPI_DGELU:
        d = v * grad(x)
    else:
        d = v
    if t.d0 is not None and fault != "d0_overwritten":
        d = d + t.d0
    store = (lambda z: truncate(z, c.dt)) if fault == "truncated_store" else (lambda z: z.to(c.dt))
    return (d if c.d_f32 else store(d)), (store(aux_out) if c.aux_out else None)


def inputs(c):
    return R.controlled_inputs(c) if c.family == "controlled" else R.make_inputs(c)


def families(dt):
    """every case family of tests/test_gpu_gemm.py that fits a CPU"""
    out = [c for a_mn, b_mn in R.LAYOUTS for N in R.SWEEP_N for c in R.sweep_cases(dt, a_mn, b_mn, N)]
    out += R.epilogue_cases(dt) + R.split_cases(dt) + R.probe_cases(dt) + R.stride_cases(dt) + [R.patch_embed_case(dt)]
    out += [R.controlled_case(dt, EPI_GELU), R.controlled_case(dt, EPI_GELU_GRAD)]
    if dt == BF16:
        out += [R.controlled_case(dt, EPI_DGELU), R.controlled_case(dt, EPI_DGELU, b_mn=True)]
    return out


def missed(fault, cases):
    """ids of the cases whose faulty emulation the comparator lets through"""
    assert cases, "the fault applies to no case"
    out = []
    for c in cases:
        t = inputs(c)
        if not R.check(c, t, *emulate(c, t, fault)):
            out.append(c.id)
    return out


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_rounding_where_the_kernel_rounds_passes(dt):
    for c in families(dt):
        t = inputs(c)
        bad = R.check(c, t, *emulate(c, t))
        assert not bad, bad


# which cases a fault changes
APPLIES = {
    "k_tail_dropped": lambda c: c.K % 64 != 0,
    "k_block_dropped": lambda c: True,
    "k_block_twice": lambda c: True,
    "bias_per_split": lambda c: c.bias and pieces(c) > 1,
    "bias_omitted": lambda c: c.bias,
    "alpha_after_bias": lambda c: c.bias and c.alpha != 1.0,
    "aux_row_off_by_one": lambda c: c.aux != "",
    "rowmap_ignored": lambda c: c.aux == "rowmap",
    "period_128": lambda c: c.aux == "period" and c.M > R.PERIOD,
    "tanh_gelu": lambda c: c.epi in (EPI_GELU, EPI_GELU_GRAD),
    "grad_without_xphi": lambda c: c.epi == EPI_DGELU or (c.epi == EPI_GELU_GRAD and c.aux_out),
    "truncated_store": lambda c: not c.d_f32,
    "aux_out_activation": lambda c: c.epi == EPI_GELU and c.aux_out,
    "d0_overwritten": lambda c: c.accumulate,
    "mn_blocks_swapped": lambda c: (c.b_mn and c.N >= 128) or (c.a_mn and c.b_mn and c.M >= 128),
}


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
@pytest.mark.parametrize("fault", sorted(APPLIES))
def test_fault_rejected(fault, dt):
    cases = [c for c in families(dt) if c.family != "controlled" and APPLIES[fault](c)]
    if fault == "truncated_store":      # one element cannot be relied on to sit where truncation costs more than an ulp
        cases = [c for c in cases if c.M * c.N >= 4096]
    m = missed(fault, cases)
    assert not m, f"{fault} not rejected at {m}"


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_gelu_faults_rejected_on_controlled_preactivations(dt):
    for fault, epi in (("tanh_gelu", EPI_GELU), ("grad_without_xphi", EPI_GELU_GRAD), ("aux_out_activation", EPI_GELU),
                       ("truncated_store", EPI_GELU)) + ((("grad_without_xphi", EPI_DGELU),) if dt == BF16 else ()):
        assert not missed(fault, [R.controlled_case(dt, epi)]), fault


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_constants_are_not_wider_than_measured(dt, monkeypatch):
    """The bound's constants cannot be widened quietly: ulp is the stored type's unit roundoff, C_ACC stays within 4x of
    the largest accumulation error measured on the H100, and with every term 4x wider a truncating store would pass."""
    assert R.ULP == {BF16: 2.0 ** -8, F16: 2.0 ** -11, F32: 0.0}
    assert R.ACC_MEASURED <= R.C_ACC <= 4 * R.ACC_MEASURED
    c = R.Case("epilogue", dt, 300, 192, 328, bias=True)
    assert missed("truncated_store", [c]) == []
    monkeypatch.setattr(R, "C_ACC", 4 * R.C_ACC)
    monkeypatch.setattr(R, "ULP", {k: 4 * v for k, v in R.ULP.items()})
    assert missed("truncated_store", [c]) == [c.id]
