"""vj_gemm / vj_gemm_f16 one launch at a time against the fp64 reference and comparator of tests/gemm_ref.py: every
schedule (64- / 128-wide ping-pong tiles, the cooperative 128 x 256 tile, the weight-gradient kernel), operand layout,
instantiated epilogue, split-K / stream-K decomposition and row stride, at ragged M, K tails and the attentive probe's
real call sites.  Every output is compared whole, lies inside a larger allocation whose guard rows and columns must stay
bit-unchanged, and starts as NaN (as d0 when accumulating, as zero for split-K).  tests/test_gemm_sensitivity_cpu.py
shows that the comparator rejects known faults on these inputs.  Run with -s for the worst err / bound per case family.
"""
import pytest
import torch

import gemm_ref as R
from gemm_ref import BF16, EPI_ADD, EPI_DGELU, EPI_GELU, EPI_GELU_GRAD, EPI_MUL, F16, F32, Case

pytestmark = pytest.mark.gpu
DTS = pytest.mark.parametrize("dt", (BF16, F16), ids=("bf16", "fp16"))
GUARD_ROWS, SENTINEL = 64, 1.5


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    yield torch.device("cuda:0")
    _lib.call("vj_set_sm_limit", 0)
    for k in sorted(R.WORST):
        acc = f"   |err| / absdot {R.WORST_ACC[k]:.3g}" if k in R.WORST_ACC else ""
        print(f"\nworst err/bound {k}: {R.WORST[k]:.3g}{acc}")


def bits(x):
    return x.view(torch.int32 if x.dtype == F32 else torch.int16)


class Out:
    """An M x N output inside a larger allocation: GUARD_ROWS rows below it and, with pad > 0, 8 guard columns to its left
    and pad - 8 to its right (the window starts 16-byte aligned).  Guards hold a finite sentinel, so that a stray
    reduce-add changes them too; the window holds `fill` (NaN unless given)."""

    def __init__(self, M, N, dtype, dev, pad=0, fill=None):
        self.full = torch.full((M + GUARD_ROWS, N + pad), SENTINEL, dtype=dtype, device=dev)
        self.window = (slice(0, M), slice(8 if pad else 0, (8 if pad else 0) + N))
        self.view = self.full[self.window]
        self.view.copy_(torch.full((M, N), float("nan"), device=dev) if fill is None else fill)
        self.before = self.full.clone()

    def guards_unchanged(self):
        now = self.full.clone()
        now[self.window] = self.before[self.window]
        return torch.equal(bits(now), bits(self.before))

    def untouched(self):
        return torch.equal(bits(self.full), bits(self.before))


def gemm_args(c, t, out, aux_out=None):
    """the C ABI's argument list for case c on device tensors (row strides from the tensors)"""
    p = lambda x: None if x is None else x.data_ptr()
    ld = lambda x: 0 if x is None else x.stride(0)
    return [p(t.a), ld(t.a), int(c.a_mn), p(t.b), ld(t.b), int(c.b_mn), p(out), ld(out), int(out.dtype == F32), c.M, c.N,
            c.K, p(t.bias), float(c.alpha), c.epi, p(t.aux), ld(t.aux), int(t.aux is not None and t.aux.dtype == F32),
            p(t.rowmap), t.period, p(aux_out), ld(aux_out), c.split_k, int(c.accumulate),
            torch.cuda.current_stream().cuda_stream]


def entry(c):
    return "vj_gemm" if c.dt == BF16 else "vj_gemm_f16"


def launch(c, t, out, aux_out=None):
    """through kernels.gemm when every tensor is contiguous (it insists), else through the C ABI"""
    from jepa_b200 import _lib, kernels as Kn
    if all(x.is_contiguous() for x in (t.a, t.b, out, t.aux, aux_out) if x is not None):
        return Kn.gemm(t.a, t.b, out, a_mn=c.a_mn, b_mn=c.b_mn, bias=t.bias, alpha=c.alpha, epi=c.epi, aux=t.aux,
                       aux_rowmap=t.rowmap, aux_period=t.period, aux_out=aux_out, split_k=c.split_k,
                       accumulate=c.accumulate)
    return _lib.call(entry(c), *gemm_args(c, t, out, aux_out))


def outputs(c, t, dev, pad):
    fill = t.d0 if c.accumulate else (torch.zeros(c.M, c.N, device=dev) if c.split_k != 1 else None)   # split-K adds
    return Out(c.M, c.N, c.out_dtype, dev, pad, fill), (Out(c.M, c.N, c.dt, dev, pad) if c.aux_out else None)


def run_case(dev, c, pad=0, t=None):
    """Launches c; returns the violations (bound, guards) and the outputs."""
    t = R.to_device(R.make_inputs(c), dev) if t is None else t
    out, xo = outputs(c, t, dev, pad)
    launch(c, t, out.view, xo.view if xo else None)
    torch.cuda.synchronize()
    bad = R.check(c, t, out.view, xo.view if xo else None)
    if not out.guards_unchanged() or (xo is not None and not xo.guards_unchanged()):
        bad.append(f"{c.id}: guard rows / columns written")
    return bad, out.view, (xo.view if xo else None)


def run_all(dev, cases):
    bad = []
    for i, c in enumerate(cases):
        bad += run_case(dev, c, pad=16 * (i % 2))[0]     # every other case with guard columns, i.e. through the C ABI
    assert not bad, "\n".join(bad)


def rejected(dev, c, t=None, override=None):
    """vj_gemm returns < 0 with a message and writes nothing.  override: position in gemm_args -> value (a pointer
    override is relative to this call's own buffers only in that it keeps their alignment)"""
    from jepa_b200 import _lib
    t = R.to_device(R.make_inputs(c), dev) if t is None else t
    out, xo = outputs(c, t, dev, 16)
    args = gemm_args(c, t, out.view, xo.view if xo else None)
    for k, v in (override or {}).items():
        args[k] = v
    lib = _lib.load()
    rc = getattr(lib, entry(c))(*args)
    torch.cuda.synchronize()
    assert rc < 0 and lib.vj_last_error_string(), f"{c.id} {override}: rc {rc}"
    assert out.untouched() and (xo is None or xo.untouched()), f"{c.id} {override}: output written"


# ------------------------------------------------------------------------------- a. schedule x layout x shape sweep
@DTS
@pytest.mark.parametrize("N", R.SWEEP_N)
@pytest.mark.parametrize("a_mn,b_mn", R.LAYOUTS, ids=("kk", "kmn", "mnmn"))
def test_sweep_plain_epilogue(dev, dt, a_mn, b_mn, N):
    run_all(dev, R.sweep_cases(dt, a_mn, b_mn, N))


# ---------------------------------------------------------------------------------- b. every instantiated epilogue
@DTS
@pytest.mark.parametrize("shape", R.EPI_SHAPES, ids=("bn64", "bn128", "coop256"))
def test_every_instantiated_epilogue(dev, dt, shape):
    run_all(dev, [c for c in R.epilogue_cases(dt) if (c.M, c.N, c.K) == shape])


@pytest.mark.parametrize("c", [
    Case("reject", BF16, 128, 128, 128, epi=EPI_GELU, d_f32=True),
    Case("reject", BF16, 128, 128, 128, b_mn=True, epi=EPI_MUL, aux="f32"),
    Case("reject", BF16, 128, 128, 128, a_mn=True),
    Case("reject", BF16, 128, 128, 128, epi=EPI_DGELU, aux="f32"),
    Case("reject", F16, 128, 128, 128, epi=EPI_DGELU, aux="16"),
    Case("reject", F16, 128, 128, 128, a_mn=True, b_mn=True),
    Case("reject", BF16, 128, 128, 128, a_mn=True, b_mn=True, epi=EPI_ADD, aux="f32", d_f32=True),
], ids=lambda c: ("bf16-" if c.dt == BF16 else "fp16-") + c.id)
def test_combination_not_instantiated_is_an_error(dev, c):
    rejected(dev, c)


# ------------------------------------------------------------------------------------ c. controlled pre-activations
@DTS
@pytest.mark.parametrize("epi", (EPI_GELU, EPI_GELU_GRAD), ids=("gelu", "gelu_grad"))
def test_gelu_on_controlled_preactivations(dev, dt, epi):
    c = R.controlled_case(dt, epi)
    t = R.to_device(R.controlled_inputs(c), dev)
    bad, d, xo = run_case(dev, c, t=t)
    assert not bad, "\n".join(bad)
    x, d, xo = t.a.double(), d.double(), xo.double()
    assert torch.isfinite(d).all() and torch.isfinite(xo).all()
    assert (d[x < 0] <= 0).all() and (d[x <= -1e4] == 0).all() and torch.equal(d[x >= 1e4], x[x >= 1e4])
    if epi == EPI_GELU:
        assert torch.equal(xo, x)            # the pre-activation, stored as it was read
    else:
        assert (xo[x >= 1e4] == 1).all() and (xo[x <= -1e4] == 0).all()


@pytest.mark.parametrize("b_mn", (False, True), ids=("kk", "kmn"))
def test_dgelu_on_controlled_preactivations(dev, b_mn):
    c = R.controlled_case(BF16, EPI_DGELU, b_mn)
    t = R.to_device(R.controlled_inputs(c), dev)
    bad, d, _ = run_case(dev, c, t=t)
    assert not bad, "\n".join(bad)
    x, a, d = t.aux.double(), t.a.double(), d.double()
    assert torch.isfinite(d).all()
    assert torch.equal(d[x >= 1e4], a[x >= 1e4]) and (d[x <= -1e4] == 0).all()


# -------------------------------------------------------------------------------- d. split-K, stream-K, accumulate
@DTS
@pytest.mark.parametrize("a_mn,b_mn", R.LAYOUTS, ids=("kk", "kmn", "mnmn"))
def test_split_k_stream_k_accumulate(dev, dt, a_mn, b_mn):
    run_all(dev, [c for c in R.split_cases(dt) if (c.a_mn, c.b_mn) == (a_mn, b_mn)])


@pytest.mark.parametrize("limit", (1, 7, 131))
def test_split_k_with_few_ctas(dev, limit):
    """vj_set_sm_limit: one CTA walks many (tile, k-range) pieces, in both kernels, classic and stream-K."""
    from jepa_b200 import _lib
    cases = [c for c in R.split_cases(BF16) if (c.N, c.K) == (192, 640) and c.split_k in (7, -1) and c.accumulate]
    cases += [c for c in R.split_cases(F16) if c.K == 1904]
    assert len(cases) == 8
    _lib.call("vj_set_sm_limit", limit)
    try:
        run_all(dev, cases)
    finally:
        _lib.call("vj_set_sm_limit", 0)


@pytest.mark.parametrize("c", [
    Case("reject", BF16, 128, 128, 256, split_k=2),                                         # 16-bit D, split-K
    Case("reject", BF16, 128, 128, 256, accumulate=True),                                   # 16-bit D, accumulate
    Case("reject", F16, 128, 128, 256, split_k=-1, accumulate=True),                        # 16-bit D, stream-K
    Case("reject", BF16, 128, 128, 256, d_f32=True, split_k=-1),                            # stream-K without accumulate
    Case("reject", BF16, 128, 128, 256, d_f32=True, epi=EPI_ADD, aux="16", split_k=2),      # 16-bit aux, split-K
    Case("reject", BF16, 128, 128, 256, d_f32=True, epi=EPI_ADD, aux="f32", split_k=2),     # every piece would add the aux
    Case("reject", F16, 128, 128, 256, d_f32=True, epi=EPI_ADD, aux="period", split_k=4, accumulate=True),
], ids=lambda c: ("bf16-" if c.dt == BF16 else "fp16-") + c.id)
def test_split_k_argument_checks(dev, c):
    rejected(dev, c)


# ---------------------------------------------------------------------------------------- e. the probe's call sites
@DTS
def test_probe_call_sites(dev, dt):
    """pooler.py's GEMMs at their real sizes, A a 16-byte-aligned slice out of a larger flat buffer as FlatParamStore hands
    the weights over; and engine.py's patch embedding (row-mapped fp32 aux into 16-bit D at K = 1536)."""
    bad = []
    for c in R.probe_cases(dt) + [R.patch_embed_case(dt)]:
        t = R.to_device(R.make_inputs(c), dev)
        flat = torch.full((t.a.numel() + 4104,), 3.0, dtype=dt, device=dev)
        flat[4096:4096 + t.a.numel()] = t.a.reshape(-1)
        t.a = flat[4096:4096 + t.a.numel()].view(t.a.shape)
        bad += run_case(dev, c, t=t)[0]
    assert not bad, "\n".join(bad)


# ------------------------------------------------------------------------------------------------- f. row strides
def window(x, dev):
    """x as a column window of a tensor 24 columns wider (8 to the left: the base stays 16-byte aligned)"""
    wide = torch.full((x.shape[0], x.shape[1] + 24), 3.0, dtype=x.dtype, device=dev)
    wide[:, 8:8 + x.shape[1]] = x
    return wide[:, 8:8 + x.shape[1]]


@DTS
@pytest.mark.parametrize("i", range(4), ids=("gelu_auxout", "add16", "dgrad_mul", "wgrad_f32"))
def test_row_strides_larger_than_the_width(dev, dt, i):
    """lda, ldb, ldd, ldaux and ldauxout each larger than the logical width, through the C ABI"""
    c = R.stride_cases(dt)[i]
    t = R.to_device(R.make_inputs(c), dev)
    t.a, t.b = window(t.a, dev), window(t.b, dev)
    if t.aux is not None:
        t.aux = window(t.aux, dev)
    bad = run_case(dev, c, pad=24, t=t)[0]
    assert not bad, "\n".join(bad)


BAD_ARGS = [      # what, fp32 D, position in the C ABI's argument list -> value (pointers: byte offset)
    ("A base 8 bytes off", False, {0: 8}), ("B base 8 bytes off", False, {3: 8}), ("D base 4 bytes off", True, {6: 4}),
    ("lda % 8", False, {1: 132}), ("ldb % 8", False, {4: 132}), ("ldd % 8, 16-bit D", False, {7: 148}),
    ("ldd % 4, fp32 D", True, {7: 146}), ("N % 64", False, {10: 96}), ("MN-major A, M % 8", True, {2: 1, 5: 1, 9: 124}),
    ("M = 0", False, {9: 0}), ("N = 0", False, {10: 0}), ("K = 0", False, {11: 0}), ("epilogue 9", False, {14: 9}),
]


@pytest.mark.parametrize("why,d_f32,override", BAD_ARGS, ids=[b[0].replace(" ", "_") for b in BAD_ARGS])
def test_bad_arguments_are_errors(dev, why, d_f32, override):
    c = Case("reject", BF16, 128, 128, 128, d_f32=d_f32)
    t = R.to_device(R.make_inputs(c), dev)
    base = gemm_args(c, t, Out(c.M, c.N, c.out_dtype, dev, 16).view)
    rejected(dev, c, t=t, override={k: base[k] + v if k in (0, 3, 6) else v for k, v in override.items()})


# ------------------------------------------------------------------------------------------------- g. determinism
@DTS
def test_non_atomic_paths_are_bitwise_reproducible(dev, dt):
    """16-bit D, and fp32 D with one piece per tile (the probe's accumulating weight gradients included): the same bits
    on a second launch and with 7 CTAs instead of one per SM; a GELU's D does not depend on aux_out being asked for."""
    from jepa_b200 import _lib
    cases = R.epilogue_cases(dt) + R.probe_cases(dt)
    cases += [c for N in (64, 128) for c in R.sweep_cases(dt, True, True, N) if c.K in (174, 4099)]
    differs = []
    for c in cases:
        assert c.split_k == 1
        t = R.to_device(R.make_inputs(c), dev)
        runs = []
        for limit in (0, 0, 7):
            _lib.call("vj_set_sm_limit", limit)
            try:
                out, xo = outputs(c, t, dev, 0)
                launch(c, t, out.view, xo.view if xo else None)
                torch.cuda.synchronize()
            finally:
                _lib.call("vj_set_sm_limit", 0)
            runs.append((out.full, xo.full if xo else None))
        if c.aux_out:
            out = Out(c.M, c.N, c.out_dtype, dev)
            launch(c, t, out.view)
            torch.cuda.synchronize()
            runs.append((out.full, runs[0][1]))
        for d, x in runs[1:]:
            if not torch.equal(bits(d), bits(runs[0][0])) or (x is not None and not torch.equal(bits(x), bits(runs[0][1]))):
                differs.append(c.id)
    assert not differs, differs


# ------------------------------------------------------------------------------ h. full step shapes, full output
@DTS
@pytest.mark.parametrize("how", ("split_k_for", "stream_k"))
@pytest.mark.parametrize("T,n_out,k_in", [(13056, 4096, 1024), (76032, 1536, 384), (76032, 384, 1536), (50200, 1024, 1024)])
def test_weight_gradient_at_step_shapes_whole_output(dev, dt, how, T, n_out, k_in):
    """grad[n_out, k_in] += dY^T X over T tokens with engine._split_k_for's split and as stream-K, every element against
    an fp64 product computed on the device 256 output rows at a time.  Peak memory about 2.5 GB at (76032, 384, 1536):
    dY and X in 16 bits (0.3 GB), X and |X| in fp64 (0.93 GB each), a 256-row block of dY in fp64 twice (0.3 GB)."""
    from jepa_b200 import kernels as Kn
    from jepa_b200.engine import _split_k_for
    g = torch.Generator(device=dev).manual_seed(T + n_out)
    dy = torch.randn(T, n_out, generator=g, device=dev).to(dt)
    x = torch.randn(T, k_in, generator=g, device=dev).to(dt)
    d0 = torch.randn(n_out, k_in, generator=g, device=dev)
    out = Out(n_out, k_in, F32, dev, fill=d0)
    Kn.gemm(dy, x, out.view, a_mn=True, b_mn=True, accumulate=True,
            split_k=_split_k_for(n_out, k_in, T) if how == "split_k_for" else -1)
    torch.cuda.synchronize()
    assert out.guards_unchanged()
    x64 = x.double()
    xabs = x64.abs()
    bad = []
    fam = f"step wgrad {how} {'bf16' if dt == BF16 else 'fp16'}"
    for r in range(0, n_out, 256):
        blk = dy[:, r:r + 256].double().t()
        R.compare(fam, out.view[r:r + 256], blk @ x64 + d0[r:r + 256].double(), blk.abs() @ xabs + d0[r:r + 256].abs().double(),
                  0.0, bad=bad)
    assert not bad, "\n".join(bad)
