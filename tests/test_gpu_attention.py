"""vj_attn_fwd / vj_attn_bwd (attn_fwd.cu, attn_bwd.cu) against an fp64 softmax reference computed on the device from
the same bf16 inputs, with the comparator of tests/attention_ref.py (whose power to reject known faults
tests/test_attention_sensitivity_cpu.py shows on these inputs).

  residue sweep      : L = 1 ... 385 over every residue mod 2, 4 and 8 and both sides of the 128-row forward tiles and
                       the backward's 128 resident / 64 streamed rows, at head dims 24 (-> 32), 64, 80 / 88 (-> 128) and
                       128, forward and backward, each sequence between poison sequences; padded lanes stay exactly 0
  ragged batches     : many sequences and heads per launch (grids of up to 1536 CTAs), long sequences, every head
  sequence isolation : several poisoned sequences per launch; one sequence first, in the middle and last among other
                       content gives bitwise the same O, lse2 and dQ / dK / dV rows
  head isolation     : head h of 16 is bitwise the same as that head's data run alone
  softmax extremes   : constant keys, one dominant key, scores spanning about +-100, late keys that move the max
  determinism        : forward and backward run twice are bitwise equal at the benchmark's shapes and a ragged batch

Run with -s to print the worst error over bound (and rel-L2) per head dim at the end of the module.
"""
import pytest
import torch

from attention_ref import (G_ATOL, GRADS, HEAD_DIMS, RESIDUE_LENS, Packed, bf, compare, plant_late_keys, random_rows,
                           reference, residue_case)

pytestmark = pytest.mark.gpu
WORST = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()  # fail loudly if the extension is missing - there is no fallback
    yield torch.device("cuda:0")
    for hd in sorted(WORST):
        print(f"\nworst at hd {hd}: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST[hd].items())))


def run(pk, dev, backward=True):
    """the kernels on a Packed: O [T, H, hdp], lse2 [H, T] and dqkv [T, 3, H, hdp] (outputs start as NaN)"""
    from jepa_b200 import kernels as Kn
    from jepa_b200.params import padded_head_dim
    q, k, v, do = pk.tensors()
    T, H, hd = q.shape
    hdp = padded_head_dim(hd)
    scale = hd ** -0.5
    qkv = torch.zeros(T, 3, H, hdp, dtype=torch.bfloat16, device=dev)
    dop = torch.zeros(T, H, hdp, dtype=torch.bfloat16, device=dev)
    for i, t in enumerate((q, k, v)):
        qkv[:, i, :, :hd] = t.to(dev)
    dop[..., :hd] = do.to(dev)
    qkv = qkv.view(T, 3 * H * hdp)
    cu = torch.tensor(pk.cu_seqlens(), dtype=torch.int32, device=dev)
    nseq, max_len = len(pk.lens), max(pk.lens)
    out = torch.full((T, H * hdp), float("nan"), dtype=torch.bfloat16, device=dev)
    lse = torch.full((H, T), float("nan"), device=dev)
    Kn.attn_fwd(qkv, out, lse, cu, nseq, max_len, H, hdp, scale)
    dqkv = None
    if backward:
        dqkv = torch.full_like(qkv, float("nan"))
        Kn.attn_bwd(qkv, out, dop.view(T, H * hdp), lse, torch.empty(H * T, device=dev), dqkv, cu, nseq, max_len, H, hdp,
                    scale)
        dqkv = dqkv.view(T, 3, H, hdp)
    return out.view(T, H, hdp), lse, dqkv


def check(pk, dev, backward=True, relax=False, grads=GRADS, k_scale=1.0):
    """every checked sequence of pk against its own fp64 reference; padded lanes exactly zero.  Keys k_scale times the
    unit scale make dQ = scale dS K, and its rounding, k_scale times larger: dQ is compared divided by k_scale."""
    out, lse, dqkv = run(pk, dev, backward)
    q, k, v, do = pk.tensors()
    hd = q.shape[-1]
    scale = hd ** -0.5
    grads = grads if backward else ()
    for off, L in pk.checked:
        rows = slice(off, off + L)
        o = out[rows, :, :hd]
        ref = reference(*(t[rows].to(dev) for t in (q, k, v)), do[rows].to(dev) if backward else None, scale, o_in=o)
        got = dict(o=o, lse2=lse[:, rows])
        if backward:
            got.update(dq=dqkv[rows, 0, :, :hd].double() / k_scale, dk=dqkv[rows, 1, :, :hd], dv=dqkv[rows, 2, :, :hd])
            ref["dq"] = ref["dq"] / k_scale
        bad = compare(got, ref, grads, relax, stats=WORST.setdefault(hd, {}))
        assert not bad, f"sequence of {L} tokens at row {off} (lens {pk.lens}): " + "; ".join(bad)
        assert bool((out[rows, :, hd:] == 0).all()), "padded lanes of O are not zero"
        if backward:
            assert bool((dqkv[rows, :, :, hd:] == 0).all()), "padded lanes of dqkv are not zero"
    return out, lse, dqkv


# --------------------------------------------------------------------------------------------- residue sweep
@pytest.mark.parametrize("hd", HEAD_DIMS)
@pytest.mark.parametrize("L", RESIDUE_LENS)
def test_residue_sweep(dev, L, hd):
    """An odd L leaves a ragged tile whose last valid key is the first of a key pair; a one-column mask error there lets
    the next sequence's first key - a poison key - into the softmax (see test_attention_sensitivity_cpu)."""
    check(residue_case(L, hd), dev)


# --------------------------------------------------------------------------------------------- ragged batches
# Many (sequence, head) CTAs per launch: 480 / 384 / 1536 forward CTAs, mixed one- and multi-tile sequences, long
# sequences (3680 at hd 32: 29 query / 58 streamed tiles), and every head checked.
@pytest.mark.parametrize("H,hd,lens", [
    (2, 64, [1568]), (2, 24, [1184, 1192]), (2, 64, [360, 48, 360]), (1, 80, [1568, 200]),
    (16, 64, [300] * 8 + [40, 513]), (16, 24, [520] + [300] * 7), (8, 128, [300] * 11 + [700]),
    (1, 32, [3680]), (2, 24, [129, 127, 256, 257, 17, 300]),
])
def test_ragged_batch(dev, H, hd, lens):
    g = torch.Generator().manual_seed(H * 1000 + hd + len(lens))
    pk = Packed()
    for L in lens:
        pk.add(random_rows(L, H, hd, g))
    check(pk, dev)


# --------------------------------------------------------------------------------------------- isolation
@pytest.mark.parametrize("hd", [24, 64, 80])
def test_poisoned_sequences_in_one_batch(dev, hd):
    g = torch.Generator().manual_seed(hd)
    pk = Packed()
    for L in (1, 64, 129, 200, 385, 63):
        rows = random_rows(L, 3, hd, g)
        pk.add_poisoned(rows, g)
    check(pk, dev)


@pytest.mark.parametrize("hd", [24, 64, 88])
def test_sequence_placement_bitwise(dev, hd):
    """The same sequence first, in the middle and last among other content (poisoned and plain, shorter and longer than
    it): O, lse2 and dQ / dK / dV of its rows are bitwise equal in every placement."""
    H, L = 3, 193
    g = torch.Generator().manual_seed(100 + hd)
    fixed = random_rows(L, H, hd, g)
    other = lambda n, s=1.0: random_rows(n, H, hd, g, k_scale=s)
    placements = [
        Packed().add(fixed).add(other(70)).add(other(300, 2.0)),
        Packed().add(other(5)).add_poisoned(fixed, g).add(other(385)),
        Packed().add(other(129, 3.0)).add(other(64)).add(fixed),
    ]
    results = []
    for pk in placements:
        out, lse, dqkv = check(pk, dev)
        off = next(o for o, n in pk.checked if n == L)
        results.append((out[off:off + L], lse[:, off:off + L], dqkv[off:off + L]))
    for i, r in enumerate(results[1:], 1):
        for name, a, b in zip(("O", "lse2", "dqkv"), results[0], r):
            assert torch.equal(a, b), f"{name} of the fixed sequence differs between placement 0 and {i}"


@pytest.mark.parametrize("hd", [24, 64, 80])
def test_head_isolation_bitwise(dev, hd):
    """Head h of an H = 16 launch equals the same data run as a single head, bit for bit (strides head * HD, H * HD and
    head * T of lse2 / delta)."""
    H = 16
    g = torch.Generator().manual_seed(200 + hd)
    lens = (1, 63, 129, 300)
    full = Packed()
    for L in lens:
        full.add(random_rows(L, H, hd, g))
    out, lse, dqkv = check(full, dev)
    tensors = full.tensors()
    for h in range(H):
        one = Packed()
        one.parts, one.lens = [[t[:, h:h + 1] for t in tensors]], list(full.lens)
        o1, l1, d1 = run(one, dev)
        assert torch.equal(o1[:, 0], out[:, h]), f"O of head {h}"
        assert torch.equal(l1[0], lse[h]), f"lse2 of head {h}"
        assert torch.equal(d1[:, :, 0], dqkv[:, :, h]), f"dqkv of head {h}"


# --------------------------------------------------------------------------------------------- softmax extremes
@pytest.mark.parametrize("hd", [24, 64, 80])
def test_constant_keys(dev, hd):
    """All keys of a sequence equal: P is uniform, lse2 = log2 L + s log2 e (one key too many or too few moves it by
    log2((L +- 1) / L), 3.7e-3 at L = 385, over the lse2 bound) and O is the mean of V to its bf16 rounding.
    dQ = scale k sum_j dS_ij is zero up to rounding (the dS of a row sum to zero), so it is held to the absolute bound
    alone."""
    H = 2
    g = torch.Generator().manual_seed(300 + hd)
    pk = Packed()
    for L in (1, 7, 129, 385):
        q, k, v, do = random_rows(L, H, hd, g)
        pk.add((q, k[:1].expand(L, H, hd).clone(), v, do))
    out, _, dqkv = check(pk, dev, grads=("dk", "dv"))
    assert float(dqkv[:, 0].abs().max()) <= G_ATOL
    v = pk.tensors()[2]
    for off, L in pk.checked:
        rows = slice(off, off + L)
        mean_v = v[rows].double().mean(0)                                        # [H, hd]
        err = (out[rows, :, :hd].cpu().double() - mean_v).abs()
        assert bool((err <= 2 ** -8 * mean_v.abs() + 1e-5).all()), f"O is not mean(V) at L = {L}: {float(err.max()):.3g}"


@pytest.mark.parametrize("hd", [24, 64, 80])
def test_one_dominant_key(dev, hd):
    """Every query has component 3 along u and key j* is 10 sqrt(hd) u: j* scores 30 above zero and the other keys'
    weights are below e^-20, so O is V[j*] up to its bf16 rounding.  j* is the first key, the last of a tile, the first
    of a tile and the last key."""
    H = 2
    g = torch.Generator().manual_seed(400 + hd)
    pk, star = Packed(), []
    for L, j in ((385, 0), (385, 127), (129, 128), (257, 256), (7, 6)):
        q, k, v, do = random_rows(L, H, hd, g)
        u = torch.nn.functional.normalize(torch.randn(H, hd, generator=g), dim=-1)
        q = bf(q - (q * u).sum(-1, keepdim=True) * u + 3.0 * u)
        k[j] = bf(10.0 * hd ** 0.5 * u)
        pk.add((q, k, v, do))
        star.append(j)
    out, _, _ = check(pk, dev)
    v = pk.tensors()[2]
    for (off, L), j in zip(pk.checked, star):
        vj = v[off + j].double()
        err = (out[off:off + L, :, :hd].cpu().double() - vj).abs()
        assert bool((err <= 2 ** -8 * vj.abs() + 1e-5).all()), f"O is not V[{j}] at L = {L}: {float(err.max()):.3g}"


@pytest.mark.parametrize("hd", [24, 64, 80])
def test_scores_spanning_100(dev, hd):
    """Keys scaled by 40: scaled scores spread over about +-100, exp2 of all but the top few keys of a row underflows, and
    the running max jumps by tens between KV tiles."""
    g = torch.Generator().manual_seed(500 + hd)
    pk = Packed()
    for L in (1, 33, 129, 385):
        pk.add(random_rows(L, 2, hd, g, k_scale=40.0))
    check(pk, dev, k_scale=40.0)


@pytest.mark.parametrize("hd,lens", [(64, [1569, 385]), (24, [1183, 1193]), (80, [1567, 129])])
def test_late_max_odd_lengths(dev, hd, lens):
    g = torch.Generator().manual_seed(600 + hd)
    pk = Packed()
    for L in lens:
        q, k, v, do = random_rows(L, 2, hd, g)
        plant_late_keys(q, k)
        pk.add((q, k, v, do))
    check(pk, dev, relax=True)


# --------------------------------------------------------------------------------------------- determinism
@pytest.mark.parametrize("H,hd,lens", [(16, 64, [1568] * 32), (16, 24, [1184] * 32),
                                       (16, 80, [1, 2, 3, 17, 63, 64, 65, 129, 255, 300, 385, 1183, 1569])],
                         ids=["bench-target-hd64", "bench-predictor-hd24", "ragged-hd80"])
def test_deterministic(dev, H, hd, lens):
    """Forward and backward twice on the same inputs: O, lse2 and dqkv bitwise equal (the backward has no atomics).
    Outputs start as NaN, so an element either run leaves unwritten fails the comparison too."""
    g = torch.Generator(device=dev).manual_seed(hd)
    T = sum(lens)
    pk = Packed()
    pk.parts = [[bf(torch.randn(T, H, hd, device=dev, generator=g)) for _ in range(4)]]
    pk.lens = list(lens)
    first = run(pk, dev)
    second = run(pk, dev)
    for name, a, b in zip(("O", "lse2", "dqkv"), first, second):
        assert torch.equal(a, b), f"{name} differs between two runs"
