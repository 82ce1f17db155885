"""Attention test inputs, an fp64 reference and the comparator, shared by tests/test_gpu_attention.py (vj_attn_fwd /
vj_attn_bwd on the GPU) and tests/test_attention_sensitivity_cpu.py (the same comparator against fp64 references of
kernels with known faults, on the same inputs).

Inputs are fp32 tensors [L, H, hd] holding bf16 values, so the reference sees exactly what the kernels read.  Checked
sequences can be packed between poison sequences: a poison sequence's keys point along the mean query of the sequence
it borders, scaled so that one leaked key takes over the softmax of most of that sequence's query rows; its queries
point along that sequence's mean key; its V and dO are +-1000.  Poison is finite on purpose: rows past a sequence's end
are multiplied by P = 0, and 0 * NaN would test a promise the kernels do not make.

The reference backward takes delta = rowsum(dO o O) from the O the backward kernel is given (the forward's bf16 output),
so the backward is checked as the function of its inputs that it is; the forward's O is checked on its own.  With the
exact O instead, rows whose softmax is nearly one-hot, where dQ and dK are small differences, would fail on the bf16
storage rounding of O alone.

Comparator bounds (those of tests/test_gpu_parity.py's attention cases, lse2 tighter):
  O                 : |err| <= 2e-2 + 1e-2 |ref|
  lse2              : |err| <= 1e-3 (largest measured on an H100 over tests/test_gpu_attention.py: 6e-5); a key
                      missing from or added to a row moves it by log2(1 -+ P of that key)
  dQ / dK / dV      : |err| <= 3e-2 + 2e-2 |ref|, and rel-L2 <= 1e-2 per tensor
  planted dominant keys (relax=True): the gradient atol grows by 2e-2 max|ref| and rel-L2 to 2e-2, because the rows of
  those keys sum hundreds of O(1) terms that each carry the bf16 rounding of P and dS
rel-L2 is skipped for a reference whose RMS is below 1e-4, i.e. zero up to cancellation (dQ and dK of a one-token
sequence, or of a softmax that is one-hot to e^-20); the elementwise bound still applies there.
"""
import math

import torch

LOG2E = 1.4426950408889634
O_ATOL, O_RTOL = 2e-2, 1e-2
LSE_ATOL = 1e-3
G_ATOL, G_RTOL, G_REL_L2 = 3e-2, 2e-2, 1e-2
G_RELAX_ATOL, G_RELAX_REL_L2 = 2e-2, 2e-2
GRADS = ("dq", "dk", "dv")

POISON = 1000.0       # |V| and |dO| of poison rows (a bf16 value)
POISON_GAIN = 32.0    # score of a poison key, in natural-log units, per unit of (query . mean query direction)
POISON_LENS = (67, 70)   # rows of the poison sequences before / after a checked one (odd start rows for the checked one)


def bf(t):
    return t.to(torch.bfloat16).to(t.dtype)


def unit(x):
    return x / x.norm(dim=-1, keepdim=True)


def random_rows(L, H, hd, g, k_scale=1.0):
    """q, k, v, dO [L, H, hd]: N(0, 1) in bf16, keys times k_scale."""
    q, k, v, do = (torch.randn(L, H, hd, generator=g) for _ in range(4))
    return bf(q), bf(k * k_scale), bf(v), bf(do)


def plant_last_key(q, k, g):
    """Every third query row (from row 0) gets +2 along a random direction d and the last key becomes a sqrt(hd) d with
    2a = ln L + 1, so that key scores about ln L + 1 for those rows and holds about half of their softmax at every L: a
    kernel that masks one valid key too many loses it."""
    L, H, hd = q.shape
    d = unit(torch.randn(H, hd, generator=g))
    rows = torch.arange(0, L, 3)
    q[rows] = bf(q[rows] + 2.0 * d)
    k[L - 1] = bf((math.log(L) + 1) / 2 * d * hd ** 0.5)


def plant_late_keys(q, k):
    """Three keys far into the sequence (70 %, 83 %, 97 %) score ~2^6..2^12 times above everything before them for every
    7th query row from row 5, so the running max of those rows moves late, more than once, by large steps."""
    L, H, hd = q.shape
    for frac, gain in ((0.70, 3.0), (0.83, 6.0), (0.97, 9.0)):
        kpos = int(frac * L)
        rows = torch.arange(5, L, 7)
        qdir = unit(q[rows].mean(0))    # [H, hd]
        k[kpos] = bf(gain * qdir * (hd ** 0.5))
        q[rows] = bf(q[rows] + 2.0 * qdir)


def poison_rows(n, q, k, g):
    """n poison rows bordering the sequence with queries q and keys k [L, H, hd] (see the module docstring)."""
    L, H, hd = q.shape
    amp = POISON_GAIN * hd ** 0.5
    kp = bf(amp * unit(q.mean(0))).expand(n, H, hd).clone()
    qp = bf(amp * unit(k.mean(0))).expand(n, H, hd).clone()
    sign = lambda: torch.randint(0, 2, (n, H, hd), generator=g).float() * 2 - 1
    return qp, kp, POISON * sign(), POISON * sign()


class Packed:
    """Sequences packed row after row, as the kernels take them; `checked` lists (first row, length) of the sequences
    the tests compare (poison sequences are computed but not compared)."""

    def __init__(self):
        self.parts, self.lens, self.checked = [], [], []

    def add(self, rows, checked=True):
        L = rows[0].shape[0]
        if checked:
            self.checked.append((sum(self.lens), L))
        self.parts.append(rows)
        self.lens.append(L)
        return self

    def add_poisoned(self, rows, g):
        """rows between a poison sequence aligned with it before and another after"""
        q, k = rows[0], rows[1]
        self.add(poison_rows(POISON_LENS[0], q, k, g), checked=False)
        self.add(rows)
        return self.add(poison_rows(POISON_LENS[1], q, k, g), checked=False)

    def tensors(self):
        """q, k, v, dO [T, H, hd]"""
        return [torch.cat([p[i] for p in self.parts]) for i in range(4)]

    def cu_seqlens(self):
        return [0] + [sum(self.lens[:i + 1]) for i in range(len(self.lens))]


# Sequence lengths of the residue sweep: every residue mod 2, 4 and 8, both sides of the forward's 128-row query / key
# tiles and of the backward's 128 resident / 64 streamed rows.  Head dims: the predictor's 24 (padded to 32), 64, ViT-H's
# 80 and ViT-g's 88 (padded to 128) and a true 128.
RESIDUE_LENS = (1, 2, 3, 5, 7, 8, 9, 15, 17, 31, 33, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 257, 383, 385)
HEAD_DIMS = (24, 64, 80, 88, 128)


def residue_case(L, hd, H=2):
    """One checked sequence of L tokens (its last key planted, see plant_last_key) between two poison sequences."""
    g = torch.Generator().manual_seed(1000 * hd + L)
    rows = random_rows(L, H, hd, g)
    plant_last_key(rows[0], rows[1], g)
    return Packed().add_poisoned(rows, g)


def reference(q, k, v, do=None, scale=None, o_in=None):
    """fp64 softmax attention of one sequence: q, do [Lq, H, hd], k, v [Lk, H, hd] -> dict with O [Lq, H, hd], lse2
    [H, Lq] (log2 domain) and, given dO, dq / dk / dv with delta from o_in (default: the fp64 O).  Runs on the inputs'
    device."""
    q, k, v = (t.double() for t in (q, k, v))
    s = torch.einsum("qhd,khd->hqk", q, k) * scale
    p = torch.softmax(s, -1)
    o = torch.einsum("hqk,khd->qhd", p, v)
    out = dict(o=o, lse2=torch.logsumexp(s, -1) * LOG2E)
    if do is not None:
        do = do.double()
        delta = (do * (o if o_in is None else o_in.double())).sum(-1).t()[..., None]    # [H, Lq, 1]
        ds = p * (torch.einsum("qhd,khd->hqk", do, v) - delta)
        out.update(dq=torch.einsum("hqk,khd->qhd", ds, k) * scale, dk=torch.einsum("hqk,qhd->khd", ds, q) * scale,
                   dv=torch.einsum("hqk,qhd->khd", p, do))
    return out


def _bound_check(bad, stats, name, got, ref, atol, rtol):
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    bound = atol + rtol * ref.abs()
    ratio = torch.nan_to_num(err / bound, nan=math.inf)
    worst = float(ratio.max())
    if stats is not None:
        stats[name] = max(stats.get(name, 0.0), worst)
    if not worst <= 1.0:
        at = tuple(int(i) for i in torch.nonzero(ratio == worst)[0])
        bad.append(f"{name}: max err {float(torch.nan_to_num(err, nan=math.inf).max()):.4g}, "
                   f"worst err/bound {worst:.4g} at {at} (got {float(got[at]):.6g}, ref {float(ref[at]):.6g})")


def compare(got, ref, grads=GRADS, relax=False, stats=None):
    """Checks got against ref (dicts as `reference` returns; got may hold bf16 / fp32 values) under the bounds of the
    module docstring.  Returns the violations (empty: pass).  stats, if given, keeps the worst err / bound per quantity
    and the worst rel-L2 per gradient."""
    bad = []
    _bound_check(bad, stats, "O", got["o"], ref["o"], O_ATOL, O_RTOL)
    _bound_check(bad, stats, "lse2", got["lse2"], ref["lse2"], LSE_ATOL, 0.0)
    for n in grads:
        r = ref[n].double()
        atol = G_ATOL + (G_RELAX_ATOL * float(r.abs().max()) if relax else 0.0)
        _bound_check(bad, stats, n, got[n], r, atol, G_RTOL)
        rn = float(r.norm())
        if rn > 1e-4 * r.numel() ** 0.5:
            e = float((got[n].double() - r).norm()) / rn
            limit = G_RELAX_REL_L2 if relax else G_REL_L2
            if stats is not None:
                stats[n + " rel-L2"] = max(stats.get(n + " rel-L2", 0.0), e)
            if not e <= limit:
                bad.append(f"{n}: rel-L2 {e:.4g} > {limit}")
    return bad
