"""Power of the attention comparator, on the CPU.  tests/test_gpu_attention.py checks vj_attn_fwd / vj_attn_bwd with
attention_ref.compare against an fp64 reference on the residue sweep's inputs.  Here the same comparator, on the same
inputs, must reject fp64 references of kernels with known faults at every sequence length where the fault changes the
result, and must pass a kernel that rounds where ours do.  Faults:
  - the forward's ragged-tile mask without its (e & 1) term (8c + 2(lane % 4) >= valid): at an odd number of valid keys
    the first key of the next sequence, a poison row, joins the softmax; the same leak in the dQ kernel's column mask;
  - the last valid key dropped (a mask one column too wide);
  - V of the last KV tile taken from the previous tile (the wrong ring stage);
  - lse2 from one thread's partial row sum instead of the quad's: the lane with lane % 4 == 0 writes lse2, and its
    partial holds keys 8c and 8c + 1 only.
"""
import pytest
import torch

from attention_ref import HEAD_DIMS, LOG2E, RESIDUE_LENS, bf, compare, reference, residue_case


def _case(L, hd):
    """the checked sequence's q, k, v, dO [L, H, hd], the first row of the poison sequence after it, and the scale"""
    pk = residue_case(L, hd)
    (off, _), = pk.checked
    rows = pk.tensors()
    return [t[off:off + L] for t in rows], [t[off + L:off + L + 1] for t in rows], hd ** -0.5


def emulate_bf16(q, k, v, do, scale):
    """Attention rounded where the kernels round: P and dS enter the MMAs as bf16, O / dQ / dK / dV are stored as bf16,
    delta = rowsum(dO o O) reads the stored O; the rest in fp64."""
    q, k, v, do = (t.double() for t in (q, k, v, do))
    s = torch.einsum("qhd,khd->hqk", q, k) * scale
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    o = bf(torch.einsum("hqk,khd->qhd", bf(p), v) / l.permute(1, 0, 2))
    lse = (m + torch.log(l))[..., 0]
    p = torch.exp(s - lse[..., None])
    dp = torch.einsum("qhd,khd->hqk", do, v)
    ds = bf(p * (dp - (do * o).sum(-1).t()[..., None]))
    return dict(o=o, lse2=lse * LOG2E, dv=bf(torch.einsum("hqk,qhd->khd", bf(p), do)),
                dk=bf(torch.einsum("hqk,qhd->khd", ds, q) * scale), dq=bf(torch.einsum("hqk,khd->qhd", ds, k) * scale))


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_bf16_rounding_passes(hd):
    for L in RESIDUE_LENS:
        (q, k, v, do), _, scale = _case(L, hd)
        got = emulate_bf16(q, k, v, do, scale)
        bad = compare(got, reference(q, k, v, do, scale, o_in=got["o"]))
        assert not bad, f"L={L}: {bad}"


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_leaked_neighbour_key_rejected(hd):
    missed = []
    for L in RESIDUE_LENS:
        if L % 2 == 0:   # an even count of valid keys masks both columns of every pair alike
            continue
        (q, k, v, do), (_, kn, vn, _), scale = _case(L, hd)
        ref = reference(q, k, v, do, scale)
        if not compare(reference(q, torch.cat([k, kn]), torch.cat([v, vn]), scale=scale), ref, grads=()):
            missed.append(("fwd", L))
        # dQ kernel: key L enters dQ = scale dS K with P from this sequence's lse2
        s = torch.einsum("qhd,khd->hqk", q.double(), kn.double()) * scale
        p = torch.exp(s - ref["lse2"][..., None] / LOG2E)
        dp = torch.einsum("qhd,khd->hqk", do.double(), vn.double())
        ds = p * (dp - (do.double() * ref["o"]).sum(-1).t()[..., None])
        dq = ref["dq"] + torch.einsum("hqk,khd->qhd", ds, kn.double()) * scale
        if not compare(dict(ref, dq=dq), ref):
            missed.append(("dq", L))
    assert not missed, f"leak not rejected at {missed}"


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_dropped_last_key_rejected(hd):
    missed = []
    for L in RESIDUE_LENS[1:]:
        (q, k, v, do), _, scale = _case(L, hd)
        if not compare(reference(q, k[:-1], v[:-1], scale=scale), reference(q, k, v, scale=scale), grads=()):
            missed.append(L)
    assert not missed, f"dropped key not rejected at L = {missed}"


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_last_v_tile_from_previous_tile_rejected(hd):
    missed = []
    for L in (L for L in RESIDUE_LENS if L > 128):
        (q, k, v, do), _, scale = _case(L, hd)
        lo = 128 * ((L - 1) // 128)
        v2 = v.clone()
        v2[lo:] = v[lo - 128:L - 128]
        if not compare(reference(q, k, v2, scale=scale), reference(q, k, v, scale=scale), grads=()):
            missed.append(L)
    assert not missed, f"stale V tile not rejected at L = {missed}"


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_lse2_from_one_thread_partial_rejected(hd):
    missed = []
    for L in (L for L in RESIDUE_LENS if L >= 3):   # up to 2 keys the partial is the whole row
        (q, k, v, do), _, scale = _case(L, hd)
        ref = reference(q, k, v, scale=scale)
        s = torch.einsum("qhd,khd->hqk", q.double(), k.double()) * scale
        m = s.amax(-1)
        mine = torch.arange(L) % 8 < 2
        partial = torch.exp(s - m[..., None])[..., mine].sum(-1)
        if not compare(dict(ref, lse2=(m + torch.log(partial)) * LOG2E), ref, grads=()):
            missed.append(L)
    assert not missed, f"partial-sum lse2 not rejected at L = {missed}"
