"""fp16 cross-attention (vj_cross_attn_*_f16) checking, shared by tests/test_gpu_probe_fp16.py (the kernels on an H100) and
tests/test_probe_fp16_cpu.py (the comparator's power, on the CPU):

  make_case    the inputs: three clips, clip 1 checked, clips 0 and 2 poison (keys that would score high against clip 1's
               queries, values of +-1000), a large late key that moves query 0's running max
  reference    fp64 forward (out, lse2) and backward (dq, dkv) of the checked clip from the kernels' own fp16 inputs
               (the backward's delta = dO . O from the fp16 out it is given, as the kernel and fp16 SDPA's backward do)
  emulate      what the kernels compute, with their roundings: fp64 arithmetic, fp16 stores of out and dkv (round to
               nearest, +-inf past 65504), fp32 lse2 and dq; `fault` swaps in one known defect
  check        the comparator: |err| <= atol + rtol |ref| everywhere, and where the fp16 rounding of the fp64 value is
               +-inf the stored value must be that inf (a saturated 65504 is an error)
"""
import math

import torch

F16, BF16, F64 = torch.float16, torch.bfloat16, torch.float64
OUT_TOL, LSE_TOL, GRAD_TOL = (2.5e-3, 1e-3), (1e-3, 0.0), (4e-3, 2.5e-3)
THREADS = 256


def key_chunk(hd):
    """Keys per CTA of the backward (xattn.cu xattn_bwd_chunk): 8 warps x (32 / (hd / 8)) lane groups x 2 keys."""
    return (THREADS // 32) * (32 // (hd // 8)) * 2


def make_case(hd, nq, S, seed, H=2):
    """fp32 sources (q [3*nq, H*hd], kv [3*S, 2*H*hd], dout [3*nq, H*hd]); the kernels read their fp16 rounding."""
    g = torch.Generator().manual_seed(seed)
    B, D = 3, H * hd
    q = torch.randn(B * nq, D, generator=g)
    kv = torch.randn(B, S, 2, H, hd, generator=g)
    qbar = q[nq:2 * nq].view(nq, H, hd).mean(0)
    kv[0, :, 0] = kv[2, :, 0] = 3.0 * hd ** 0.5 * qbar / qbar.norm(dim=-1, keepdim=True)   # high scores for clip 1's queries
    kv[0, :, 1], kv[2, :, 1] = -1000.0, 1000.0
    q1 = q[nq].view(H, hd)                                # query 0 of clip 1
    kv[1, S - 1, 0] = 4.0 * hd ** 0.5 * q1 / q1.norm(dim=-1, keepdim=True) ** 2    # score 4: a new running max
    dout = 16.0 * torch.randn(B * nq, D, generator=g)     # key gradients of ~16 / S stand well above the bound's atol
    return dict(q=q, kv=kv.reshape(B * S, 2 * D), dout=dout, B=B, nq=nq, S=S, H=H, hd=hd, scale=hd ** -0.5)


def _fwd_bwd(q, kv, dout, nq, S, H, hd, scale, out=None, drop=None):
    """fp64 forward and backward of one clip.  The backward takes delta = dO . O from `out`, the 16-bit output the
    backward kernel is given (the exact O when None); `drop` removes one key from the backward only."""
    qd, dd = q.to(F64).view(nq, H, hd), dout.to(F64).view(nq, H, hd)
    k, v = kv.to(F64).view(S, 2, H, hd)[:, 0], kv.to(F64).view(S, 2, H, hd)[:, 1]
    s = torch.einsum("nhd,shd->hns", qd, k) * scale
    p = torch.softmax(s, -1)
    o = torch.einsum("hns,shd->nhd", p, v)
    lse2 = (torch.logsumexp(s, -1) / math.log(2.0)).T
    delta = (dd * (o if out is None else out.to(F64).view(nq, H, hd))).sum(-1).T[:, :, None]
    ds = p * (torch.einsum("nhd,shd->hns", dd, v) - delta)
    if drop is not None:
        p, ds = p.clone(), ds.clone()
        p[:, :, drop] = ds[:, :, drop] = 0.0
    dq = scale * torch.einsum("hns,shd->nhd", ds, k)
    dkv = torch.stack([scale * torch.einsum("hns,nhd->shd", ds, qd), torch.einsum("hns,nhd->shd", p, dd)], 1)
    return o.reshape(nq, H * hd), lse2, dq.reshape(nq, H * hd), dkv.reshape(S, 2 * H * hd)


def checked(c, t, rows):
    """Clip 1's rows of a [3 * rows, ...] tensor."""
    return t[rows:2 * rows]


def reference(c, q, kv, dout, out):
    """fp64 results of clip 1 from the 16-bit inputs the kernels read (out: clip 1's output the backward is given)."""
    nq, S = c["nq"], c["S"]
    return _fwd_bwd(checked(c, q, nq), checked(c, kv, S), checked(c, dout, nq), nq, S, c["H"], c["hd"], c["scale"], out)


def emulate(c, fault=None):
    """(out, lse2, dq, dkv) of clip 1 as the fp16 kernels compute them, or with one known fault:
      'bf16'       today's bf16 probe: bf16 inputs and bf16 stores at the same places
      'leak'       the first key of the next clip is attended to as well
      'drop_chunk' the backward loses the last key of the first key chunk (no dk / dv row, no dq term)
      'satfinite'  fp16 stores saturate at +-65504 instead of becoming +-inf"""
    nq, S, H, hd, scale = c["nq"], c["S"], c["H"], c["hd"], c["scale"]
    e = BF16 if fault == "bf16" else F16
    q, kv, dout = (checked(c, c[k].to(e), n) for k, n in (("q", nq), ("kv", S), ("dout", nq)))
    store = (lambda t: t.clamp(-65504.0, 65504.0).to(e)) if fault == "satfinite" else (lambda t: t.to(e))
    if fault == "leak":
        kv = torch.cat([kv, c["kv"].to(e)[2 * S:2 * S + 1]])
    n = kv.shape[0]
    o, l2, _, _ = _fwd_bwd(q, kv, dout, nq, n, H, hd, scale)
    out = store(o)
    drop = key_chunk(hd) - 1 if fault == "drop_chunk" and S >= key_chunk(hd) else None
    _, _, dq, dkv = _fwd_bwd(q, kv, dout, nq, n, H, hd, scale, out=out, drop=drop)
    return out, l2.float(), dq.float(), store(dkv[:S])


def worst(got, ref, atol, rtol, f16=False):
    """Largest |err| / (atol + rtol |ref|); with f16, entries whose fp16 rounding overflows must equal that inf."""
    got, ref = got.to(F64), ref.to(F64)
    ratio = torch.nan_to_num((got - ref).abs() / (atol + rtol * ref.abs()), nan=math.inf)
    if f16:
        inf = torch.isinf(ref.to(F16))
        ratio = torch.where(inf, torch.where(got == ref.to(F16).to(F64), 0.0, math.inf), ratio)
    return float(ratio.max()) if ratio.numel() else 0.0


def check(c, out, lse2, dq, dkv, ref):
    """{quantity: worst err / bound} of clip 1's results against `ref` = reference(...)."""
    o, l2, gq, gkv = ref
    return {"out": worst(out, o, *OUT_TOL, f16=True), "lse2": worst(lse2, l2, *LSE_TOL),
            "dq": worst(dq, gq, *GRAD_TOL), "dkv": worst(dkv, gkv, *GRAD_TOL, f16=True)}


def overflow_case(hd=64, H=1):
    """One key and three queries with upstream gradients of 60000: p = 1, so dv = 3 x 60000 must store as +inf."""
    nq, S = 3, 1
    c = dict(q=torch.ones(3 * nq, H * hd), kv=torch.ones(3 * S, 2 * H * hd), dout=torch.full((3 * nq, H * hd), 6e4),
             B=3, nq=nq, S=S, H=H, hd=hd, scale=hd ** -0.5)
    return c
