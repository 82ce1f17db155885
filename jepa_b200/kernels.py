"""Tensor-level wrappers over the C ABI: marshal torch CUDA tensors into raw pointers + sizes.

PyTorch is only the allocator / stream provider here; every op below is one of our own sm_90a
kernels.  All functions enqueue on torch's current stream and never synchronise.
"""
import ctypes

import torch

from . import _lib

EPI_NONE, EPI_GELU, EPI_ADD, EPI_DGELU, EPI_MUL, EPI_GELU_GRAD = 0, 1, 2, 3, 4, 5
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32


def compute_dtype():
    """Element type of the tensor-core operands for the caller's autocast state: fp16 inside
    torch.autocast('cuda', dtype=torch.float16) (or the deprecated torch.cuda.amp.autocast(dtype=torch.float16)), as the
    reference's eval loops run their frozen encoder; bf16 everywhere else (no autocast, or bf16 autocast)."""
    if torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == F16:
        return F16
    return BF16


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _chk(t, dtype=None, name="tensor"):
    if not t.is_cuda:
        raise _lib.VJError(f"{name} must live on a CUDA device (the hot path has no CPU fallback)")
    if not t.is_contiguous():
        raise _lib.VJError(f"{name} must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise _lib.VJError(f"{name} must be {dtype}, got {t.dtype}")
    return t


def _isf32(t):
    if t.dtype == F32:
        return 1
    if t.dtype == BF16:
        return 0
    raise _lib.VJError(f"unsupported dtype {t.dtype}")


def _dtcode(t):
    """The dtype flag of the entry points that also take fp16 (x_f32 / y_f32 / dst_f32): 0 bf16, 1 fp32, 2 fp16."""
    return 2 if t.dtype == F16 else _isf32(t)


def _f16(name, t):
    """Entry point `name`, or its fp16 twin `name_f16` when the 16-bit operand t is fp16."""
    if t.dtype == F16:
        return name + "_f16"
    if t.dtype != BF16:
        raise _lib.VJError(f"{name}: 16-bit operand must be bf16 or fp16, got {t.dtype}")
    return name


def gemm(a, b, out, *, a_mn=False, b_mn=False, bias=None, alpha=1.0, epi=EPI_NONE, aux=None, aux_rowmap=None,
         aux_period=0, aux_out=None, split_k=1, accumulate=False):
    """out[M,N] = epi(alpha * A @ B^T).  a: [M,K] (or [K,M] if a_mn); b: [N,K] (or [K,N] if b_mn).
    a and b are both bf16 or both fp16; a 16-bit out / aux / aux_out has their dtype."""
    name = _f16("vj_gemm", a)
    dt = a.dtype
    _chk(a, dt, "a"); _chk(b, dt, "b"); _chk(out, None, "out")
    if out.dtype not in (dt, F32):
        raise _lib.VJError(f"gemm: out must be {dt} or fp32, got {out.dtype}")
    if a_mn:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    if K != Kb or tuple(out.shape) != (M, N):
        raise _lib.VJError(f"gemm shape mismatch a={tuple(a.shape)} b={tuple(b.shape)} out={tuple(out.shape)}")
    if bias is not None:
        _chk(bias, F32, "bias")
    if aux is not None:
        _chk(aux, None, "aux")
        if aux.dtype not in (dt, F32):
            raise _lib.VJError(f"gemm: aux must be {dt} or fp32, got {aux.dtype}")
    if aux_rowmap is not None:
        _chk(aux_rowmap, torch.int32, "aux_rowmap")
    if aux_out is not None:
        _chk(aux_out, dt, "aux_out")
    _lib.call(name, _p(a), a.stride(0), int(a_mn), _p(b), b.stride(0), int(b_mn), _p(out), out.stride(0),
              int(out.dtype == F32), M, N, K, _p(bias), float(alpha), int(epi), _p(aux),
              aux.stride(0) if aux is not None else 0, int(aux is not None and aux.dtype == F32), _p(aux_rowmap),
              int(aux_period), _p(aux_out), aux_out.stride(0) if aux_out is not None else 0, int(split_k),
              int(accumulate), _s())
    return out


def attn_fwd(qkv, out, lse2, cu_seqlens, nseq, max_len, H, HD, scale):
    """qkv and out bf16, or both fp16."""
    name = _f16("vj_attn_fwd", qkv)
    _chk(qkv, None, "qkv"); _chk(out, qkv.dtype, "out"); _chk(lse2, F32, "lse2"); _chk(cu_seqlens, torch.int32, "cu_seqlens")
    T = qkv.shape[0]
    _lib.call(name, _p(qkv), _p(out), _p(lse2), _p(cu_seqlens), nseq, max_len, H, HD, T, float(scale), _s())
    return out


def attn_bwd(qkv, out, dout, lse2, delta_ws, dqkv, cu_seqlens, nseq, max_len, H, HD, scale, dq_acc_ws=None):
    for t, n in ((qkv, "qkv"), (out, "out"), (dout, "dout"), (dqkv, "dqkv")):
        _chk(t, BF16, n)
    _chk(lse2, F32, "lse2"); _chk(delta_ws, F32, "delta_ws")
    T = qkv.shape[0]
    if dq_acc_ws is not None:
        _chk(dq_acc_ws, F32, "dq_acc_ws")
    _lib.call("vj_attn_bwd", _p(qkv), _p(out), _p(dout), _p(lse2), _p(delta_ws), _p(dqkv), _p(dq_acc_ws), _p(cu_seqlens),
              nseq, max_len, H, HD, T, float(scale), _s())
    return dqkv


def layernorm_fwd(x, y, gamma, beta, eps, mean=None, rstd=None):
    _chk(x, None, "x"); _chk(y, None, "y"); _chk(gamma, F32, "gamma"); _chk(beta, F32, "beta")
    T, D = x.shape
    _lib.call("vj_layernorm_fwd", _p(x), _dtcode(x), _p(y), _dtcode(y), _p(gamma), _p(beta), _p(mean), _p(rstd), T, D,
              float(eps), _s())
    return y


_ln_ws = {}


def layernorm_bwd(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta):
    """dy bf16 with x / dres / dx bf16 or fp32; or dy fp16 with x / dres / dx fp32 (vj_layernorm_bwd_f16)."""
    _chk(dy, None, "dy"); _chk(x, None, "x"); _chk(dx, x.dtype, "dx")
    _chk(dgamma, F32, "dgamma"); _chk(dbeta, F32, "dbeta")
    if dy.dtype == F16:
        _chk(x, F32, "x (with an fp16 dy)")
        if dres is not None:
            _chk(dres, F32, "dres (with an fp16 dy)")
    elif dy.dtype != BF16:
        raise _lib.VJError(f"layernorm_bwd: dy must be bf16 or fp16, got {dy.dtype}")
    T, D = x.shape
    need = _lib.load().vj_layernorm_bwd_workspace(T, D)
    key = (x.device.index, torch.cuda.current_stream().cuda_stream)
    ws = _ln_ws.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=x.device)
        _ln_ws[key] = ws
    if dy.dtype == F16:
        _lib.call("vj_layernorm_bwd_f16", _p(dy), _p(x), _p(gamma), _p(mean), _p(rstd), _p(dres), _p(dx), _p(dgamma),
                  _p(dbeta), _p(ws), ws.numel(), T, D, _s())
    else:
        _lib.call("vj_layernorm_bwd", _p(dy), _p(x), _isf32(x), _p(gamma), _p(mean), _p(rstd), _p(dres), _p(dx),
                  _p(dgamma), _p(dbeta), _p(ws), ws.numel(), T, D, _s())
    return dx


def colsum(x, out, period=0, lo=0, hi=0):
    """out[N] += column sums of x [T, N] (bf16, fp16 or fp32) over rows r with lo <= r % period < hi."""
    _chk(x, None, "x"); _chk(out, F32, "out")
    T, N = x.shape
    if x.dtype == F16:
        _lib.call("vj_colsum_f16", _p(x), _p(out), T, N, x.stride(0), period, lo, hi, _s())
    else:
        _lib.call("vj_colsum", _p(x), _isf32(x), _p(out), T, N, x.stride(0), period, lo, hi, _s())
    return out


def im2col_tubelets(clips, patches, idx, tubelet, patch):
    """patches bf16, or fp16."""
    name = _f16("vj_im2col_tubelets", patches)
    _chk(clips, F32, "clips"); _chk(patches, None, "patches")
    B, C, T, H, W = clips.shape
    K = 0
    if idx is not None:
        _chk(idx, torch.int64, "idx")
        K = idx.shape[1]
    _lib.call(name, _p(clips), _p(patches), _p(idx), B, C, T, H, W, tubelet, patch, K, _s())
    return patches


def pos_interp(table, out, scales, mode):
    """interpolate_pos_encoding (vision_transformer.py:197-246) on the GPU: table fp32 [Nt, Nh, Nw, D] -> out fp32
    [T', H', W', D], bit-exact with torch's CPU F.interpolate at scale_factor `scales` = (st, sh, sw).
    mode 3: trilinear (video); mode 2: bicubic over [1, Nh, Nw, D] (images, st ignored)."""
    _chk(table, F32, "table"); _chk(out, F32, "out")
    Nt, Nh, Nw, D = table.shape
    T, H, W, Do = out.shape
    if Do != D:
        raise _lib.VJError(f"pos_interp: width mismatch table={tuple(table.shape)} out={tuple(out.shape)}")
    st, sh, sw = (float(s) for s in scales)
    _lib.call("vj_pos_interp", _p(table), _p(out), Nt, Nh, Nw, T, H, W, D, st, sh, sw, int(mode), _s())
    return out


def gather_rows(x, idx, out=None):
    """apply_masks for one mask: x [B,N,D], idx int64 [B,K] -> [B,K,D] (bit-exact row copy)."""
    _chk(x, None, "x"); _chk(idx, torch.int64, "idx")
    B, N, D = x.shape
    K = idx.shape[1]
    if out is None:
        out = torch.empty(B, K, D, dtype=x.dtype, device=x.device)
    _lib.call("vj_gather_rows", _p(x), _p(out), _p(idx), B, N, K, D * x.element_size(), _s())
    return out


def scatter_rows_add(dy, dx, idx):
    _chk(dy, None, "dy"); _chk(dx, dy.dtype, "dx"); _chk(idx, torch.int64, "idx")
    B, N, D = dx.shape
    K = idx.shape[1]
    _lib.call("vj_scatter_rows_add", _p(dy), _p(dx), _p(idx), B, N, K, D, _isf32(dx), _s())
    return dx


def target_ln_gather(x, idx, gamma, beta, eps_norm, eps_target, out=None):
    _chk(x, BF16, "x"); _chk(idx, torch.int64, "idx")
    B, N, D = x.shape
    K = idx.shape[1]
    if out is None:
        out = torch.empty(B, K, D, dtype=F32, device=x.device)
    _lib.call("vj_target_ln_gather", _p(x), _p(out), _p(idx), _p(gamma), _p(beta), B, N, K, D, float(eps_norm),
              float(eps_target), _s())
    return out


def pred_assemble_fwd(emb, pos, mask_token, idx_ctx, idx_tgt, x, B, Ke, Kp, Dp):
    _chk(emb, BF16, "emb"); _chk(pos, F32, "pos"); _chk(mask_token, F32, "mask_token"); _chk(x, None, "x")
    _lib.call("vj_pred_assemble_fwd", _p(emb), _p(pos), _p(mask_token), _p(idx_ctx), _p(idx_tgt), _p(x), _isf32(x),
              B, Ke, Kp, Dp, _s())
    return x


def pred_assemble_bwd(dx, demb, dmask_token, B, Ke, Kp, Dp):
    _chk(dx, None, "dx"); _chk(demb, BF16, "demb"); _chk(dmask_token, F32, "dmask_token")
    _lib.call("vj_pred_assemble_bwd", _p(dx), _isf32(dx), _p(demb), _p(dmask_token), B, Ke, Kp, Dp, _s())


def seq_slice(src, dst, B, Ke, Kp, D, scatter=False, zero_ctx=False):
    _chk(src, None, "src"); _chk(dst, src.dtype, "dst")
    _lib.call("vj_seq_slice", _p(src), _p(dst), _isf32(src), B, Ke, Kp, D, int(scatter), int(zero_ctx), _s())
    return dst


def l1_loss_fwd(z, h, loss_sum, weight):
    _chk(z, BF16, "z"); _chk(h, F32, "h"); _chk(loss_sum, F32, "loss_sum")
    _lib.call("vj_l1_loss_fwd", _p(z), _p(h), _p(loss_sum), z.numel(), float(weight), _s())


def l1_loss_bwd(z, h, grad_scale, scale, dz):
    _chk(z, BF16, "z"); _chk(h, F32, "h"); _chk(dz, BF16, "dz")
    _lib.call("vj_l1_loss_bwd", _p(z), _p(h), _p(grad_scale), float(scale), _p(dz), z.numel(), _s())
    return dz


def lp_loss_fwd(z, h, loss_sum, weight, p):
    _chk(z, BF16, "z"); _chk(h, F32, "h"); _chk(loss_sum, F32, "loss_sum")
    _lib.call("vj_lp_loss_fwd", _p(z), _p(h), _p(loss_sum), z.numel(), float(weight), float(p), _s())


def lp_loss_bwd(z, h, grad_scale, scale, dz, p):
    _chk(z, BF16, "z"); _chk(h, F32, "h"); _chk(dz, BF16, "dz")
    _lib.call("vj_lp_loss_bwd", _p(z), _p(h), _p(grad_scale), float(scale), _p(dz), z.numel(), float(p), _s())
    return dz


def token_std_bwd(z, pstd_total, grad_scale, scale, dz, weight, eps=1e-4):
    _chk(z, BF16, "z"); _chk(pstd_total, F32, "pstd_total"); _chk(dz, BF16, "dz")
    B, K, D = z.shape
    _lib.call("vj_token_std_bwd", _p(z), _p(pstd_total), _p(grad_scale), float(scale), _p(dz), B, K, D, float(eps),
              float(weight), _s())
    return dz


def cross_attn_fwd(q, kv, out, B, nq, S, H, hd, scale):
    """softmax(q k^T scale) v for nq query tokens per clip over S keys (attentive probe, modules.py:138-153).
    q, kv and out are all bf16 or all fp16."""
    name = _f16("vj_cross_attn_fwd", q)
    _chk(q, None, "q"); _chk(kv, q.dtype, "kv"); _chk(out, q.dtype, "out")
    _lib.call(name, _p(q), _p(kv), _p(out), B, nq, S, H, hd, float(scale), _s())
    return out


def cross_attn_fwd_lse(q, kv, out, lse2, B, nq, S, H, hd, scale):
    """cross_attn_fwd that also writes the softmax statistics lse2 fp32 [B*nq, H] (log2 domain) for the backward."""
    name = _f16("vj_cross_attn_fwd_lse", q)
    _chk(q, None, "q"); _chk(kv, q.dtype, "kv"); _chk(out, q.dtype, "out"); _chk(lse2, F32, "lse2")
    _lib.call(name, _p(q), _p(kv), _p(out), _p(lse2), B, nq, S, H, hd, float(scale), _s())
    return out


def cross_attn_bwd(q, kv, out, dout, lse2, dq, dkv, B, nq, S, H, hd, scale):
    """dq fp32 [B*nq, H*hd] and dkv [B*S, 2*H*hd] of cross_attn_fwd_lse; q, kv, out, dout and dkv are all bf16 or all
    fp16."""
    name = _f16("vj_cross_attn_bwd", q)
    for t, n in ((q, "q"), (kv, "kv"), (out, "out"), (dout, "dout"), (dkv, "dkv")):
        _chk(t, q.dtype, n)
    _chk(lse2, F32, "lse2"); _chk(dq, F32, "dq")
    need = _lib.load().vj_cross_attn_bwd_workspace(B, nq, S, H, hd)
    ws = torch.empty(max(need, 4), dtype=torch.uint8, device=q.device)
    _lib.call(name, _p(q), _p(kv), _p(out), _p(dout), _p(lse2), _p(dq), _p(dkv), _p(ws), ws.numel(),
              B, nq, S, H, hd, float(scale), _s())
    return dq, dkv


def token_std_accum(z, pstd, weight, eps=1e-4):
    _chk(z, BF16, "z"); _chk(pstd, F32, "pstd")
    B, K, D = z.shape
    _lib.call("vj_token_std_accum", _p(z), _p(pstd), B, K, D, float(eps), float(weight), _s())


def cast_f32_bf16(src, dst):
    _chk(src, F32, "src"); _chk(dst, BF16, "dst")
    _lib.call("vj_cast_f32_bf16", _p(src), _p(dst), src.numel(), _s())
    return dst


def cast_f32_f16(src, dst):
    _chk(src, F32, "src"); _chk(dst, F16, "dst")
    _lib.call("vj_cast_f32_f16", _p(src), _p(dst), src.numel(), _s())
    return dst


def head_pad(src, dst, outer, G, hd, hdp, inner, unpad_add=False):
    _chk(src, None, "src"); _chk(dst, None, "dst")
    _lib.call("vj_head_pad", _p(src), _isf32(src), _p(dst), _dtcode(dst), outer, G, hd, hdp, inner, int(unpad_add), _s())
    return dst


def ema_update(k_flat, q_flat, m):
    _chk(k_flat, F32, "k"); _chk(q_flat, F32, "q")
    _lib.call("vj_ema_update", _p(k_flat), _p(q_flat), k_flat.numel(), float(m), float(1.0 - m), _s())


def adamw_step(p, g, m, v, lr, beta1, beta2, eps, wd, step, inv_scale=None, found_inf=None):
    _lib.call("vj_adamw_step", _p(p), _p(g), _p(m), _p(v), p.numel(), float(lr), float(beta1), float(beta2),
              float(eps), float(wd), int(step), _p(inv_scale), _p(found_inf), _s())


def adamw_flat(p, g, m, v, group_ids, lr, wd, beta1, beta2, eps, step_dev, shadow, inv_scale=None, found_inf=None):
    """AdamW over a whole flat buffer in one launch: group_ids (uint8 per 64 elements) pick (lr[i], wd[i]) of at most 4
    groups, id 255 is skipped; step_dev is the device step counter, shadow receives the bf16 copy of the update."""
    _chk(p, F32, "p"); _chk(g, F32, "g"); _chk(m, F32, "m"); _chk(v, F32, "v")
    _chk(group_ids, torch.uint8, "group_ids"); _chk(step_dev, F32, "step_dev"); _chk(shadow, BF16, "shadow")
    lr4 = (ctypes.c_float * 4)(*map(float, lr))      # unused entries stay 0
    wd4 = (ctypes.c_float * 4)(*map(float, wd))
    _lib.call("vj_adamw_flat", _p(p), _p(g), _p(m), _p(v), _p(group_ids), p.numel(), ctypes.cast(lr4, ctypes.c_void_p),
              ctypes.cast(wd4, ctypes.c_void_p), float(beta1), float(beta2), float(eps), 0, _p(inv_scale), _p(found_inf),
              _p(step_dev), _p(shadow), _s())


def sumsq(x, out):
    _chk(x, F32, "x"); _chk(out, F32, "out")
    _lib.call("vj_sumsq", _p(x), x.numel(), _p(out), _s())


def ema_update_shadow(k_flat, q_flat, m, shadow):
    _chk(k_flat, F32, "k"); _chk(q_flat, F32, "q"); _chk(shadow, BF16, "shadow")
    _lib.call("vj_ema_update_shadow", _p(k_flat), _p(q_flat), k_flat.numel(), float(m), float(1.0 - m), _p(shadow), _s())


def grad_unscale_stats(gflat, seg, sumsq_out, inv_scale=None, found_inf=None, write_back=True):
    """One pass over a flat fp32 gradient buffer: optional in-place unscale, non-finite flag, per-tensor sum of squares."""
    _chk(gflat, F32, "gflat"); _chk(seg, torch.uint16, "seg"); _chk(sumsq_out, F32, "sumsq_out")
    _lib.call("vj_grad_unscale_stats", _p(gflat), _p(seg), gflat.numel(), _p(inv_scale), _p(found_inf), _p(sumsq_out),
              int(bool(write_back)), _s())


def seg_abs_sum(x, seg, out):
    _chk(x, F32, "x"); _chk(seg, torch.uint16, "seg"); _chk(out, F32, "out")
    _lib.call("vj_seg_abs_sum", _p(x), _p(seg), x.numel(), _p(out), _s())


def clip_coef(sumsq, max_norm, total_norm_out, coef_out):
    _chk(sumsq, F32, "sumsq")
    _lib.call("vj_clip_coef", _p(sumsq), sumsq.numel(), float(max_norm), _p(total_norm_out), _p(coef_out), _s())


def scale_flat(x, coef_dev):
    _chk(x, F32, "x"); _chk(coef_dev, F32, "coef")
    _lib.call("vj_scale_flat", _p(x), x.numel(), _p(coef_dev), _s())
