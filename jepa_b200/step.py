"""The V-JEPA train-step pieces that live as closures inside app/vjepa/train.py:414-498 in the
reference: target forward (+ LN + gather), L1 latent loss, variance regulariser, EMA update.
Each is a thin host wrapper over fused kernels; `app/vjepa/train.py` and `bench.py` both call these.
"""
import torch
import torch.nn.functional as F

from . import engine
from . import kernels as K
from .models import _common_base, _token_views, MultiMaskWrapper, PredictorMultiMaskWrapper

from .distributed import DistributedDataParallel as _FlatDDP  # noqa: E402

TARGET_LN_EPS = 1e-5  # F.layer_norm default eps, app/vjepa/train.py:426


def unwrap(module):
    """Strip DistributedDataParallel / multi-mask wrappers down to the backbone."""
    m = module
    if hasattr(m, "module") and isinstance(m, (torch.nn.parallel.DistributedDataParallel, _FlatDDP)):
        m = m.module
    if isinstance(m, (MultiMaskWrapper, PredictorMultiMaskWrapper)):
        m = m.backbone
    return m


@torch.no_grad()
def forward_target(target_encoder, clips, masks_pred):
    """forward_target (train.py:419-429): h = LN_noaffine(target_encoder(clips)) gathered at masks_pred.

    Runs the no-grad encoder over all N tokens, then ONE fused kernel per mask applies the final
    encoder LayerNorm, the affine-free F.layer_norm and the gather, touching only the kept rows.
    Returns a list of fp32 [B, Kp_i, D] views of one contiguous buffer.
    """
    bb = unwrap(target_encoder)
    x, grid = bb._check_input(clips)
    raw, _, _ = engine.encoder_forward(bb, x, None, save=False, final_norm=False, grid=grid)
    B, N, D = x.shape[0], grid[0] * grid[1] * grid[2], bb.embed_dim
    raw = raw.view(B, N, D)
    store = bb._store
    sizes = [int(m.shape[1]) for m in masks_pred]
    h_cat = torch.empty(sum(B * k for k in sizes), D, dtype=torch.float32, device=clips.device)
    off = 0
    for m, k in zip(masks_pred, sizes):
        K.target_ln_gather(raw, m.contiguous(), store.f32("norm.weight"), store.f32("norm.bias"), engine.LN_EPS,
                           TARGET_LN_EPS, out=h_cat[off:off + B * k].view(B, k, D))
        off += B * k
    return _token_views(h_cat, B, sizes)


class _LpLossFn(torch.autograd.Function):
    """(1/M) sum_i mean(|z_i - h_i|^p) / p over the concatenated token rows of all masks; p = 1 takes the L1 kernels."""

    @staticmethod
    def forward(ctx, z_cat, h_cat, row_counts, p):
        n_masks = len(row_counts)
        D = z_cat.shape[1]
        loss = torch.zeros(1, dtype=torch.float32, device=z_cat.device)
        off = 0
        for rows in row_counts:
            w = 1.0 / (n_masks * rows * D)
            if p == 1.0:
                K.l1_loss_fwd(z_cat[off:off + rows], h_cat[off:off + rows], loss, w)
            else:
                K.lp_loss_fwd(z_cat[off:off + rows], h_cat[off:off + rows], loss, w / p, p)
            off += rows
        ctx.save_for_backward(z_cat, h_cat)
        ctx.row_counts, ctx.p = row_counts, p
        return loss.view(())

    @staticmethod
    def backward(ctx, g):
        z_cat, h_cat = ctx.saved_tensors
        n_masks = len(ctx.row_counts)
        D = z_cat.shape[1]
        g = g.detach().to(torch.float32).contiguous()
        dz = torch.empty_like(z_cat)
        off = 0
        for rows in ctx.row_counts:
            w = 1.0 / (n_masks * rows * D)
            if ctx.p == 1.0:
                K.l1_loss_bwd(z_cat[off:off + rows], h_cat[off:off + rows], g, w, dz[off:off + rows])
            else:
                K.lp_loss_bwd(z_cat[off:off + rows], h_cat[off:off + rows], g, w, dz[off:off + rows], ctx.p)
            off += rows
        return dz, None, None, None


def _cat_rows(views, dtype):
    base = _common_base(views)
    if base is None:
        base = torch.cat([t.reshape(-1, t.shape[-1]) for t in views], dim=0)
    return base if base.dtype == dtype else base.to(dtype)


def jepa_loss(z, h, loss_exp=1.0):
    """loss_fn (train.py:440-446): (1/M) sum_i mean(|z_i - h_i|^p) / p; p = loss_exp (1.0 in every shipped config)."""
    p = float(loss_exp)
    if not p >= 1.0:
        raise ValueError(f"loss_exp must be >= 1 (got {loss_exp}): |z - h|^p has no finite gradient at z = h otherwise")
    zb, hb = _cat_rows(z, torch.bfloat16), _cat_rows(h, torch.float32)
    rows = tuple(int(t.shape[0] * t.shape[1]) for t in z)
    return _LpLossFn.apply(zb.contiguous(), hb.contiguous(), rows, p)


class _RegLossFn(torch.autograd.Function):
    """reg_fn + relu-mean (train.py:448-449,458-459): mean(relu(1 - (1/M) sum_i sqrt(var_unbiased(z_i, dim=1) + 1e-4)))."""

    @staticmethod
    def forward(ctx, z_cat, B, sizes):
        D = z_cat.shape[1]
        pstd = torch.zeros(B, D, dtype=torch.float32, device=z_cat.device)
        off = 0
        for k in sizes:
            K.token_std_accum(z_cat[off:off + B * k].view(B, k, D), pstd, 1.0 / len(sizes))
            off += B * k
        ctx.save_for_backward(z_cat, pstd)
        ctx.B, ctx.sizes = B, sizes
        return torch.mean(F.relu(1. - pstd))          # [B, D] epilogue of the regulariser (the kernels did the token reduction)

    @staticmethod
    def backward(ctx, g):
        z_cat, pstd = ctx.saved_tensors
        B, sizes, D = ctx.B, ctx.sizes, z_cat.shape[1]
        g = g.detach().to(torch.float32).reshape(1).contiguous()
        dz = torch.empty_like(z_cat)
        off = 0
        for k in sizes:
            K.token_std_bwd(z_cat[off:off + B * k].view(B, k, D), pstd, g, 1.0, dz[off:off + B * k].view(B, k, D),
                            1.0 / len(sizes))
            off += B * k
        return dz, None, None


def reg_loss(z, with_grad=False):
    """reg_fn + relu-mean (train.py:448-449,458-459).  with_grad=False (reg_coeff = 0, every shipped config): the value is
    only logged; with_grad=True: differentiable through the hand-written backward kernel (reg_coeff != 0)."""
    B = int(z[0].shape[0])
    sizes = tuple(int(t.shape[1]) for t in z)
    zb = _cat_rows(z, torch.bfloat16).contiguous()
    if with_grad and zb.requires_grad:
        return _RegLossFn.apply(zb, B, sizes)
    with torch.no_grad():
        return _RegLossFn.apply(zb.detach(), B, sizes)


@torch.no_grad()
def ema_update(encoder, target_encoder, m):
    """Momentum update (train.py:484-487) as ONE kernel over the flat parameter buffers."""
    q, k = unwrap(encoder), unwrap(target_encoder)
    qs, ks = q._store.adopt(q), k._store.adopt(k)
    if qs.offsets != ks.offsets:
        raise RuntimeError("encoder / target_encoder parameter layouts differ")
    # the bf16 tensor-core operands of the target's next forward leave in the same pass (no separate cast launch)
    K.ema_update_shadow(ks.flat, qs.flat, m, ks.shadow)
    ks.mark_shadow_fresh(complete=True)   # the EMA pass walks the WHOLE flat buffer (frozen tensors and padding included)


@torch.no_grad()
def clip_grad_norm_(module, max_norm):
    """torch.nn.utils.clip_grad_norm_(module.parameters(), max_norm) (L2; app/vjepa/train.py:468-471) for a network whose
    gradients live in one flat buffer: per-tensor sums of squares (reused from the unscale pass of this step when
    current) -> total norm and clip coefficient ON THE DEVICE -> one scaling pass that exits immediately when no
    clipping is needed.  Returns the total norm as a device scalar (float() it like the reference does)."""
    from .logging_utils import _flat_grad_sumsq
    bb = unwrap(module)
    named = [(n, p) for n, p in bb.named_parameters() if p.grad is not None]
    if not named:
        return torch.zeros((), device=next(bb.parameters()).device)
    flat = _flat_grad_sumsq(named)
    if flat is None or len(flat) != len(named):
        return torch.nn.utils.clip_grad_norm_([p for _, p in named], max_norm)
    sumsq = next(iter(flat.values()))[0]
    store = named[0][1]._vj_store
    out = torch.empty(2, dtype=torch.float32, device=sumsq.device)
    K.clip_coef(sumsq, max_norm, out[0:1], out[1:2])
    p0 = named[0][1]
    base_off = store.offsets[p0._vj_name][0]
    gflat = torch.as_strided(p0.grad, (store.total,), (1,), storage_offset=p0.grad.storage_offset() - base_off)
    K.scale_flat(gflat, out[1:2])
    store._grad_sumsq = None          # the cached statistics describe the unclipped gradients
    return out[0]
