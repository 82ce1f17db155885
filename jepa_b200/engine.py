"""Forward / backward schedules of the V-JEPA networks on top of the sm_90a kernels.

This is the GPU-first replacement for the autograd graph PyTorch builds over
src/models/vision_transformer.py:159-195, src/models/predictor.py:174-239 and
src/models/utils/modules.py:61-120 in the reference: tokens of ALL masks of a step are
concatenated into one token-major [T, D] matrix (only attention needs the sequence boundaries, via
cu_seqlens), every Linear is one wgmma GEMM launch with its bias / GELU / residual fused in the
epilogue, and the backward is scheduled by hand - dgrad and wgrad GEMMs read the saved activations
in place (MN-major descriptors, no transposes) and the wgrads reduce straight into a flat fp32
gradient buffer.
"""

import math

import torch

from . import kernels as K
from .params import padded_head_dim

BF16, F32 = torch.bfloat16, torch.float32
LN_EPS = 1e-6  # norm_layer=partial(nn.LayerNorm, eps=1e-6): vision_transformer.py:252, predictor.py:244


def _empty(shape, dtype, dev):
    return torch.empty(shape, dtype=dtype, device=dev)


_cu_cache = {}


def cu_seqlens_for(segments, device):
    """segments: list of (n_sequences, length).  Returns (cu int32 [nseq+1] on device, nseq, max_len, T)."""
    key = (tuple(segments), device.index)
    hit = _cu_cache.get(key)
    if hit is None:
        cu = [0]
        for n, l in segments:
            for _ in range(n):
                cu.append(cu[-1] + l)
        t = torch.tensor(cu, dtype=torch.int32).to(device, non_blocking=True)
        hit = (t, len(cu) - 1, max(l for _, l in segments), cu[-1])
        if len(_cu_cache) > 256:
            _cu_cache.clear()
        _cu_cache[key] = hit
    return hit


import os as _os
_STREAM_K = _os.environ.get("VJ_GEMM_STREAMK", "0") == "1"     # "1": stream-K wgrads instead of the wave-filling split-K


def _split_k_for(m_out, n_in, k_tokens, sms=132):
    """Split-K factor of a weight-gradient GEMM [m_out, n_in] += dY^T X over k_tokens: the output has 18..128 tiles for 132
    SMs, so pick the split whose work-item count fills whole waves best (a mild penalty per split: every piece reduce-adds
    a full fp32 tile).  Stream-K stays available as split_k = -1 but loses the L2 sharing of the operand tiles between
    co-scheduled pieces.  Weight-gradient tiles are at most 128 columns wide (gemm.cu, kPromoteKB)."""
    bn = 128 if n_in % 128 == 0 else 64
    tiles = ((m_out + 127) // 128) * (n_in // bn)
    kb = (k_tokens + 63) // 64
    best, best_score = 1, -1.0
    for s in range(1, min(kb, 16) + 1):
        items = tiles * s
        waves = (items + sms - 1) // sms
        score = items / (waves * sms) - 0.02 * (s - 1)
        if score > best_score + 1e-9:
            best, best_score = s, score
    return best


class BlockWeights:
    """Per-step view of one transformer Block's tensors (bf16 shadows + fp32 bias / LN params)."""
    __slots__ = ("prefix", "n1w", "n1b", "qkv_w", "qkv_b", "proj_w", "proj_b", "n2w", "n2b", "fc1_w", "fc1_b", "fc2_w",
                 "fc2_b")


class StackSpec:
    """Static geometry of a stack of Blocks."""

    def __init__(self, dim, heads, hidden, depth, block_prefix):
        self.dim, self.heads, self.hidden, self.depth = dim, heads, hidden, depth
        self.hd = dim // heads
        self.hdp = padded_head_dim(self.hd)
        self.padded = self.hdp != self.hd
        self.inner = heads * self.hdp          # width of q (and of the attention output)
        self.scale = self.hd ** -0.5
        self.block_prefix = block_prefix       # e.g. "blocks" / "predictor_blocks"


def gather_block_weights(store, spec, scratch):
    """Collect bf16 weights for every block; builds head-padded copies when hd is not a tile size."""
    out = []
    dev = store.flat.device
    for i in range(spec.depth):
        pre = f"{spec.block_prefix}.{i}."
        w = BlockWeights()
        w.prefix = pre
        w.n1w, w.n1b = store.f32(pre + "norm1.weight"), store.f32(pre + "norm1.bias")
        w.n2w, w.n2b = store.f32(pre + "norm2.weight"), store.f32(pre + "norm2.bias")
        w.fc1_w, w.fc1_b = store.bf16(pre + "mlp.fc1.weight"), store.f32(pre + "mlp.fc1.bias")
        w.fc2_w, w.fc2_b = store.bf16(pre + "mlp.fc2.weight"), store.f32(pre + "mlp.fc2.bias")
        w.proj_b = store.f32(pre + "attn.proj.bias")
        if not spec.padded:
            w.qkv_w, w.qkv_b = store.bf16(pre + "attn.qkv.weight"), store.f32(pre + "attn.qkv.bias")
            w.proj_w = store.bf16(pre + "attn.proj.weight")
        else:
            H, hd, hdp, D = spec.heads, spec.hd, spec.hdp, spec.dim
            key = ("pad", i)
            bufs = scratch.get(key)
            if bufs is None:
                bufs = (_empty((3 * H * hdp, D), BF16, dev), _empty((3 * H * hdp,), F32, dev),
                        _empty((D, H * hdp), BF16, dev))
                scratch[key] = bufs
            K.head_pad(store.f32(pre + "attn.qkv.weight"), bufs[0], 1, 3 * H, hd, hdp, D)
            K.head_pad(store.f32(pre + "attn.qkv.bias"), bufs[1], 1, 3 * H, hd, hdp, 1)
            K.head_pad(store.f32(pre + "attn.proj.weight"), bufs[2], D, H, hd, hdp, 1)
            w.qkv_w, w.qkv_b, w.proj_w = bufs
        out.append(w)
    return out


class BlockSaved:
    __slots__ = ("x_in", "mean1", "rstd1", "ln1", "qkv", "attn", "lse", "x_mid", "mean2", "rstd2", "ln2", "h", "g")


def blocks_forward(spec, weights, x, seq, save, tap=None):
    """Run the Block stack over token matrix x [T, dim] (bf16).  Returns (x_out, saved list or None).

    Block.forward (modules.py:114-120): x = x + proj(attn(LN1(x))); x = x + fc2(gelu(fc1(LN2(x)))).
    tap(i, x): called with the residual stream after block i (multi-layer feature taps, vision_transformer.py:186-187).
    """
    cu, nseq, max_len, T = seq
    dev = x.device
    D, Hd, W = spec.dim, spec.hidden, spec.inner
    saved = [] if save else None
    # scratch reused across layers when nothing has to be kept for a backward
    ln = qkv = attn = lse = g = None
    for w in weights:
        if save or ln is None:
            ln = _empty((T, D), BF16, dev)
            qkv = _empty((T, 3 * W), BF16, dev)
            attn = _empty((T, W), BF16, dev)
            lse = _empty((spec.heads, T), F32, dev)
            g = _empty((T, Hd), BF16, dev)
        s = None
        if save:
            s = BlockSaved()
            s.x_in = x
            s.mean1, s.rstd1 = _empty((T,), F32, dev), _empty((T,), F32, dev)
            s.mean2, s.rstd2 = _empty((T,), F32, dev), _empty((T,), F32, dev)
        K.layernorm_fwd(x, ln, w.n1w, w.n1b, LN_EPS, s.mean1 if save else None, s.rstd1 if save else None)
        K.gemm(ln, w.qkv_w, qkv, bias=w.qkv_b)
        K.attn_fwd(qkv, attn, lse, cu, nseq, max_len, spec.heads, spec.hdp, spec.scale)
        x_mid = _empty((T, D), BF16, dev)
        K.gemm(attn, w.proj_w, x_mid, bias=w.proj_b, epi=K.EPI_ADD, aux=x)
        ln2 = _empty((T, D), BF16, dev) if save else ln
        K.layernorm_fwd(x_mid, ln2, w.n2w, w.n2b, LN_EPS, s.mean2 if save else None, s.rstd2 if save else None)
        h = _empty((T, Hd), BF16, dev) if save else None
        # training: keep gelu'(pre-activation) (bf16) instead of the pre-activation itself, computed in the same epilogue
        K.gemm(ln2, w.fc1_w, g, bias=w.fc1_b, epi=K.EPI_GELU_GRAD if save else K.EPI_GELU, aux_out=h)
        x_out = _empty((T, D), BF16, dev)
        K.gemm(g, w.fc2_w, x_out, bias=w.fc2_b, epi=K.EPI_ADD, aux=x_mid)
        if save:
            s.ln1, s.qkv, s.attn, s.lse, s.x_mid, s.ln2, s.h, s.g = ln, qkv, attn, lse, x_mid, ln2, h, g
            saved.append(s)
        x = x_out
        if tap is not None:
            tap(len(saved) - 1 if save else tap.count, x)
            tap.count += 1
    return x, saved


def _wgrad(dy, act, grad_out, bias_grad, tokens):
    """grad_out[N_out, K_in] += dy^T act ; bias_grad[N_out] += colsum(dy)."""
    n_out, k_in = grad_out.shape
    # stream-K (split_k = -1): 32..128 output tiles for 132 SMs - every SM gets the same number of k-blocks instead of a
    # ragged second wave; all pieces reduce-add into the flat fp32 gradient buffer anyway
    K.gemm(dy, act, grad_out, a_mn=True, b_mn=True, accumulate=True,
           split_k=-1 if _STREAM_K else _split_k_for(n_out, k_in, tokens))
    if bias_grad is not None:
        K.colsum(dy, bias_grad)


def _sync_begin(mod, gflat):
    """Data-parallel gradient exchange (jepa_b200.distributed.FlatGradSync) attached to this network, or None."""
    sync = getattr(mod, "_vj_grad_sync", None)
    if sync is not None:
        sync.begin(gflat)
    return sync


def blocks_backward(spec, weights, saved, dx, seq, store, gflat, scratch, sync=None):
    """Backward through the Block stack.  dx [T, dim] bf16 is d(loss)/d(stack output); returns d/d(input).
    `sync`: told after every block that the flat gradients from that block's first parameter upwards are final."""
    cu, nseq, max_len, T = seq
    dev = dx.device
    D, Hd, W = spec.dim, spec.hidden, spec.inner
    H, hd, hdp = spec.heads, spec.hd, spec.hdp
    gv = lambda name: store.grad_view(gflat, name)
    delta_ws = _empty((H * T,), F32, dev)
    for w, s in zip(reversed(weights), reversed(saved)):
        pre = w.prefix
        # ---- MLP: x_out = x_mid + fc2(gelu(fc1(ln2)))
        dh = _empty((T, Hd), BF16, dev)
        K.gemm(dx, w.fc2_w, dh, b_mn=True, epi=K.EPI_MUL, aux=s.h)               # (dx W2) * gelu'(h), s.h holds gelu'(h)
        _wgrad(dx, s.g, gv(pre + "mlp.fc2.weight"), gv(pre + "mlp.fc2.bias"), T)
        dln2 = _empty((T, D), BF16, dev)
        K.gemm(dh, w.fc1_w, dln2, b_mn=True)
        _wgrad(dh, s.ln2, gv(pre + "mlp.fc1.weight"), gv(pre + "mlp.fc1.bias"), T)
        dx_mid = _empty((T, D), BF16, dev)
        K.layernorm_bwd(dln2, s.x_mid, w.n2w, s.mean2, s.rstd2, dx, dx_mid, gv(pre + "norm2.weight"),
                        gv(pre + "norm2.bias"))
        # ---- attention: x_mid = x_in + proj(attn(qkv(ln1)))
        dattn = _empty((T, W), BF16, dev)
        K.gemm(dx_mid, w.proj_w, dattn, b_mn=True)
        dqkv = _empty((T, 3 * W), BF16, dev)
        K.attn_bwd(s.qkv, s.attn, dattn, s.lse, delta_ws, dqkv, cu, nseq, max_len, H, hdp, spec.scale)
        dln1 = _empty((T, D), BF16, dev)
        K.gemm(dqkv, w.qkv_w, dln1, b_mn=True)
        if not spec.padded:
            _wgrad(dx_mid, s.attn, gv(pre + "attn.proj.weight"), gv(pre + "attn.proj.bias"), T)
            _wgrad(dqkv, s.ln1, gv(pre + "attn.qkv.weight"), gv(pre + "attn.qkv.bias"), T)
        else:
            pw = scratch.get("pad_grad")
            if pw is None:   # three padded fp32 gradient scratch tensors carved out of ONE buffer: one memset per layer
                n0, n1, n2 = D * H * hdp, 3 * H * hdp * D, 3 * H * hdp
                flat = _empty((n0 + n1 + n2,), F32, dev)
                pw = (flat[:n0].view(D, H * hdp), flat[n0:n0 + n1].view(3 * H * hdp, D), flat[n0 + n1:].view(3 * H * hdp), flat)
                scratch["pad_grad"] = pw
            pw[3].zero_()
            _wgrad(dx_mid, s.attn, pw[0], gv(pre + "attn.proj.bias"), T)
            _wgrad(dqkv, s.ln1, pw[1], pw[2], T)
            K.head_pad(pw[0], gv(pre + "attn.proj.weight"), D, H, hd, hdp, 1, unpad_add=True)
            K.head_pad(pw[1], gv(pre + "attn.qkv.weight"), 1, 3 * H, hd, hdp, D, unpad_add=True)
            K.head_pad(pw[2], gv(pre + "attn.qkv.bias"), 1, 3 * H, hd, hdp, 1, unpad_add=True)
        dx_in = _empty((T, D), BF16, dev)
        K.layernorm_bwd(dln1, s.x_in, w.n1w, s.mean1, s.rstd1, dx_mid, dx_in, gv(pre + "norm1.weight"),
                        gv(pre + "norm1.bias"))
        dx = dx_in
        if sync is not None:
            sync.ready_down_to(store.offsets[pre + "norm1.weight"][0])
    return dx


# =================================================================================================
# Encoder (VisionTransformer)
# =================================================================================================
class EncoderSaved:
    pass


class _LayerTaps:
    """Collects norm(x) after the requested blocks (out_layers, vision_transformer.py:183-190)."""

    def __init__(self, layers, store):
        self.layers, self.store, self.count, self.outs = set(int(i) for i in layers), store, 0, []

    def __call__(self, i, x):
        if i in self.layers:
            y = torch.empty_like(x)
            K.layernorm_fwd(x, y, self.store.f32("norm.weight"), self.store.f32("norm.bias"), LN_EPS, None, None)
            self.outs.append(y)


def pos_interp_scales(grid0, grid, video):
    """scale_factor that interpolate_pos_encoding (vision_transformer.py:197-246) hands to F.interpolate to take the
    table of token grid `grid0` to `grid`: (T'/Nt, H'/Nh, W'/Nw) for video, sqrt(npatch / N) on both axes for images."""
    if video:
        return tuple(g / n for g, n in zip(grid, grid0))
    s = math.sqrt((grid[1] * grid[2]) / (grid0[1] * grid0[2]))
    return (1.0, s, s)


def encoder_pos(mod, store, grid, dev):
    """The positional embedding added to the tokens of a `grid` = (T', H', W') input, fp32 [N', D].  At the grid the
    encoder was built for this is pos_embed itself (no launch); otherwise vj_pos_interp resamples pos_embed into a new
    buffer on every call, as the reference's interpolate_pos_encoding does (pos_embed may have changed since)."""
    D = mod.embed_dim
    n = grid[0] * grid[1] * grid[2]
    if tuple(grid) == mod.grid:
        return store.f32("pos_embed").view(n, D)
    table = store.f32("pos_embed").view(*mod.grid, D)
    out = _empty((*grid, D), F32, dev)
    K.pos_interp(table, out, pos_interp_scales(mod.grid, grid, mod.is_video), 3 if mod.is_video else 2)
    return out.view(n, D)


def encoder_forward(mod, clips, masks, save, final_norm=True, out_layers=None, grid=None):
    """VisionTransformer.forward (vision_transformer.py:159-195) for all masks at once.

    clips fp32 [B,3,T,H,W] holding whole patches of the token grid `grid` = (T', H', W') (default: the grid the encoder
    was built for); masks: None or list of int64 [B,K_i] indexing that grid.  Returns (out, saved) where out is
    bf16 [sum_i B*K_i, D] (normalised if final_norm else the raw residual stream).
    """
    store = mod._store.adopt(mod)
    store.refresh_shadow()
    spec = mod._spec
    dev = clips.device
    B = clips.shape[0]
    grid = mod.grid if grid is None else tuple(grid)
    N, D = grid[0] * grid[1] * grid[2], mod.embed_dim
    P = mod.patch_embed.proj.weight[0].numel()
    weights = gather_block_weights(store, spec, mod._scratch)
    clips = clips.contiguous()
    if clips.dtype != F32:
        clips = clips.float()
    if masks is None:
        segments = [(B, N)]
        seq = cu_seqlens_for(segments, dev)
        T = seq[3]
        patches = _empty((T, P), BF16, dev)
        K.im2col_tubelets(clips, patches, None, mod.tubelet_size, mod.patch_size)
        rowmap, period = None, N
    else:
        masks = [m.contiguous() for m in masks]
        segments = [(B, int(m.shape[1])) for m in masks]
        seq = cu_seqlens_for(segments, dev)
        T = seq[3]
        patches = _empty((T, P), BF16, dev)
        off = 0
        for m in masks:
            n = B * m.shape[1]
            K.im2col_tubelets(clips, patches[off:off + n], m, mod.tubelet_size, mod.patch_size)
            off += n
        rowmap = torch.cat([m.reshape(-1) for m in masks]).to(torch.int32)
        period = 0
    x = _empty((T, D), BF16, dev)
    w_pe = store.bf16("patch_embed.proj.weight").view(D, P)
    pos = encoder_pos(mod, store, grid, dev)
    K.gemm(patches, w_pe, x, bias=store.f32("patch_embed.proj.bias"), epi=K.EPI_ADD, aux=pos, aux_rowmap=rowmap,
           aux_period=period)
    if out_layers is not None:      # frozen-encoder feature taps (evals): list of normalised per-layer outputs
        if save:
            raise RuntimeError("out_layers is an inference-time feature (frozen encoder); run it under torch.no_grad()")
        taps = _LayerTaps(out_layers, store)
        blocks_forward(spec, weights, x, seq, False, tap=taps)
        return taps.outs, None, segments
    x, bsaved = blocks_forward(spec, weights, x, seq, save)
    out = x
    sv = None
    if save:
        sv = EncoderSaved()
        sv.patches, sv.seq, sv.blocks, sv.weights, sv.x_final, sv.store = patches, seq, bsaved, weights, x, store
    if final_norm:
        out = _empty((T, D), BF16, dev)
        mean = _empty((T,), F32, dev) if save else None
        rstd = _empty((T,), F32, dev) if save else None
        K.layernorm_fwd(x, out, store.f32("norm.weight"), store.f32("norm.bias"), LN_EPS, mean, rstd)
        if save:
            sv.mean, sv.rstd = mean, rstd
    return out, sv, segments


def encoder_backward(mod, sv, dout):
    """dout bf16 [T, D] = grad wrt the normalised encoder output.  Returns the flat fp32 grad buffer."""
    store = sv.store
    spec = mod._spec
    gflat = store.new_grad_buffer()
    gv = lambda name: store.grad_view(gflat, name)
    T, D = dout.shape
    dev = dout.device
    dx = _empty((T, D), BF16, dev)
    K.layernorm_bwd(dout.contiguous(), sv.x_final, store.f32("norm.weight"), sv.mean, sv.rstd, None, dx,
                    gv("norm.weight"), gv("norm.bias"))
    sync = _sync_begin(mod, gflat)
    dx = blocks_backward(spec, sv.weights, sv.blocks, dx, sv.seq, store, gflat, mod._scratch, sync)
    P = sv.patches.shape[1]
    _wgrad(dx, sv.patches, gv("patch_embed.proj.weight").view(D, P), gv("patch_embed.proj.bias"), T)
    if sync is not None:
        sync.finish()
    return gflat


# =================================================================================================
# Predictor (VisionTransformerPredictor)
# =================================================================================================
class PredictorSaved:
    pass


def predictor_forward(mod, z_cat, masks_ctxt, masks_tgt, mask_indices, save):
    """VisionTransformerPredictor.forward (predictor.py:174-239) for all masks at once.

    z_cat bf16 [sum_i B*Ke_i, D_enc]: context tokens of every mask, concatenated in mask order.
    Returns (pred bf16 [sum_i B*Kp_i, D_enc], saved).
    """
    store = mod._store.adopt(mod)
    store.refresh_shadow()
    spec = mod._spec
    dev = z_cat.device
    Dp = spec.dim
    Denc = z_cat.shape[1]
    N = mod.num_patches
    B = masks_ctxt[0].shape[0]
    weights = gather_block_weights(store, spec, mod._scratch)
    masks_ctxt = [m.contiguous() for m in masks_ctxt]
    masks_tgt = [m.contiguous() for m in masks_tgt]
    Ke = [int(m.shape[1]) for m in masks_ctxt]
    Kp = [int(m.shape[1]) for m in masks_tgt]
    Tc = sum(B * k for k in Ke)
    if z_cat.shape[0] != Tc:
        raise RuntimeError(f"predictor: got {z_cat.shape[0]} context rows, masks imply {Tc}")
    z_cat = z_cat.contiguous()
    emb = _empty((Tc, Dp), BF16, dev)
    K.gemm(z_cat, store.bf16("predictor_embed.weight"), emb, bias=store.f32("predictor_embed.bias"))
    segments = [(B, ke + kp) for ke, kp in zip(Ke, Kp)]
    seq = cu_seqlens_for(segments, dev)
    T = seq[3]
    x = _empty((T, Dp), BF16, dev)
    pos = store.f32("predictor_pos_embed").view(N, Dp)
    eo = xo = 0
    for i, (mc, mt) in enumerate(zip(masks_ctxt, masks_tgt)):
        tok = store.f32(f"mask_tokens.{mask_indices[i]}").view(Dp)
        n = B * (Ke[i] + Kp[i])
        K.pred_assemble_fwd(emb[eo:eo + B * Ke[i]], pos, tok, mc, mt, x[xo:xo + n], B, Ke[i], Kp[i], Dp)
        eo += B * Ke[i]
        xo += n
    x, bsaved = blocks_forward(spec, weights, x, seq, save)
    ln = _empty((T, Dp), BF16, dev)
    mean = _empty((T,), F32, dev) if save else None
    rstd = _empty((T,), F32, dev) if save else None
    K.layernorm_fwd(x, ln, store.f32("predictor_norm.weight"), store.f32("predictor_norm.bias"), LN_EPS, mean, rstd)
    Tt = sum(B * k for k in Kp)
    tgt = _empty((Tt, Dp), BF16, dev)
    to = xo = 0
    for i in range(len(Ke)):
        n = B * (Ke[i] + Kp[i])
        K.seq_slice(ln[xo:xo + n], tgt[to:to + B * Kp[i]], B, Ke[i], Kp[i], Dp)
        to += B * Kp[i]
        xo += n
    out = _empty((Tt, Denc), BF16, dev)
    K.gemm(tgt, store.bf16("predictor_proj.weight"), out, bias=store.f32("predictor_proj.bias"))
    sv = None
    if save:
        sv = PredictorSaved()
        sv.store, sv.weights, sv.blocks, sv.seq = store, weights, bsaved, seq
        sv.z_cat, sv.tgt, sv.x_final, sv.mean, sv.rstd = z_cat, tgt, x, mean, rstd
        sv.B, sv.Ke, sv.Kp, sv.mask_indices = B, Ke, Kp, list(mask_indices)
    return out, sv


def predictor_backward(mod, sv, dout):
    """dout bf16 [sum B*Kp_i, D_enc].  Returns (dz_cat bf16 [sum B*Ke_i, D_enc], flat grad buffer)."""
    store = sv.store
    spec = mod._spec
    dev = dout.device
    Dp = spec.dim
    B, Ke, Kp = sv.B, sv.Ke, sv.Kp
    T = sv.seq[3]
    Tt, Denc = dout.shape
    gflat = store.new_grad_buffer()
    gv = lambda name: store.grad_view(gflat, name)
    dout = dout.contiguous()
    # predictor_proj
    dtgt = _empty((Tt, Dp), BF16, dev)
    K.gemm(dout, store.bf16("predictor_proj.weight"), dtgt, b_mn=True)
    _wgrad(dout, sv.tgt, gv("predictor_proj.weight"), gv("predictor_proj.bias"), Tt)
    # x[:, Ke:] slice -> scatter back (context rows get zero gradient from this path)
    dln = _empty((T, Dp), BF16, dev)
    to = xo = 0
    for i in range(len(Ke)):
        n = B * (Ke[i] + Kp[i])
        K.seq_slice(dtgt[to:to + B * Kp[i]], dln[xo:xo + n], B, Ke[i], Kp[i], Dp, scatter=True, zero_ctx=True)
        to += B * Kp[i]
        xo += n
    dx = _empty((T, Dp), BF16, dev)
    K.layernorm_bwd(dln, sv.x_final, store.f32("predictor_norm.weight"), sv.mean, sv.rstd, None, dx,
                    gv("predictor_norm.weight"), gv("predictor_norm.bias"))
    sync = _sync_begin(mod, gflat)
    dx = blocks_backward(spec, sv.weights, sv.blocks, dx, sv.seq, store, gflat, mod._scratch, sync)
    # input assembly: context rows -> d(embed out); target rows -> d(mask token)
    Tc = sum(B * k for k in Ke)
    demb = _empty((Tc, Dp), BF16, dev)
    eo = xo = 0
    for i in range(len(Ke)):
        n = B * (Ke[i] + Kp[i])
        K.pred_assemble_bwd(dx[xo:xo + n], demb[eo:eo + B * Ke[i]], gv(f"mask_tokens.{sv.mask_indices[i]}").view(Dp),
                            B, Ke[i], Kp[i], Dp)
        eo += B * Ke[i]
        xo += n
    dz = _empty((Tc, Denc), BF16, dev)
    K.gemm(demb, store.bf16("predictor_embed.weight"), dz, b_mn=True)
    _wgrad(demb, sv.z_cat, gv("predictor_embed.weight"), gv("predictor_embed.bias"), Tc)
    if sync is not None:
        sync.finish()       # overlaps with the context encoder's backward; waited for at the end of the backward pass
    return dz, gflat
