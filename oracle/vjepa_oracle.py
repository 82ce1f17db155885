"""ORACLE - TEST INFRASTRUCTURE ONLY.  Never imported by the product path (jepa_b200/, src/, app/).

CPU restatement of the reference's V-JEPA pre-training hot path in plain torch tensor algebra
(matmul / exp / sum; no nn.Module, no F.scaled_dot_product_attention, no CUDA), parameterised by a
state dict with the reference's own keys.  Runs in float32 or float64.  Gradients come from torch
autograd over these primitive ops.

Pinning: the reference has no tests or golden vectors of its own (SURVEY.md section 4), so this file
is pinned against the reference ITSELF: tests/golden/make_golden.py imports a reference checkout, runs its
unmodified modules on seeded inputs and commits the outputs to tests/golden/*.json|*.pt;
tests/test_oracle_cpu.py checks every function below against those fixtures.

Each function cites the reference lines it restates (paths relative to the reference repository root).
"""
import math

import numpy as np
import torch


# ---------------------------------------------------------------------------------------------
# positional table  (src/models/utils/pos_embs.py:11-44,82-99)
# ---------------------------------------------------------------------------------------------
def sincos_1d(dim, pos):
    omega = np.arange(dim // 2, dtype=float) / (dim / 2.)
    omega = 1. / 10000 ** omega
    out = np.einsum('m,d->md', pos.reshape(-1), omega)
    return np.concatenate([np.sin(out), np.cos(out)], axis=1)


def pos_embed_3d(embed_dim, grid_size, grid_depth, uniform_power=True):
    gd = np.arange(grid_depth, dtype=float)
    gh = np.arange(grid_size, dtype=float)
    gw = np.arange(grid_size, dtype=float)
    gh, gd, gw = np.meshgrid(gh, gd, gw)
    if uniform_power:
        dh = dw = dd = int(np.ceil(embed_dim / 6) * 2)
    else:
        dh = dw = embed_dim // 4
        dd = embed_dim // 2
    emb = np.concatenate([sincos_1d(dd, gd), sincos_1d(dh, gh), sincos_1d(dw, gw)], axis=1)
    return emb[:, :embed_dim]


# ---------------------------------------------------------------------------------------------
# primitives
# ---------------------------------------------------------------------------------------------
# FUSED = True swaps the hand-written primitives for torch's fused CPU operators (F.layer_norm, F.gelu,
# F.scaled_dot_product_attention) - exactly the library calls the reference itself makes - so the CPU
# timing legs of bench.py run at the reference's own CPU speed.  tests/test_oracle_cpu.py checks that
# both modes agree; parity tests always use the plain (FUSED = False) restatement.
FUSED = False


def layer_norm(x, w, b, eps):
    """nn.LayerNorm / F.layer_norm over the last dim (biased variance)."""
    if FUSED:
        return torch.nn.functional.layer_norm(x, (x.shape[-1],), w, b, eps)
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    y = (x - mu) / torch.sqrt(var + eps)
    if w is not None:
        y = y * w + b
    return y


def gelu(x):
    """nn.GELU() exact erf form (src/models/utils/modules.py:26)."""
    if FUSED:
        return torch.nn.functional.gelu(x)
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def linear(x, w, b):
    if FUSED:
        return torch.nn.functional.linear(x, w, b)
    return x @ w.t() + b


def apply_masks(x, masks, concat=True):
    """src/masks/utils.py:11-23: out[b,k,:] = x[b, idx[b,k], :] per mask, concatenated on batch."""
    outs = []
    for m in masks:
        B, Kk = m.shape
        rows = torch.arange(B).unsqueeze(1).expand(B, Kk)
        outs.append(x[rows, m])
    return torch.cat(outs, dim=0) if concat else outs


def repeat_interleave_batch(x, B, repeat):
    """src/utils/tensors.py:65-71."""
    N = len(x) // B
    return torch.cat([torch.cat([x[i * B:(i + 1) * B] for _ in range(repeat)], dim=0) for i in range(N)], dim=0)


def patch_embed_3d(clips, w, b):
    """PatchEmbed3D (src/models/utils/patch_embed.py:47-57): Conv3d k=s=(tub,ps,ps) as unfold + matmul.

    Token order (t', h', w') row-major; patch vector order (c, dt, dh, dw)."""
    D, C, tub, ps, _ = w.shape
    B, _, T, H, W = clips.shape
    x = clips.reshape(B, C, T // tub, tub, H // ps, ps, W // ps, ps)
    x = x.permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(B, (T // tub) * (H // ps) * (W // ps), C * tub * ps * ps)
    return x @ w.reshape(D, -1).t() + b


def attention(x, S, pre, heads):
    """Attention.forward (modules.py:61-78): dense softmax(q k^T / sqrt(hd)) v; the mask arg is unused."""
    B, N, C = x.shape
    hd = C // heads
    qkv = linear(x, S[pre + 'qkv.weight'], S[pre + 'qkv.bias']).reshape(B, N, 3, heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    if FUSED:
        y = torch.nn.functional.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, C)
        return linear(y, S[pre + 'proj.weight'], S[pre + 'proj.bias'])
    att = (q @ k.transpose(-2, -1)) * (hd ** -0.5)
    att = att - att.amax(dim=-1, keepdim=True)
    att = torch.exp(att)
    att = att / att.sum(dim=-1, keepdim=True)
    y = (att @ v).transpose(1, 2).reshape(B, N, C)
    return linear(y, S[pre + 'proj.weight'], S[pre + 'proj.bias'])


def block(x, S, pre, heads, eps=1e-6):
    """Block.forward (modules.py:114-120)."""
    x = x + attention(layer_norm(x, S[pre + 'norm1.weight'], S[pre + 'norm1.bias'], eps), S, pre + 'attn.', heads)
    h = layer_norm(x, S[pre + 'norm2.weight'], S[pre + 'norm2.bias'], eps)
    h = linear(gelu(linear(h, S[pre + 'mlp.fc1.weight'], S[pre + 'mlp.fc1.bias'])), S[pre + 'mlp.fc2.weight'],
               S[pre + 'mlp.fc2.bias'])
    return x + h


# ---------------------------------------------------------------------------------------------
# networks
# ---------------------------------------------------------------------------------------------
def encoder(S, clips, masks, depth, heads, eps=1e-6, out_layers=None):
    """VisionTransformer.forward (src/models/vision_transformer.py:159-195); S uses backbone-level keys.
    out_layers: list of block indices -> list of norm(x) after those blocks (:183-190)."""
    x = patch_embed_3d(clips, S['patch_embed.proj.weight'], S['patch_embed.proj.bias'])
    x = x + S['pos_embed']
    if masks is not None:
        x = apply_masks(x, masks)
    outs = []
    for i in range(depth):
        x = block(x, S, f'blocks.{i}.', heads, eps)
        if out_layers is not None and i in out_layers:
            outs.append(layer_norm(x, S['norm.weight'], S['norm.bias'], eps))
    if out_layers is not None:
        return outs
    return layer_norm(x, S['norm.weight'], S['norm.bias'], eps)


def predictor(S, ctxt, masks_ctxt, masks_tgt, mask_index, depth, heads, eps=1e-6):
    """VisionTransformerPredictor.forward with mask tokens (src/models/predictor.py:174-239), one mask pair."""
    B = ctxt.shape[0]
    x = linear(ctxt, S['predictor_embed.weight'], S['predictor_embed.bias'])
    n_ctxt = x.shape[1]
    pos = S['predictor_pos_embed'].expand(B, -1, -1)
    x = x + apply_masks(pos, [masks_ctxt])
    n_tok = len([k for k in S if k.startswith('mask_tokens.')])
    tok = S[f'mask_tokens.{mask_index % n_tok}']
    pred = apply_masks(tok.expand(B, pos.shape[1], -1), [masks_tgt]) + apply_masks(pos, [masks_tgt])
    x = torch.cat([x, pred], dim=1)
    for i in range(depth):
        x = block(x, S, f'predictor_blocks.{i}.', heads, eps)
    x = layer_norm(x, S['predictor_norm.weight'], S['predictor_norm.bias'], eps)
    return linear(x[:, n_ctxt:], S['predictor_proj.weight'], S['predictor_proj.bias'])


# ---------------------------------------------------------------------------------------------
# train step pieces  (app/vjepa/train.py:414-498)
# ---------------------------------------------------------------------------------------------
def forward_target(S_tgt, clips, masks_pred, depth, heads):
    """train.py:419-429: no-grad target encoder, affine-free layer_norm (eps 1e-5), gather targets."""
    with torch.no_grad():
        h = encoder(S_tgt, clips, None, depth, heads)
        h = layer_norm(h, None, None, 1e-5)
        return apply_masks(h, masks_pred, concat=False)


def forward_context(S_enc, S_pred, clips, masks_enc, masks_pred, depth, heads, pred_depth, pred_heads):
    """train.py:431-438 with MultiMaskWrapper / PredictorMultiMaskWrapper loops (multimask.py:17-48)."""
    z = [encoder(S_enc, clips, [m], depth, heads) for m in masks_enc]
    return [predictor(S_pred, zi, mc, mt, i, pred_depth, pred_heads)
            for i, (zi, mc, mt) in enumerate(zip(z, masks_enc, masks_pred))]


def loss_fn(z, h, loss_exp=1.0):
    """train.py:440-446."""
    loss = 0.
    for zi, hi in zip(z, h):
        loss = loss + torch.mean(torch.abs(zi - hi) ** loss_exp) / loss_exp
    return loss / len(z)


def reg_fn(z):
    """train.py:448-449 and :458-459: mean(relu(1 - mean_i sqrt(var_unbiased(z_i, dim=1) + 1e-4)))."""
    pstd = sum(torch.sqrt(zi.var(dim=1) + 0.0001) for zi in z) / len(z)
    return torch.mean(torch.relu(1. - pstd))


def ema(S_tgt, S_enc, m):
    """train.py:484-487: k <- k*m + (1-m)*q, in place, every parameter (incl. pos_embed)."""
    with torch.no_grad():
        for k in S_tgt:
            S_tgt[k].mul_(m).add_((1. - m) * S_enc[k].detach())


# ---------------------------------------------------------------------------------------------
# input pipeline  (app/vjepa/transforms.py:86-117,140-153; src/datasets/utils/video/transforms.py:545-577,160-190)
# ---------------------------------------------------------------------------------------------
def video_transform(buffer_u8, box, flip, crop_size, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
    """VideoTransform.__call__ on its non-auto-augment path with the random decisions (crop box, flip) given:
    uint8 [T,H,W,3] -> float -> [3,T,H,W] -> crop -> bilinear resize (align_corners=False, no antialias; written out
    explicitly: src = max(0, (dst + 0.5) * in/out - 0.5)) -> flip -> (x - 255 mean) / (255 std).  Returns fp32 [3,T,S,S]."""
    x = torch.as_tensor(np.asarray(buffer_u8)).to(torch.float32).permute(3, 0, 1, 2)
    i, j, h, w = box
    x = x[:, :, i:i + h, j:j + w]
    S = crop_size

    def axis(n_in):
        src = (torch.arange(S, dtype=torch.float32) + 0.5) * (torch.tensor(float(n_in)) / float(S)) - 0.5
        src = torch.clamp(src, min=0.0)
        i0 = src.floor().to(torch.int64).clamp(max=n_in - 1)
        i1 = (i0 + 1).clamp(max=n_in - 1)
        l1 = src - i0.to(torch.float32)
        return i0, i1, 1.0 - l1, l1

    y0, y1, hy, ly = axis(h)
    x0, x1, hx, lx = axis(w)
    top = x[:, :, y0][:, :, :, x0] * hx + x[:, :, y0][:, :, :, x1] * lx
    bot = x[:, :, y1][:, :, :, x0] * hx + x[:, :, y1][:, :, :, x1] * lx
    out = hy[:, None] * top + ly[:, None] * bot
    if flip:
        out = out.flip(-1)
    m = torch.tensor(mean, dtype=torch.float32) * 255.
    s = torch.tensor(std, dtype=torch.float32) * 255.
    return (out - m[:, None, None, None]) / s[:, None, None, None]


# ---------------------------------------------------------------------------------------------
# attentive probe of the frozen-encoder evaluations (SURVEY section 8 row f4)
# ---------------------------------------------------------------------------------------------
def cross_attention(S, pre, q, x, heads):
    """CrossAttention.forward (src/models/utils/modules.py:138-153): q/kv projections, softmax(q k^T hd^-0.5) v per head.
    NOTE the reference never applies `proj` in this forward (modules.py:152-153) - neither does this restatement."""
    B, n, C = q.shape
    hd = C // heads
    qh = linear(q, S[pre + "q.weight"], S[pre + "q.bias"]).reshape(B, n, heads, hd).permute(0, 2, 1, 3)
    N = x.shape[1]
    kv = linear(x, S[pre + "kv.weight"], S[pre + "kv.bias"]).reshape(B, N, 2, heads, hd).permute(2, 0, 3, 1, 4)
    k, v = kv[0], kv[1]
    att = torch.softmax((qh @ k.transpose(-2, -1)) * hd ** -0.5, dim=-1)
    return (att @ v).transpose(1, 2).reshape(B, n, C)


def attentive_pooler(S, x, heads, complete_block=True, pre="pooler."):
    """AttentivePooler.forward (src/models/attentive_pooler.py:96-102), depth = 1; CrossAttentionBlock.forward
    (modules.py:178-182): q = q + xattn(q, norm1(x)); q = q + mlp(norm2(q)); nn.LayerNorm default eps 1e-5."""
    q = S[pre + "query_tokens"].repeat(len(x), 1, 1)
    b = pre + "cross_attention_block."
    if not complete_block:
        return cross_attention(S, b, q, x, heads)
    y = cross_attention(S, b + "xattn.", q, layer_norm(x, S[b + "norm1.weight"], S[b + "norm1.bias"], 1e-5), heads)
    q = q + y
    h = gelu(linear(layer_norm(q, S[b + "norm2.weight"], S[b + "norm2.bias"], 1e-5), S[b + "mlp.fc1.weight"],
                    S[b + "mlp.fc1.bias"]))
    return q + linear(h, S[b + "mlp.fc2.weight"], S[b + "mlp.fc2.bias"])


def attentive_classifier(S, x, heads, complete_block=True):
    """AttentiveClassifier.forward (attentive_pooler.py:133-136)."""
    return linear(attentive_pooler(S, x, heads, complete_block).squeeze(1), S["linear.weight"], S["linear.bias"])
