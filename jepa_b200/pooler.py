"""Frozen-encoder evaluation side of V-JEPA on the sm_90a kernels (SURVEY section 8, row f4): the attentive probe
(src/models/attentive_pooler.py:21-136, CrossAttention / CrossAttentionBlock of src/models/utils/modules.py:122-182) and
the clip aggregation wrapper (evals/video_classification_frozen/utils.py:86-159).

Same constructor arguments, parameter names, initialisation and `state_dict` keys as the reference, so a probe checkpoint
written by the reference's eval loop loads here unchanged.  The accelerated path is INFERENCE: `forward` runs under
no-grad on the hand-written kernels (LayerNorm, wgmma GEMMs with fused bias / GELU / residual epilogues, and
`vj_cross_attn_fwd` for the query-token attention); training the probe is the evals' job and stays with the reference
(`forward` raises if a gradient is requested).  There is no CPU fallback.
"""
import math

import torch
import torch.nn as nn

from . import kernels as K
from .models import MLP
from .pos_embs import get_1d_sincos_pos_embed
from .tensors import apply_masks, trunc_normal_

BF16, F32 = torch.bfloat16, torch.float32
LN_EPS = 1e-5   # nn.LayerNorm default: AttentivePooler is built with norm_layer=nn.LayerNorm (attentive_pooler.py:30)


def _pad_rows(n, mult):
    return (n + mult - 1) // mult * mult


class _Shadow:
    """bf16 copies of the probe's Linear weights (the GEMM B operands), refreshed when a parameter changes."""

    def __init__(self):
        self._cache = {}

    def get(self, p, pad_rows_to=None):
        key = id(p)
        hit = self._cache.get(key)
        if hit is not None and hit[0] == p._version and hit[1].device == p.device:
            return hit[1]
        w = p.detach()
        if pad_rows_to is not None and w.shape[0] % pad_rows_to:
            w = torch.cat([w, w.new_zeros(_pad_rows(w.shape[0], pad_rows_to) - w.shape[0], *w.shape[1:])])
        w = w.to(BF16).contiguous()
        self._cache[key] = (p._version, w)
        return w


class CrossAttention(nn.Module):
    """modules.py:122-153.  `proj` is constructed (and checkpointed) but never applied by the reference's forward."""

    def __init__(self, dim, num_heads=12, qkv_bias=False, use_sdpa=True):
        super().__init__()
        self.num_heads = num_heads
        head_dim = dim // num_heads
        self.scale = head_dim ** -0.5
        self.q = nn.Linear(dim, dim, bias=qkv_bias)
        self.kv = nn.Linear(dim, int(dim * 2), bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.use_sdpa = use_sdpa


class CrossAttentionBlock(nn.Module):
    """modules.py:156-182: q = q + xattn(q, norm1(x)); q = q + mlp(norm2(q))."""

    def __init__(self, dim, num_heads, mlp_ratio=4., qkv_bias=False, act_layer=nn.GELU, norm_layer=nn.LayerNorm):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.xattn = CrossAttention(dim, num_heads=num_heads, qkv_bias=qkv_bias)
        self.norm2 = norm_layer(dim)
        self.mlp = MLP(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer)


class AttentivePooler(nn.Module):
    """attentive_pooler.py:21-102."""

    def __init__(self, num_queries=1, embed_dim=768, num_heads=12, mlp_ratio=4.0, depth=1, norm_layer=nn.LayerNorm,
                 init_std=0.02, qkv_bias=True, complete_block=True):
        super().__init__()
        if depth != 1:
            raise NotImplementedError("AttentivePooler depth > 1 (extra self-attention blocks over the query tokens) is not "
                                      "used by the frozen evaluations (eval.py:182-187 builds depth=1)")
        if embed_dim % num_heads or (embed_dim // num_heads) not in (32, 64, 80, 128):
            raise NotImplementedError(f"head dim {embed_dim // num_heads}: vj_cross_attn_fwd supports 32 / 64 / 80 / 128")
        self.query_tokens = nn.Parameter(torch.zeros(1, num_queries, embed_dim))
        self.complete_block = complete_block
        if complete_block:
            self.cross_attention_block = CrossAttentionBlock(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio,
                                                             qkv_bias=qkv_bias, norm_layer=norm_layer)
        else:
            self.cross_attention_block = CrossAttention(dim=embed_dim, num_heads=num_heads, qkv_bias=qkv_bias)
        self.blocks = None
        self.init_std = init_std
        self.embed_dim, self.num_heads, self.num_queries = embed_dim, num_heads, num_queries
        trunc_normal_(self.query_tokens, std=self.init_std)
        self.apply(self._init_weights)
        self._rescale_blocks()
        self._shadow = _Shadow()

    def _rescale_blocks(self):
        def rescale(param, layer_id):
            param.div_(math.sqrt(2.0 * layer_id))

        if self.complete_block:
            rescale(self.cross_attention_block.xattn.proj.weight.data, 1)
            rescale(self.cross_attention_block.mlp.fc2.weight.data, 1)
        else:
            rescale(self.cross_attention_block.proj.weight.data, 1)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=self.init_std)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def forward(self, x):
        """x [B, S, D] encoder tokens -> pooled query tokens fp32 [B, num_queries, D]."""
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            if x.requires_grad:
                raise NotImplementedError("the accelerated attentive probe is inference-only: run it under torch.no_grad()")
        with torch.no_grad():
            return self._forward(x)

    def _forward(self, x):
        if not x.is_cuda:
            raise RuntimeError("AttentivePooler: CUDA tensors only (there is no CPU fallback)")
        B, S, D = x.shape
        H, nq, dev = self.num_heads, self.num_queries, x.device
        hd = D // H
        sh = self._shadow
        blk = self.cross_attention_block
        xa = blk.xattn if self.complete_block else blk
        x2 = x.reshape(B * S, D).contiguous()
        if x2.dtype not in (BF16, F32):
            x2 = x2.float()
        # keys / values: kv(norm1(x)) - one LayerNorm pass and one [B*S, 2D] GEMM (bias in the epilogue)
        if self.complete_block:
            xn = torch.empty(B * S, D, dtype=BF16, device=dev)
            K.layernorm_fwd(x2, xn, blk.norm1.weight.detach().float(), blk.norm1.bias.detach().float(), blk.norm1.eps)
        else:
            xn = x2 if x2.dtype == BF16 else x2.to(BF16)
        kv = torch.empty(B * S, 2 * D, dtype=BF16, device=dev)
        K.gemm(xn, sh.get(xa.kv.weight), kv, bias=None if xa.kv.bias is None else xa.kv.bias.detach().float())
        # queries: the learned tokens, identical for every clip -> project once, repeat (rows padded to 8 for 16-byte rows)
        q0 = self.query_tokens.detach().reshape(nq, D).float()
        q0b = torch.zeros(_pad_rows(nq, 8), D, dtype=BF16, device=dev)
        q0b[:nq] = q0.to(BF16)
        qp = torch.empty(_pad_rows(nq, 8), D, dtype=BF16, device=dev)
        K.gemm(q0b, sh.get(xa.q.weight), qp, bias=None if xa.q.bias is None else xa.q.bias.detach().float())
        qrep = qp[:nq].repeat(B, 1).contiguous()                       # [B*nq, D], row b*nq + j = query j of clip b
        att = torch.empty(B * nq, D, dtype=BF16, device=dev)
        K.cross_attn_fwd(qrep, kv, att, B, nq, S, H, hd, xa.scale)
        if not self.complete_block:
            return att.float().view(B, nq, D)
        # q = q + y ; q = q + fc2(gelu(fc1(norm2(q))))   (fp32 residual stream: it is only B*nq rows)
        q1 = q0.repeat(B, 1) + att.float()
        M = _pad_rows(B * nq, 8)
        q1p = torch.zeros(M, D, dtype=F32, device=dev)
        q1p[:B * nq] = q1
        ln2 = torch.empty(M, D, dtype=BF16, device=dev)
        K.layernorm_fwd(q1p, ln2, blk.norm2.weight.detach().float(), blk.norm2.bias.detach().float(), blk.norm2.eps)
        hid = blk.mlp.fc1.weight.shape[0]
        g = torch.empty(M, hid, dtype=BF16, device=dev)
        K.gemm(ln2, sh.get(blk.mlp.fc1.weight), g, bias=blk.mlp.fc1.bias.detach().float(), epi=K.EPI_GELU)
        q2 = torch.empty(M, D, dtype=F32, device=dev)
        K.gemm(g, sh.get(blk.mlp.fc2.weight), q2, bias=blk.mlp.fc2.bias.detach().float(), epi=K.EPI_ADD, aux=q1p)
        return q2[:B * nq].view(B, nq, D)


class AttentiveClassifier(nn.Module):
    """attentive_pooler.py:105-136: pooler (one query token) + linear head."""

    def __init__(self, embed_dim=768, num_heads=12, mlp_ratio=4.0, depth=1, norm_layer=nn.LayerNorm, init_std=0.02,
                 qkv_bias=True, num_classes=1000, complete_block=True):
        super().__init__()
        self.pooler = AttentivePooler(num_queries=1, embed_dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio,
                                      depth=depth, norm_layer=norm_layer, init_std=init_std, qkv_bias=qkv_bias,
                                      complete_block=complete_block)
        self.linear = nn.Linear(embed_dim, num_classes, bias=True)
        self._shadow = _Shadow()

    def forward(self, x):
        pooled = self.pooler(x).squeeze(1)                              # [B, D] fp32
        with torch.no_grad():
            B, D = pooled.shape
            C = self.linear.out_features
            M, Cp = _pad_rows(B, 8), _pad_rows(C, 64)                   # GEMM N must be a multiple of 64: zero weight rows
            a = torch.zeros(M, D, dtype=BF16, device=pooled.device)
            a[:B] = pooled.to(BF16)
            bias = torch.zeros(Cp, dtype=F32, device=pooled.device)
            bias[:C] = self.linear.bias.detach().float()
            out = torch.empty(M, Cp, dtype=F32, device=pooled.device)
            K.gemm(a, self._shadow.get(self.linear.weight, pad_rows_to=64), out, bias=bias)
            return out[:B, :C]


class ClipAggregation(nn.Module):
    """Frozen-encoder feature extraction for multi-clip / multi-view evaluation
    (evals/video_classification_frozen/utils.py:86-159): every clip and view goes through the encoder in ONE batch, the
    token sets come back grouped per view, and - with attend_across_segments - the temporal segments of a view are strung
    together (optionally tagged with the 1-D sin-cos position of their frames) so that the probe attends across them."""

    def __init__(self, model, tubelet_size=2, max_frames=10000, use_pos_embed=False, attend_across_segments=False):
        super().__init__()
        self.model = model
        self.tubelet_size = tubelet_size
        self.embed_dim = model.embed_dim
        self.num_heads = model.num_heads
        self.attend_across_segments = attend_across_segments
        self.pos_embed = None
        if use_pos_embed:
            steps = max_frames // tubelet_size
            table = torch.from_numpy(get_1d_sincos_pos_embed(self.embed_dim, steps)).float()
            self.pos_embed = nn.Parameter(table.unsqueeze(0), requires_grad=False)

    def forward(self, x, clip_indices=None):
        """x: list (clips) of lists (views) of [B, C, T, H, W]; returns per view either the list of per-clip token sets
        [B, N, D] or (attend_across_segments) one [B, clips*N, D] tensor."""
        n_clips, n_views = len(x), len(x[0])
        B, frames = x[0][0].shape[0], x[0][0].shape[2]
        tokens = self.model(torch.cat([view for clip in x for view in clip], dim=0))      # clip-major, view-minor batch order
        D = tokens.shape[-1]
        t_tok = frames // self.tubelet_size                 # temporal tokens of one clip
        s_tok = tokens.shape[1] // t_tok                    # spatial tokens per temporal step
        per_view = [[tokens[(c * n_views + v) * B:(c * n_views + v + 1) * B] for c in range(n_clips)] for v in range(n_views)]
        if not self.attend_across_segments:
            return per_view
        tags = None
        if self.pos_embed is not None and clip_indices is not None:
            # temporal position of every tubelet of every clip (frame index / tubelet_size picks a row of the sin-cos table)
            steps = [idx[:, ::self.tubelet_size] for idx in clip_indices]
            rows = apply_masks(self.pos_embed.expand(B, -1, -1), steps, concat=False)       # list of [B, t_tok, D]
            tags = torch.cat(rows, dim=1).unsqueeze(2).expand(-1, -1, s_tok, -1).flatten(1, 2)
        merged = []
        for clips in per_view:
            seq = torch.cat([c.reshape(B, t_tok, s_tok, D) for c in clips], dim=1).flatten(1, 2)
            merged.append(seq if tags is None else seq + tags.to(seq.dtype))
        return merged
