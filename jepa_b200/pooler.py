"""Frozen-encoder evaluation side of V-JEPA on the sm_90a kernels (SURVEY section 8, row f4): the attentive probe
(src/models/attentive_pooler.py:21-136, CrossAttention / CrossAttentionBlock of src/models/utils/modules.py:122-182) and
the clip and frame aggregation wrappers (evals/video_classification_frozen/utils.py:23-159).

Same constructor arguments, parameter names, initialisation and `state_dict` keys as the reference, so a probe checkpoint
written by the reference's eval loop loads here unchanged.  Everything runs on the hand-written kernels (LayerNorm, wgmma
GEMMs with fused bias / GELU / residual epilogues, `vj_cross_attn_fwd` / `vj_cross_attn_bwd` for the query-token
attention); there is no CPU fallback.

Training the probe (the frozen evaluations' job, eval.py:317-373): with parameters that require grad, `forward` saves
what the backward needs and returns outputs with a grad_fn.  The probe's parameters live in one FlatParamStore (fp32
master weights, bf16 GEMM operands in its shadow) and the backward writes ONE flat fp32 gradient buffer, so FlatAdamW,
FlatGradScaler and step.clip_grad_norm_ each take one launch over it.  Several probe calls in one step (one per temporal
segment without attend_across_segments) accumulate into the same buffer.  `proj` gets no gradient: the reference builds
it but never applies it (modules.py:152-153).  Gradients into the encoder's tokens (fine-tuning) and depth > 1 are not
implemented.

Precision: the probe computes bf16 x bf16 -> fp32 by default, inside an autocast region or not.  Built with
`follow_autocast=True`, it follows an fp16 autocast (torch.autocast('cuda', dtype=torch.float16) or
torch.cuda.amp.autocast(dtype=torch.float16), as the reference's eval loops open, eval.py:323): every 16-bit operand and
activation is then fp16 (the fp16 shadow of the store, vj_gemm_f16, vj_cross_attn_*_f16, vj_layernorm_bwd_f16,
vj_colsum_f16), while the residual stream, the LayerNorm statistics, lse2, dq and every weight gradient stay fp32.  The
outputs then have the dtypes the reference's modules return under that autocast: fp16 logits from AttentiveClassifier,
fp32 from AttentivePooler(complete_block=True), fp16 from AttentivePooler(complete_block=False).  Outside autocast, or
under a bf16 autocast, such a probe computes in bf16 as by default.
"""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import kernels as K
from .models import MLP, VisionTransformer
from .params import FlatParamStore
from .pos_embs import get_1d_sincos_pos_embed
from .tensors import apply_masks, trunc_normal_

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32


def _pad_rows(n, mult):
    return (n + mult - 1) // mult * mult


def _store_of(module, anchor):
    """The FlatParamStore that holds every parameter of `module` (adopting them into module._store if none does) and
    the name prefix of `module`'s parameters inside it.  A classifier's store holds its pooler too ('pooler.' prefix),
    so calling clf.pooler directly reuses it instead of moving the parameters."""
    st = getattr(anchor, "_vj_store", None)
    if st is None or not all(st.owns(p) for p in module.parameters()):
        st = module._store.adopt(module)
    return st, anchor._vj_name[:-len("query_tokens")] if anchor._vj_name.endswith("query_tokens") else ""


def _grad_buffer(store, members):
    """The flat gradient buffer of this step: the one the members' .grad already alias (an earlier probe call of the
    same step), else a new zero buffer."""
    if all(p.grad is not None for _, p in members):
        gflat = store.grad_buffer(p for _, p in members)
        if gflat is not None:
            store.grads_changed()
            return gflat
    gflat = store.new_grad_buffer()
    for n, p in members:
        p.grad = store.grad_view(gflat, n)
    return gflat


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
                 init_std=0.02, qkv_bias=True, complete_block=True, follow_autocast=False):
        super().__init__()
        self.follow_autocast = follow_autocast       # a plain attribute: not a parameter, not in the state_dict
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
        self._store = FlatParamStore()

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

    def _load_from_state_dict(self, *args, **kwargs):
        nn.Module._load_from_state_dict(self, *args, **kwargs)
        _invalidate(self)

    def forward(self, x):
        """x [B, S, D] encoder tokens -> pooled query tokens [B, num_queries, D], fp32 (fp16 with complete_block=False
        under an fp16 autocast that the probe follows)."""
        return _run_probe(self, self, x, head=False)


def _invalidate(module):
    """Parameters changed behind the optimizer's back (load_state_dict): re-cast the bf16 operands at the next forward."""
    for p in module.parameters():
        st = getattr(p, "_vj_store", None)
        if st is not None:
            st.invalidate_shadow()
    module._store.invalidate_shadow()


def _inside_torch_ddp(module):
    """True while torch's own DistributedDataParallel runs `module`'s forward.  Its reducer waits for per-parameter
    gradient hooks, which the probe's flat-buffer backward never fires, so the replicas would silently drift apart."""
    active = getattr(torch.nn.parallel.DistributedDataParallel, "_active_ddp_module", None)
    return active is not None and getattr(active, "module", None) is module


def _run_probe(module, pooler, x, head):
    if _inside_torch_ddp(module):
        raise NotImplementedError("the attentive probe cannot be wrapped in torch.nn.parallel.DistributedDataParallel "
                                  "(its backward writes one flat gradient buffer and never fires the reducer's hooks); "
                                  "wrap it in src.utils.distributed.DistributedDataParallel")
    if not x.is_cuda:
        raise RuntimeError("AttentivePooler: CUDA tensors only (there is no CPU fallback)")
    train = torch.is_grad_enabled() and any(p.requires_grad for p in module.parameters())
    if torch.is_grad_enabled() and x.requires_grad:
        raise NotImplementedError("the accelerated attentive probe trains the probe only: gradients into the encoder's "
                                  "tokens (fine-tuning) are not implemented - pass detached tokens")
    store, prefix = _store_of(module, pooler.query_tokens)
    dt = K.compute_dtype() if getattr(module, "follow_autocast", False) else BF16
    store.refresh_shadow(dt)
    if not train:
        with torch.no_grad():
            y, _ = _probe_forward(pooler, store, prefix, x, head, save=False, dt=dt)
        return y
    return _ProbeFn.apply(pooler, store, prefix, x, head, dt, getattr(module, "_vj_probe_sync", None),
                          *module.parameters())


class _ProbeFn(torch.autograd.Function):
    """forward: the probe on the kernels, saving its activations.  backward: accumulates every trainable parameter's
    gradient into the store's flat gradient buffer of this step (and points .grad at its slices) - a flat buffer that two
    probe calls of one step can share, which autograd's per-tensor accumulation would break apart - and returns None for
    the parameters.  proj is left without a gradient, as in the reference."""

    @staticmethod
    def forward(ctx, pooler, store, prefix, x, head, dt, sync, *params):
        y, sv = _probe_forward(pooler, store, prefix, x, head, save=True, dt=dt)
        ctx.pooler, ctx.store, ctx.prefix, ctx.sv, ctx.head, ctx.params = pooler, store, prefix, sv, head, params
        ctx.sync = sync
        return y

    @staticmethod
    def backward(ctx, dy):
        pooler, store, prefix, sv = ctx.pooler, ctx.store, ctx.prefix, ctx.sv
        members = [(p._vj_name, p) for p in ctx.params if p.requires_grad and ".proj." not in p._vj_name]
        if members:
            gflat = _grad_buffer(store, members)
            _probe_backward(pooler, store, prefix, sv, dy, ctx.head, gflat)
            if ctx.sync is not None:       # data parallel: average the buffer once, at the end of this backward pass
                ctx.sync.mark(gflat)
        n = len(ctx.params)
        ctx.sv = ctx.params = ctx.sync = None
        return (None,) * 7 + (None,) * n


def _names(pooler, prefix):
    blk = prefix + "cross_attention_block."
    return blk, (blk + "xattn." if pooler.complete_block else blk)


def _probe_forward(pooler, store, prefix, x, head, save, dt=BF16):
    """Pooler (+ linear head) forward with 16-bit operands of dtype dt (bf16, or fp16 under an fp16 autocast the probe
    follows).  Returns (pooled [B, nq, D] or logits [B, C], saved activations): fp32, except the fp16 logits and the fp16
    pooled tokens of complete_block=False when dt is fp16."""
    B, S, D = x.shape
    H, nq, dev = pooler.num_heads, pooler.num_queries, x.device
    hd = D // H
    blk, xa = _names(pooler, prefix)
    w = lambda name: store.w16(name, dt)
    f = store.f32
    has_qkv_bias = (xa + "kv.bias") in store.offsets
    x2 = x.detach().reshape(B * S, D).contiguous()
    # fp16 LayerNorm reads fp16 or fp32 only (under autocast the encoder hands fp32); training in fp16 reads fp16 tokens
    # as fp32 (exact), because the LayerNorm backward pairs its fp16 dy with an fp32 x
    if x2.dtype not in (dt, F32) or (dt == F16 and save and x2.dtype == F16):
        x2 = x2.float()
    sv = SimpleNamespace(B=B, S=S, x2=x2, dt=dt) if save else None
    # keys / values: kv(norm1(x)) - one LayerNorm pass and one [B*S, 2D] GEMM (bias in the epilogue)
    if pooler.complete_block:
        xn = torch.empty(B * S, D, dtype=dt, device=dev)
        mean1 = torch.empty(B * S, dtype=F32, device=dev) if save else None
        rstd1 = torch.empty(B * S, dtype=F32, device=dev) if save else None
        K.layernorm_fwd(x2, xn, f(blk + "norm1.weight"), f(blk + "norm1.bias"), pooler.cross_attention_block.norm1.eps,
                        mean1, rstd1)
    else:
        xn = x2 if x2.dtype == dt else x2.to(dt)
        mean1 = rstd1 = None
    kv = torch.empty(B * S, 2 * D, dtype=dt, device=dev)
    K.gemm(xn, w(xa + "kv.weight"), kv, bias=f(xa + "kv.bias") if has_qkv_bias else None)
    # queries: the learned tokens, identical for every clip -> project once, repeat (rows padded to 8 for 16-byte rows)
    q0 = f(prefix + "query_tokens").reshape(nq, D)
    q0b = torch.zeros(_pad_rows(nq, 8), D, dtype=dt, device=dev)
    q0b[:nq] = q0.to(dt)
    qp = torch.empty(_pad_rows(nq, 8), D, dtype=dt, device=dev)
    K.gemm(q0b, w(xa + "q.weight"), qp, bias=f(xa + "q.bias") if has_qkv_bias else None)
    qrep = qp[:nq].repeat(B, 1).contiguous()                       # [B*nq, D], row b*nq + j = query j of clip b
    att = torch.empty(B * nq, D, dtype=dt, device=dev)
    if save:
        lse2 = torch.empty(B * nq, H, dtype=F32, device=dev)
        K.cross_attn_fwd_lse(qrep, kv, att, lse2, B, nq, S, H, hd, pooler.cross_attention_block.xattn.scale
                             if pooler.complete_block else pooler.cross_attention_block.scale)
        sv.xn, sv.mean1, sv.rstd1, sv.kv, sv.q0b, sv.qrep, sv.att, sv.lse2 = xn, mean1, rstd1, kv, q0b, qrep, att, lse2
    else:
        K.cross_attn_fwd(qrep, kv, att, B, nq, S, H, hd, pooler.cross_attention_block.xattn.scale
                         if pooler.complete_block else pooler.cross_attention_block.scale)
    M = _pad_rows(B * nq, 8)
    if not pooler.complete_block:
        pooled = att.clone() if dt == F16 else att.float()     # SDPA's output dtype under fp16 autocast (att is saved)
    else:
        # q = q + y ; q = q + fc2(gelu(fc1(norm2(q))))   (fp32 residual stream: it is only B*nq rows)
        q1p = torch.zeros(M, D, dtype=F32, device=dev)
        q1p[:B * nq] = q0.repeat(B, 1) + att.float()
        ln2 = torch.empty(M, D, dtype=dt, device=dev)
        mean2 = torch.empty(M, dtype=F32, device=dev) if save else None
        rstd2 = torch.empty(M, dtype=F32, device=dev) if save else None
        K.layernorm_fwd(q1p, ln2, f(blk + "norm2.weight"), f(blk + "norm2.bias"), pooler.cross_attention_block.norm2.eps,
                        mean2, rstd2)
        hid = store.offsets[blk + "mlp.fc1.weight"][2][0]
        g = torch.empty(M, hid, dtype=dt, device=dev)
        # training keeps gelu'(pre-activation) from the same epilogue: the fc1 dgrad is then a plain multiply
        h = torch.empty(M, hid, dtype=dt, device=dev) if save else None
        K.gemm(ln2, w(blk + "mlp.fc1.weight"), g, bias=f(blk + "mlp.fc1.bias"), epi=K.EPI_GELU_GRAD if save else K.EPI_GELU,
               aux_out=h)
        q2 = torch.empty(M, D, dtype=F32, device=dev)
        K.gemm(g, w(blk + "mlp.fc2.weight"), q2, bias=f(blk + "mlp.fc2.bias"), epi=K.EPI_ADD, aux=q1p)
        pooled = q2[:B * nq]
        if save:
            sv.q1p, sv.ln2, sv.mean2, sv.rstd2, sv.h, sv.g = q1p, ln2, mean2, rstd2, h, g
    if not head:
        return pooled.view(B, nq, D), sv
    # linear head as logits^T [C, Np] = W [C, D] . pooled^T: the GEMM's N is the (padded) batch, so the weight is read
    # straight from the store for any class count; the bias comes in through the residual epilogue
    C = store.offsets["linear.weight"][2][0]
    Np = _pad_rows(B, 64)
    pb = torch.zeros(Np, D, dtype=dt, device=dev)
    pb[:B] = pooled
    bias_t = f("linear.bias").unsqueeze(1).expand(C, Np).contiguous()
    lt = torch.empty(C, Np, dtype=F32, device=dev)
    K.gemm(w("linear.weight"), pb, lt, epi=K.EPI_ADD, aux=bias_t)
    if save:
        sv.pb = pb
    logits = lt[:, :B].t()
    # nn.Linear under fp16 autocast returns fp16: the fp32 accumulator plus bias, rounded once (past 65504: +-inf)
    return (logits.to(F16) if dt == F16 else logits).contiguous(), sv


def _probe_backward(pooler, store, prefix, sv, dy, head, gflat):
    B, S, D, dt = sv.B, sv.S, sv.x2.shape[1], sv.dt
    H, nq, dev = pooler.num_heads, pooler.num_queries, gflat.device
    hd = D // H
    blk, xa = _names(pooler, prefix)
    w = lambda name: store.w16(name, dt)
    f = store.f32
    gv = lambda name: store.grad_view(gflat, name)
    has_qkv_bias = (xa + "kv.bias") in store.offsets
    M, Mp = B * nq, _pad_rows(B * nq, 8)
    if head:
        # dlogits [B, C] -> dW += dlogits^T pooled, db += column sums, dpooled = dlogits W
        C = store.offsets["linear.weight"][2][0]
        Np = sv.pb.shape[0]
        dl = dy.detach().to(F32)
        dlt = torch.zeros(C, Np, dtype=dt, device=dev)
        dlt[:, :B] = dl.t()
        K.gemm(dlt, sv.pb, gv("linear.weight"), b_mn=True, accumulate=True)
        Cp = _pad_rows(C, 8)      # colsum works on 8-column groups: the bias slice is followed by store padding
        dlp = torch.zeros(B, Cp, dtype=F32, device=dev)
        dlp[:, :C] = dl
        boff = store.offsets["linear.bias"][0]
        K.colsum(dlp, gflat[boff:boff + Cp])
        dpooled = torch.empty(Np, D, dtype=F32, device=dev)
        K.gemm(dlt, w("linear.weight"), dpooled, a_mn=True, b_mn=True)
        dq2 = torch.zeros(Mp, D, dtype=F32, device=dev)
        dq2[:M] = dpooled[:B]
    else:
        dq2 = torch.zeros(Mp, D, dtype=F32, device=dev)
        dq2[:M] = dy.detach().reshape(M, D)
    if pooler.complete_block:
        # MLP: q2 = q1 + fc2(gelu(fc1(ln2(q1))))
        dq2b = dq2.to(dt)
        _wgrad(dq2b, sv.g, gv(blk + "mlp.fc2.weight"), gv(blk + "mlp.fc2.bias"), Mp)
        hid = sv.g.shape[1]
        dpre = torch.empty(Mp, hid, dtype=dt, device=dev)
        K.gemm(dq2b, w(blk + "mlp.fc2.weight"), dpre, b_mn=True, epi=K.EPI_MUL, aux=sv.h)
        _wgrad(dpre, sv.ln2, gv(blk + "mlp.fc1.weight"), gv(blk + "mlp.fc1.bias"), Mp)
        dln2 = torch.empty(Mp, D, dtype=dt, device=dev)
        K.gemm(dpre, w(blk + "mlp.fc1.weight"), dln2, b_mn=True)
        dq1 = torch.empty(Mp, D, dtype=F32, device=dev)
        K.layernorm_bwd(dln2, sv.q1p, f(blk + "norm2.weight"), sv.mean2, sv.rstd2, dq2, dq1, gv(blk + "norm2.weight"),
                        gv(blk + "norm2.bias"))
    else:
        dq1 = dq2
    # cross-attention
    datt = dq1[:M].to(dt)
    dqrep = torch.empty(M, D, dtype=F32, device=dev)
    dkv = torch.empty(B * S, 2 * D, dtype=dt, device=dev)
    scale = pooler.cross_attention_block.xattn.scale if pooler.complete_block else pooler.cross_attention_block.scale
    K.cross_attn_bwd(sv.qrep, sv.kv, sv.att, datt, sv.lse2, dqrep, dkv, B, nq, S, H, hd, scale)
    # the query projection is shared by all clips: sum its gradient over them (row b*nq + j -> query j)
    dqp = torch.zeros(_pad_rows(nq, 8), D, dtype=F32, device=dev)
    gq = gv(prefix + "query_tokens").view(nq, D)
    for j in range(nq):
        K.colsum(dqrep, dqp[j], period=nq, lo=j, hi=j + 1)
        if pooler.complete_block:      # residual path q1 = q0 + y
            K.colsum(dq1[:M], gq[j], period=nq, lo=j, hi=j + 1)
    dqpb = dqp.to(dt)
    _wgrad(dqpb, sv.q0b, gv(xa + "q.weight"), None, dqpb.shape[0])
    if has_qkv_bias:
        K.colsum(dqp, gv(xa + "q.bias"))
    K.gemm(dqpb[:nq], w(xa + "q.weight"), gq, b_mn=True, accumulate=True)
    # keys / values: kv = xn W_kv^T + b over all B*S tokens
    _wgrad(dkv, sv.xn, gv(xa + "kv.weight"), gv(xa + "kv.bias") if has_qkv_bias else None, B * S)
    if pooler.complete_block:
        # norm1's affine parameters only: the gradient into the frozen encoder's tokens goes to scratch
        dxn = torch.empty(B * S, D, dtype=dt, device=dev)
        K.gemm(dkv, w(xa + "kv.weight"), dxn, b_mn=True)
        dx = torch.empty_like(sv.x2)
        K.layernorm_bwd(dxn, sv.x2, f(blk + "norm1.weight"), sv.mean1, sv.rstd1, None, dx, gv(blk + "norm1.weight"),
                        gv(blk + "norm1.bias"))


def _wgrad(dy, act, grad_out, bias_grad, tokens):
    """grad_out[N_out, K_in] += dy^T act over `tokens` rows; bias_grad[N_out] += colsum(dy).  One CTA per output tile
    (split_k = 1: no reduce-add of split pieces, so the weight gradients are bitwise reproducible); the probe's weight
    gradients have 64 .. 256 output tiles, which fills the GPU without splitting the token range."""
    K.gemm(dy, act, grad_out, a_mn=True, b_mn=True, accumulate=True, split_k=1)
    if bias_grad is not None:
        K.colsum(dy, bias_grad)


class AttentiveClassifier(nn.Module):
    """attentive_pooler.py:105-136: pooler (one query token) + linear head."""

    def __init__(self, embed_dim=768, num_heads=12, mlp_ratio=4.0, depth=1, norm_layer=nn.LayerNorm, init_std=0.02,
                 qkv_bias=True, num_classes=1000, complete_block=True, follow_autocast=False):
        super().__init__()
        self.follow_autocast = follow_autocast       # a plain attribute: not a parameter, not in the state_dict
        self.pooler = AttentivePooler(num_queries=1, embed_dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio,
                                      depth=depth, norm_layer=norm_layer, init_std=init_std, qkv_bias=qkv_bias,
                                      complete_block=complete_block, follow_autocast=follow_autocast)
        self.linear = nn.Linear(embed_dim, num_classes, bias=True)
        self._store = FlatParamStore()

    def _load_from_state_dict(self, *args, **kwargs):
        nn.Module._load_from_state_dict(self, *args, **kwargs)
        _invalidate(self)

    def forward(self, x):
        """x [B, S, D] encoder tokens -> logits [B, num_classes]: fp32, or fp16 under an fp16 autocast the classifier
        follows."""
        return _run_probe(self, self.pooler, x, head=True)


class FrameAggregation(nn.Module):
    """An image encoder evaluated on video (evals/video_classification_frozen/utils.py:23-83, used when the pre-training
    config has frames_per_clip == 1): every frame of every segment and view goes through the encoder in ONE batch, and
    each view comes back as one sequence [B, frames * segments * N, D], segments strung together along time - optionally
    tagged with the 1-D sin-cos position of each frame's clip index.  As in the reference, attend_across_segments is
    accepted but has no effect: the output is always one sequence per view.

    `model` must be an image encoder of jepa_b200.models (VisionTransformer with num_frames == 1), the encoder that runs
    the frames on the kernels; any other module (a video encoder, an eager PyTorch model) raises NotImplementedError."""

    def __init__(self, model, max_frames=10000, use_pos_embed=False, attend_across_segments=False):
        super().__init__()
        if not isinstance(model, VisionTransformer) or model.is_video:
            what = "a video encoder (num_frames > 1)" if isinstance(model, VisionTransformer) else type(model).__name__
            raise NotImplementedError(
                f"FrameAggregation runs an image encoder of jepa_b200.models (VisionTransformer, num_frames=1) frame by "
                f"frame on the sm_90a kernels; wrapping {what} is not implemented")
        self.model = model
        self.embed_dim = model.embed_dim
        self.num_heads = model.num_heads
        self.attend_across_segments = attend_across_segments
        self.pos_embed = None
        if use_pos_embed:
            table = torch.from_numpy(get_1d_sincos_pos_embed(self.embed_dim, max_frames)).float()
            self.pos_embed = nn.Parameter(table.unsqueeze(0), requires_grad=False)

    def forward(self, x, clip_indices=None):
        """x: list (segments) of lists (views) of [B, C, T, H, W]; returns per view [B, segments * T * N, D]."""
        n_views = len(x[0])
        clips = torch.cat([torch.cat(views, dim=0) for views in x], dim=2)     # views on batch, segments along time
        VB, C, T, H, W = clips.shape
        tokens = self.model(clips.transpose(1, 2).reshape(VB * T, C, H, W))  # frame-major within each clip
        N, D = tokens.shape[1], tokens.shape[2]
        tokens = tokens.view(VB, T * N, D)
        B = VB // n_views
        tags = None
        if self.pos_embed is not None and clip_indices is not None:
            rows = apply_masks(self.pos_embed.expand(B, -1, -1), list(clip_indices), concat=False)    # [B, T_s, D] each
            tags = torch.cat(rows, dim=1).unsqueeze(2).expand(-1, -1, N, -1).flatten(1, 2)
        views = [tokens[v * B:(v + 1) * B] for v in range(n_views)]
        return views if tags is None else [o + tags.to(o.dtype) for o in views]


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
