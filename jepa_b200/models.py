"""Host-side mirror of the reference model API (src/models/*) on top of the sm_90a engine.

Class names, constructor kwargs, parameter names / shapes and state_dict keys follow
src/models/vision_transformer.py, src/models/predictor.py, src/models/utils/{modules,patch_embed,
multimask}.py so reference checkpoints load and app/vjepa/utils.py-style factories work
unchanged.  The nn.Modules here only OWN parameters; all math runs in jepa_b200.engine through the
C-ABI kernels.  There is deliberately no eager / CPU implementation: calling forward without a CUDA
device raises.
"""
import math
from functools import partial

import torch
import torch.nn as nn

from . import engine
from .params import FlatParamStore
from .pos_embs import get_2d_sincos_pos_embed, get_3d_sincos_pos_embed
from .tensors import trunc_normal_


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(
            f"jepa_b200: {what} needs CUDA tensors - the V-JEPA hot path is implemented only as sm_90a "
            "kernels (no CPU or eager-PyTorch fallback).")


# -------------------------------------------------------------------------------------------------
# parameter containers (modules.py:13-120, patch_embed.py:13-57)
# -------------------------------------------------------------------------------------------------
class MLP(nn.Module):
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        if drop != 0.:
            raise NotImplementedError("dropout is not part of the accelerated path (all V-JEPA configs use 0)")
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features, out_features)


class Attention(nn.Module):
    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0., proj_drop=0., use_sdpa=True):
        super().__init__()
        if attn_drop != 0. or proj_drop != 0.:
            raise NotImplementedError("dropout is not part of the accelerated path (all V-JEPA configs use 0)")
        if not qkv_bias:
            raise NotImplementedError("qkv_bias=False is not used by any V-JEPA factory")
        if qk_scale:      # None or False (AttentivePooler's Blocks) mean the default hd^-0.5, as `qk_scale or ...` does
            raise NotImplementedError("qk_scale override is not supported")
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.use_sdpa = use_sdpa


class Block(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio=4., qkv_bias=False, qk_scale=None, drop=0., attn_drop=0.,
                 act_layer=nn.GELU, norm_layer=nn.LayerNorm, grid_size=None, grid_depth=None):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale, attn_drop=attn_drop,
                              proj_drop=drop)
        self.norm2 = norm_layer(dim)
        self.mlp = MLP(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer, drop=drop)


class PatchEmbed(nn.Module):
    def __init__(self, patch_size=16, in_chans=3, embed_dim=768):
        super().__init__()
        self.patch_size = patch_size
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)


class PatchEmbed3D(nn.Module):
    def __init__(self, patch_size=16, tubelet_size=2, in_chans=3, embed_dim=768):
        super().__init__()
        self.patch_size = patch_size
        self.tubelet_size = tubelet_size
        self.proj = nn.Conv3d(in_channels=in_chans, out_channels=embed_dim,
                              kernel_size=(tubelet_size, patch_size, patch_size),
                              stride=(tubelet_size, patch_size, patch_size))


def _check_ln_eps(norm_layer, dim):
    ln = norm_layer(dim)
    if not isinstance(ln, nn.LayerNorm) or abs(ln.eps - engine.LN_EPS) > 1e-12:
        raise NotImplementedError("the accelerated path implements nn.LayerNorm(eps=1e-6) (all V-JEPA factories)")


def _token_views(flat, B, sizes):
    """Split a [sum B*K_i, D] matrix into per-mask [B, K_i, D] views that remember their base."""
    outs, off = [], 0
    for k in sizes:
        v = flat[off:off + B * k].view(B, k, flat.shape[1])
        v._vj_base = (flat, off)
        outs.append(v)
        off += B * k
    return outs


def _common_base(tensors):
    """If `tensors` are the consecutive views produced by _token_views, return their base matrix."""
    base, expect = None, 0
    for t in tensors:
        info = getattr(t, "_vj_base", None)
        if info is None:
            return None
        b, off = info
        if base is None:
            base = b
        if b is not base or off != expect:
            return None
        expect += t.shape[0] * t.shape[1]
    if base is None or expect != base.shape[0]:
        return None
    return base


# -------------------------------------------------------------------------------------------------
# autograd glue
# -------------------------------------------------------------------------------------------------
def _live_grad_buffer(mod, store):
    """The flat buffer the .grads of every trainable parameter of `mod` already alias (a backward since zero_grad(): the
    earlier micro-batches of gradient accumulation), or None."""
    return store.live_grad_buffer(p for p in mod.parameters() if p.requires_grad)


def _param_grads(mod, store, gflat, live):
    """What the backward hands autograd for mod's parameters: views of the new buffer `gflat` (AccumulateGrad makes them
    the .grads), or nothing when the backward added into the live buffer the .grads already are."""
    if live is not None:
        return [None] * len(list(mod.parameters()))
    return [store.grad_view(gflat, n) if p.requires_grad else None for n, p in mod.named_parameters()]


class _EncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mod, clips, masks, final_norm, grid, grad_enabled, *params):
        # needs_input_grad follows requires_grad even under torch.no_grad(): a forward there keeps nothing for a backward
        save = grad_enabled and any(ctx.needs_input_grad[6:])
        out, sv, _ = engine.encoder_forward(mod, clips, masks, save, final_norm=final_norm, grid=grid)
        if save and not final_norm:
            raise RuntimeError("training through the un-normalised encoder output is not supported")
        ctx.mod, ctx.sv = mod, sv
        return out

    @staticmethod
    def backward(ctx, dout):
        mod, sv = ctx.mod, ctx.sv
        live = _live_grad_buffer(mod, sv.store)
        gflat = engine.encoder_backward(mod, sv, dout, live)
        ctx.sv = None
        return (None, None, None, None, None, None, *_param_grads(mod, sv.store, gflat, live))


class _PredictorFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mod, z_cat, masks_ctxt, masks_tgt, mask_indices, *params):
        save = any(ctx.needs_input_grad)
        out, sv = engine.predictor_forward(mod, z_cat, masks_ctxt, masks_tgt, mask_indices, save)
        ctx.mod, ctx.sv = mod, sv
        return out

    @staticmethod
    def backward(ctx, dout):
        mod, sv = ctx.mod, ctx.sv
        live = _live_grad_buffer(mod, sv.store)
        dz, gflat = engine.predictor_backward(mod, sv, dout, live)
        ctx.sv = None
        return (None, dz if ctx.needs_input_grad[1] else None, None, None, None,
                *_param_grads(mod, sv.store, gflat, live))


# -------------------------------------------------------------------------------------------------
# VisionTransformer (vision_transformer.py:21-246)
# -------------------------------------------------------------------------------------------------
class VisionTransformer(nn.Module):
    """ Vision Transformer encoder; parameters and API of the reference, math on sm_90a kernels. """

    def __init__(self, img_size=224, patch_size=16, num_frames=1, tubelet_size=2, in_chans=3, embed_dim=768, depth=12,
                 num_heads=12, mlp_ratio=4.0, qkv_bias=True, qk_scale=None, drop_rate=0.0, attn_drop_rate=0.0,
                 norm_layer=nn.LayerNorm, init_std=0.02, out_layers=None, uniform_power=False, **kwargs):
        super().__init__()
        self.num_features = self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.out_layers = out_layers     # evals: return [norm(x_i) for i in out_layers] (frozen encoder, no grad)
        self.input_size = img_size
        self.patch_size = patch_size
        self.num_frames = num_frames
        self.tubelet_size = tubelet_size if num_frames > 1 else 1
        self.is_video = num_frames > 1
        grid_size = self.input_size // self.patch_size
        grid_depth = self.num_frames // tubelet_size
        _check_ln_eps(norm_layer, embed_dim)

        if self.is_video:
            self.patch_embed = PatchEmbed3D(patch_size=patch_size, tubelet_size=tubelet_size, in_chans=in_chans,
                                            embed_dim=embed_dim)
            self.num_patches = (num_frames // tubelet_size) * (img_size // patch_size) * (img_size // patch_size)
        else:
            self.patch_embed = PatchEmbed(patch_size=patch_size, in_chans=in_chans, embed_dim=embed_dim)
            self.num_patches = (img_size // patch_size) * (img_size // patch_size)

        self.uniform_power = uniform_power
        self.pos_embed = nn.Parameter(torch.zeros(1, self.num_patches, embed_dim), requires_grad=False)
        self.blocks = nn.ModuleList([
            Block(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, qk_scale=qk_scale,
                  drop=drop_rate, act_layer=nn.GELU, grid_size=grid_size, grid_depth=grid_depth,
                  attn_drop=attn_drop_rate, norm_layer=norm_layer) for _ in range(depth)])
        self.norm = norm_layer(embed_dim)

        self._init_pos_embed(self.pos_embed.data)
        self.init_std = init_std
        self.apply(self._init_weights)
        self._rescale_blocks()

        self._store = FlatParamStore()
        self._scratch = {}
        self._spec = engine.StackSpec(embed_dim, num_heads, int(embed_dim * mlp_ratio), depth, "blocks")

    def _load_from_state_dict(self, *args, **kwargs):
        nn.Module._load_from_state_dict(self, *args, **kwargs)   # (explicit base: the predictor class reuses this function)
        self._store.invalidate_shadow()      # parameters changed behind the optimizer's back: re-cast the bf16 operands

    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k == "_scratch":
                new.__dict__[k] = {}
            else:
                new.__dict__[k] = copy.deepcopy(v, memo)
        return new

    def _init_pos_embed(self, pos_embed):
        embed_dim = pos_embed.size(-1)
        grid_size = self.input_size // self.patch_size
        if self.is_video:
            grid_depth = self.num_frames // self.tubelet_size
            sincos = get_3d_sincos_pos_embed(embed_dim, grid_size, grid_depth, cls_token=False,
                                             uniform_power=self.uniform_power)
        else:
            sincos = get_2d_sincos_pos_embed(embed_dim, grid_size, cls_token=False)
        pos_embed.copy_(torch.from_numpy(sincos).float().unsqueeze(0))

    def _init_weights(self, m):
        if isinstance(m, (nn.Linear, nn.Conv2d, nn.Conv3d)):
            trunc_normal_(m.weight, std=self.init_std)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def _rescale_blocks(self):
        for layer_id, layer in enumerate(self.blocks):
            layer.attn.proj.weight.data.div_(math.sqrt(2.0 * (layer_id + 1)))
            layer.mlp.fc2.weight.data.div_(math.sqrt(2.0 * (layer_id + 1)))

    def get_num_layers(self):
        return len(self.blocks)

    def no_weight_decay(self):
        return {}

    @property
    def grid(self):
        """Token grid (T', H', W') the positional embedding was built for (T' = 1 for an image encoder)."""
        g = self.input_size // self.patch_size
        return (self.num_frames // self.tubelet_size if self.is_video else 1, g, g)

    def token_grid(self, shape):
        """Token grid of an input of `shape` ([B,C,T,H,W] video, [B,C,H,W] image): (T // tubelet, H // patch,
        W // patch), flooring like the reference's Conv3d / Conv2d patch embedding.  Raises ValueError for a size the
        reference's interpolate_pos_encoding (vision_transformer.py:197-246) cannot serve either."""
        ps = self.patch_size
        if self.is_video:
            _, _, T, H, W = shape
            grid = (T // self.tubelet_size, H // ps, W // ps)
        else:
            _, _, H, W = shape
            grid = (1, H // ps, W // ps)
        if min(grid) < 1:
            raise ValueError(f"input {tuple(shape)} is smaller than one {self.tubelet_size}x{ps}x{ps} patch")
        if grid != self.grid:
            n0 = self.grid
            if self.is_video:
                scales = engine.pos_interp_scales(n0, grid, True)
                out = tuple(int(n * s) for n, s in zip(n0, scales))
            else:
                if grid[1] != grid[2]:
                    raise ValueError(
                        f"image of {H}x{W} pixels: a {grid[1]}x{grid[2]} patch grid is not square; the reference's "
                        "bicubic interpolate_pos_encoding resamples a square table and then fails at x += pos_embed")
                s = engine.pos_interp_scales(n0, grid, False)[1]
                out = (1, int(n0[1] * s), int(n0[2] * s))
            if out != grid:
                raise ValueError(f"input {tuple(shape)}: interpolate_pos_encoding's scale factors give a {out} table "
                                 f"for a {grid} token grid (floating-point rounding); the reference fails on it too")
        return grid

    def _check_input(self, x):
        """Returns (x as a [B,C,T,H,W] clip cropped to whole patches, token grid (T', H', W'))."""
        _require_cuda(x, "VisionTransformer.forward")
        if self.is_video:
            if x.dim() != 5:
                raise ValueError(f"expected a video batch [B,C,T,H,W], got {tuple(x.shape)}")
        elif x.dim() != 4:
            raise ValueError(f"expected an image batch [B,C,H,W], got {tuple(x.shape)}")
        grid = self.token_grid(tuple(x.shape))
        if not self.is_video:
            x = x.unsqueeze(2)
        T, H, W = grid[0] * self.tubelet_size, grid[1] * self.patch_size, grid[2] * self.patch_size
        if x.shape[2:] != (T, H, W):       # the strided patch embedding ignores the remainder
            x = x[:, :, :T, :H, :W]
        return x, grid

    @torch.no_grad()
    def _forward_out_layers(self, x, masks):
        """vision_transformer.py:183-190 with out_layers set: list of norm(x) after the chosen blocks, each [B, N, D]
        (or [len(masks)*B, K, D]).  Inference only - the evals use it on the frozen encoder."""
        xv, grid = self._check_input(x)
        if masks is not None and len({int(m.shape[1]) for m in masks}) != 1:
            raise ValueError("out_layers with masks of different sizes cannot be concatenated along batch")
        outs, _, _ = engine.encoder_forward(self, xv, masks, save=False, out_layers=self.out_layers, grid=grid)
        B = xv.shape[0] * (1 if masks is None else len(masks))
        return [o.view(B, -1, self.embed_dim) for o in outs]

    def forward_multi(self, x, masks, final_norm=True):
        """All masks in one fused pass.  Returns list of [B, K_i, D] bf16 views (one per mask)."""
        x, grid = self._check_input(x)
        params = [p for _, p in self.named_parameters()]
        out = _EncoderFn.apply(self, x, list(masks), final_norm, grid, torch.is_grad_enabled(), *params)
        return _token_views(out, x.shape[0], [int(m.shape[1]) for m in masks])

    def forward(self, x, masks=None):
        """
        :param x: input image/video
        :param masks: indices of patch tokens to keep (tensor or list of tensors [B, K])
        Returns [B, N, D] (masks=None) or the batch-concatenated [len(masks)*B, K, D] like the reference.
        """
        if masks is not None and not isinstance(masks, list):
            masks = [masks]
        if self.out_layers is not None:
            return self._forward_out_layers(x, masks)
        if masks is None:
            xv, grid = self._check_input(x)
            params = [p for _, p in self.named_parameters()]
            out = _EncoderFn.apply(self, xv, None, True, grid, torch.is_grad_enabled(), *params)
            return out.view(xv.shape[0], grid[0] * grid[1] * grid[2], self.embed_dim)
        sizes = {int(m.shape[1]) for m in masks}
        if len(sizes) != 1:
            raise ValueError("VisionTransformer.forward(x, masks=[...]) concatenates along batch and needs equal K; "
                             "use forward_multi / MultiMaskWrapper for masks of different sizes")
        outs = self.forward_multi(x, masks)
        if len(outs) == 1:
            return outs[0]
        base = _common_base(outs)
        k = sizes.pop()
        return base.view(len(masks) * x.shape[0], k, self.embed_dim)


def vit_tiny(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=192, depth=12, num_heads=3, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_small(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=384, depth=12, num_heads=6, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_base(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_large(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=1024, depth=24, num_heads=16, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_huge(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=1280, depth=32, num_heads=16, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_giant(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=1408, depth=40, num_heads=16, mlp_ratio=48 / 11,
                             qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_gigantic(patch_size=14, **kwargs):
    # the reference passes a misspelt `mpl_ratio` here (vision_transformer.py:293), i.e. mlp_ratio stays 4.0
    return VisionTransformer(patch_size=patch_size, embed_dim=1664, depth=48, num_heads=16, mpl_ratio=64 / 13,
                             qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


VIT_EMBED_DIMS = {
    'vit_tiny': 192, 'vit_small': 384, 'vit_base': 768, 'vit_large': 1024, 'vit_huge': 1280, 'vit_giant': 1408,
    'vit_gigantic': 1664,
}


# -------------------------------------------------------------------------------------------------
# Predictor (predictor.py:23-246)
# -------------------------------------------------------------------------------------------------
class VisionTransformerPredictor(nn.Module):
    """ Narrow ViT predicting target-token latents from context tokens + positional mask tokens. """

    def __init__(self, img_size=224, patch_size=16, num_frames=1, tubelet_size=2, embed_dim=768,
                 predictor_embed_dim=384, depth=6, num_heads=12, mlp_ratio=4.0, qkv_bias=True, qk_scale=None,
                 drop_rate=0.0, attn_drop_rate=0.0, norm_layer=nn.LayerNorm, init_std=0.02, uniform_power=False,
                 use_mask_tokens=False, num_mask_tokens=2, zero_init_mask_tokens=True, **kwargs):
        super().__init__()
        self.predictor_embed = nn.Linear(embed_dim, predictor_embed_dim, bias=True)
        self.mask_tokens = None
        self.num_mask_tokens = 0
        if use_mask_tokens:
            self.num_mask_tokens = num_mask_tokens
            self.mask_tokens = nn.ParameterList([
                nn.Parameter(torch.zeros(1, 1, predictor_embed_dim)) for _ in range(num_mask_tokens)])
        self.input_size = img_size
        self.patch_size = patch_size
        self.num_frames = num_frames
        self.tubelet_size = tubelet_size
        self.is_video = num_frames > 1
        grid_size = self.input_size // self.patch_size
        grid_depth = self.num_frames // self.tubelet_size
        _check_ln_eps(norm_layer, predictor_embed_dim)
        if self.is_video:
            self.num_patches = (num_frames // tubelet_size) * (img_size // patch_size) * (img_size // patch_size)
        else:
            self.num_patches = (img_size // patch_size) * (img_size // patch_size)
        self.uniform_power = uniform_power
        self.predictor_pos_embed = nn.Parameter(torch.zeros(1, self.num_patches, predictor_embed_dim),
                                                requires_grad=False)
        self.predictor_blocks = nn.ModuleList([
            Block(dim=predictor_embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias,
                  qk_scale=qk_scale, drop=drop_rate, act_layer=nn.GELU, attn_drop=attn_drop_rate,
                  grid_size=grid_size, grid_depth=grid_depth, norm_layer=norm_layer) for _ in range(depth)])
        self.predictor_norm = norm_layer(predictor_embed_dim)
        self.predictor_proj = nn.Linear(predictor_embed_dim, embed_dim, bias=True)

        self._init_pos_embed(self.predictor_pos_embed.data)
        self.init_std = init_std
        if not zero_init_mask_tokens:
            for mt in self.mask_tokens:
                trunc_normal_(mt, std=init_std)
        self.apply(self._init_weights)
        self._rescale_blocks()

        self.embed_dim = embed_dim
        self._store = FlatParamStore()
        self._scratch = {}
        self._spec = engine.StackSpec(predictor_embed_dim, num_heads, int(predictor_embed_dim * mlp_ratio), depth,
                                      "predictor_blocks")

    __deepcopy__ = VisionTransformer.__deepcopy__
    _load_from_state_dict = VisionTransformer._load_from_state_dict

    def _init_pos_embed(self, pos_embed):
        embed_dim = pos_embed.size(-1)
        grid_size = self.input_size // self.patch_size
        if self.is_video:
            grid_depth = self.num_frames // self.tubelet_size
            sincos = get_3d_sincos_pos_embed(embed_dim, grid_size, grid_depth, cls_token=False,
                                             uniform_power=self.uniform_power)
        else:
            sincos = get_2d_sincos_pos_embed(embed_dim, grid_size, cls_token=False)
        pos_embed.copy_(torch.from_numpy(sincos).float().unsqueeze(0))

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=self.init_std)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def _rescale_blocks(self):
        for layer_id, layer in enumerate(self.predictor_blocks):
            layer.attn.proj.weight.data.div_(math.sqrt(2.0 * (layer_id + 1)))
            layer.mlp.fc2.weight.data.div_(math.sqrt(2.0 * (layer_id + 1)))

    def diffusion(self, x, noise_beta=(0.5, 1.0), steps=1000):
        raise NotImplementedError("the diffusion-noise target path (use_mask_tokens=False, predictor.py:154-172) is "
                                  "not used by any pre-training config and is outside the accelerated path")

    def forward_multi(self, ctxt, masks_ctxt, masks_tgt, mask_indices):
        """All (context, target) mask pairs in one fused pass; returns list of [B, Kp_i, D] bf16 views."""
        if self.mask_tokens is None:
            self.diffusion(None)
        base = _common_base(ctxt)
        if base is None:
            base = torch.cat([c.reshape(-1, c.shape[-1]) for c in ctxt], dim=0)
        _require_cuda(base, "VisionTransformerPredictor.forward")
        if base.dtype != torch.bfloat16:
            base = base.to(torch.bfloat16)
        params = [p for _, p in self.named_parameters()]
        idx = [i % self.num_mask_tokens for i in mask_indices]
        out = _PredictorFn.apply(self, base, list(masks_ctxt), list(masks_tgt), idx, *params)
        return _token_views(out, masks_tgt[0].shape[0], [int(m.shape[1]) for m in masks_tgt])

    def forward(self, ctxt, tgt, masks_ctxt, masks_tgt, mask_index=1):
        """
        :param ctxt: context tokens [B, Ke, D]
        :param tgt: target tokens (only its batch length is used when mask tokens are on)
        :param masks_ctxt: indices of context tokens in input
        :params masks_tgt: indices of target tokens in input
        """
        assert (masks_ctxt is not None) and (masks_tgt is not None), 'Cannot run predictor without mask indices'
        if isinstance(masks_ctxt, list):
            if len(masks_ctxt) != 1:
                raise NotImplementedError("use PredictorMultiMaskWrapper / forward_multi for several mask pairs")
            masks_ctxt = masks_ctxt[0]
        if isinstance(masks_tgt, list):
            if len(masks_tgt) != 1:
                raise NotImplementedError("use PredictorMultiMaskWrapper / forward_multi for several mask pairs")
            masks_tgt = masks_tgt[0]
        return self.forward_multi([ctxt], [masks_ctxt], [masks_tgt], [mask_index])[0]


def vit_predictor(**kwargs):
    return VisionTransformerPredictor(mlp_ratio=4, qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6),
                                      **kwargs)


# -------------------------------------------------------------------------------------------------
# multi-mask wrappers (multimask.py:11-48)
# -------------------------------------------------------------------------------------------------
class MultiMaskWrapper(nn.Module):
    def __init__(self, backbone):
        super().__init__()
        self.backbone = backbone

    def forward(self, x, masks=None):
        if masks is None:
            return self.backbone(x)
        if not isinstance(masks, list):
            masks = [masks]
        return self.backbone.forward_multi(x, masks)


class PredictorMultiMaskWrapper(nn.Module):
    def __init__(self, backbone):
        super().__init__()
        self.backbone = backbone

    def forward(self, ctxt, tgt, masks_ctxt, masks_tgt):
        if type(ctxt) is not list:
            ctxt = [ctxt]
        if type(tgt) is not list:
            tgt = [tgt]
        if type(masks_ctxt) is not list:
            masks_ctxt = [masks_ctxt]
        if type(masks_tgt) is not list:
            masks_tgt = [masks_tgt]
        n = min(len(ctxt), len(tgt), len(masks_ctxt), len(masks_tgt))
        return self.backbone.forward_multi(ctxt[:n], masks_ctxt[:n], masks_tgt[:n], list(range(n)))
