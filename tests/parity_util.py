"""Shared harness for the parity tests and __graft_entry__.smoke(): one C1-shaped V-JEPA step through
(a) the CUDA product path and (b) the CPU oracle, on identical seeded weights / clips / masks."""
import copy
import os

import torch

from common import C1, synth_clips, synth_state

HERE = os.path.dirname(os.path.abspath(__file__))
EMA_M = 0.998


def c1_masks(batch):
    g = torch.load(os.path.join(HERE, "golden", "golden_masks.pt"))["c1_call0"]
    return [m[:batch].clone() for m in g["enc"]], [m[:batch].clone() for m in g["pred"]]


# 2-block slices of the BASELINE networks (SURVEY section 8c(ii)): full width / heads / sequence lengths of ViT-L/16 and
# ViT-H/16 at 16x224^2, one clip, the C2 / C4 seeded masks (first collator call at the config's batch size, first row)
VITL_2B = dict(model_name='vit_large', crop_size=224, patch_size=16, num_frames=16, tubelet_size=2, batch=1,
               pred_depth=2, pred_embed_dim=384, depth=2, heads=16, embed_dim=1024, mask_batch=32)
VITH_2B = dict(model_name='vit_huge', crop_size=224, patch_size=16, num_frames=16, tubelet_size=2, batch=1,
               pred_depth=2, pred_embed_dim=384, depth=2, heads=16, embed_dim=1280, mask_batch=24)


def cfg_masks(cfg, batch):
    """Masks of a step config: C1 -> the committed reference-generated fixture; others -> the (bit-exact, sha-pinned)
    product collator seeded like BASELINE.md section 2, first `batch` rows."""
    if cfg is C1:
        return c1_masks(batch)
    from common import VITL16_MASKS
    from jepa_b200.masks import MultiBlock3DMaskCollator as MaskCollator
    torch.manual_seed(0)
    coll = MaskCollator(cfgs_mask=VITL16_MASKS, crop_size=cfg["crop_size"], num_frames=cfg["num_frames"],
                        patch_size=cfg["patch_size"], tubelet_size=cfg["tubelet_size"])
    _, me, mp = coll([torch.zeros(1) for _ in range(cfg["mask_batch"])])
    return [m[:batch].clone() for m in me], [m[:batch].clone() for m in mp]


def _shapes(depth, pred_depth, cfg=C1):
    """state-dict shapes of the networks (optionally shallower), derived from the product modules on CPU."""
    from jepa_b200.models import VisionTransformer, vit_predictor
    from functools import partial
    import torch.nn as nn
    enc = VisionTransformer(img_size=cfg["crop_size"], patch_size=cfg["patch_size"], num_frames=cfg["num_frames"],
                            tubelet_size=cfg["tubelet_size"], embed_dim=cfg["embed_dim"], depth=depth, num_heads=cfg["heads"],
                            mlp_ratio=4, qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), uniform_power=True)
    pred = vit_predictor(img_size=cfg["crop_size"], use_mask_tokens=True, patch_size=cfg["patch_size"],
                         num_frames=cfg["num_frames"], tubelet_size=cfg["tubelet_size"], embed_dim=cfg["embed_dim"],
                         predictor_embed_dim=cfg["pred_embed_dim"], depth=pred_depth, num_heads=cfg["heads"],
                         uniform_power=True, num_mask_tokens=2, zero_init_mask_tokens=True)
    return enc, pred


def build_states(depth_limit=None, cfg=C1):
    depth = depth_limit or cfg["depth"]
    pdepth = depth_limit or cfg["pred_depth"]
    enc, pred = _shapes(depth, pdepth, cfg)
    enc_shapes = {k: tuple(v.shape) for k, v in enc.state_dict().items()}
    pred_shapes = {k: tuple(v.shape) for k, v in pred.state_dict().items()}
    s_enc = synth_state(enc_shapes, seed=11, keep=("pos_embed",))
    s_pred = synth_state(pred_shapes, seed=12, keep=("pos_embed",))
    s_tgt = synth_state(enc_shapes, seed=13, keep=("pos_embed",))
    return enc, pred, s_enc, s_pred, s_tgt, depth, pdepth


def run_c1_step_cuda(device, batch=None, depth_limit=None, cfg=C1):
    from jepa_b200 import step as vj
    from jepa_b200.models import MultiMaskWrapper, PredictorMultiMaskWrapper
    C1 = cfg
    batch = batch or cfg["batch"]
    enc, pred, s_enc, s_pred, s_tgt, depth, pdepth = build_states(depth_limit, cfg)
    enc.load_state_dict(s_enc, strict=False)
    pred.load_state_dict(s_pred, strict=False)
    tgt = copy.deepcopy(enc)
    tgt.load_state_dict(s_tgt, strict=False)
    enc, pred, tgt = MultiMaskWrapper(enc).to(device), PredictorMultiMaskWrapper(pred).to(device), MultiMaskWrapper(tgt).to(device)
    for p in tgt.parameters():
        p.requires_grad = False
    clips = synth_clips(batch, C1["num_frames"], C1["crop_size"], C1["crop_size"], seed=0).to(device)
    me, mp = cfg_masks(cfg, batch)
    me, mp = [m.to(device) for m in me], [m.to(device) for m in mp]

    h = vj.forward_target(tgt, clips, mp)
    z_enc = enc(clips, me)
    z = pred(z_enc, h, me, mp)
    loss = vj.jepa_loss(z, h)
    loss_reg = vj.reg_loss(z)
    loss.backward()
    out = dict(loss_jepa=float(loss), loss_reg=float(loss_reg))
    out["h"] = [t.detach().float().cpu() for t in h]
    out["z"] = [t.detach().float().cpu() for t in z]
    out["z_enc"] = [t.detach().float().cpu() for t in z_enc]
    out["enc_grad"] = {n: p.grad.detach().float().cpu() for n, p in enc.backbone.named_parameters() if p.grad is not None}
    out["pred_grad"] = {n: p.grad.detach().float().cpu() for n, p in pred.backbone.named_parameters() if p.grad is not None}
    vj.ema_update(enc, tgt, EMA_M)
    torch.cuda.synchronize()
    out["ema"] = {n: p.detach().float().cpu() for n, p in tgt.backbone.named_parameters()}
    return out


def run_c1_step_oracle(batch=None, depth_limit=None, dtype=torch.float32, cfg=C1):
    from oracle import vjepa_oracle as O
    C1 = cfg
    batch = batch or cfg["batch"]
    _, _, s_enc, s_pred, s_tgt, depth, pdepth = build_states(depth_limit, cfg)
    enc_mod, pred_mod = _shapes(depth, pdepth, cfg)

    def with_pos(state, mod, key):
        full = {k: v.clone().to(dtype) for k, v in state.items()}
        full[key] = mod.state_dict()[key].clone().to(dtype)
        return full

    S_enc = with_pos(s_enc, enc_mod, "pos_embed")
    S_tgt = with_pos(s_tgt, enc_mod, "pos_embed")
    S_pred = with_pos(s_pred, pred_mod, "predictor_pos_embed")
    for S, frozen in ((S_enc, "pos_embed"), (S_pred, "predictor_pos_embed")):
        for k, v in S.items():
            if k != frozen:
                v.requires_grad_(True)
    clips = synth_clips(batch, C1["num_frames"], C1["crop_size"], C1["crop_size"], seed=0).to(dtype)
    me, mp = cfg_masks(cfg, batch)
    heads = C1["heads"]
    h = O.forward_target(S_tgt, clips, mp, depth, heads)
    z_enc = [O.encoder(S_enc, clips, [m], depth, heads) for m in me]
    z = [O.predictor(S_pred, zi, mc, mt, i, pdepth, heads) for i, (zi, mc, mt) in enumerate(zip(z_enc, me, mp))]
    loss = O.loss_fn(z, h)
    loss_reg = O.reg_fn(z)
    loss.backward()
    out = dict(loss_jepa=float(loss), loss_reg=float(loss_reg))
    out["h"] = [t.detach().float() for t in h]
    out["z"] = [t.detach().float() for t in z]
    out["z_enc"] = [t.detach().float() for t in z_enc]
    out["enc_grad"] = {n: p.grad.detach().float() for n, p in S_enc.items() if p.grad is not None}
    out["pred_grad"] = {n: p.grad.detach().float() for n, p in S_pred.items() if p.grad is not None}
    S_q = {k: v.detach().float() for k, v in S_enc.items()}
    S_k = {k: v.detach().float().clone() for k, v in S_tgt.items()}
    O.ema(S_k, S_q, EMA_M)
    out["ema"] = S_k
    return out


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


# tolerances (north_star: "within a stated fp tolerance"): bf16-operand / fp32-accumulate kernels against
# the fp32 oracle, 12+12 layer networks.
TOL_ACT = 2e-2      # rel-L2 on encoder / predictor / target outputs
TOL_GRAD = 3e-2     # rel-L2 per parameter gradient
TOL_LOSS = 3e-3     # absolute, loss ~ 0.9


def compare_step(got, ref, verbose=False, tol_act=TOL_ACT, tol_grad=TOL_GRAD, tol_loss=TOL_LOSS):
    worst = {}
    for key in ("h", "z_enc", "z"):
        for i, (a, b) in enumerate(zip(got[key], ref[key])):
            assert a.shape == b.shape, (key, a.shape, b.shape)
            e = rel_l2(a, b)
            worst[f"{key}[{i}]"] = e
            assert e <= tol_act, f"{key}[{i}] rel-L2 {e:.4f} > {tol_act}"
    assert abs(got["loss_jepa"] - ref["loss_jepa"]) <= tol_loss, (got["loss_jepa"], ref["loss_jepa"])
    assert abs(got["loss_reg"] - ref["loss_reg"]) <= 2e-2, (got["loss_reg"], ref["loss_reg"])
    for key in ("enc_grad", "pred_grad"):
        assert set(got[key]) == set(ref[key]), set(got[key]) ^ set(ref[key])
        for n in ref[key]:
            a, b = got[key][n], ref[key][n]
            assert a.shape == b.shape, (n, a.shape, b.shape)
            e = rel_l2(a, b)
            worst[f"{key}.{n}"] = e
            assert e <= tol_grad, f"{key} {n} rel-L2 {e:.4f} > {tol_grad} (|ref|={float(b.norm()):.3e})"
    for n, b in ref["ema"].items():
        a = got["ema"][n]
        assert torch.equal(a, b), f"EMA of {n} not bit-exact (max diff {float((a - b).abs().max()):.3e})"
    if verbose:
        top = sorted(worst.items(), key=lambda kv: -kv[1])[:8]
        print("worst rel-L2:", ", ".join(f"{k}={v:.4f}" for k, v in top))
    return worst
