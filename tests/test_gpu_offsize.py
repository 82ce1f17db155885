"""Encoder inputs at a size other than the configured one, on the GPU (-m gpu): vj_pos_interp against the reference's
interpolate_pos_encoding (golden_offsize.pt digests: bit for bit), the encoder at off sizes against the reference's
outputs and the fp32 / fp64 oracle (forward with and without masks, out_layers, backward), the image encoder,
FrameAggregation, and an image encoder evaluated on video through evals.scaffold.main."""
import hashlib
import math
import os
import sys
from functools import partial

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from common import synth_clips, synth_state
from parity_util import TOL_ACT, TOL_GRAD, rel_l2

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import posinterp_numpy as PN  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(HERE, "golden", "golden_offsize.pt")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


def _sha(t):
    return hashlib.sha256(t.detach().float().contiguous().cpu().numpy().tobytes()).hexdigest()[:16]


def _max_ulps(a, b):
    ia = a.float().cpu().numpy().view(np.int32).astype(np.int64)
    ib = b.float().cpu().numpy().view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int(np.abs(ia - ib).max())


def _vit(D, depth, heads, num_frames, img_size=224, **kw):
    from jepa_b200.models import VisionTransformer
    if num_frames > 1:
        kw.setdefault("tubelet_size", 2)
    return VisionTransformer(img_size=img_size, patch_size=16, num_frames=num_frames, embed_dim=D, depth=depth,
                             num_heads=heads, mlp_ratio=4, qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6),
                             uniform_power=True, **kw)


def _seeded(mod, seed):
    mod.load_state_dict(synth_state({k: tuple(v.shape) for k, v in mod.state_dict().items()}, seed=seed,
                                    keep=("pos_embed",)), strict=False)
    return mod


# ------------------------------------------------------------------------------------------------------------------
# vj_pos_interp
# ------------------------------------------------------------------------------------------------------------------
def test_pos_interp_bitwise_reference_tables(dev, gold):
    """Every table of the fixture, bit for bit.  On a mismatch the message carries the largest difference in ulps against
    torch's CPU F.interpolate on this machine."""
    from jepa_b200 import kernels as K
    from jepa_b200.engine import pos_interp_scales
    for case in gold["tables"]["video"] + gold["tables"]["image"]:
        D = case["D"]
        video = "thw" in case
        m = _vit(D, 0, D // 64, 16 if video else 1)
        grid = m.token_grid((1, 3) + (case["thw"] if video else (case["size"], case["size"])))
        src = m.pos_embed.detach().view(*m.grid, D)
        assert _sha(src) == case["src_sha"]
        if grid == m.grid:          # (16, 230, 230): the reference interpolates at scale 1, a copy
            assert _sha(src) == case["sha"]
            continue
        scales = pos_interp_scales(m.grid, grid, video)
        out = torch.empty(*grid, D, device=dev)
        K.pos_interp(src.to(dev).contiguous(), out, scales, 3 if video else 2)
        torch.cuda.synchronize()
        if _sha(out) != case["sha"]:
            if video:
                want = F.interpolate(src.unsqueeze(0).permute(0, 4, 1, 2, 3), scale_factor=scales,
                                     mode="trilinear").permute(0, 2, 3, 4, 1)[0]
            else:
                want = F.interpolate(src.view(1, *m.grid[1:], D).permute(0, 3, 1, 2), scale_factor=scales[1],
                                     mode="bicubic").permute(0, 2, 3, 1)
            pytest.fail(f"{case}: not bit-exact, max {_max_ulps(out.view(-1), want.reshape(-1))} ulps from F.interpolate")


@pytest.mark.parametrize("mode,shape,scales", [
    (3, (3, 5, 6), (1.7, 0.6, 1.33)), (3, (5, 9, 3), (0.45, 2.31, 3.0)), (3, (8, 24, 24), (2.0, 1.0, 1.0)),
    (2, (1, 9, 9), (1.0, 0.34, 0.34)), (2, (1, 4, 4), (1.0, 3.5625, 3.5625)), (2, (1, 20, 20), (1.0, 0.55, 0.55))])
def test_pos_interp_matches_restatement_on_odd_shapes(dev, mode, shape, scales):
    """Scales below 1, odd sizes, copies along an axis: the kernel equals the numpy restatement (which equals torch's CPU
    kernels, tests/test_offsize_cpu.py) bit for bit."""
    from jepa_b200 import kernels as K
    D = 20
    table = torch.randn(*shape, D, generator=torch.Generator().manual_seed(5))
    if mode == 3:
        want = PN.trilinear(table.numpy(), scales)
    else:
        want = PN.bicubic(table[0].numpy(), scales[1])[None]
    out = torch.empty(*want.shape, device=dev)
    K.pos_interp(table.to(dev), out, scales, mode)
    got = out.cpu().numpy()
    assert np.array_equal(got, want), _max_ulps(out.cpu(), torch.from_numpy(want))


def test_pos_interp_argument_checks(dev):
    from jepa_b200 import _lib
    from jepa_b200 import kernels as K
    t = torch.zeros(8, 14, 14, 64, device=dev)
    with pytest.raises(_lib.VJError, match="floor"):
        K.pos_interp(t, torch.empty(16, 20, 19, 64, device=dev), (2.0, 20 / 14, 20 / 14), 3)
    with pytest.raises(_lib.VJError, match="mode"):
        K.pos_interp(t, torch.empty(16, 20, 20, 64, device=dev), (2.0, 20 / 14, 20 / 14), 1)
    with pytest.raises(_lib.VJError, match="multiple of 4"):
        K.pos_interp(torch.zeros(8, 14, 14, 6, device=dev), torch.empty(16, 20, 20, 6, device=dev), (2.0, 20 / 14, 20 / 14), 3)
    with pytest.raises(_lib.VJError, match="2-D"):
        K.pos_interp(t, torch.empty(16, 20, 20, 64, device=dev), (2.0, 20 / 14, 20 / 14), 2)


# ------------------------------------------------------------------------------------------------------------------
# encoder at off sizes
# ------------------------------------------------------------------------------------------------------------------
def _rows(out, idx):
    return out.reshape(-1, out.shape[-1]).float().cpu()[idx]


def test_encoder_offsize_matches_reference(dev, gold):
    """ViT-Tiny (12 blocks) at 32x224^2, 16x320^2, 16x224x320, 8x288x160 and 16x230^2: forward, forward with masks,
    MultiMaskWrapper / forward_multi and out_layers against the reference's outputs."""
    from jepa_b200.models import MultiMaskWrapper
    enc = _seeded(_vit(192, 12, 3, 16), 21).to(dev).eval()
    enc_ol = _seeded(_vit(192, 12, 3, 16, out_layers=[3, 7, 11]), 21).to(dev).eval()
    mm = MultiMaskWrapper(enc)
    for case in gold["encoder"]:
        T, H, W = case["thw"]
        x = synth_clips(case["B"], T, H, W, seed=case["clip_seed"]).to(dev)
        with torch.no_grad():
            if case["kind"] == "plain":
                out = enc(x)
            elif case["kind"] == "masked":
                masks = [m.to(dev) for m in case["masks"]]
                out = enc(x, masks)
                multi = mm(x, masks)
                assert torch.equal(torch.cat(multi, 0), out)
            else:
                out = enc_ol(x)[int(case["kind"][5:])]
        assert tuple(out.shape) == case["shape"], (case["thw"], case["kind"])
        e = rel_l2(_rows(out, case["rows"]), case["out"])
        assert e <= TOL_ACT, (case["thw"], case["kind"], e)


def test_image_encoder_matches_reference(dev, gold):
    """The image encoder (num_frames=1: Conv2d patch embedding, 2-D sin-cos) at its own size and, bicubic, at 320."""
    from jepa_b200 import _lib
    lib = _lib.load()
    enc = _seeded(_vit(192, 12, 3, 1), 21).to(dev).eval()
    for case in gold["image_encoder"]:
        S = case["size"]
        x = synth_clips(case["B"], 1, S, S, seed=case["clip_seed"])[:, :, 0].to(dev)
        with torch.no_grad():
            out = enc(x)
        assert tuple(out.shape) == case["shape"]
        e = rel_l2(_rows(out, case["rows"]), case["out"])
        assert e <= TOL_ACT, (S, e)
    with pytest.raises(ValueError, match="not square"):
        enc(torch.zeros(1, 3, 224, 320, device=dev))
    assert lib.vj_launch_count() > 0


def _launches(fn):
    from jepa_b200 import _lib
    lib = _lib.load()
    n0 = lib.vj_launch_count()
    fn()
    torch.cuda.synchronize()
    return lib.vj_launch_count() - n0


def test_configured_size_launches_no_interpolation(dev):
    """At the configured size the table is pos_embed itself; an off-size call adds exactly one launch (the resample),
    recomputed on every call (no cache: pos_embed may change between calls, as the EMA does)."""
    enc = _seeded(_vit(192, 2, 3, 16), 21).to(dev).eval()
    x0 = synth_clips(1, 16, 224, 224, seed=1).to(dev)
    x1 = synth_clips(1, 16, 320, 320, seed=1).to(dev)
    with torch.no_grad():
        enc(x0)
        enc(x1)
        n0 = _launches(lambda: enc(x0))
        n1 = _launches(lambda: enc(x1))
        a = enc(x1)
        enc.pos_embed.data.mul_(2.0)
        enc._store.invalidate_shadow()
        b = enc(x1)
    assert n1 == n0 + 1, (n0, n1)
    assert not torch.equal(a, b)


def _oracle_state(enc, grid, dtype):
    """The module's parameters as oracle tensors, pos_embed replaced by torch's CPU interpolation of it to `grid`."""
    from jepa_b200.engine import pos_interp_scales
    S = {k: v.detach().cpu().clone().to(dtype) for k, v in enc.state_dict().items()}
    D = enc.embed_dim
    src = enc.pos_embed.detach().cpu().view(*enc.grid, D)
    pos = F.interpolate(src.unsqueeze(0).permute(0, 4, 1, 2, 3), scale_factor=pos_interp_scales(enc.grid, grid, True),
                        mode="trilinear").permute(0, 2, 3, 4, 1).reshape(1, -1, D)
    S["pos_embed"] = pos.to(dtype)
    return S


def _masks(n, B, K, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.stack([torch.randperm(n, generator=g)[:K].sort().values for _ in range(B)]) for _ in range(2)]


def test_vitl_2block_offsize_masked_vs_oracle(dev):
    """2-block ViT-L/16 (full width, 16 heads) at 16x320^2 with two context masks, against the fp32 oracle."""
    from oracle import vjepa_oracle as O
    enc = _seeded(_vit(1024, 2, 16, 16), 11).to(dev).eval()
    grid = (8, 20, 20)
    x = synth_clips(1, 16, 320, 320, seed=0)
    masks = _masks(8 * 20 * 20, 1, 1200, seed=3)
    with torch.no_grad():
        got = enc(x.to(dev), [m.to(dev) for m in masks]).float().cpu()
    S = _oracle_state(enc, grid, torch.float32)
    with torch.no_grad():
        want = torch.cat([O.encoder(S, x, [m], 2, 16) for m in masks], 0)
    assert got.shape == want.shape
    e = rel_l2(got, want)
    assert e <= TOL_ACT, e


def test_offsize_backward_vs_fp64_oracle(dev):
    """Gradients through _EncoderFn at 16x224x320 with a mask (and at a non-multiple size, 16x230x330): every parameter
    against the fp64 oracle (pos_embed has no gradient, so only the token count changes)."""
    from oracle import vjepa_oracle as O
    for (T, H, W), seed in (((16, 224, 320), 4), ((16, 230, 330), 5)):
        enc = _seeded(_vit(192, 2, 3, 16), 11).to(dev)
        grid = enc.token_grid((1, 3, T, H, W))
        n = grid[0] * grid[1] * grid[2]
        x = synth_clips(2, T, H, W, seed=seed)
        m = _masks(n, 2, n // 2, seed=seed)[0]
        R = torch.randn(2, n // 2, 192, generator=torch.Generator().manual_seed(seed))
        out = enc(x.to(dev), m.to(dev))
        (out.float() * R.to(dev)).sum().backward()
        got = {k: p.grad.detach().float().cpu() for k, p in enc.named_parameters() if p.grad is not None}
        S = _oracle_state(enc, grid, torch.float64)
        for k, v in S.items():
            if k != "pos_embed":
                v.requires_grad_(True)
        xc = x[:, :, :grid[0] * 2, :grid[1] * 16, :grid[2] * 16].double()
        (O.encoder(S, xc, [m], 2, 3) * R.double()).sum().backward()
        assert set(got) == {k for k, v in S.items() if v.grad is not None}
        for k, g in got.items():
            e = rel_l2(g, S[k].grad.float())
            assert e <= TOL_GRAD, ((T, H, W), k, e)


# ------------------------------------------------------------------------------------------------------------------
# FrameAggregation
# ------------------------------------------------------------------------------------------------------------------
def test_frame_aggregation_matches_reference(dev, gold):
    from jepa_b200.pooler import FrameAggregation
    fa = gold["frameagg"]
    img = _seeded(_vit(192, 12, 3, 1, img_size=64), 22).to(dev).eval()
    g = torch.Generator().manual_seed(fa["seed"])
    B, Fr, V, NSEG = fa["B"], fa["frames"], fa["views"], fa["segments"]
    xs = [[torch.randn(B, 3, Fr, 64, 64, generator=g) for _ in range(V)] for _ in range(NSEG)]
    idx = [torch.stack([torch.randint(0, 64, (Fr,), generator=g) for _ in range(B)]) for _ in range(NSEG)]
    xs = [[v.to(dev) for v in seg] for seg in xs]
    idx = [i.to(dev) for i in idx]
    n_calls = []
    img.register_forward_pre_hook(lambda mod, inp: n_calls.append(tuple(inp[0].shape)))
    for pos, key in ((False, "out"), (True, "out_pos")):
        agg = FrameAggregation(img, max_frames=fa["max_frames"], use_pos_embed=pos).to(dev).eval()
        with torch.no_grad():
            out = agg(xs, clip_indices=idx)
        assert len(out) == V
        for o, w in zip(out, fa[key]):
            assert o.shape == w.shape
            e = rel_l2(o.float().cpu(), w.float())
            assert e <= TOL_ACT, (key, e)
    assert n_calls == [(V * B * NSEG * Fr, 3, 64, 64)] * 2          # one encoder call per forward


# ------------------------------------------------------------------------------------------------------------------
# an image encoder evaluated on video, end to end
# ------------------------------------------------------------------------------------------------------------------
def _image_checkpoint(folder):
    """A pre-training checkpoint of an image ViT-Tiny (frames_per_clip 1) in the reference's format."""
    enc = _seeded(_vit(192, 12, 3, 1), 31)
    sd = {f"module.backbone.{k}": v for k, v in enc.state_dict().items()}
    torch.save({"encoder": sd, "predictor": {}, "target_encoder": sd, "opt": None, "scaler": None, "epoch": 1,
                "loss": 0.0, "batch_size": 8, "world_size": 1, "lr": 0.0}, os.path.join(folder, "jepa-latest.pth.tar"))


@pytest.mark.parametrize("dataset_type", ["synthetic", "synthetic_uint8"])
def test_image_encoder_video_eval_end_to_end(dev, tmp_path, dataset_type):
    from evals.scaffold import main as eval_main
    from test_gpu_eval import _check_run, _eval_cfg
    _image_checkpoint(tmp_path)
    cfg = _eval_cfg(tmp_path, "img", True, dataset_type=dataset_type)
    cfg["pretrain"].update(frames_per_clip=1)
    cfg["data"].update(frames_per_clip=4)
    if dataset_type == "synthetic_uint8":
        cfg["data"]["gpu_augment"] = True       # the training transform (RandAugment, random erasing) on the GPU
    eval_main("video_classification_frozen", cfg)
    body, ck = _check_run(tmp_path, "video_classification_frozen", "img", 2)
    assert [r[0] for r in body] == ["1", "2"]
    assert all(0.0 <= float(r[1]) <= 100.0 and 0.0 <= float(r[2]) <= 100.0 for r in body), body
    if dataset_type == "synthetic":
        # on uint8 frames the probe trains through RandAugment and random erasing, which two short epochs do not fit
        assert float(body[-1][1]) == 100.0, body


def test_image_encoder_eval_needs_attend_across_segments(dev, tmp_path):
    from evals.scaffold import main as eval_main
    from test_gpu_eval import _eval_cfg
    _image_checkpoint(tmp_path)
    cfg = _eval_cfg(tmp_path, "img", False)
    cfg["pretrain"].update(frames_per_clip=1)
    with pytest.raises(ValueError, match="attend_across_segments"):
        eval_main("video_classification_frozen", cfg)
