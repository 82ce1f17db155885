"""ViT-G/14 on the GPU (-m gpu): vj_im2col_tubelets at 14-pixel patches (padded rows, pad columns zero), a 2-block
ViT-G/14 training step against the CPU oracle, the image ViT-G/14 frozen forward in bf16 and fp16 against fp64, and
the frozen evaluations end to end for a 2-block vit_giant (video) and vit_gigantic (image) encoder."""
import csv
import os
from functools import partial

import pytest
import torch

from parity_util import TOL_ACT, compare_step, run_c1_step_cuda, run_c1_step_oracle
from test_patch14_cpu import im2col_ref

pytestmark = pytest.mark.gpu
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32

# 2+2-block slice of ViT-G/14 at full width / heads / token count (16 x 224^2: 8 x 16 x 16 = 2048 tokens).  MLP 4 x 1664:
# the reference's vit_gigantic passes a misspelt `mpl_ratio`, so mlp_ratio keeps its default.
VITG14_2B = dict(model_name='vit_gigantic', crop_size=224, patch_size=14, num_frames=16, tubelet_size=2, batch=1,
                 pred_depth=2, pred_embed_dim=384, depth=2, heads=16, embed_dim=1664, mlp_ratio=4, mask_batch=32)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


@pytest.mark.parametrize("dt", [BF16, F16])
@pytest.mark.parametrize("kind", ["video", "image"])
def test_im2col_patch14_bit_exact(dev, kind, dt):
    """Rows of P_pad = 1216 (video) / 640 (image) elements; W = 70 px (5 patches: rows not 16-byte aligned in the clip);
    with and without a gather index (repeated tokens included).  The buffer starts as NaN, so the pad must be written."""
    from jepa_b200 import _lib, kernels as Kn
    from jepa_b200.params import padded_patch_dim
    g = torch.Generator().manual_seed(14)
    tub = 2 if kind == "video" else 1
    clips = torch.randn(2, 3, 2 * tub, 56, 70, generator=g).to(dev)       # grid (2 | 1) x 4 x 5
    n = (2 * tub // tub) * 4 * 5
    idx = torch.stack([torch.randperm(n, generator=g)[:7] for _ in range(2)])
    idx[1, 3] = idx[1, 0]
    for ix in (None, idx.to(dev)):
        want = im2col_ref(clips, tub, 14, ix).to(dt)
        assert want.shape[1] == (1216 if kind == "video" else 640)
        got = torch.full_like(want, float("nan"))
        Kn.im2col_tubelets(clips, got, ix, tub, 14)
        assert torch.equal(got, want)
        assert not got[:, 3 * tub * 196:].any()
    with pytest.raises(_lib.VJError):       # rows of the unpadded length
        Kn.im2col_tubelets(clips, torch.empty(2 * n, 3 * tub * 196, dtype=dt, device=dev), None, tub, 14)
    with pytest.raises(_lib.VJError):       # odd patch (56 x 70 px is 8 x 10 patches of 7)
        rows = 2 * (2 * tub // tub) * 8 * 10
        Kn.im2col_tubelets(clips, torch.empty(rows, padded_patch_dim(3 * tub * 49), dtype=dt, device=dev), None, tub, 7)


def test_vitg14_step_vs_oracle(dev):
    """One 2+2-block ViT-G/14 V-JEPA step (context / target encoders, predictor and mask collator at patch 14) against the
    fp32 CPU oracle at test_baseline_width_step_vs_oracle's bounds: every output, the loss, every gradient - the
    patch-embedding weight gradient included, which runs at N = 1216 and keeps only its first 1176 columns - and the
    bit-exact EMA."""
    got = run_c1_step_cuda(dev, cfg=VITG14_2B)
    ref = run_c1_step_oracle(cfg=VITG14_2B)
    assert got["enc_grad"]["patch_embed.proj.weight"].shape == (1664, 3, 2, 14, 14)
    compare_step(got, ref, verbose=True)


def _vitg14(dev, num_frames, depth=2):
    from jepa_b200.models import VisionTransformer
    return VisionTransformer(img_size=224, patch_size=14, num_frames=num_frames, tubelet_size=2, embed_dim=1664,
                             depth=depth, num_heads=16, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(torch.nn.LayerNorm, eps=1e-6)).to(dev).eval()


@pytest.mark.parametrize("kind", ["image", "video"])
def test_vitg14_frozen_forward_bf16_fp16_vs_fp64(dev, kind):
    """The frozen ViT-G/14 forward (2 blocks, full width) with and without fp16 autocast against fp64 from the fp32
    master weights: bf16 within TOL_ACT, fp16 within test_vit_under_f16_autocast's bounds; a 237 px image floors to
    the same 16 x 16 grid."""
    from test_gpu_fp16 import _encoder_fp64, _rel
    torch.manual_seed(3)
    mod = _vitg14(dev, 1 if kind == "image" else 16)
    x = torch.randn(*((2, 3, 224, 224) if kind == "image" else (1, 3, 16, 224, 224))).to(dev)
    with torch.no_grad():
        ref = _encoder_fp64(mod, x)
        plain = mod(x)
        with torch.autocast("cuda", dtype=F16):
            half = mod(x)
    assert plain.dtype == BF16 and half.dtype == F32 and plain.shape == (x.shape[0], 256 * (8 if kind == "video" else 1), 1664)
    e_bf, e16 = _rel(plain, ref), _rel(half, ref)
    print(f"\nViT-G/14 {kind}: rel-L2 vs fp64: bf16 {e_bf:.3g}, fp16 {e16:.3g}")
    assert e_bf < TOL_ACT and e16 <= 4e-3 and e16 <= 0.5 * e_bf
    if kind == "image":
        with torch.no_grad():
            big = torch.nn.functional.pad(x, (0, 13, 0, 13), value=7.0)
            assert torch.equal(mod(big), plain)


# ------------------------------------------------------------------------------------------------------ end to end
# widths of the reference's factories (tests/test_patch14_cpu.py holds the real factories' state dicts to the reference's)
WIDTHS = {"vit_giant": dict(embed_dim=1408, num_heads=16, mlp_ratio=48 / 11),
          "vit_gigantic": dict(embed_dim=1664, num_heads=16, mlp_ratio=4)}


def _two_block(name):
    """The factory `name` with depth 2: full width, heads and MLP; the patch size comes from the config."""
    from jepa_b200.models import VisionTransformer
    return partial(VisionTransformer, depth=2, qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6),
                   **WIDTHS[name])


def _pretrained(folder, name, frames, patch):
    enc = _two_block(name)(img_size=224, patch_size=patch, num_frames=frames, tubelet_size=2, uniform_power=True)
    torch.save({"target_encoder": enc.state_dict(), "epoch": 1}, os.path.join(folder, "jepa-latest.pth.tar"))


def _cfg(folder, name, patch, frames):
    from test_eval_cpu import _video_cfg
    cfg = _video_cfg(folder, "synthetic")
    cfg["pretrain"].update(model_name=name, patch_size=patch, frames_per_clip=frames)
    cfg["data"].update(num_classes=3, synthetic_length=16, frames_per_clip=frames if frames > 1 else 16)
    cfg["optimization"].update(batch_size=4, num_epochs=1)
    return cfg


def _check(folder, eval_name, tag, multihead):
    out = os.path.join(folder, eval_name, tag)
    with open(os.path.join(out, "jepa_r0.csv")) as f:
        rows = [r for r in csv.reader(f)]
    assert rows[0] == (["epoch", "head", "loss", "acc"] if multihead else ["epoch", "loss", "acc"])
    assert len(rows) == (3 if multihead else 2), rows
    ck = torch.load(os.path.join(out, "jepa-latest.pth.tar"), map_location="cpu")
    assert ck["epoch"] == 1
    sd = ck["classifiers"][0] if multihead else ck["classifier"]
    assert sd["module.pooler.cross_attention_block.xattn.kv.weight"].shape == (2 * sd["module.linear.weight"].shape[1],
                                                                               sd["module.linear.weight"].shape[1])


def test_eval_vit_giant_video_end_to_end(dev, tmp_path, monkeypatch):
    """vit_giant (patch 16, 16 heads of 88) as a 2-block video encoder: the probe trains at head dim 88, one head, bf16."""
    import src.models.vision_transformer as vit
    from evals.scaffold import main as eval_main
    monkeypatch.setitem(vit.__dict__, "vit_giant", _two_block("vit_giant"))
    _pretrained(tmp_path, "vit_giant", 16, 16)
    cfg = _cfg(tmp_path, "vit_giant", 16, 16)
    cfg["data"].update(num_segments=1, num_views_per_segment=1)
    eval_main("video_classification_frozen", cfg)
    _check(tmp_path, "video_classification_frozen", "t", multihead=False)


def test_eval_vit_gigantic_image_end_to_end(dev, tmp_path, monkeypatch):
    """vit_gigantic (patch 14, 16 heads of 104) as a 2-block image encoder: two probes (multihead_kwargs) under fp16
    autocast."""
    import src.models.vision_transformer as vit
    from evals.scaffold import main as eval_main
    monkeypatch.setitem(vit.__dict__, "vit_gigantic", _two_block("vit_gigantic"))
    _pretrained(tmp_path, "vit_gigantic", 1, 14)
    cfg = _cfg(tmp_path, "vit_gigantic", 14, 1)
    cfg["eval_name"] = "image_classification_frozen"
    cfg["data"] = dict(dataset_name="synthetic", num_classes=3, resolution=224, synthetic_length=16)
    cfg["optimization"].update(fp16_autocast=True, multihead_kwargs=[dict(lr=1e-3), dict(lr=3e-3)])
    eval_main("image_classification_frozen", cfg)
    _check(tmp_path, "image_classification_frozen", "t", multihead=True)
