"""Encoder inputs at a size other than the configured one, without a GPU: the numpy restatement of the positional-
embedding resampling (tests/posinterp_numpy.py, the rules vj_pos_interp implements) against torch's CPU F.interpolate
and the reference-generated digests of golden_offsize.pt, the token-grid and error rules of VisionTransformer, and
FrameAggregation's keys and regrouping."""
import hashlib
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import posinterp_numpy as PN  # noqa: E402

GOLD = os.path.join(HERE, "golden", "golden_offsize.pt")


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()[:16]


def _torch_tri(table, scales):
    x = torch.from_numpy(table).unsqueeze(0).permute(0, 4, 1, 2, 3)
    return F.interpolate(x, scale_factor=scales, mode="trilinear").permute(0, 2, 3, 4, 1)[0].numpy()


def _torch_cubic(table, scale):
    x = torch.from_numpy(table).unsqueeze(0).permute(0, 3, 1, 2)
    return F.interpolate(x, scale_factor=scale, mode="bicubic").permute(0, 2, 3, 1)[0].numpy()


TRI_CASES = [((8, 14, 14), (2.0, 20 / 14, 20 / 14)), ((8, 14, 14), (4 / 8, 18 / 14, 10 / 14)), ((3, 5, 6), (1.7, 0.6, 1.33)),
             ((4, 7, 7), (2.0, 1.5, 1.5)), ((8, 24, 24), (2.0, 1.0, 1.0)), ((5, 9, 3), (0.45, 2.31, 3.0)),
             ((2, 2, 2), (1.5, 0.5, 3.7)), ((8, 14, 14), (16 / 8, 14 / 14, 20 / 14))]
CUBIC_CASES = [(14, math.sqrt(256 / 196)), (14, math.sqrt(400 / 196)), (14, math.sqrt(576 / 196)), (7, 1.5), (5, 0.7),
               (9, 0.34), (4, 3.5625), (3, 3.25), (13, 1.0), (20, 0.55)]


@pytest.mark.parametrize("shape,scales", TRI_CASES)
def test_numpy_trilinear_equals_torch(shape, scales):
    table = torch.randn(*shape, 24, generator=torch.Generator().manual_seed(sum(shape))).numpy()
    want = _torch_tri(table, scales)
    got = PN.trilinear(table, scales)
    assert got.shape == want.shape and np.array_equal(got, want), np.abs(got - want).max()


@pytest.mark.parametrize("n,scale", CUBIC_CASES)
def test_numpy_bicubic_equals_torch(n, scale):
    table = torch.randn(n, n, 24, generator=torch.Generator().manual_seed(n)).numpy()
    want = _torch_cubic(table, scale)
    got = PN.bicubic(table, scale)
    assert got.shape == want.shape and np.array_equal(got, want), np.abs(got - want).max()


def test_fma32_is_correctly_rounded():
    from fractions import Fraction
    g = np.random.default_rng(0)
    a, b, c = (g.standard_normal(3000).astype(np.float32) for _ in range(3))
    c[::3] = -(a[::3] * b[::3])          # near-cancellation, where a double rounding would show
    got = PN.fma32(a, b, c)
    for i in range(len(a)):
        q = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        r = np.float32(float(q))
        cands = [r, np.nextafter(r, np.float32(np.inf)), np.nextafter(r, np.float32(-np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - q), int(np.float32(v).view(np.int32)) & 1))
        assert got[i] == best, i


def _tables():
    from jepa_b200.pos_embs import get_2d_sincos_pos_embed, get_3d_sincos_pos_embed
    return (lambda D: get_3d_sincos_pos_embed(D, 14, 8, cls_token=False, uniform_power=True).astype(np.float32),
            lambda D: get_2d_sincos_pos_embed(D, 14, cls_token=False).astype(np.float32))


def test_fixture_tables_reproduced_by_restatement():
    """The reference's interpolate_pos_encoding outputs (sha digests) follow from our sin-cos tables and the restated
    rules - the same bit-exact target the GPU kernel is held to."""
    g = torch.load(GOLD)
    video, image = _tables()
    for case in g["tables"]["video"]:
        D, (T, H, W) = case["D"], case["thw"]
        src = video(D)
        assert _sha(src) == case["src_sha"]
        grid = (T // 2, H // 16, W // 16)
        out = src.reshape(8, 14, 14, D) if grid == (8, 14, 14) else PN.trilinear(src.reshape(8, 14, 14, D),
                                                                                  PN.video_scales((8, 14, 14), grid))
        assert (1,) + (out.size // D, D) == case["shape"] and _sha(out) == case["sha"], (D, T, H, W)
    for case in g["tables"]["image"]:
        D, S = case["D"], case["size"]
        src = image(D)
        assert _sha(src) == case["src_sha"]
        out = PN.bicubic(src.reshape(14, 14, D), PN.image_scale(14, S // 16))
        assert (1,) + (out.size // D, D) == case["shape"] and _sha(out) == case["sha"], (D, S)


def _vit(num_frames=16, **kw):
    from functools import partial
    from jepa_b200.models import VisionTransformer
    return VisionTransformer(img_size=224, num_frames=num_frames, tubelet_size=2, embed_dim=192, depth=1, num_heads=3,
                             norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), uniform_power=True, **kw)


def test_token_grid_rules():
    v = _vit()
    assert v.grid == (8, 14, 14)
    assert v.token_grid((2, 3, 16, 224, 224)) == (8, 14, 14)
    assert v.token_grid((2, 3, 32, 224, 224)) == (16, 14, 14)
    assert v.token_grid((2, 3, 16, 224, 320)) == (8, 14, 20)
    assert v.token_grid((1, 3, 16, 230, 230)) == (8, 14, 14)         # non-multiples floor, as Conv3d does
    assert v.token_grid((1, 3, 17, 239, 250)) == (8, 14, 15)
    with pytest.raises(ValueError, match="smaller than one"):
        v.token_grid((1, 3, 1, 224, 224))
    im = _vit(num_frames=1)
    assert im.grid == (1, 14, 14) and im.tubelet_size == 1
    assert im.token_grid((4, 3, 224, 224)) == (1, 14, 14)
    assert im.token_grid((4, 3, 320, 320)) == (1, 20, 20)
    assert im.token_grid((4, 3, 230, 239)) == (1, 14, 14)
    with pytest.raises(ValueError, match="not square"):
        im.token_grid((4, 3, 224, 320))
    with pytest.raises(RuntimeError, match="CUDA"):
        v(torch.zeros(1, 3, 16, 320, 320))


def test_grid_rejects_sizes_the_reference_cannot_serve():
    """Where the reference's own scale factor floors to a table smaller than the token grid (x += pos_embed fails
    there), the encoder raises instead of adding a mismatched table."""
    v, im = _vit(), _vit(num_frames=1)
    bad = [h for h in range(1, 80) if int(14 * (h / 14)) != h]
    bad_im = [h for h in range(1, 80) if int(14 * math.sqrt(h * h / 196)) != h]
    assert bad and bad_im
    for h in bad[:3]:
        with pytest.raises(ValueError, match="rounding"):
            v.token_grid((1, 3, 16, 16 * h, 224))
    for h in bad_im[:3]:
        with pytest.raises(ValueError, match="rounding"):
            im.token_grid((1, 3, 16 * h, 16 * h))


def test_frame_aggregation_keys_match_reference():
    from evals.video_classification_frozen.utils import FrameAggregation
    from jepa_b200.models import vit_tiny
    g = torch.load(GOLD)["frameagg"]
    enc = vit_tiny(img_size=64, num_frames=1, uniform_power=True)
    assert list(FrameAggregation(enc).state_dict().keys()) == g["keys"]
    agg = FrameAggregation(enc, max_frames=g["max_frames"], use_pos_embed=True)
    assert list(agg.state_dict().keys()) == g["keys_pos"]
    assert agg.embed_dim == 192 and agg.num_heads == 3 and not agg.pos_embed.requires_grad


def _frames_encoder():
    """Stand-in image encoder: a VisionTransformer (4 x 4 images, 2 x 2 patches, width 8, no blocks) whose forward is a
    cheap CPU map [B, C, H, W] -> [B, 4, 8] of tokens that identify the image."""
    from functools import partial
    from jepa_b200.models import VisionTransformer

    class _Frames(VisionTransformer):
        def forward(self, x):
            B, C, H, W = x.shape
            t = x.reshape(B, C, 2, H // 2, 2, W // 2).mean(dim=(3, 5)).flatten(2).transpose(1, 2)     # [B, 4, C]
            return torch.cat([t, 2 * t, t[..., :2]], dim=-1)

    return _Frames(img_size=4, patch_size=2, num_frames=1, embed_dim=8, depth=0, num_heads=2,
                   norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def test_frame_aggregation_wraps_only_image_encoders():
    """FrameAggregation runs the frames through an image encoder of jepa_b200.models; a video encoder or another module
    is refused instead of being run frame by frame outside the kernels."""
    from jepa_b200.pooler import FrameAggregation
    with pytest.raises(NotImplementedError, match="video encoder"):
        FrameAggregation(_vit(num_frames=16))
    with pytest.raises(NotImplementedError, match="Identity"):
        FrameAggregation(torch.nn.Identity())
    assert FrameAggregation(_vit(num_frames=1)).embed_dim == 192


def test_frame_aggregation_regroups_like_reference():
    """The reference's forward (utils.py:50-83) restated: views on batch, segments along time, frames on batch through
    the encoder, per-view token sequences, 1-D sin-cos rows of each frame's clip index added to its tokens."""
    from jepa_b200.pooler import FrameAggregation
    from jepa_b200.pos_embs import get_1d_sincos_pos_embed
    g = torch.Generator().manual_seed(3)
    B, Fr, V, S = 2, 3, 2, 2
    xs = [[torch.randn(B, 3, Fr, 4, 4, generator=g) for _ in range(V)] for _ in range(S)]
    idx = [torch.randint(0, 20, (B, Fr), generator=g) for _ in range(S)]
    enc = _frames_encoder()
    x = torch.cat([torch.cat(v, dim=0) for v in xs], dim=2)
    VB, C, T, H, W = x.shape
    tok = enc(x.permute(0, 2, 1, 3, 4).reshape(VB * T, C, H, W))
    N, D = tok.shape[1:]
    tok = tok.reshape(VB, T, N, D).flatten(1, 2)
    table = torch.from_numpy(get_1d_sincos_pos_embed(D, 20)).float()
    pos = torch.cat([table[i] for i in idx], dim=1).unsqueeze(2).repeat(1, 1, N, 1).flatten(1, 2)
    want_nopos = [tok[v * B:(v + 1) * B] for v in range(V)]
    got = FrameAggregation(enc)(xs, clip_indices=idx)
    assert len(got) == V and all(torch.equal(a, b) for a, b in zip(got, want_nopos))
    got = FrameAggregation(enc, max_frames=20, use_pos_embed=True)(xs, clip_indices=idx)
    assert all(torch.equal(a, b + pos) for a, b in zip(got, want_nopos))


def test_eval_wraps_image_encoders_in_frame_aggregation():
    import inspect
    import evals.video_classification_frozen.eval as ev
    src = inspect.getsource(ev.main)
    assert "FrameAggregation(encoder)" in src and "pretrain_frames_per_clip == 1" in src
