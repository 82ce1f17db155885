"""14-pixel patches (ViT-G/14) on the CPU: the padded patch-row length, the patch-vector order vj_im2col_tubelets
writes (restated here and held against the unmodified reference's PatchEmbed3D / PatchEmbed, tests/golden/
golden_patch14.pt), and the state-dict keys and shapes of vit_giant / vit_gigantic against the reference's."""
import os

import pytest
import torch

from common import synth_state

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "golden_patch14.pt")


def im2col_ref(clips, tub, ps, idx=None):
    """What vj_im2col_tubelets writes, restated: clips [B,C,T,H,W] -> [B*K, P_pad], columns (c, dt, dh, dw), rows the
    (t', h', w') tokens (or idx[b]), columns P.. P_pad-1 zero."""
    from jepa_b200.params import padded_patch_dim
    B, C, T, H, W = clips.shape
    x = clips.reshape(B, C, T // tub, tub, H // ps, ps, W // ps, ps).permute(0, 2, 4, 6, 1, 3, 5, 7)
    x = x.reshape(B, -1, C * tub * ps * ps)
    if idx is not None:
        x = torch.stack([x[b, idx[b]] for b in range(B)])
    P = x.shape[-1]
    out = torch.zeros(x.shape[0] * x.shape[1], padded_patch_dim(P), dtype=x.dtype, device=x.device)
    out[:, :P] = x.reshape(-1, P)
    return out


def test_padded_patch_dim():
    from jepa_b200.params import padded_patch_dim
    assert [padded_patch_dim(p) for p in (3 * 2 * 16 * 16, 3 * 16 * 16, 3 * 2 * 14 * 14, 3 * 14 * 14, 1, 64, 65)] == \
        [1536, 768, 1216, 640, 64, 64, 128]


@pytest.mark.parametrize("kind", ["video", "image"])
def test_patch_order_matches_reference(kind):
    """Padded patch rows times the zero-padded [D, P_pad] weight are the reference's Conv3d / Conv2d patch embedding."""
    from jepa_b200.models import PatchEmbed, PatchEmbed3D
    from jepa_b200.params import padded_patch_dim
    gold = torch.load(GOLD)[kind]
    x, want = gold["x"], gold["y"]
    mod = PatchEmbed3D(patch_size=14, tubelet_size=2, embed_dim=64) if kind == "video" else PatchEmbed(14, embed_dim=64)
    mod.load_state_dict(synth_state({k: tuple(v.shape) for k, v in mod.state_dict().items()},
                                    seed=53 if kind == "video" else 54))
    w, b = mod.proj.weight.detach(), mod.proj.bias.detach()
    D, P = w.shape[0], w[0].numel()
    Pp = padded_patch_dim(P)
    assert Pp > P
    clips = x if kind == "video" else x.unsqueeze(2)
    rows = im2col_ref(clips, 2 if kind == "video" else 1, 14)
    assert rows.shape == (want.shape[0] * want.shape[1], Pp) and not rows[:, P:].any()
    w_pad = torch.zeros(D, Pp)
    w_pad[:, :P] = w.reshape(D, P)
    got = (rows.double() @ w_pad.double().t() + b.double()).view_as(want)
    torch.testing.assert_close(got, want.double(), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("name", ["vit_giant", "vit_gigantic"])
@pytest.mark.parametrize("frames", [16, 1])
def test_state_dict_matches_reference(name, frames):
    from jepa_b200 import models
    ref = torch.load(GOLD)["shapes"][(name, frames)]
    with torch.device("meta"):
        m = models.__dict__[name](img_size=224, num_frames=frames, tubelet_size=2, uniform_power=True)
    sd = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    assert len(sd) == ref["n_keys"] and len(m.blocks) == ref["depth"]
    kept = [kv for kv in sd if not kv[0].startswith("blocks.") or kv[0].startswith("blocks.0.")]
    assert kept == ref["keys"]
    block0 = [(k[len("blocks.0."):], s) for k, s in sd if k.startswith("blocks.0.")]
    for i in range(len(m.blocks)):
        assert [(k[len(f"blocks.{i}."):], s) for k, s in sd if k.startswith(f"blocks.{i}.")] == block0
    D, ps = (1664, 14) if name == "vit_gigantic" else (1408, 16)
    assert dict(sd)["patch_embed.proj.weight"] == ((D, 3, 2, ps, ps) if frames > 1 else (D, 3, ps, ps))
