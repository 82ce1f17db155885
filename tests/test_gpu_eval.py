"""The frozen evaluations on the GPU (-m gpu): vj_clip_views against the reference's own evaluation views
(tests/golden/golden_eval_views.pt: fp32 bit for bit, bf16 = round-to-nearest of it), and the drop-in entry points end
to end - `app.scaffold.main('vjepa', cfg)` pre-trains ViT-Tiny and writes jepa-latest.pth.tar, then
`evals.scaffold.main(...)` evaluates that checkpoint (video with and without attend_across_segments, 2 segments x 3
validation views; image) with the reference's CSV rows and checkpoint keys, and resumes from its own checkpoint."""
import csv
import os

import pytest
import torch

from parity_util import TOL_ACT, rel_l2
from test_eval_cpu import _cases, _video_cfg, synth_frames
from test_gpu_train_entry import _cfg as pretrain_cfg

pytestmark = pytest.mark.gpu
MEAN = torch.tensor((0.485, 0.456, 0.406))[:, None, None, None]
STD = torch.tensor((0.229, 0.224, 0.225))[:, None, None, None]
N_ITEMS = 320          # synthetic items per split: 40 steps per epoch at batch 8


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


def _expected(u8):
    """ClipToTensor + Normalize of the reference's uint8 views, in fp32 as the reference computes them."""
    return (u8.float() / 255 - MEAN) / STD


def test_clip_views_match_reference_fixture(dev):
    from jepa_b200.transforms import preprocess_views
    for c in _cases():
        frames = torch.from_numpy(synth_frames(c["seed"], c["shape"]))
        want = torch.stack([_expected(u) for u in c["u8"]])
        if "out" in c:
            assert torch.equal(want, c["out"])
        got = preprocess_views([frames[None]], dev, c["crop"], c["views"])
        assert len(got) == 1 and len(got[0]) == c["views"]
        for v in range(c["views"]):
            assert torch.equal(got[0][v][0].cpu(), want[v]), (c["seed"], v)
        got = preprocess_views([frames[None]], dev, c["crop"], c["views"], dtype=torch.bfloat16)
        for v in range(c["views"]):
            assert torch.equal(got[0][v][0].cpu(), want[v].to(torch.bfloat16)), (c["seed"], v)


def test_clip_views_batch_of_mixed_frame_sizes(dev):
    """One launch for 2 segments x 3 views x 2 clips whose frame sizes all differ (landscape, portrait, square, no-resize)."""
    from jepa_b200.transforms import preprocess_views
    cases = [c for c in _cases() if c["crop"] == 32 and c["views"] == 3 and c["shape"][0] == 2]
    clips = [torch.from_numpy(synth_frames(c["seed"], c["shape"])) for c in cases]
    got = preprocess_views([clips[:2], clips[2:]], dev, 32, 3)
    for k, c in enumerate(cases):
        s, b = divmod(k, 2)
        for v in range(3):
            assert torch.equal(got[s][v][b].cpu(), _expected(c["u8"][v])), (c["seed"], v)


def test_uint8_validation_logits_match_cpu_views(dev):
    """Validation fed by uint8 frames through vj_clip_views and by the reference's CPU-transformed views give the same
    logits (within DESIGN section 5's activation tolerance)."""
    from jepa_b200.models import vit_tiny
    from jepa_b200.pooler import AttentiveClassifier, ClipAggregation
    from jepa_b200.transforms import preprocess_views
    torch.manual_seed(0)
    c = next(c for c in _cases() if c["seed"] == 1)                  # T 2, crop 32, 3 views
    enc = vit_tiny(img_size=32, patch_size=16, num_frames=2, tubelet_size=2, uniform_power=True).to(dev).eval()
    encoder = ClipAggregation(enc, tubelet_size=2)
    clf = AttentiveClassifier(embed_dim=192, num_heads=3, depth=1, num_classes=5).to(dev).eval()
    cpu_views = [[_expected(u)[None].to(dev) for u in c["u8"]]]
    gpu_views = preprocess_views([torch.from_numpy(synth_frames(c["seed"], c["shape"]))[None]], dev, 32, 3)
    with torch.no_grad():
        a = [clf(o[0]) for o in encoder(cpu_views)]
        b = [clf(o[0]) for o in encoder(gpu_views)]
    for x, y in zip(a, b):
        assert rel_l2(y.float().cpu(), x.float().cpu()) < TOL_ACT


# ------------------------------------------------------------------------------------------------------------------
# pre-train, then evaluate through the drop-in entry points
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pretrained(dev, tmp_path_factory):
    from app.scaffold import main as app_main
    folder = tmp_path_factory.mktemp("pretrain")
    app_main("vjepa", pretrain_cfg(folder, epochs=1, load=False))
    assert os.path.exists(os.path.join(folder, "jepa-latest.pth.tar"))
    return folder


def _eval_cfg(folder, tag, attend, epochs=2, dataset_type="synthetic"):
    cfg = _video_cfg(folder, dataset_type)
    cfg["tag"] = tag
    cfg["data"].update(num_classes=3, synthetic_length=N_ITEMS)
    cfg["optimization"].update(batch_size=8, num_epochs=epochs, attend_across_segments=attend, lr=5e-3, start_lr=5e-3,
                               final_lr=1e-3, warmup=0.)
    return cfg


def _csv(path):
    with open(path) as f:
        return [r for r in csv.reader(f)]


def _check_run(folder, eval_name, tag, epochs):
    out = os.path.join(folder, eval_name, tag)
    rows = _csv(os.path.join(out, "jepa_r0.csv"))
    assert rows[0] == ["epoch", "loss", "acc"]
    body = [r for r in rows if r and r[0] != "epoch"]
    ck = torch.load(os.path.join(out, "jepa-latest.pth.tar"), map_location="cpu")
    assert set(ck) == {"classifier", "opt", "scaler", "epoch", "batch_size", "world_size", "lr"}
    assert ck["epoch"] == epochs and ck["world_size"] == 1
    assert all(k.startswith("module.") for k in ck["classifier"])
    assert "module.pooler.cross_attention_block.xattn.kv.weight" in ck["classifier"] and "module.linear.weight" in ck["classifier"]
    assert len(ck["opt"]["param_groups"]) == 2 and ck["opt"]["param_groups"][1]["WD_exclude"]
    return body, ck


@pytest.mark.parametrize("attend", [False, True])
def test_video_eval_end_to_end(pretrained, attend):
    from evals.scaffold import main as eval_main
    tag = f"attend{int(attend)}"
    eval_main("video_classification_frozen", _eval_cfg(pretrained, tag, attend))
    body, ck = _check_run(pretrained, "video_classification_frozen", tag, 2)
    assert [r[0] for r in body] == ["1", "2"]
    train_acc = [float(r[1]) for r in body]
    assert train_acc[-1] == 100.0, body
    assert all(0.0 <= float(r[2]) <= 100.0 for r in body)
    ipe = N_ITEMS // 8
    assert float(next(iter(ck["opt"]["state"].values()))["step"]) == 2 * ipe

    if attend:
        return
    # resume: a third epoch continues from the saved one with the saved optimizer state
    from evals.video_classification_frozen.eval import init_opt, load_checkpoint
    from jepa_b200.distributed import DistributedDataParallel
    from jepa_b200.pooler import AttentiveClassifier
    out = os.path.join(pretrained, "video_classification_frozen", tag, "jepa-latest.pth.tar")
    clf = AttentiveClassifier(embed_dim=192, num_heads=3, depth=1, num_classes=3).cuda()
    opt, scaler, _, _ = init_opt(clf, iterations_per_epoch=ipe, start_lr=5e-3, ref_lr=5e-3, warmup=0., num_epochs=3,
                                 use_bfloat16=True)
    clf = DistributedDataParallel(clf, static_graph=True)
    clf, opt, scaler, epoch = load_checkpoint(torch.device("cuda:0"), out, clf, opt, scaler)
    assert epoch == 2
    sd = opt.state_dict()
    for k, st in ck["opt"]["state"].items():
        for name, t in st.items():
            assert torch.equal(torch.as_tensor(sd["state"][k][name]).cpu(), torch.as_tensor(t)), (k, name)
    assert torch.equal(clf.module.linear.weight.detach().cpu(), ck["classifier"]["module.linear.weight"])

    cfg = _eval_cfg(pretrained, tag, attend, epochs=3)
    cfg["resume_checkpoint"] = True
    eval_main("video_classification_frozen", cfg)
    body, ck3 = _check_run(pretrained, "video_classification_frozen", tag, 3)
    assert [r[0] for r in body] == ["1", "2", "3"]
    assert float(next(iter(ck3["opt"]["state"].values()))["step"]) == 3 * ipe


def test_video_eval_uint8_validation(pretrained):
    """dataset_type synthetic_uint8: validation frames stay uint8 through the loader and vj_clip_views makes the 3 views
    per segment; the training loader of the same config raises (RandAugment / random erasing), so the probe trains on
    the pre-normalised set and is then validated on uint8 frames."""
    from evals.scaffold import main as eval_main
    from evals.video_classification_frozen import eval as ve
    with pytest.raises(NotImplementedError, match="RandAugment"):
        eval_main("video_classification_frozen", _eval_cfg(pretrained, "u8", False, dataset_type="synthetic_uint8"))
    from jepa_b200 import _lib
    lib = _lib.load()
    loader = ve.make_dataloader(root_path=["v"], batch_size=4, world_size=1, rank=0, dataset_type="synthetic_uint8",
                                resolution=224, frames_per_clip=8, num_segments=2, num_views_per_segment=3,
                                training=False, num_classes=3, synthetic_length=8)
    data = next(iter(loader))
    n0 = lib.vj_launch_count()
    clips = ve.load_clips(data, torch.device("cuda:0"), loader)
    assert lib.vj_launch_count() - n0 == 1
    assert len(clips) == 2 and all(len(s) == 3 and tuple(v.shape) == (4, 3, 8, 224, 224) for s in clips for v in s)
    assert all(torch.isfinite(v).all() for s in clips for v in s)


def test_image_eval_end_to_end(pretrained):
    from evals.scaffold import main as eval_main
    cfg = _eval_cfg(pretrained, "img", False)
    cfg["eval_name"] = "image_classification_frozen"
    cfg["data"] = dict(dataset_name="synthetic", num_classes=3, resolution=224, synthetic_length=N_ITEMS)
    eval_main("image_classification_frozen", cfg)
    body, _ = _check_run(pretrained, "image_classification_frozen", "img", 2)
    assert [r[0] for r in body] == ["1", "2"]
    assert float(body[-1][1]) == 100.0, body
