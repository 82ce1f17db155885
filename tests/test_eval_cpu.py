"""Frozen-evaluation host side without a GPU: the evaluation-view geometry and OpenCV coefficient tables against the
reference's own output (tests/golden/golden_eval_views.pt), the `evals` entry points, the synthetic evaluation items'
collated structure, and the guards (RandAugment / random erasing, FrameAggregation, torch's own DDP around the probe)."""
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _cases():
    return torch.load(os.path.join(HERE, "golden", "golden_eval_views.pt"))


def synth_frames(seed, shape):
    """make_golden_eval_views.synth_frames: the fixture's inputs, regenerated from the seed."""
    T, H, W = shape
    return np.random.RandomState(2000 + seed).randint(0, 256, size=(T, H, W, 3), dtype=np.uint8)


def emulate_views(frames, crop_size, num_views):
    """The kernel's integer arithmetic in numpy over the host tables: uint8 [V, 3, T, S, S]."""
    from jepa_b200.transforms import resize_axis_coefs, view_geometry
    f = frames.astype(np.int64)
    T, H, W, _ = frames.shape
    S = crop_size
    rh, rw, wins = view_geometry(H, W, S, num_views)
    yt, xt = resize_axis_coefs(H, rh, False), resize_axis_coefs(W, rw, True)
    out = []
    for oy, ox in wins:
        ry, cx = yt[oy:oy + S].astype(np.int64), xt[ox:ox + S].astype(np.int64)

        def hpass(rows):
            return f[:, rows][:, :, cx[:, 0]] * cx[None, None, :, 2, None] + f[:, rows][:, :, cx[:, 1]] * cx[None, None, :, 3, None]
        h0, h1 = hpass(ry[:, 0]), hpass(ry[:, 1])
        u = ((((ry[None, :, None, 2, None] * (h0 >> 4)) >> 16) + ((ry[None, :, None, 3, None] * (h1 >> 4)) >> 16) + 2) >> 2) & 255
        out.append(u.astype(np.uint8).transpose(3, 0, 1, 2))
    return torch.from_numpy(np.stack(out))


def test_view_geometry_matches_reference():
    from jepa_b200.transforms import view_geometry
    for c in _cases():
        T, H, W = c["shape"]
        rh, rw, wins = view_geometry(H, W, c["crop"], c["views"])
        assert (rh, rw) == tuple(c["resized"]), c["seed"]
        assert wins == [tuple(w) for w in c["windows"]], c["seed"]
        assert tuple(c["u8"].shape) == (c["views"], 3, T, c["crop"], c["crop"])


def test_opencv_tables_reproduce_reference_views():
    """Host coefficient tables + the kernel's fixed-point expression give the reference's uint8 views exactly (landscape,
    portrait, square, no-resize, upscale, 1 and 3 views, crop 32 and 224); ClipToTensor + Normalize of them is the
    reference's fp32 output bit for bit."""
    mean = torch.tensor((0.485, 0.456, 0.406))[:, None, None, None]
    std = torch.tensor((0.229, 0.224, 0.225))[:, None, None, None]
    for c in _cases():
        u8 = emulate_views(synth_frames(c["seed"], c["shape"]), c["crop"], c["views"])
        assert torch.equal(u8, c["u8"]), c["seed"]
        if "out" in c:
            assert torch.equal((u8.float() / 255 - mean) / std, c["out"]), c["seed"]


def test_pack_views_job_table():
    from jepa_b200.transforms import pack_views, resize_axis_coefs, view_geometry
    cases = [c for c in _cases() if c["crop"] == 32 and c["views"] == 3 and c["shape"][0] == 2]
    clips = [torch.from_numpy(synth_frames(c["seed"], c["shape"])) for c in cases]
    buf, jobs, tab = pack_views(clips, 32, 3, n_segments=2)
    B, V, T, S = 2, 3, 2, 32
    assert jobs.shape == (2 * V * B, 4) and jobs.dtype == torch.int64 and tab.shape[1] == 4
    j32 = jobs.numpy().view(np.int32).reshape(-1, 8)          # {int64 src, int64 out, int32 H, W, ytab, xtab}
    for k, (c, clip) in enumerate(zip(cases, clips)):
        s, b = divmod(k, B)
        _, H, W = c["shape"]
        for v, (oy, ox) in enumerate(view_geometry(H, W, S, V)[2]):
            j = (s * V + v) * B + b
            src = int(jobs[j, 0])
            assert torch.equal(buf[src:src + clip.numel()], clip.reshape(-1))
            assert int(jobs[j, 1]) == j * 3 * T * S * S
            assert (j32[j, 4], j32[j, 5]) == (H, W)
            rh, rw, _ = view_geometry(H, W, S, V)
            assert torch.equal(tab[j32[j, 6]:j32[j, 6] + S], torch.from_numpy(resize_axis_coefs(H, rh, False)[oy:oy + S]))
            assert torch.equal(tab[j32[j, 7]:j32[j, 7] + S], torch.from_numpy(resize_axis_coefs(W, rw, True)[ox:ox + S]))


def _video_cfg(folder, dataset_type="synthetic"):
    return {
        "eval_name": "video_classification_frozen", "resume_checkpoint": False, "tag": "t",
        "pretrain": dict(model_name="vit_tiny", checkpoint_key="target_encoder", clip_duration=None, frames_per_clip=8,
                         tubelet_size=2, uniform_power=True, use_silu=False, tight_silu=False, use_sdpa=True,
                         patch_size=16, folder=str(folder), checkpoint="jepa-latest.pth.tar", write_tag="jepa"),
        "data": dict(dataset_type=dataset_type, dataset_train="x", dataset_val="y", num_classes=3, frames_per_clip=8,
                     num_segments=2, num_views_per_segment=3),
        "optimization": dict(resolution=224, batch_size=4, num_epochs=2, weight_decay=0.01, lr=1e-3, start_lr=1e-3,
                             final_lr=0.0, warmup=0., use_bfloat16=True, attend_across_segments=False),
    }


def test_evals_entry_points_need_cuda(tmp_path, monkeypatch):
    import evals.main  # noqa: F401
    import evals.scaffold
    import evals.video_classification_frozen.utils as vu
    assert vu.ClipAggregation is not None and callable(vu.make_transforms)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA"):
        evals.scaffold.main("video_classification_frozen", _video_cfg(tmp_path))
    cfg = _video_cfg(tmp_path)
    cfg["data"] = dict(dataset_name="synthetic", num_classes=3, resolution=224)
    with pytest.raises(RuntimeError, match="CUDA"):
        evals.scaffold.main("image_classification_frozen", cfg)


def test_synthetic_eval_items_collate_to_reference_structure():
    from src.datasets.data_manager import init_data
    B, T, S, n_seg, V = 4, 4, 32, 2, 3
    loader, _ = init_data(batch_size=B, data="synthetic", clip_len=T, num_clips=n_seg, crop_size=S, num_workers=0,
                          training=False, num_classes=3, num_views_per_clip=V, synthetic_length=8, pin_mem=False)
    data = next(iter(loader))
    assert len(data[0]) == n_seg and all(len(seg) == V for seg in data[0])
    assert all(tuple(v.shape) == (B, 3, T, S, S) and v.dtype == torch.float32 for seg in data[0] for v in seg)
    assert tuple(data[1].shape) == (B,) and int(data[1].min()) >= 0 and int(data[1].max()) < 3
    assert len(data[2]) == n_seg and all(tuple(i.shape) == (B, T) for i in data[2])
    # the class pattern is shared by items of one class: same-label views correlate, different labels do not
    ds = loader.dataset
    a, b, c = ds[0][0][0][0], ds[3][0][0][0], ds[1][0][0][0]      # labels 0, 0, 1
    corr = lambda x, y: float(torch.corrcoef(torch.stack([x.flatten(), y.flatten()]))[0, 1])
    assert corr(a, b) > 0.6 and abs(corr(a, c)) < 0.1

    from jepa_b200.transforms import make_eval_transforms
    tf = make_eval_transforms(training=False, num_views_per_clip=V, crop_size=S)
    loader, _ = init_data(batch_size=B, data="synthetic_uint8", transform=tf, clip_len=T, num_clips=n_seg, crop_size=S,
                          num_workers=0, training=False, num_classes=3, num_views_per_clip=V, synthetic_length=8)
    data = next(iter(loader))
    assert len(data[0]) == n_seg and all(seg.dtype == torch.uint8 and tuple(seg.shape) == (B, T, 36, 42, 3)
                                         for seg in data[0])

    loader, _ = init_data(batch_size=B, data="synthetic", crop_size=S, num_workers=0, training=True, num_classes=5,
                          images=True, synthetic_length=8, pin_mem=False)
    imgs, labels = next(iter(loader))
    assert tuple(imgs.shape) == (B, 3, S, S) and tuple(labels.shape) == (B,)


def test_pretraining_synthetic_items_unchanged():
    from src.datasets.data_manager import SyntheticVideoDataset, init_data
    loader, _ = init_data(batch_size=2, data="synthetic", clip_len=4, num_clips=1, crop_size=32, num_workers=0,
                          synthetic_length=4, pin_mem=False)
    assert isinstance(loader.dataset, SyntheticVideoDataset)
    clips, label, idx = loader.dataset[1]
    assert label == 0 and idx == [list(range(4))] and tuple(clips[0].shape) == (3, 4, 32, 32)


def test_uint8_training_loader_raises():
    from evals.video_classification_frozen.eval import make_dataloader
    with pytest.raises(NotImplementedError, match="RandAugment.*random erasing"):
        make_dataloader(root_path=["x"], batch_size=2, world_size=1, rank=0, dataset_type="synthetic_uint8",
                        resolution=32, frames_per_clip=4, num_segments=1, training=True, num_classes=3)


def test_frame_aggregation_not_implemented():
    from evals.video_classification_frozen.utils import FrameAggregation
    with pytest.raises(NotImplementedError, match="FrameAggregation"):
        FrameAggregation(torch.nn.Identity())


def test_probe_refuses_torch_ddp():
    """torch's own DDP never sees the probe's gradients (its backward writes the flat buffer, the reducer's hooks never
    fire): the forward refuses to run under it instead of training unsynchronised replicas."""
    import torch.distributed as dist
    from jepa_b200.pooler import AttentiveClassifier
    if dist.is_initialized():
        pytest.skip("a process group is already initialised")
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        clf = AttentiveClassifier(embed_dim=64, num_heads=2, depth=1, num_classes=3)
        ddp = torch.nn.parallel.DistributedDataParallel(clf)
        with pytest.raises(NotImplementedError, match="torch.nn.parallel.DistributedDataParallel"):
            ddp(torch.zeros(2, 4, 64))
    finally:
        dist.destroy_process_group()
