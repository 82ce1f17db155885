"""The frozen image evaluation's GPU transforms, host side, without a GPU: the numpy restatement of csrc/image.cu's
resampling (tests/image_numpy.py) equals PIL's Image.resize bit for bit; the validation geometry and crops equal
torchvision's; the training sampler reproduces the reference's decisions and RNG states
(tests/golden/golden_image_transforms.pt); the AutoAugment table equals torchvision's ImageNet policy; ImageFolder trees
load through init_data; and the new entry points reject bad arguments."""
import ctypes
import hashlib
import os
import random
import sys

import numpy as np
import pytest
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from image_numpy import apply_tables, pil_resize, synth_image  # noqa: E402
from jepa_b200 import image_transforms as it  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(HERE, "golden", "golden_image_transforms.pt"), weights_only=False)


def _pil(img, box, out_hw, bicubic):
    i, j, h, w = box
    return np.asarray(Image.fromarray(img).crop((j, i, j + w, i + h)).resize(
        (out_hw[1], out_hw[0]), Image.BICUBIC if bicubic else Image.BILINEAR))


RESAMPLE_SIZES = [(37, 50), (50, 37), (7, 9), (64, 64), (6, 200), (129, 3)]


def resample_cases(H, W):
    """(box, out_hw): x1/16 .. x8, identity, one axis only, odd sizes, crops touching each border, 1-pixel boxes."""
    full = (0, 0, H, W)
    outs = [(H, W), (H * 8, W * 8), (max(1, H // 16), max(1, W // 16)), (H, W * 3), (H * 2 + 1, W), (13, 17), (1, 1),
            (max(1, H // 3), W * 2)]
    boxes = [full, (0, 0, max(1, H // 2), max(1, W // 2)), (H - max(1, H // 3), W - max(1, W // 4), max(1, H // 3),
                                                            max(1, W // 4)), (0, W - 1, H, 1), (H - 1, 0, 1, W),
             (H // 2, W // 2, 1, 1)]
    return [(b, o) for b in boxes for o in outs]


@pytest.mark.parametrize("bicubic", [False, True])
def test_numpy_resample_equals_pil(bicubic):
    n = 0
    for k, (H, W) in enumerate(RESAMPLE_SIZES):
        img = synth_image(k, H, W)
        for box, out_hw in resample_cases(H, W):
            want = _pil(img, box, out_hw, bicubic)
            got = pil_resize(img, box, out_hw, bicubic)
            assert np.array_equal(got, want), (H, W, box, out_hw, bicubic)
            n += 1
    assert n == len(RESAMPLE_SIZES) * 48


def _val_window(img, S):
    H, W = img.shape[:2]
    rh, rw, top, left = it.eval_geometry(H, W, S)
    return apply_tables(img, *it.resample_spec(H, W, (0, 0, H, W), (rh, rw), (top, left), S, False))


def test_validation_geometry_equals_torchvision():
    from torchvision import transforms as T
    from torchvision.transforms import functional as F
    for S in (32, 224, 384):
        for H, W in [(375, 500), (500, 375), (256, 300), (300, 256), (41, 500), (480, 640), (333, 333), (227, 5000)]:
            rh, rw, top, left = it.eval_geometry(H, W, S)
            img = Image.new("RGB", (W, H))
            r = T.Resize(int(S * 256 / 224))(img)
            assert (r.height, r.width) == (rh, rw)
            assert F.get_dimensions(T.CenterCrop(S)(r))[1:] == [S, S]
            assert (top, left) == (int(round((rh - S) / 2.0)), int(round((rw - S) / 2.0)))
    assert it.eval_geometry(375, 500, 224) == (256, 341, 16, 58)             # (341 - 224) / 2 = 58.5 -> 58


def test_validation_crops_equal_fixture(golden):
    for c in golden["val"]:
        img = synth_image(100 + c["seed"], c["H"], c["W"])
        assert np.array_equal(_val_window(img, c["S"]), c["u8"].numpy()), c


def test_policy_table_equals_torchvision():
    from torchvision.transforms import AutoAugment, AutoAugmentPolicy
    tv = AutoAugment(AutoAugmentPolicy.IMAGENET).policies
    ours = [tuple((("Posterize" if n == "PosterizeOriginal" else n), p, m) for n, p, m in sp) for sp in it.AA_POLICY]
    assert [tuple(tuple(op) for op in sp) for sp in tv] == ours
    assert len(it.AA_POLICY) == 25
    assert it.fill_color(it.DEFAULT_NORMALIZE[0]) == (124, 116, 104)


def _digests():
    py = hashlib.sha256(repr(random.getstate()).encode()).hexdigest()
    th = hashlib.sha256(torch.get_rng_state().numpy().tobytes()).hexdigest()
    return py, th


def run_sequence(seq):
    """The GPU training transform over a fixture sequence: [(ticket, fixture item)]."""
    tf = it.GpuImageTransform(crop_size=seq["S"])
    random.seed(seq["seed"])
    np.random.seed(seq["seed"])
    torch.manual_seed(seq["seed"])
    out = []
    for k, ((H, W), d) in enumerate(zip(seq["sizes"], seq["items"])):
        t = tf(Image.fromarray(synth_image(seq["seed"] * 1000 + k, H, W)))
        out.append((t, d, _digests()))
    return out


def test_sampler_matches_reference_decisions_and_rng_state(golden):
    seen, n_erase = set(), 0
    for seq in golden["train"]:
        for t, d, dig in run_sequence(seq):
            assert tuple(t.box) == tuple(d["box"]) and t.flip == d["flip"] and t.policy == d["policy"]
            assert [(n, tuple(a)) for n, a in t.applied] == [(n, tuple(a)) for n, a in d["applied"]]
            assert (t.erase is None) == (d["erase"] is None)
            if t.erase is not None:
                n_erase += 1
                assert tuple(t.erase) == tuple(d["erase"]) and tuple(t.noise.shape) == (3, *d["erase"][2:])
            assert dig == (d["py_state"], d["torch_state"])
            seen.add(t.policy)
    assert seen == set(range(25)) and n_erase >= 10


def test_fallback_crop_and_tiny_images():
    random.seed(0)
    for _ in range(20):
        assert it.rrc_params(6, 200) == (0, 96, 6, 8)            # never fits: central crop at the widest ratio
    assert it.rrc_params(200, 6)[2:] == (8, 6)


def test_training_resample_equals_pil_crop_resize_flip(golden):
    for seq in golden["train"][:2]:
        S = seq["S"]
        for (t, d, _), (H, W) in zip(run_sequence(seq)[:12], seq["sizes"]):
            img = t.image.numpy()
            got = apply_tables(img, *it.resample_spec(H, W, t.box, (S, S), (0, 0), S, True))
            want = _pil(img, t.box, (S, S), True)
            assert np.array_equal(got, want)


def test_image_tickets_collate():
    tf = it.GpuImageEvalTransform(32)
    items = [(tf(synth_image(k, 20 + k, 30)), k) for k in range(3)]
    tickets, labels = it.collate_image_tickets(items)
    assert len(tickets) == 3 and all(isinstance(t, it.ImageTicket) for t in tickets)
    assert labels.tolist() == [0, 1, 2]
    pk, jobs_off, coefs_off, tmp = it.pack_resample([t.image for t in tickets],
                                                    [((0, 0, 20 + k, 30), (32, 40), (0, 0), False, False)
                                                     for k in range(3)], 32)
    assert jobs_off % 64 == 0 and coefs_off % 64 == 0 and tmp > 0


def _png_tree(root, sizes=((40, 30), (30, 44)), classes=("cat", "dog")):
    for split in ("train", "val"):
        for c, name in enumerate(classes):
            d = os.path.join(root, "imgs", split, name)
            os.makedirs(d, exist_ok=True)
            for k, (H, W) in enumerate(sizes):
                Image.fromarray(synth_image(10 * c + k, H, W)).save(os.path.join(d, f"{k}.png"))
            Image.fromarray(synth_image(7, 24, 36)[..., 0]).save(os.path.join(d, "gray.png"))          # mode L
            rgba = np.concatenate([synth_image(8, 33, 21), np.full((33, 21, 1), 200, np.uint8)], -1)
            Image.fromarray(rgba).save(os.path.join(d, "rgba.png"))                                   # mode RGBA


def test_image_folder_through_init_data(tmp_path):
    from src.datasets.data_manager import init_data
    _png_tree(str(tmp_path))
    for training in (True, False):
        tf = it.GpuImageTransform(32) if training else it.GpuImageEvalTransform(32)
        loader, sampler = init_data(batch_size=4, transform=tf, data="ImageNet", root_path=str(tmp_path),
                                    image_folder="imgs", training=training, num_workers=0, crop_size=32, num_classes=2,
                                    images=True, drop_last=False, pin_mem=False)
        ds = loader.dataset
        assert ds.classes == ["cat", "dog"] and len(ds) == 8
        assert ds.root.rstrip("/").endswith(os.path.join("imgs", "train" if training else "val"))
        batches = list(loader)
        assert sum(len(b[0]) for b in batches) == 8
        for tickets, labels in batches:
            assert all(isinstance(t, it.ImageAugmentTicket if training else it.ImageTicket) for t in tickets)
            assert all(t.image.dtype == torch.uint8 and t.image.shape[-1] == 3 for t in tickets)
            assert labels.dtype == torch.int64
    ds = init_data(batch_size=2, transform=it.GpuImageEvalTransform(32), data="iNat21", root_path=str(tmp_path),
                   image_folder="imgs", training=False, num_workers=0, num_classes=2, images=True, pin_mem=False)[0].dataset
    gray = next(k for k, (p, _) in enumerate(ds.samples) if p.endswith("gray.png"))
    t, _ = ds[gray]
    g = synth_image(7, 24, 36)[..., 0]
    assert np.array_equal(t.image.numpy(), np.stack([g, g, g], -1))
    rgba = next(k for k, (p, _) in enumerate(ds.samples) if p.endswith("rgba.png"))
    assert np.array_equal(ds[rgba][0].image.numpy(), synth_image(8, 33, 21))


def test_synthetic_uint8_images_vary_in_size():
    from src.datasets.data_manager import init_data
    loader, _ = init_data(batch_size=4, transform=it.GpuImageEvalTransform(32), data="synthetic_uint8", training=False,
                          num_workers=0, crop_size=32, num_classes=3, images=True, synthetic_length=8, pin_mem=False)
    tickets, labels = next(iter(loader))
    shapes = {tuple(t.image.shape) for t in tickets}
    assert len(shapes) > 1 and any(h > w for h, w, _ in shapes) and any(h < w for h, w, _ in shapes)
    assert labels.tolist() == [0, 1, 2, 0]


def test_image_entry_points_argument_checks_without_gpu():
    from jepa_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p
    f3 = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    fill = (ctypes.c_ubyte * 3)(124, 116, 104)
    fl = (ctypes.c_int * 2)(1, 1)
    views = [p(4096), p(8192), p(16384), p(32768), p(65536), 1, 2, 32, ctypes.cast(f3, p), ctypes.cast(f3, p), None]
    bad = list(views)
    bad[1] = None
    assert lib.vj_image_views(*bad) != 0 and b"null pointer" in lib.vj_last_error_string()
    bad = list(views)
    bad[1] = p(8192 + 8)
    assert lib.vj_image_views(*bad) != 0 and b"aligned" in lib.vj_last_error_string()
    bad = list(views)
    bad[6] = 70000
    assert lib.vj_image_views(*bad) != 0 and b"65535" in lib.vj_last_error_string()
    aug = [p(4096), p(8192), p(16384), p(32768), p(65536), p(1 << 17), p(1 << 18), p(1 << 19), p(1 << 20),
           ctypes.cast(fl, p), 2, p(1 << 21), p(1 << 22), 1, 2, 32, ctypes.cast(f3, p), ctypes.cast(f3, p),
           ctypes.cast(fill, p), None]
    bad = list(aug)
    bad[18] = None
    assert lib.vj_image_augment(*bad) != 0 and b"null pointer" in lib.vj_last_error_string()
    bad = list(aug)
    bad[6] = p((1 << 18) + 4)
    assert lib.vj_image_augment(*bad) != 0 and b"aligned" in lib.vj_last_error_string()
    bad = list(aug)
    bad[10] = 17
    assert lib.vj_image_augment(*bad) != 0 and b"n_layers" in lib.vj_last_error_string()
    bad = list(aug)
    bad[15] = 0
    assert lib.vj_image_augment(*bad) != 0 and b"empty" in lib.vj_last_error_string()
