"""The frozen image evaluation's GPU transforms on an H100 (-m gpu): vj_image_views / vj_image_augment against PIL,
torchvision and the reference (tests/golden/golden_image_transforms.pt).  Resampling equals PIL's Image.resize exactly in
one mixed-size batch; validation equals torchvision's fp32 output bit for bit (bf16 is its rounding); training equals
the reference's fp32 output bit for bit, erase box included; every AutoAugment op equals PIL with the (124, 116, 104)
fill; launch counts stay within 2 (validation) and 7 (training); and the image evaluation runs from evals.scaffold.main
on synthetic uint8 images and on a PNG ImageFolder tree."""
import hashlib
import os

import numpy as np
import pytest
import torch
from PIL import Image, ImageEnhance, ImageOps

from image_numpy import synth_image
from jepa_b200 import _lib
from jepa_b200 import image_transforms as it
from test_gpu_eval import N_ITEMS, _check_run, _eval_cfg, pretrained  # noqa: F401  (module fixture)
from test_image_transforms_cpu import RESAMPLE_SIZES, _pil, _png_tree, resample_cases, run_sequence

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MEAN = torch.tensor(it.DEFAULT_NORMALIZE[0]).view(3, 1, 1)
STD = torch.tensor(it.DEFAULT_NORMALIZE[1]).view(3, 1, 1)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    _lib.load()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(HERE, "golden", "golden_image_transforms.pt"), weights_only=False)


def _launches():
    return _lib.load().vj_launch_count()


def _to_tensor_normalise(u8):
    """torchvision ToTensor + Normalize of uint8 [H, W, 3], on the CPU in fp32."""
    return (torch.as_tensor(np.ascontiguousarray(u8)).permute(2, 0, 1).float().div(255) - MEAN) / STD


def test_resample_equals_pil_in_one_mixed_size_batch(dev):
    S, images, specs, want = 8, [], [], []
    for k, (H, W) in enumerate(RESAMPLE_SIZES):
        img = synth_image(k, H, W)
        for bicubic in (False, True):
            for box, (oh, ow) in resample_cases(H, W):
                if oh < S or ow < S:
                    continue
                ref = _pil(img, box, (oh, ow), bicubic)
                for top, left in ((0, 0), (oh - S, ow - S)):
                    images.append(torch.from_numpy(img))
                    specs.append((box, (oh, ow), (top, left), bicubic, False))
                    want.append(ref[top:top + S, left:left + S])
    n0 = _launches()
    got = it.resample_images(images, specs, S, dev).cpu().numpy()
    torch.cuda.synchronize()
    assert _launches() - n0 <= 3 and len(want) > 200
    bad = [s for s, g, w in zip(specs, got, want) if not np.array_equal(g, w)]
    assert not bad, bad[:5]


@pytest.mark.parametrize("S", [224, 384])
def test_validation_equals_torchvision(dev, S):
    from torchvision import transforms as T
    tf = T.Compose([T.Resize(int(S * 256 / 224)), T.CenterCrop(S), T.ToTensor(), T.Normalize(*it.DEFAULT_NORMALIZE)])
    sizes = [(375, 500), (500, 375), (256, 300), (300, 256), (438, 600), (480, 640), (333, 333), (227, 1000)]
    pils = [Image.fromarray(synth_image(k, H, W)) for k, (H, W) in enumerate(sizes)]
    want = torch.stack([tf(p) for p in pils])
    gt = it.GpuImageEvalTransform(S)
    tickets = [gt(p) for p in pils]
    n0 = _launches()
    got = gt.batch(tickets, dev).cpu()
    assert _launches() - n0 == 2
    assert torch.equal(got, want)
    assert torch.equal(gt.batch(tickets, dev, torch.bfloat16).cpu(), want.to(torch.bfloat16))


def test_validation_crops_equal_fixture(dev, golden):
    for S in (32, 64, 224):
        cases = [c for c in golden["val"] if c["S"] == S]
        got = it.image_views_batch([torch.from_numpy(synth_image(100 + c["seed"], c["H"], c["W"])) for c in cases], dev, S)
        for c, g in zip(cases, got.cpu()):
            assert torch.equal(g, _to_tensor_normalise(c["u8"].numpy())), c


def _sha(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def test_training_equals_reference(dev, golden):
    """Every image of every fixture sequence: the uint8 AutoAugment output and the fp32 output equal the reference's
    (sha256 digests), so every op is checked through the composed path at every S; the stored tensors too."""
    for seq in golden["train"]:
        S = seq["S"]
        run = run_sequence(seq)
        tickets = [t for t, _, _ in run]
        n0 = _launches()
        out, u8 = it.image_augment_batch(tickets, dev, S, with_images=True)
        assert _launches() - n0 <= 7
        out, u8 = out.cpu(), u8.cpu()
        bf = it.image_augment_batch(tickets, dev, S, dtype=torch.bfloat16).cpu()
        assert torch.equal(bf, out.to(torch.bfloat16))
        bad = [(k, d["applied"]) for k, (t, d, _) in enumerate(run) if _sha(u8[k]) != d["u8_sha"]]
        assert not bad, (S, bad[:5])
        bad = [(k, t.erase) for k, (t, d, _) in enumerate(run) if _sha(out[k]) != d["out_sha"]]
        assert not bad, (S, bad[:5])
        for k, (t, d, _) in enumerate(run):
            if "u8" in d:
                assert torch.equal(u8[k], d["u8"]), (S, k)
            if "out" in d:
                assert torch.equal(out[k], d["out"]), (S, k)


def _pil_op(img, name, arg, fill):
    kw = dict(resample=Image.BICUBIC, fillcolor=fill)
    if name == "Rotate":
        return img.rotate(arg, **kw)
    if name == "ShearX":
        return img.transform(img.size, Image.AFFINE, (1, arg, 0, 0, 1, 0), **kw)
    if name == "PosterizeOriginal":
        return ImageOps.posterize(img, arg) if arg < 8 else img
    if name == "Solarize":
        return ImageOps.solarize(img, arg)
    if name in ("Color", "Contrast", "Sharpness"):
        return getattr(ImageEnhance, name)(img).enhance(arg)
    return {"AutoContrast": ImageOps.autocontrast, "Equalize": ImageOps.equalize, "Invert": ImageOps.invert}[name](img)


def test_every_autoaugment_op_with_fill(dev):
    fill = it.fill_color(it.DEFAULT_NORMALIZE[0])
    S, images, specs, ops, want, names = 40, [], [], [], [], []
    for k in range(3):
        img = synth_image(200 + k, S, S)
        for sp in it.AA_POLICY:
            for name, _, mag in sp:
                for sgn in ((1, -1) if name in ("Rotate", "ShearX") else (1,)):
                    level = mag or 0
                    code = it.RA_OPS.index(it.AA_KERNEL_OP[name])
                    fval, ival, m, arg = 0.0, 0, None, None
                    if name == "Rotate":
                        arg = sgn * (level / 10.0) * 30.0
                        m = it.rotate_matrix(arg, S, S)
                    elif name == "ShearX":
                        arg = sgn * (level / 10.0) * 0.3
                        m = (1.0, arg, 0.0, 0.0, 1.0, 0.0)
                    elif name == "PosterizeOriginal":
                        arg = ival = int((level / 10.0) * 4) + 4
                    elif name == "Solarize":
                        arg = ival = int((level / 10.0) * 256)
                    elif name in ("Color", "Contrast", "Sharpness"):
                        arg = fval = (level / 10.0) * 1.8 + 0.1
                    images.append(torch.from_numpy(img))
                    specs.append(((0, 0, S, S), (S, S), (0, 0), True, False))
                    ops.append([(code, fval, ival, m)])
                    want.append(np.asarray(_pil_op(Image.fromarray(img), name, arg, fill)))
                    names.append((name, arg, k))
    got = it.resample_images(images, specs, S, dev, ops=ops, fill=fill).cpu().numpy()
    bad = [n for n, g, w in zip(names, got, want) if not np.array_equal(g, w)]
    assert not bad, bad
    assert {n[0] for n in names} == set(it.AA_KERNEL_OP)


# ------------------------------------------------------------------------------------------------------------------
def test_image_eval_trains_on_uint8_images(pretrained):  # noqa: F811
    """Labels stay in step with the device batch, training uses the augmenting transform and validation the
    deterministic one: the probe learns the augmented training images (rising accuracy; a few augmented images, such as
    small crops that keep one stripe, stay ambiguous) and classifies the deterministic validation crops far better than
    the augmented training images (labels out of step would give chance, the training transform on validation about
    the training accuracy)."""
    from evals.scaffold import main as eval_main
    cfg = _eval_cfg(pretrained, "img_u8", False, epochs=3)
    cfg["eval_name"] = "image_classification_frozen"
    cfg["data"] = dict(dataset_name="synthetic_uint8", num_classes=3, resolution=224, synthetic_length=N_ITEMS)
    eval_main("image_classification_frozen", cfg)
    body, _ = _check_run(pretrained, "image_classification_frozen", "img_u8", 3)
    assert [r[0] for r in body] == ["1", "2", "3"]
    train_acc, val_acc = [float(r[1]) for r in body], [float(r[2]) for r in body]
    assert train_acc[0] < train_acc[-1] and train_acc[-1] >= 90.0 and val_acc[-1] >= 99.0, body


def test_image_eval_on_png_image_folder(pretrained, tmp_path):  # noqa: F811
    from evals.scaffold import main as eval_main
    _png_tree(str(tmp_path))
    cfg = _eval_cfg(pretrained, "img_folder", False, epochs=1)
    cfg["eval_name"] = "image_classification_frozen"
    cfg["data"] = dict(dataset_name="ImageNet", num_classes=2, resolution=224, root_path=str(tmp_path),
                       image_folder="imgs")
    eval_main("image_classification_frozen", cfg)
    body, ck = _check_run(pretrained, "image_classification_frozen", "img_folder", 1)
    assert [r[0] for r in body] == ["1"]
    assert ck["classifier"]["module.linear.weight"].shape[0] == 2
