"""The GPU training transform on an H100 (-m gpu): vj_clip_augment against PIL and the reference
(tests/golden/golden_randaugment.pt).  Every RandAugment op equals PIL's uint8 output exactly, in one mixed-frame-size
batch; the end-to-end transforms match the reference's fp32 output outside the erase box and the erase box itself; the
erase noise is N(0, 1), uncorrelated between frames and reproducible; bf16 is the rounding of fp32; and both drop-in
entry points train with gpu_augment on synthetic_uint8 frames."""
import math
import os
import random

import numpy as np
import pytest
import torch

from jepa_b200 import _lib
from randaugment_numpy import op_cases
from test_randaugment_cpu import NORMALIZE, make_transform, run_sampler

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(HERE, "golden", "golden_randaugment.pt"), weights_only=False)


def test_every_op_equals_pil_in_one_mixed_size_batch(dev, golden):
    from jepa_b200 import transforms as tr
    cases = list(op_cases(golden))
    tickets = [tr.AugmentTicket(x[None].contiguous(), (0, 0, x.shape[0], x.shape[1]), False,
                                [(c["code"], c["fval"], c["ival"], c["m"])], None, 0) for c, x, _ in cases]
    n0 = _lib.load().vj_launch_count()
    _, frames = tr.augment_batch(tickets, dev, 8, with_frames=True)
    torch.cuda.synchronize()
    assert _lib.load().vj_launch_count() - n0 <= 3          # one layer: histogram + apply, then the crop pass
    bad = [(c["name"], c["args"], c["frame"]) for (c, _, y), f in zip(cases, frames) if not torch.equal(f[0].cpu(), y)]
    assert not bad, bad


def _outside(out, erase):
    keep = torch.ones(out.shape[-2:], dtype=torch.bool)
    if erase is not None:
        top, left, h, w = erase
        keep[top:top + h, left:left + w] = False
    return keep


def test_end_to_end_matches_reference(dev, golden):
    from jepa_b200 import transforms as tr
    for c in golden["e2e"]:
        t = run_sampler(c)
        tf = make_transform(c["pipeline"], c["crop"])
        n0 = _lib.load().vj_launch_count()
        out = tf.batch([t], dev)[0].cpu()
        assert _lib.load().vj_launch_count() - n0 <= 2 * tr.RA_LAYERS + 1
        ref = c["out"]
        keep = _outside(ref, c["erase"])
        assert torch.equal(torch.isnan(ref[0, 0]), ~keep)
        err = (out - ref)[..., keep].abs().max().item()
        assert err <= 5e-5, (c["pipeline"], c["seed"], err)
        if c["erase"] is not None:
            assert torch.isfinite(out).all() and tuple(t.erase) == tuple(c["erase"])


def _big_erase_tickets(T=8, S=224, B=2):
    from jepa_b200 import transforms as tr
    g = torch.Generator().manual_seed(5)
    return [tr.AugmentTicket(torch.randint(0, 256, (T, 256, 300, 3), dtype=torch.uint8, generator=g), (10, 20, 200, 260),
                             b == 1, None, (2, 3, 200, 210), 1234 + b) for b in range(B)]


def test_erase_noise_statistics_and_reproducibility(dev):
    from jepa_b200 import transforms as tr
    tickets = _big_erase_tickets()
    out = tr.augment_batch(tickets, dev, 224, NORMALIZE[0], NORMALIZE[1])
    again = tr.augment_batch(tickets, dev, 224, NORMALIZE[0], NORMALIZE[1])
    bf = tr.augment_batch(tickets, dev, 224, NORMALIZE[0], NORMALIZE[1], dtype=torch.bfloat16)
    assert torch.equal(out, again)
    assert torch.equal(bf, out.to(torch.bfloat16))
    box = out[:, :, :, 2:202, 3:213].float()
    assert abs(box.mean().item()) < 0.01 and abs(box.std().item() - 1) < 0.01
    flat = box[0].permute(1, 0, 2, 3).reshape(box.shape[2], -1)          # [T, 3 * area] of clip 0
    r = torch.corrcoef(flat)
    off = r[~torch.eye(r.shape[0], dtype=torch.bool, device=r.device)]
    assert off.abs().max().item() < 0.02
    assert not torch.equal(out[0, :, :, 2:202, 3:213], out[1, :, :, 2:202, 3:213])       # per-clip seeds


def test_same_seeds_give_same_batch(dev):
    from jepa_b200 import transforms as tr

    def run():
        tf = make_transform("pretrain", 64)
        random.seed(3)
        np.random.seed(3)
        torch.manual_seed(3)
        g = torch.Generator().manual_seed(9)
        tickets = [tf(torch.randint(0, 256, (4, 72 + 8 * b, 96 - 4 * b, 3), dtype=torch.uint8, generator=g).numpy())
                   for b in range(8)]
        return tr.augment_batch(tickets, dev, 64)
    assert torch.equal(run(), run())


# ------------------------------------------------------------------------------------------------------------------
def test_app_main_with_gpu_augment(tmp_path):
    from app.scaffold import main as app_main
    from test_gpu_train_entry import _cfg, _rows
    cfg = _cfg(tmp_path, epochs=1, load=False)
    cfg["data"]["dataset_type"] = "synthetic_uint8"
    cfg["data_aug"].update(auto_augment=True, reprob=0.25, gpu_augment=True)
    cfg["optimization"]["ipe"] = 2
    app_main("vjepa", cfg)
    body = [r for r in _rows(tmp_path) if r and r[0] != "epoch"]
    assert len(body) == 2 and all(math.isfinite(float(r[2])) for r in body), body


def test_video_eval_trains_with_gpu_augment(dev, tmp_path_factory):
    from app.scaffold import main as app_main
    from evals.scaffold import main as eval_main
    from test_gpu_eval import _check_run, _eval_cfg
    from test_gpu_train_entry import _cfg as pretrain_cfg
    folder = tmp_path_factory.mktemp("pretrain_aug")
    app_main("vjepa", pretrain_cfg(folder, epochs=1, load=False))
    cfg = _eval_cfg(folder, "u8aug", False, dataset_type="synthetic_uint8")
    cfg["data"]["gpu_augment"] = True
    cfg["data"]["synthetic_length"] = 32
    eval_main("video_classification_frozen", cfg)
    body, ck = _check_run(folder, "video_classification_frozen", "u8aug", 2)
    assert len(body) == 2 and all(math.isfinite(float(r[1])) for r in body), body
