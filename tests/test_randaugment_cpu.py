"""The GPU training transform's host side, without a GPU: the numpy restatement of the RandAugment ops
(tests/randaugment_numpy.py) equals PIL's output bit for bit on every per-op case of golden_randaugment.pt, the sampler
reproduces the reference's decisions and leaves `random` / `np.random` in the reference's states, the synthetic_uint8
training loader collates augmenting tickets, and vj_clip_augment rejects bad arguments."""
import os
import random
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import randaugment_numpy as RN  # noqa: E402
from jepa_b200 import transforms as tr  # noqa: E402

NORMALIZE = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(HERE, "golden", "golden_randaugment.pt"), weights_only=False)


def test_numpy_ops_equal_pil(golden):
    names = set()
    for c, x, y in RN.op_cases(golden):
        got = RN.apply_op(x.numpy(), (c["code"], c["fval"], c["ival"], c["m"]))
        assert np.array_equal(got, y.numpy()), (c["name"], c["args"], c["frame"])
        names.add(c["name"])
    assert names == set(tr.RA_OPS)


def make_transform(pipeline, crop, gpu_augment=True):
    if pipeline == "eval":
        return tr.make_eval_transforms(training=True, random_horizontal_flip=False, random_resize_aspect_ratio=(0.75, 4 / 3),
                                       random_resize_scale=(0.08, 1.0), reprob=0.25, auto_augment=True, motion_shift=False,
                                       crop_size=crop, normalize=NORMALIZE, gpu_augment=gpu_augment)
    return tr.make_transforms(random_horizontal_flip=True, random_resize_aspect_ratio=(0.75, 4 / 3),
                              random_resize_scale=(0.3, 1.0), reprob=0.25, auto_augment=True, motion_shift=False,
                              crop_size=crop, normalize=NORMALIZE, gpu_augment=gpu_augment)


def synth_clip(seed, shape):       # tests/golden/make_golden_randaugment.py
    T, H, W = shape
    rs = np.random.RandomState(3000 + seed)
    y, x = np.mgrid[:H, :W]
    base = np.stack([(x * 255 // max(W - 1, 1)), (y * 255 // max(H - 1, 1)), ((x + y) * 7) % 256], -1)
    return np.clip(base[None] + rs.randint(-40, 41, size=(T, H, W, 3)), 0, 255).astype(np.uint8)


def run_sampler(case):
    tf = make_transform(case["pipeline"], case["crop"])
    random.seed(case["seed"])
    np.random.seed(case["seed"])
    torch.manual_seed(case["seed"])
    return tf(synth_clip(case["seed"], case["shape"]))


def reference_args(op):
    """The level arguments the reference passes to the op function, from a sampled op record."""
    code, fval, ival, m = op
    name = tr.RA_OPS[code]
    if name in ("AutoContrast", "Equalize", "Invert"):
        return ()
    if name in ("PosterizeIncreasing", "SolarizeIncreasing", "SolarizeAdd"):
        return (float(ival),)
    if name.endswith("Increasing"):
        return (fval,)
    return None          # geometric: checked through the matrix


def test_sampler_matches_reference_decisions_and_rng_state(golden):
    n_erase = 0
    for c in golden["e2e"]:
        t = run_sampler(c)
        assert isinstance(t, tr.AugmentTicket)
        applied = [op for op in t.ops if op is not None]
        assert [tr.RA_OPS[op[0]] for op in applied] == [a[0] for a in c["applied"]], c["seed"]
        T, H, W = c["shape"]
        for op, (name, args) in zip(applied, c["applied"]):
            want = reference_args(op)
            if want is not None:
                assert want == args, (name, want, args)
            elif name == "Rotate":
                assert op[3] == tr.rotate_matrix(args[0], W, H)
            else:
                k = {"ShearX": 1, "ShearY": 3, "TranslateXRel": 2, "TranslateYRel": 5}[name]
                scale = {"TranslateXRel": W, "TranslateYRel": H}.get(name, 1)
                assert op[3][k] == args[0] * scale
        assert tuple(t.box) == tuple(c["box"])
        assert (t.erase is None) == (c["erase"] is None)
        if t.erase is not None:
            n_erase += 1
            assert tuple(t.erase) == tuple(c["erase"])
        assert RN.rng_digests() == (c["py_state"], c["np_state"]), c["seed"]
    assert n_erase >= 2


def test_without_gpu_augment_the_raises_stay():
    with pytest.raises(NotImplementedError, match="RandAugment.*random erasing"):
        make_transform("eval", 32, gpu_augment=False)
    with pytest.raises(NotImplementedError, match="RandAugment.*random erasing"):
        make_transform("pretrain", 32, gpu_augment=False)
    with pytest.raises(NotImplementedError, match="motion_shift"):
        tr.make_transforms(motion_shift=True, gpu_augment=True)


def test_uint8_training_loader_yields_ticket_batches():
    from src.datasets.data_manager import init_data
    tf = make_transform("eval", 32)
    loader, _ = init_data(batch_size=3, transform=tf, data="synthetic_uint8", training=True, clip_len=4, num_clips=2,
                          num_workers=0, crop_size=32, num_classes=5, synthetic_length=6, pin_mem=False)
    data = next(iter(loader))
    segs, labels = data[0], data[1]
    assert len(segs) == 2 and all(len(s) == 3 for s in segs)
    assert all(isinstance(t, tr.AugmentTicket) for s in segs for t in s)
    assert labels.shape == (3,)
    buf, frame_bytes, L, flags = tr.pack_augment([t for s in segs for t in s])
    assert L == 4 and frame_bytes % 64 == 0 and buf.numel() == frame_bytes + 64 * 6 * (1 + L)


def test_pack_augment_tracks_buffers():
    fr = torch.zeros(2, 8, 9, 3, dtype=torch.uint8)
    inv, post = tr.RA_OPS.index("Invert"), tr.RA_OPS.index("Equalize")
    rot0 = (tr.RA_OPS.index("Rotate"), 0.0, 0, None)          # rotation by 0 degrees: PIL copies
    t1 = tr.AugmentTicket(fr, (0, 0, 8, 9), False, [(inv, 0.0, 0, None), None, rot0, (post, 0.0, 0, None)], None, 0)
    t2 = tr.AugmentTicket(fr, (1, 1, 4, 4), True, [None, None, None, None], (1, 2, 3, 4), 99)
    buf, frame_bytes, L, flags = tr.pack_augment([t1, t2])
    tabs = buf[frame_bytes:].numpy().tobytes()
    clips = np.frombuffer(tabs[:128], tr.AUG_CLIP)
    ops = np.frombuffer(tabs[128:], tr.AUG_OP).reshape(L, 2)
    assert list(ops["code"][:, 0]) == [inv, -1, -1, post] and list(ops["in_buf"][:, 0]) == [0, 1, 1, 1]
    assert (ops["code"][:, 1] == -1).all()
    assert list(flags) == [1, 0, 0, 3]
    assert list(clips["final_buf"]) == [0, 0]
    assert tuple(clips[1][["etop", "eleft", "eh", "ew"]].item()) == (1, 2, 3, 4) and clips[1]["seed"] == 99


def test_clip_augment_argument_checks_without_gpu():
    import ctypes
    from jepa_b200 import _lib
    lib = _lib.load()
    f3 = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    fl = (ctypes.c_int * 1)(1)
    p = ctypes.c_void_p
    args = [p(4096), p(8192), p(16384), p(32768), p(65536), ctypes.cast(fl, p), 1, p(1 << 20), 1, 2, 2, 8,
            ctypes.cast(f3, p), ctypes.cast(f3, p), None]
    bad = list(args)
    bad[0] = None
    assert lib.vj_clip_augment(*bad) != 0
    assert b"null pointer" in lib.vj_last_error_string()
    bad = list(args)
    bad[2] = p(16384 + 8)
    assert lib.vj_clip_augment(*bad) != 0
    assert b"aligned" in lib.vj_last_error_string()
    bad = list(args)
    bad[9] = 70000
    assert lib.vj_clip_augment(*bad) != 0
    assert b"65535" in lib.vj_last_error_string()
    bad = list(args)
    bad[6] = 17
    assert lib.vj_clip_augment(*bad) != 0
