"""Gradient accumulation on the GPU (-m gpu): two half-batch micro-batches, each scaled by 1/2, accumulated into the
live flat gradient buffer against one full-batch backward, on ViT-Tiny (C1) and a 2-block ViT-L/16 slice; the buffer
arithmetic, memory and aliasing of the second backward; and app.vjepa.train.main with `optimization.accum_iter: 2`."""
import copy
import os

import pytest
import torch

from common import C1, synth_clips
from parity_util import VITL_2B, build_states, cfg_masks, rel_l2

pytestmark = pytest.mark.gpu
F32_EPS = torch.finfo(torch.float32).eps


def _nets(cfg, depth, dev):
    from jepa_b200.models import MultiMaskWrapper, PredictorMultiMaskWrapper
    enc, pred, s_enc, s_pred, s_tgt, _, _ = build_states(depth, cfg)
    enc.load_state_dict(s_enc, strict=False)
    pred.load_state_dict(s_pred, strict=False)
    tgt = copy.deepcopy(enc)
    tgt.load_state_dict(s_tgt, strict=False)
    enc, pred, tgt = MultiMaskWrapper(enc).to(dev), PredictorMultiMaskWrapper(pred).to(dev), MultiMaskWrapper(tgt).to(dev)
    for p in tgt.parameters():
        p.requires_grad = False
    return enc, pred, tgt


def _inputs(cfg, B, dev):
    """B clips and fixed [B, K] masks of one seeded collator call; rows b of clips and masks belong together."""
    clips = synth_clips(B, cfg["num_frames"], cfg["crop_size"], cfg["crop_size"], seed=0).to(dev)
    me, mp = cfg_masks(cfg, B)
    return clips, [m.to(dev) for m in me], [m.to(dev) for m in mp]


def _half(inputs, i, B):
    clips, me, mp = inputs
    s = slice(i * (B // 2), (i + 1) * (B // 2))
    return clips[s], [m[s] for m in me], [m[s] for m in mp]


def _backward(nets, inputs, scale):
    from jepa_b200 import step as vj
    enc, pred, tgt = nets
    clips, me, mp = inputs
    h = vj.forward_target(tgt, clips, mp)
    loss = vj.jepa_loss(pred(enc(clips, me), h, me, mp), h)
    (loss * scale if scale != 1.0 else loss).backward()
    return float(loss.detach())


def _grads(nets):
    enc, pred, _ = nets
    return {(i, n): p.grad.detach().clone() for i, net in enumerate((enc, pred)) for n, p in net.named_parameters()
            if p.grad is not None}


def _zero(nets):
    for net in nets[:2]:
        net.zero_grad(set_to_none=True)


def _buffers(nets):
    """The flat gradient buffer of the encoder and of the predictor (every trainable .grad is a slice of it)."""
    out = []
    for net in nets[:2]:
        st = net.backbone._store
        g = st.grad_buffer(p for p in net.parameters() if p.requires_grad)
        assert g is not None
        for n, p in net.backbone.named_parameters():
            if p.requires_grad:
                assert p.grad.data_ptr() == g.data_ptr() + 4 * st.offsets[n][0], n
        out.append(g)
    return out


@pytest.mark.parametrize("cfg,depth,B", [(C1, 2, 2), (VITL_2B, None, 2)], ids=["vit_tiny_c1", "vit_large_2block"])
def test_two_half_batches_match_the_full_batch(cfg, depth, B):
    dev = torch.device("cuda:0")
    nets = _nets(cfg, depth, dev)
    inputs = _inputs(cfg, B, dev)
    loss_full = _backward(nets, inputs, 1.0)
    want = _grads(nets)
    _zero(nets)
    losses = [_backward(nets, _half(inputs, i, B), 0.5) for i in range(2)]
    torch.cuda.synchronize()
    got = _grads(nets)
    assert set(got) == set(want)
    worst = max(rel_l2(got[k], want[k]) for k in want)
    assert worst <= 1e-5, worst
    assert abs(sum(losses) / 2 - loss_full) <= 1e-5 * abs(loss_full), (losses, loss_full)


def test_accumulated_buffer_is_the_sum_of_the_half_batch_buffers():
    dev = torch.device("cuda:0")
    B = 2
    nets = _nets(C1, 2, dev)
    inputs = _inputs(C1, B, dev)
    _backward(nets, _half(inputs, 0, B), 1.0)
    g1 = [g.clone() for g in _buffers(nets)]
    _backward(nets, _half(inputs, 1, B), 1.0)            # adds into the live buffers
    acc = [g.clone() for g in _buffers(nets)]
    _zero(nets)
    _backward(nets, _half(inputs, 1, B), 1.0)
    g2 = [g.clone() for g in _buffers(nets)]
    torch.cuda.synchronize()
    for a, x, y in zip(acc, g1, g2):
        # a few fp32 ulps of |g1| + |g2|: the second backward's weight-gradient pieces reduce-add onto g1 instead of
        # onto zero; where the two cancel, the bound is taken at 1e-3 of the buffer's largest magnitude
        mag = torch.maximum(x.abs() + y.abs(), 1e-3 * (x.abs() + y.abs()).max())
        err = float(((a - (x + y)).abs() / (F32_EPS * mag)).max())
        assert err <= 16, err


def test_second_micro_batch_allocates_no_gradient_buffer():
    dev = torch.device("cuda:0")
    B = 2
    nets = _nets(C1, 2, dev)
    inputs = _inputs(C1, B, dev)
    _backward(nets, _half(inputs, 0, B), 0.5)
    torch.cuda.synchronize()
    bufs = [g.data_ptr() for g in _buffers(nets)]
    mem0 = torch.cuda.memory_allocated()
    _backward(nets, _half(inputs, 1, B), 0.5)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - mem0
    assert [g.data_ptr() for g in _buffers(nets)] == bufs         # every .grad still a slice of the first buffers
    smallest = min(net.backbone._store.total for net in nets[:2]) * 4
    assert grown < smallest, (grown, smallest)


def test_app_main_accum_iter_train_save_resume(tmp_path):
    from app.scaffold import main as app_main
    from jepa_b200 import _lib
    from test_gpu_train_entry import _cfg, _rows
    lib = _lib.load()
    cfg = _cfg(tmp_path, epochs=1, load=False)
    cfg["optimization"]["accum_iter"] = 2
    n0 = lib.vj_launch_count()
    app_main("vjepa", cfg)
    assert lib.vj_launch_count() - n0 > 600
    body = [r for r in _rows(tmp_path) if r and r[0] != "epoch"]
    assert [r[:2] for r in body] == [["1", "0"], ["1", "1"], ["1", "2"]]       # one row per optimizer step
    assert all(0.1 < float(r[2]) < 3.0 for r in body), body
    ck = torch.load(os.path.join(tmp_path, "jepa-latest.pth.tar"), map_location="cpu")
    assert ck["accum_iter"] == 2 and ck["batch_size"] == 2 and ck["epoch"] == 1
    assert float(next(iter(ck["opt"]["state"].values()))["step"]) == 3.0      # AdamW stepped once per 2 micro-batches

    cfg = _cfg(tmp_path, epochs=2, load=True)
    cfg["optimization"]["accum_iter"] = 2
    app_main("vjepa", cfg)
    body = [r for r in _rows(tmp_path) if r and r[0] != "epoch"]
    assert [r[:2] for r in body] == [["1", "0"], ["1", "1"], ["1", "2"], ["2", "0"], ["2", "1"], ["2", "2"]]
    ck2 = torch.load(os.path.join(tmp_path, "jepa-latest.pth.tar"), map_location="cpu")
    assert ck2["epoch"] == 2 and float(next(iter(ck2["opt"]["state"].values()))["step"]) == 6.0
    k = "module.backbone.blocks.1.mlp.fc1.weight"
    assert not torch.equal(ck["encoder"][k], ck2["encoder"][k])
