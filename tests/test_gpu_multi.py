"""2-GPU NCCL test of the data-parallel path (skipped on a 1-GPU box; `pytest tests/test_gpu_multi.py -m gpu` on a 2-GPU one):
the flat-buffer gradient exchange run inside the backward pass must leave on every rank the mean of the per-rank gradients
of the same step computed without any exchange."""
import copy
import os
import socket
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _step(enc, pred, tgt, clips, me, mp):
    from jepa_b200 import step as vj
    h = vj.forward_target(tgt, clips, mp)
    z = pred(enc(clips, me), h, me, mp)
    loss = vj.jepa_loss(z, h)
    loss.backward()
    return float(loss)


def _worker(rank, world, port, q):
    try:
        _worker_body(rank, world, port, q)
    except Exception:       # surface the failure in the parent instead of letting it wait for the queue
        import traceback
        q.put((rank, "error", traceback.format_exc()))


def _worker_body(rank, world, port, q):
    import torch.distributed as dist
    from common import C1, synth_clips
    from parity_util import build_states, c1_masks
    from jepa_b200.distributed import DistributedDataParallel
    from jepa_b200.models import MultiMaskWrapper, PredictorMultiMaskWrapper
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    device = torch.device("cuda", rank)
    torch.cuda.set_device(device)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
    enc, pred, s_enc, s_pred, s_tgt, _, _ = build_states(depth_limit=3)
    enc.load_state_dict(s_enc, strict=False)
    pred.load_state_dict(s_pred, strict=False)
    tgt = copy.deepcopy(enc)
    tgt.load_state_dict(s_tgt, strict=False)
    enc, pred, tgt = MultiMaskWrapper(enc).to(device), PredictorMultiMaskWrapper(pred).to(device), MultiMaskWrapper(tgt).to(device)
    for p in tgt.parameters():
        p.requires_grad = False
    B = C1["batch"]
    clips = synth_clips(B, C1["num_frames"], C1["crop_size"], C1["crop_size"], seed=100 + rank).to(device)
    me, mp = c1_masks(B)
    me, mp = [m.to(device) for m in me], [m.to(device) for m in mp]

    # (1) local gradients, no exchange
    _step(enc, pred, tgt, clips, me, mp)
    local = {("e", n): p.grad.clone() for n, p in enc.named_parameters() if p.grad is not None}
    local.update({("p", n): p.grad.clone() for n, p in pred.named_parameters() if p.grad is not None})
    enc.zero_grad(set_to_none=True)
    pred.zero_grad(set_to_none=True)
    want = {}
    for k, g in local.items():
        parts = [torch.empty_like(g) for _ in range(world)]
        dist.all_gather(parts, g)
        want[k] = sum(parts) / world

    # (2) same step through the data-parallel wrappers, small buckets so several all-reduces overlap the backward
    d_enc = DistributedDataParallel(enc, static_graph=True, bucket_cap_mb=4)
    d_pred = DistributedDataParallel(pred, static_graph=True, bucket_cap_mb=1)
    d_tgt = DistributedDataParallel(tgt)
    _step(d_enc, d_pred, d_tgt, clips, me, mp)
    torch.cuda.synchronize()
    worst, n_calls = 0.0, []
    for m in list(enc.modules()) + list(pred.modules()):
        if hasattr(m, "_vj_grad_sync"):
            n_calls.append(m._vj_grad_sync.n_calls)
    got = {("e", n): p.grad for n, p in enc.named_parameters() if p.grad is not None}
    got.update({("p", n): p.grad for n, p in pred.named_parameters() if p.grad is not None})
    assert set(got) == set(want)
    for k in want:
        err = float((got[k] - want[k]).abs().max() / (want[k].abs().max() + 1e-20))
        worst = max(worst, err)
    q.put((rank, worst, n_calls))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_flat_grad_sync_nccl_two_gpus():
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = []
    for _ in range(world):
        r = q.get(timeout=240)
        assert r[1] != "error", r[2]
        res.append(r)
    res.sort()
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, worst, n_calls in res:
        # wgrads are TMA reduce-adds into fp32 (summation order varies run to run), so not bit-exact: 1e-3 of the max
        assert worst < 1e-3, (rank, worst)
        assert len(n_calls) == 2 and all(n >= 2 for n in n_calls), n_calls
