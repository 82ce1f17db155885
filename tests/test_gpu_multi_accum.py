"""2-GPU NCCL test of gradient accumulation under data parallel (skipped on a 1-GPU box; `pytest
tests/test_gpu_multi_accum.py -m gpu` on a 2-GPU one): two micro-batches per rank, the first under no_sync(); the
exchanged buffer is the rank mean of the per-rank accumulated sums, only the last backward all-reduces, replicas stay
bitwise equal over accumulated AdamW steps, and an inf in one micro-batch of one rank skips the step everywhere."""
import copy
import os

import pytest
import torch

from test_gpu_multi import _free_port

pytestmark = pytest.mark.gpu


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
    from app.vjepa.utils import init_opt
    from jepa_b200 import step as vj
    from jepa_b200.distributed import DistributedDataParallel
    from jepa_b200.models import MultiMaskWrapper, PredictorMultiMaskWrapper
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    device = torch.device("cuda", rank)
    torch.cuda.set_device(device)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
    enc, pred, s_enc, s_pred, s_tgt, _, _ = build_states(depth_limit=2)
    enc.load_state_dict(s_enc, strict=False)
    pred.load_state_dict(s_pred, strict=False)
    tgt = copy.deepcopy(enc)
    tgt.load_state_dict(s_tgt, strict=False)
    enc, pred, tgt = MultiMaskWrapper(enc).to(device), PredictorMultiMaskWrapper(pred).to(device), MultiMaskWrapper(tgt).to(device)
    for p in tgt.parameters():
        p.requires_grad = False
    B = C1["batch"]
    me, mp = c1_masks(B)
    me, mp = [m.to(device) for m in me], [m.to(device) for m in mp]
    micro = [synth_clips(B, C1["num_frames"], C1["crop_size"], C1["crop_size"], seed=100 + 10 * rank + i).to(device)
             for i in range(2)]
    nets = [enc, pred]

    def backward(e, p, t, clips):
        h = vj.forward_target(t, clips, mp)
        (vj.jepa_loss(p(e(clips, me), h, me, mp), h) / 2).backward()

    def flat_grads():
        return torch.cat([q.grad.reshape(-1) for n in nets for q in n.parameters() if q.grad is not None]).clone()

    # (1) local accumulated sum, no exchange, and its rank mean
    for clips in micro:
        backward(enc, pred, tgt, clips)
    want = flat_grads()
    dist.all_reduce(want, op=dist.ReduceOp.AVG)
    for n in nets:
        n.zero_grad(set_to_none=True)

    # (2) the same two micro-batches through the wrappers: only the last backward exchanges
    d_enc = DistributedDataParallel(enc, static_graph=True, bucket_cap_mb=4)
    d_pred = DistributedDataParallel(pred, static_graph=True, bucket_cap_mb=1)
    d_tgt = DistributedDataParallel(tgt)
    syncs = [m._vj_grad_sync for n in nets for m in n.modules() if hasattr(m, "_vj_grad_sync")]
    with d_enc.no_sync(), d_pred.no_sync():
        backward(d_enc, d_pred, d_tgt, micro[0])
    calls_first = [s.n_calls for s in syncs]
    backward(d_enc, d_pred, d_tgt, micro[1])
    torch.cuda.synchronize()
    calls_last = [s.n_calls for s in syncs]
    got = flat_grads()
    err = float((got - want).norm() / want.norm())
    for n in nets:
        n.zero_grad(set_to_none=True)

    # (3) accumulated AdamW steps: replicas stay bitwise equal; an inf in one micro-batch of rank 1 skips the step
    opt, scaler, sch, wds = init_opt(enc, pred, iterations_per_epoch=10, start_lr=1e-4, ref_lr=1e-3, warmup=1,
                                     num_epochs=1, wd=0.04, final_wd=0.4, mixed_precision=True)
    skipped = None
    for it in range(4):
        sch.step(); wds.step()
        for i, clips in enumerate(micro):
            if i == 0:
                with d_enc.no_sync(), d_pred.no_sync():
                    h = vj.forward_target(d_tgt, clips, mp)
                    scaler.scale(vj.jepa_loss(d_pred(d_enc(clips, me), h, me, mp), h) / 2).backward()
                if it == 2 and rank == 1:      # a host-side write into this rank's accumulating gradient buffer
                    enc.backbone.blocks[0].mlp.fc1.weight.grad[3, 5] = float("inf")
            else:
                h = vj.forward_target(d_tgt, clips, mp)
                scaler.scale(vj.jepa_loss(d_pred(d_enc(clips, me), h, me, mp), h) / 2).backward()
        scale_before = float(scaler.get_scale())
        before = torch.cat([p.detach().reshape(-1) for p in enc.parameters()]).clone() if it == 2 else None
        scaler.unscale_(opt)
        scaler.step(opt)
        scaler.update()
        opt.zero_grad()
        vj.ema_update(d_enc, d_tgt, 0.998)
        if it == 2:
            after = torch.cat([p.detach().reshape(-1) for p in enc.parameters()])
            skipped = (bool(torch.equal(before, after)), float(scaler.get_scale()) / scale_before)
    flat = torch.cat([p.detach().reshape(-1).float() for n in (enc, pred, tgt) for p in n.parameters()])
    parts = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(parts, flat)
    same = all(torch.equal(parts[0], p) for p in parts[1:])
    q.put((rank, err, calls_first, calls_last, skipped, same))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_accumulation_under_data_parallel_two_gpus():
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = []
    for _ in range(world):
        r = q.get(timeout=300)
        assert r[1] != "error", r[2]
        res.append(r)
    res.sort()
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, err, calls_first, calls_last, skipped, same in res:
        # wgrads are TMA reduce-adds into fp32 (summation order varies run to run): not bit-exact
        assert err < 1e-5, (rank, err)
        assert len(calls_first) == 2 and calls_first == [0, 0], calls_first        # no_sync: nothing exchanged
        assert all(n >= 2 for n in calls_last), calls_last                         # last backward: the bucket schedule
        assert skipped == (True, 0.5), skipped     # inf on one rank only: step skipped on every rank, scale halved
        assert same, rank
