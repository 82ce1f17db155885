"""2-GPU NCCL test of data-parallel multi-head probe training (skipped on a 1-GPU box; `pytest
tests/test_gpu_multi_multihead.py -m gpu` on a 2-GPU one), as tests/test_gpu_multi_probe.py checks one probe: three
heads built as the evaluation drivers build them (build_heads, one src.utils.distributed.DistributedDataParallel each)
see the same per-rank batch; each head's gradient is replaced by the mean of the per-rank gradients through its own
all-reduce, and after several FlatAdamW steps with per-head learning rates every head is bitwise identical on both ranks
while the heads differ from each other."""
import os

import pytest
import torch

from test_gpu_multi import _free_port

pytestmark = pytest.mark.gpu
CE = torch.nn.CrossEntropyLoss()
LRS = (1e-3, 3e-3, 0.0)


def _worker(rank, world, port, q):
    try:
        _worker_body(rank, world, port, q)
    except Exception:       # surface the failure in the parent instead of letting it wait for the queue
        import traceback
        q.put((rank, "error", traceback.format_exc()))


def _grads(clf, xs, labels):
    loss = sum(CE(clf(x), labels) for x in xs) / len(xs)
    loss.backward()


def _worker_body(rank, world, port, q):
    import torch.distributed as dist
    from evals.video_classification_frozen.eval import build_heads
    from jepa_b200.distributed import DistributedDataParallel
    from jepa_b200.optim import FlatAdamW
    from jepa_b200.pooler import AttentiveClassifier
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    device = torch.device("cuda", rank)
    torch.cuda.set_device(device)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
    torch.manual_seed(0)
    clfs = build_heads(lambda: AttentiveClassifier(embed_dim=256, num_heads=4, depth=1, num_classes=7).to(device).train(),
                       len(LRS))
    g = torch.Generator().manual_seed(100 + rank)                  # different data on every rank
    B, S = 4, 96

    def batch():
        xs = [torch.randn(B, S, 256, generator=g).to(device, torch.bfloat16) for _ in range(2)]
        return xs, torch.randint(0, 7, (B,), generator=g).to(device)

    xs, labels = batch()
    # (1) every head's local gradient of a step with two classifier calls, no exchange
    want = []
    for clf in clfs:
        _grads(clf, xs, labels)
        local = {n: p.grad.clone() for n, p in clf.named_parameters() if p.grad is not None}
        clf.zero_grad(set_to_none=True)
        mean = {}
        for n, t in local.items():
            parts = [torch.empty_like(t) for _ in range(world)]
            dist.all_gather(parts, t)
            mean[n] = sum(parts) / world
        want.append(mean)

    # (2) the same step through one wrapper per head: one averaging all-reduce per head and backward
    dclfs = [DistributedDataParallel(clf, static_graph=True) for clf in clfs]
    syncs = [clf._vj_probe_sync for clf in clfs]
    worst, n_first = 0.0, []
    for clf, dclf, sync, w in zip(clfs, dclfs, syncs, want):
        _grads(dclf, xs, labels)
        torch.cuda.synchronize()
        n_first.append(sync.n_calls)
        got = {n: p.grad for n, p in clf.named_parameters() if p.grad is not None}
        assert set(got) == set(w)
        worst = max([worst] + [float((got[n] - w[n]).abs().max() / (w[n].abs().max() + 1e-20)) for n in w])
        dclf.zero_grad(set_to_none=True)

    # (3) several optimizer steps per head on per-rank data: the replicas stay bitwise identical, the heads differ
    opts = [FlatAdamW([{"params": list(clf.parameters())}], lr=lr, weight_decay=0.01) for clf, lr in zip(clfs, LRS)]
    for i in range(4):
        xs, labels = batch()
        for dclf, opt in zip(dclfs, opts):
            _grads(dclf, xs[:1] if i % 2 else xs, labels)
            opt.step()
            opt.zero_grad()
    same, flats = [], []
    for clf in clfs:
        flat = torch.cat([p.detach().reshape(-1).float() for p in clf.parameters()])
        parts = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(parts, flat)
        same.append(all(torch.equal(parts[0], p) for p in parts[1:]))
        flats.append(flat)
    distinct = not torch.equal(flats[0], flats[1]) and not torch.equal(flats[1], flats[2])
    q.put((rank, worst, n_first, [s.n_calls for s in syncs], same, distinct))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_multihead_grad_sync_nccl_two_gpus():
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
    for rank, worst, n_first, n_total, same, distinct in res:
        assert worst < 1e-6, (rank, worst)           # mean of two fp32 buffers: NCCL AVG vs (a + b) / 2
        assert n_first == [1, 1, 1], n_first         # each head: two classifier calls, one exchange
        assert n_total == [5, 5, 5], n_total         # each head: one per backward
        assert all(same), (rank, same)
        assert distinct, rank
