"""2-GPU NCCL test of data-parallel training of a DEEPER probe (skipped on a 1-GPU box; `pytest
tests/test_gpu_multi_probe_depth.py -m gpu` on a 2-GPU one): AttentiveClassifier(depth=3) in
src.utils.distributed.DistributedDataParallel.  The two Blocks' parameters are members of the flat gradient buffer the
probe's single all-reduce averages: in a step with two classifier calls every gradient - each blocks.* one included - is
the mean of the per-rank gradients, and after several FlatAdamW steps on per-rank data the classifier weights are bitwise
identical on both ranks."""
import os

import pytest
import torch

from test_gpu_multi import _free_port

pytestmark = pytest.mark.gpu
CE = torch.nn.CrossEntropyLoss()
DEPTH = 3


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
    from jepa_b200.optim import FlatAdamW
    from jepa_b200.pooler import AttentiveClassifier
    from src.utils.distributed import DistributedDataParallel
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    device = torch.device("cuda", rank)
    torch.cuda.set_device(device)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
    torch.manual_seed(0)
    clf = AttentiveClassifier(embed_dim=256, num_heads=4, depth=DEPTH, num_classes=7).to(device).train()
    g = torch.Generator().manual_seed(100 + rank)                  # different data on every rank
    B, S = 4, 96

    def batch():
        xs = [torch.randn(B, S, 256, generator=g).to(device, torch.bfloat16) for _ in range(2)]
        return xs, torch.randint(0, 7, (B,), generator=g).to(device)

    xs, labels = batch()
    # (1) local gradient of a step with two classifier calls, no exchange
    _grads(clf, xs, labels)
    local = {n: p.grad.clone() for n, p in clf.named_parameters() if p.grad is not None}
    clf.zero_grad(set_to_none=True)
    want = {}
    for n, t in local.items():
        parts = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(parts, t)
        want[n] = sum(parts) / world
    n_block_grads = sum(".blocks." in n for n in want)
    differ = all(not torch.equal(local[n], want[n]) for n in want if ".blocks." in n)

    # (2) the same step through the wrapper: one averaging all-reduce of the flat buffer at the end of the backward
    dclf = DistributedDataParallel(clf, static_graph=True)
    sync = clf._vj_probe_sync
    _grads(dclf, xs, labels)
    torch.cuda.synchronize()
    n_calls = sync.n_calls
    got = {n: p.grad for n, p in clf.named_parameters() if p.grad is not None}
    assert set(got) == set(want)
    worst = max(float((got[n] - want[n]).abs().max() / (want[n].abs().max() + 1e-20)) for n in want)
    dclf.zero_grad(set_to_none=True)

    # (3) several optimizer steps on per-rank data: the replicas stay bitwise identical
    opt = FlatAdamW([{"params": list(clf.parameters())}], lr=1e-3, weight_decay=0.01)
    for i in range(4):
        xs, labels = batch()
        _grads(dclf, xs[:1] if i % 2 else xs, labels)
        opt.step()
        opt.zero_grad()
    flat = torch.cat([p.detach().reshape(-1).float() for p in clf.parameters()])
    parts = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(parts, flat)
    same = all(torch.equal(parts[0], p) for p in parts[1:])
    q.put((rank, worst, n_calls, sync.n_calls, same, n_block_grads, differ))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_deep_probe_grad_sync_nccl_two_gpus():
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
    for rank, worst, n_first, n_total, same, n_block_grads, differ in res:
        assert n_block_grads == 12 * (DEPTH - 1), n_block_grads   # norm1 2, qkv 2, proj 2, norm2 2, fc1 2, fc2 2
        assert differ, rank                          # per-rank data: the local Block gradients are not the mean
        assert worst < 1e-6, (rank, worst)           # mean of two fp32 buffers: NCCL AVG vs (a + b) / 2
        assert n_first == 1, n_first                 # two classifier calls, one exchange
        assert n_total == 5, n_total                 # one per backward
        assert same, rank
