"""Process-group bootstrap and autograd-aware collectives (src/utils/distributed.py).

One process per GPU, NCCL over NVLink 5 / NVSwitch.  `init_distributed` keeps the reference's
behaviour (early return if a group exists, SLURM variables, port 37123, fall back to (1, 0) on
failure); the backend is NCCL when CUDA is present and gloo otherwise so the host logic can be
exercised on CPU-only machines.
"""
import os
from logging import getLogger

import torch
import torch.distributed as dist

logger = getLogger()


def nccl_pg_options():
    """ProcessGroupNCCL options for the gradient exchange.  The step's GEMM / attention kernels are persistent (one CTA per
    SM); NCCL's copy/reduce CTAs have to squeeze in between them.  VJ_NCCL_MAX_CTAS / VJ_NCCL_MIN_CTAS / VJ_NCCL_CGA bound
    how many SMs a collective may occupy (ncclConfig_t maxCTAs / minCTAs / cgaClusterSize); unset = NCCL's defaults."""
    if not (torch.cuda.is_available() and dist.is_nccl_available()):
        return None
    keys = {"VJ_NCCL_MAX_CTAS": "max_ctas", "VJ_NCCL_MIN_CTAS": "min_ctas", "VJ_NCCL_CGA": "cga_cluster_size"}
    if not any(k in os.environ for k in keys):
        return None
    opts = dist.ProcessGroupNCCL.Options()
    for env, attr in keys.items():
        if env in os.environ:
            setattr(opts.config, attr, int(os.environ[env]))
    return opts


def _active():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def init_distributed(port=37123, rank_and_world_size=(None, None)):
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    rank, world_size = rank_and_world_size
    os.environ.setdefault('MASTER_ADDR', 'localhost')
    if (rank is None) or (world_size is None):
        try:
            world_size = int(os.environ['SLURM_NTASKS'])
            rank = int(os.environ['SLURM_PROCID'])
            os.environ['MASTER_ADDR'] = os.environ['HOSTNAME']
        except Exception:
            logger.info('SLURM vars not set (distributed training not available)')
            return 1, 0
    try:
        os.environ['MASTER_PORT'] = str(port)
        backend = 'nccl' if torch.cuda.is_available() else 'gloo'
        dist.init_process_group(backend=backend, world_size=world_size, rank=rank,
                                pg_options=nccl_pg_options() if backend == 'nccl' else None)
    except Exception as e:
        world_size, rank = 1, 0
        logger.info(f'Rank: {rank}. Distributed training not available {e}')
    return world_size, rank


class AllGather(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        if _active():
            x = x.contiguous()
            parts = [torch.zeros_like(x) for _ in range(dist.get_world_size())]
            dist.all_gather(parts, x)
            return torch.cat(parts, 0)
        return x

    @staticmethod
    def backward(ctx, grads):
        if _active():
            per = grads.shape[0] // dist.get_world_size()
            grads = grads.contiguous()
            dist.all_reduce(grads)
            return grads[per * dist.get_rank(): per * (dist.get_rank() + 1)]
        return grads


class AllReduceSum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        if _active():
            x = x.contiguous()
            dist.all_reduce(x)
        return x

    @staticmethod
    def backward(ctx, grads):
        return grads


class AllReduce(torch.autograd.Function):
    """Average across ranks; identity gradient."""

    @staticmethod
    def forward(ctx, x):
        if _active():
            x = x.contiguous() / dist.get_world_size()
            dist.all_reduce(x)
        return x

    @staticmethod
    def backward(ctx, grads):
        return grads


# -------------------------------------------------------------------------------------------------
# Data-parallel gradient exchange over the flat gradient buffers
# -------------------------------------------------------------------------------------------------
_pending = []           # NCCL work handles of all-reduces issued during the current backward pass
_callback_queued = [False]
_SM_RESERVE = int(os.environ.get("VJ_SM_RESERVE", "0"))   # SMs left to NCCL while gradient buckets are in flight


def _set_sm_reserve(on):
    """Shrink (or restore) the grid of the persistent GEMM / attention kernels by VJ_SM_RESERVE SMs: NCCL's CTAs then
    always find a free SM and a persistent grid never queues behind a resident NCCL CTA (pair with VJ_NCCL_MAX_CTAS)."""
    if _SM_RESERVE <= 0 or not torch.cuda.is_available():
        return
    try:
        from . import _lib
        fn = _lib.load().vj_set_sm_limit
    except Exception:
        return
    n = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    fn(int(max(1, n - _SM_RESERVE)) if on else 0)


def _wait_pending():
    """Make the compute stream wait for every outstanding gradient all-reduce (stream-side wait, no host sync)."""
    _callback_queued[0] = False
    while _pending:
        _pending.pop().wait()
    _set_sm_reserve(False)


class FlatGradSync:
    """Bucketed, asynchronous averaging all-reduce of one FlatParamStore gradient buffer.

    The backward of a network writes its flat fp32 gradient buffer from the END towards the START (parameters are
    laid out in registration order, backward visits them in reverse), so "everything at or above offset `lo` is final"
    is all the engine has to report (`ready_down_to`).  Each time at least `bucket_bytes` have become final that suffix
    slice is all-reduced in place on NCCL's stream while the compute stream goes on with the earlier layers; the
    compute stream waits for the handles once, in an end-of-backward callback.  No bucket copies: the optimiser reads
    the same buffer (torch DDP's role in app/vjepa/train.py:193-195 of the reference).
    """

    def __init__(self, process_group=None, bucket_bytes=96 << 20):
        self.group = process_group
        self.bucket_elems = max(1, bucket_bytes // 4)
        self.gflat = None
        self.hi = 0         # everything in [hi, total) has been handed to NCCL already
        self.lo = 0         # everything in [lo, hi) is final but not yet sent
        self.n_calls = 0    # all-reduces issued for the current buffer (tests / launch accounting)

    def begin(self, gflat):
        # a backward that raised after queueing its end-of-backward callback would leave the flag set and make every
        # later backward skip the stream wait; re-arming here costs at most one redundant (idempotent) callback
        _callback_queued[0] = False
        _set_sm_reserve(True)
        self.gflat = gflat
        self.hi = self.lo = gflat.numel()
        self.n_calls = 0

    def _issue(self, lo, hi):
        if hi <= lo:
            return
        world = dist.get_world_size(self.group)
        chunk = self.gflat[lo:hi]
        if dist.get_backend(self.group) == 'nccl':
            work = dist.all_reduce(chunk, op=dist.ReduceOp.AVG, group=self.group, async_op=True)
        else:  # gloo (CPU tests): no AVG
            chunk.div_(world)
            work = dist.all_reduce(chunk, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
        self.n_calls += 1
        _pending.append(work)
        if not _callback_queued[0]:
            try:
                torch.autograd.Variable._execution_engine.queue_callback(_wait_pending)
                _callback_queued[0] = True
            except RuntimeError:    # not inside a backward pass: caller must use finish(wait=True)
                pass

    def ready_down_to(self, lo):
        """Gradients at flat offsets >= lo are final."""
        if self.gflat is None or lo >= self.lo:
            return
        self.lo = lo
        if self.hi - self.lo >= self.bucket_elems:
            self._issue(self.lo, self.hi)
            self.hi = self.lo

    def finish(self, wait=False):
        """The whole buffer is final: send what is left; optionally wait right here instead of at end of backward."""
        if self.gflat is None:
            return
        self._issue(0, self.hi)
        self.hi = self.lo = 0
        self.gflat = None
        if wait or not _callback_queued[0]:
            _wait_pending()


class ProbeGradSync:
    """Gradient exchange of a trainable attentive probe (jepa_b200.pooler): ONE averaging all-reduce of the probe's whole
    flat fp32 gradient buffer per backward pass, issued from an end-of-backward callback.  The probe's backward writes
    that buffer in one piece (no per-layer readiness to overlap with), and several probe calls of one step (one per
    temporal segment without attend_across_segments) add into the same buffer first, so they are exchanged once."""

    def __init__(self, process_group=None):
        self.group = process_group
        self.gflat = None
        self.n_calls = 0    # all-reduces issued (tests)

    def mark(self, gflat):
        """Called by every probe backward with the buffer it accumulated into.  Each call queues an end-of-backward
        callback; the first one to run exchanges the buffer and the others find nothing left to do, so a pass issues
        exactly one all-reduce (and a backward that raised part-way leaves nothing armed for the next one)."""
        self.gflat = gflat
        torch.autograd.Variable._execution_engine.queue_callback(self._exchange)

    def _exchange(self):
        g, self.gflat = self.gflat, None
        if g is None or not _active():
            return
        if dist.get_backend(self.group) == 'nccl':
            dist.all_reduce(g, op=dist.ReduceOp.AVG, group=self.group)
        else:  # gloo (CPU tests): no AVG
            g.div_(dist.get_world_size(self.group))
            dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group)
        self.n_calls += 1


class DistributedDataParallel(torch.nn.Module):
    """Data-parallel wrapper with torch DDP's surface (`.module`, `module.`-prefixed state dict, forward passthrough,
    parameters broadcast from rank 0 at construction) whose gradient exchange is FlatGradSync on the flat gradient
    buffers instead of reducer buckets (encoder / predictor), or ProbeGradSync for an attentive probe (a module with a
    flat store but no layer-stack spec).  Frozen modules (the target encoder) only get the broadcast."""

    def __init__(self, module, device_ids=None, static_graph=False, process_group=None, bucket_cap_mb=96, **_ignored):
        super().__init__()
        self.module = module
        self.process_group = process_group
        if _active():
            with torch.no_grad():
                for t in list(module.parameters()) + list(module.buffers()):
                    dist.broadcast(t.data, 0, group=process_group)
            if any(p.requires_grad for p in module.parameters()):
                probe_sync = None
                for m in module.modules():
                    if hasattr(m, '_store') and hasattr(m, '_spec'):
                        m._vj_grad_sync = FlatGradSync(process_group, bucket_cap_mb << 20)
                    elif hasattr(m, '_store'):
                        # a classifier and its pooler share one store (and one buffer): one exchange object for both
                        probe_sync = probe_sync or ProbeGradSync(process_group)
                        m._vj_probe_sync = probe_sync

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def no_sync(self):
        """torch DDP's gradient-accumulation context is NOT supported: every backward writes a fresh flat gradient buffer
        and all-reduces it in place while the backward is still running, so a second backward before zero_grad() would
        accumulate into partially reduced data.  The reference never accumulates (app/vjepa/train.py:462-483)."""
        raise NotImplementedError("jepa_b200 DistributedDataParallel: gradient accumulation / no_sync() is not supported")
