"""Gradient accumulation on CPU (kernels stubbed, gloo for the collectives): DistributedDataParallel.no_sync() over the
flat-buffer exchanges, backwards that add into the live gradient buffer, and the step / schedule bookkeeping of
`optimization.accum_iter` in app.vjepa.train.main."""
import copy
import csv
import os
from types import SimpleNamespace

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from common import C1
from parity_util import c1_masks
from test_distributed_cpu import _FakeStore, _free_port
import test_dryrun_cpu
from test_dryrun_cpu import dry  # noqa: F401  (pytest fixture)


# ---------------------------------------------------------------------------------------------------------------------
# no_sync() on two gloo ranks
# ---------------------------------------------------------------------------------------------------------------------
class _Net(torch.nn.Module):
    """A layer stack as DistributedDataParallel sees one: a flat store and a spec -> FlatGradSync."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(4))
        self._store, self._spec = _FakeStore(), object()


class _Probe(torch.nn.Module):
    """A store without a layer-stack spec (the attentive probe) -> ProbeGradSync."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(4))
        self._store = object()


class _AddBackward(torch.autograd.Function):
    """Adds `fill`-valued gradients into a flat buffer back to front, the way engine.encoder_backward does, and drives
    the exchange attached to `net` through engine._sync_begin; or marks the buffer for a probe's exchange."""

    @staticmethod
    def forward(ctx, x, net, gflat, fill):
        ctx.args = (net, gflat, fill)
        return x.sum()

    @staticmethod
    def backward(ctx, g):
        from jepa_b200 import engine
        net, gflat, fill = ctx.args
        probe = getattr(net, "_vj_probe_sync", None)
        if probe is not None:
            gflat += fill
            probe.mark(gflat)
            return g.expand(4), None, None, None
        store = net._store
        o = store.offsets["norm.weight"][0]
        gflat[o:] += fill
        sync = engine._sync_begin(net, gflat)
        for i in (2, 1, 0):
            lo = store.offsets[f"blocks.{i}.norm1.weight"][0]
            gflat[lo:lo + 50] += fill * (i + 1)
            if sync is not None:
                sync.ready_down_to(lo)
        gflat[:40] += fill * 10
        if sync is not None:
            sync.finish()
        return g.expand(4), None, None, None


def _backward(net, gflat, fill):
    x = torch.ones(4, requires_grad=True)
    _AddBackward.apply(x, net, gflat, fill).backward()


def _no_sync_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    from jepa_b200 import distributed as D
    D.init_distributed(port=port, rank_and_world_size=(rank, world))
    out = {}
    net, probe = _Net(), _Probe()
    dnet = D.DistributedDataParallel(net, bucket_cap_mb=0)    # the smallest bucket: one all-reduce per block
    dprobe = D.DistributedDataParallel(probe)
    fsync, psync = net._vj_grad_sync, probe._vj_probe_sync
    total = net._store.total
    for name, ddp, sync in (("flat", dnet, fsync), ("probe", dprobe, psync)):
        mod = ddp.module
        gflat = torch.zeros(total)
        with ddp.no_sync():
            with ddp.no_sync():                               # nested
                _backward(mod, gflat, float(rank + 1))
            _backward(mod, gflat, float(rank + 1))
            inside = (sync.n_calls, gflat.clone(), D._callback_queued[0], sync.paused)
        base = sync.n_calls
        _backward(mod, gflat, 3.0 * (rank + 1))
        out[name] = dict(inside_calls=inside[0], inside=inside[1].tolist(), queued=inside[2], paused_inside=inside[3],
                         calls=sync.n_calls - base if name == "probe" else sync.n_calls, result=gflat.tolist())
        # an exception inside the context disarms it: the next backward exchanges again
        try:
            with ddp.no_sync():
                raise KeyError("boom")
        except KeyError:
            pass
        g2 = torch.zeros(total)
        n0 = psync.n_calls
        _backward(mod, g2, float(rank + 1))
        out[name]["after_exc"] = (sync.paused, sync.n_calls - n0 if name == "probe" else sync.n_calls, g2.tolist())
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def _per_rank_sum(store, fill):
    """What _AddBackward adds for `fill`, as a flat tensor."""
    g = torch.zeros(store.total)
    g[store.offsets["norm.weight"][0]:] += fill
    for i in (2, 1, 0):
        lo = store.offsets[f"blocks.{i}.norm1.weight"][0]
        g[lo:lo + 50] += fill * (i + 1)
    g[:40] += fill * 10
    return g


def test_no_sync_two_ranks():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_no_sync_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    store = _FakeStore()
    for name in ("flat", "probe"):
        sums = []
        for rank in range(world):
            r = res[rank][name]
            f = float(rank + 1)
            local = (torch.full((store.total,), 2 * f) if name == "probe" else 2 * _per_rank_sum(store, f))
            assert r["inside_calls"] == 0 and not r["queued"] and r["paused_inside"] == 1, (name, r)   # inner exited
            assert r["inside"] == local.tolist(), name                  # two backwards accumulated, nothing exchanged
            sums.append(local + (torch.full((store.total,), 3 * f) if name == "probe" else _per_rank_sum(store, 3 * f)))
        want = (sums[0] + sums[1]) / world                               # rank mean of the per-rank sums
        for rank in range(world):
            r = res[rank][name]
            # one exchange round, as without accumulation: the probe's one all-reduce, the stack's bucket schedule
            assert r["calls"] == (1 if name == "probe" else 4), (name, r["calls"])      # 4: one bucket per block
            assert r["result"] == want.tolist(), name
            paused, calls, g2 = r["after_exc"]
            assert paused == 0 and calls == r["calls"], (name, paused, calls)
            one = (torch.full((store.total,), 1.0) if name == "probe" else _per_rank_sum(store, 1.0))
            assert g2 == ((one + 2 * one) / world).tolist(), name


# ---------------------------------------------------------------------------------------------------------------------
# backward into the live gradient buffer (kernels stubbed)
# ---------------------------------------------------------------------------------------------------------------------
def _adopt_on_cpu(monkeypatch):
    """test_dryrun_cpu's CPU adoption, plus the parameter -> (store, name) links FlatParamStore.adopt leaves behind
    (grad_buffer reads them to find a live buffer)."""
    from jepa_b200 import params
    test_dryrun_cpu._adopt_on_cpu(monkeypatch)
    cpu_adopt = params.FlatParamStore.adopt

    def adopt(self, module):
        st = cpu_adopt(self, module)
        for n, p in module.named_parameters():
            p._vj_store, p._vj_name = st, n
        return st

    monkeypatch.setattr(params.FlatParamStore, "adopt", adopt)


def _models(monkeypatch):
    _adopt_on_cpu(monkeypatch)
    from app.vjepa.utils import init_video_model
    enc, pred = init_video_model(device=torch.device("cpu"), patch_size=16, num_frames=C1["num_frames"], tubelet_size=2,
                                 model_name="vit_tiny", crop_size=C1["crop_size"], pred_depth=2, pred_embed_dim=384,
                                 uniform_power=True, use_mask_tokens=True, num_mask_tokens=2, use_sdpa=True)
    tgt = copy.deepcopy(enc)
    for p in tgt.parameters():
        p.requires_grad = False
    return enc, pred, tgt


def test_second_backward_adds_into_the_first_buffer(dry, monkeypatch):
    from jepa_b200 import params
    from jepa_b200 import step as vj
    enc, pred, tgt = _models(monkeypatch)
    n_new = []
    orig = params.FlatParamStore.new_grad_buffer

    def counting(self):
        n_new.append(self)
        return orig(self)

    monkeypatch.setattr(params.FlatParamStore, "new_grad_buffer", counting)
    B = 2
    clips = torch.zeros(B, 3, C1["num_frames"], C1["crop_size"], C1["crop_size"])
    me, mp_ = c1_masks(B)
    ptrs = []
    for micro in range(2):
        h = vj.forward_target(tgt, clips, mp_)
        (vj.jepa_loss(pred(enc(clips, me), h, me, mp_), h) / 2).backward()
        ptrs.append({(id(net), n): p.grad.data_ptr() for net in (enc, pred) for n, p in net.named_parameters()
                     if p.requires_grad})
        if micro == 0:
            assert len(n_new) == 2                       # encoder and predictor: one fresh buffer each
    assert len(n_new) == 2, "the second backward allocated a gradient buffer"
    assert ptrs[0] == ptrs[1]                            # every .grad still the slice of the first buffer
    for net in (enc, pred):
        st = net.backbone._store
        g = st.grad_buffer(p for p in net.parameters() if p.requires_grad)
        assert g is not None
        for n, p in net.backbone.named_parameters():
            if p.requires_grad:
                assert p.grad.data_ptr() == g.data_ptr() + 4 * st.offsets[n][0], n
            else:
                assert p.grad is None, n


# ---------------------------------------------------------------------------------------------------------------------
# app.vjepa.train.main with accum_iter, on CPU with every kernel stubbed
# ---------------------------------------------------------------------------------------------------------------------
MASKS = [
    dict(aspect_ratio=[0.75, 1.5], num_blocks=8, spatial_scale=[0.15, 0.15], temporal_scale=[1.0, 1.0],
         max_temporal_keep=1.0, max_keep=None),
    dict(aspect_ratio=[0.75, 1.5], num_blocks=2, spatial_scale=[0.7, 0.7], temporal_scale=[1.0, 1.0],
         max_temporal_keep=1.0, max_keep=None),
]


def _cfg(folder, epochs, load, **opt):
    o = dict(ipe=3, ipe_scale=1.25, clip_grad=10.0, weight_decay=0.04, final_weight_decay=0.4, epochs=epochs, warmup=1,
             start_lr=0.0002, lr=0.000625, final_lr=1e-6, ema=[0.998, 1.0])
    o.update(opt)
    return {
        "meta": dict(load_checkpoint=load, read_checkpoint=None, seed=234, use_sdpa=True, dtype="bfloat16"),
        "mask": MASKS,
        "model": dict(model_name="vit_tiny", pred_depth=2, pred_embed_dim=384, uniform_power=True, use_mask_tokens=True,
                      zero_init_mask_tokens=True),
        "data": dict(dataset_type="synthetic", datasets=[], batch_size=2, num_clips=1, num_frames=8, tubelet_size=2,
                     sampling_rate=4, crop_size=224, patch_size=16, pin_mem=False, num_workers=0),
        "data_aug": dict(auto_augment=False, motion_shift=False, random_resize_aspect_ratio=[0.75, 1.35],
                         random_resize_scale=[0.3, 1.0], reprob=0.0),
        "loss": dict(loss_exp=1.0, reg_coeff=0.0),
        "optimization": o,
        "logging": dict(folder=str(folder), write_tag="jepa"),
    }


class _Loader:
    """The synthetic loader's shape of data: `length` batches, each through the run's mask collator."""

    def __init__(self, collator, batch_size, length, frames, crop):
        self.collator, self.batch_size, self.length = collator, batch_size, length
        self.sample = ([torch.zeros(3, frames, crop, crop)], 0, [0])
        self.drawn = 0

    def __len__(self):
        return self.length

    def __iter__(self):
        for _ in range(self.length):
            self.drawn += 1
            yield self.collator([self.sample] * self.batch_size)


def _dry_main(monkeypatch, cfg):
    """Run app.vjepa.train.main on CPU tensors: device plumbing pointed at the CPU, data from _Loader, checkpoints saved
    synchronously.  Returns counters of what the loop did."""
    import app.vjepa.train as T
    from jepa_b200 import step as vj
    _adopt_on_cpu(monkeypatch)

    class _Torch:
        def __getattr__(self, name):
            return getattr(torch, name)

    tproxy = _Torch()
    tproxy.device = lambda *a: torch.device("cpu")
    tproxy.cuda = SimpleNamespace(is_available=lambda: True, set_device=lambda d: None, max_memory_allocated=lambda: 0)
    monkeypatch.setattr(T, "torch", tproxy)
    rec = SimpleNamespace(sched=0, wd_sched=0, momenta=[], loader=None)

    def init_data(*, batch_size, collator, ipe, crop_size, clip_len, **_):
        rec.loader = _Loader(collator, batch_size, ipe, clip_len, crop_size)
        return rec.loader, SimpleNamespace(set_epoch=lambda e: None)

    real_init_opt = T.init_opt

    def init_opt(**kw):
        opt, scaler, sch, wds = real_init_opt(**kw)
        s0, w0 = sch.step, wds.step

        def sch_step():
            rec.sched += 1
            return s0()

        def wds_step():
            rec.wd_sched += 1
            return w0()

        sch.step, wds.step = sch_step, wds_step
        return opt, scaler, sch, wds

    real_ema = vj.ema_update

    def ema_update(enc, tgt, m):
        rec.momenta.append(m)
        return real_ema(enc, tgt, m)

    class Checkpointer:
        error = None

        def save(self, d, path):
            torch.save(d, path)

        def wait(self):
            pass

    monkeypatch.setattr(T, "init_data", init_data)
    monkeypatch.setattr(T, "init_opt", init_opt)
    monkeypatch.setattr(vj, "ema_update", ema_update)
    monkeypatch.setattr(T, "AsyncCheckpointer", Checkpointer)
    T.main(cfg)
    rec.collator_steps = rec.loader.collator.mask_generators[0]._counter._v.value + 1
    return rec


def _csv(folder):
    with open(os.path.join(folder, "jepa_r0.csv")) as f:
        return [r for r in csv.reader(f) if r and r[0] != "epoch"]


def test_accum_iter_one_is_the_default_loop(dry, monkeypatch, tmp_path):
    runs = []
    for sub, extra in (("absent", {}), ("one", dict(accum_iter=1))):
        dry.clear()
        (tmp_path / sub).mkdir()
        rec = _dry_main(monkeypatch, _cfg(tmp_path / sub, epochs=1, load=False, **extra))
        runs.append((list(dry), rec.sched, list(rec.momenta), rec.collator_steps, len(_csv(tmp_path / sub))))
        assert "accum_iter" not in torch.load(tmp_path / sub / "jepa-latest.pth.tar", weights_only=False)
    assert runs[0][0] and runs[0][0] == runs[1][0]       # the same library calls, in the same order
    assert runs[0][1:] == runs[1][1:] == (3, runs[0][2], 3, 3)


def test_accum_iter_bookkeeping_and_resume(dry, monkeypatch, tmp_path):
    k, ipe, ipe_scale, ema = 2, 3, 1.25, (0.998, 1.0)
    rec = _dry_main(monkeypatch, _cfg(tmp_path, epochs=1, load=False, accum_iter=k))
    # ipe counts optimizer steps: one LR / WD / EMA step each, k loader batches (and collator draws) each
    assert rec.sched == rec.wd_sched == ipe
    assert rec.loader.drawn == ipe * k and rec.collator_steps == ipe * k
    assert rec.momenta == [ema[0] + i * (ema[1] - ema[0]) / (ipe * 1 * ipe_scale) for i in range(ipe)]
    rows = _csv(tmp_path)
    assert [r[:2] for r in rows] == [["1", str(i)] for i in range(ipe)]      # one row per optimizer step
    ck = torch.load(tmp_path / "jepa-latest.pth.tar", weights_only=False)
    assert ck["accum_iter"] == k and ck["batch_size"] == 2 and ck["epoch"] == 1

    # resume into a second epoch: schedules fast-forwarded by start_epoch * ipe, the collator by start_epoch * ipe * k
    rec = _dry_main(monkeypatch, _cfg(tmp_path, epochs=2, load=True, accum_iter=k))
    assert rec.sched == rec.wd_sched == 2 * ipe
    assert rec.collator_steps == 2 * ipe * k and rec.loader.drawn == ipe * k
    assert rec.momenta == [ema[0] + i * (ema[1] - ema[0]) / (ipe * 2 * ipe_scale) for i in range(ipe, 2 * ipe)]
    assert [r[:2] for r in _csv(tmp_path)] == [["1", str(i)] for i in range(ipe)] + [["2", str(i)] for i in range(ipe)]


def test_accum_iter_rejects_bad_values(monkeypatch, tmp_path):
    import pytest

    import app.vjepa.train as T
    for bad in (0, -1, 1.5, "2", True):
        with pytest.raises(ValueError, match="accum_iter"):
            T.main(_cfg(tmp_path, epochs=1, load=False, accum_iter=bad))
