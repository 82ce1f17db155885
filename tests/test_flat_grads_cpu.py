"""Pin which kernel entry points the flat-gradient consumers launch: the GradScaler unscale hook, grad_logger,
clip_grad_norm_ and the optimizer step, on CPU tensors with every entry point replaced by a recorder.  A network whose
gradients are slices of its FlatParamStore's one flat buffer takes one launch per consumer, the per-tensor sums of
squares of the unscale pass are reused until the buffer changes, and a gradient outside the buffer turns every consumer
onto its per-tensor fallback.  No numerics are checked here (the kernels' outputs are never written)."""
import weakref

import pytest
import torch
import torch.nn as nn


@pytest.fixture()
def calls(monkeypatch):
    from jepa_b200 import _lib, params
    rec = []

    def fake_call(name, *args):
        rec.append(name)
        return 0

    class FakeLib:
        @staticmethod
        def vj_layernorm_bwd_workspace(T, D):
            return 4 * D * 4 * 2

        @staticmethod
        def vj_cross_attn_bwd_workspace(B, nq, S, H, hd):
            return 1 << 20

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(_lib, "load", lambda: FakeLib)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: type("S", (), {"cuda_stream": 0})())

    def adopt(self, module):
        # FlatParamStore.adopt without its CUDA-only check
        named = [(n, p) for n, p in module.named_parameters()]
        if self._aliases(named):
            return self
        off, offsets = 0, {}
        for n, p in named:
            offsets[n] = (off, p.numel(), tuple(p.shape))
            off += (p.numel() + params.ALIGN - 1) // params.ALIGN * params.ALIGN
        flat = torch.zeros(off)
        with torch.no_grad():
            for n, p in named:
                o, cnt, shape = offsets[n]
                v = flat[o:o + cnt].view(shape)
                v.copy_(p.data)
                p.data = v
                p._vj_store, p._vj_name = self, n
        self.flat, self.offsets, self.total, self._params = flat, offsets, off, named
        self.shadow = torch.empty(off, dtype=torch.bfloat16)
        self._shadow_fresh = self._shadow_complete = False
        self._seg = None
        return self

    monkeypatch.setattr(params.FlatParamStore, "adopt", adopt)
    with torch.random.fork_rng(devices=[]):      # the tests seed and draw: leave the global generator as it was
        yield rec


def _linear_stack():
    """Two linear layers in a store, their gradients slices of one new flat buffer (what the backbones' backward does)."""
    from jepa_b200.params import FlatParamStore
    torch.manual_seed(0)
    net = nn.Sequential(nn.Linear(8, 16), nn.Linear(16, 4))
    store = FlatParamStore().adopt(net)
    gflat = store.new_grad_buffer()
    for n, p in net.named_parameters():
        p.grad = store.grad_view(gflat, n)
        p.grad.normal_()
    return net, store


def _scaler_args():
    return torch.ones(1), torch.zeros(1)


def _grad_bases(module):
    return {p.grad.data_ptr() - 4 * p._vj_store.offsets[p._vj_name][0] for p in module.parameters() if p.grad is not None}


def test_linear_stack_one_launch_per_consumer(calls):
    from jepa_b200.logging_utils import grad_logger
    from jepa_b200.optim import FlatAdamW
    from jepa_b200.step import clip_grad_norm_
    net, _ = _linear_stack()
    opt = FlatAdamW(net.parameters(), lr=1e-3)
    assert opt.unscale_flat_(*_scaler_args()) == []
    assert calls == ["vj_grad_unscale_stats"]
    grad_logger(net.named_parameters())                      # the unscale pass's sums are current
    assert calls == ["vj_grad_unscale_stats"]
    clip_grad_norm_(net, 1.0)
    assert calls[1:] == ["vj_clip_coef", "vj_scale_flat"]
    grad_logger(net.named_parameters())                      # clipping changed the buffer: one stats pass
    assert calls[3:] == ["vj_grad_unscale_stats"]
    opt.step()
    assert calls[4:] == ["vj_adamw_flat"]
    buf = weakref.ref(net[0].weight.grad._base)
    opt.zero_grad(set_to_none=True)                          # the cached statistics keep no gradient buffer alive
    assert buf() is None


def test_probe_backward_accumulates_into_one_buffer(calls):
    from jepa_b200.logging_utils import grad_logger
    from jepa_b200.optim import FlatAdamW
    from jepa_b200.pooler import AttentiveClassifier
    torch.manual_seed(0)
    clf = AttentiveClassifier(embed_dim=64, num_heads=2, num_classes=10)
    x = torch.zeros(2, 16, 64, dtype=torch.bfloat16)
    clf(x).sum().backward()
    proj = clf.pooler.cross_attention_block.xattn.proj
    for n, p in clf.named_parameters():
        assert (p.grad is None) == (".proj." in n), n
    bases = _grad_bases(clf)
    assert len(bases) == 1
    opt = FlatAdamW(clf.parameters(), lr=1e-3)
    del calls[:]
    assert opt.unscale_flat_(*_scaler_args()) == []
    grad_logger(clf.named_parameters())
    assert calls == ["vj_grad_unscale_stats"]
    clf(x).sum().backward()                                  # a second probe call of the same step
    assert _grad_bases(clf) == bases and proj.weight.grad is None
    del calls[:]
    grad_logger(clf.named_parameters())
    assert calls == ["vj_grad_unscale_stats"]


@pytest.mark.parametrize("kind", ["own", "bf16", "strided"])
def test_gradient_outside_the_buffer_falls_back(calls, kind):
    from jepa_b200.logging_utils import grad_logger
    from jepa_b200.optim import FlatAdamW
    from jepa_b200.step import clip_grad_norm_
    net, _ = _linear_stack()
    w = net[0].weight
    if kind == "own":
        w.grad = w.grad.clone()
    elif kind == "bf16":
        w.grad.data = w.grad.data.to(torch.bfloat16)
    else:
        w.grad = w.grad.t().contiguous().t()
    assert (w.grad.dtype == torch.float32) == (kind != "bf16") and w.grad.is_contiguous() == (kind != "strided")
    opt = FlatAdamW(net.parameters(), lr=1e-3)
    assert opt.unscale_flat_(*_scaler_args()) == list(net.parameters())
    grad_logger(net.named_parameters())
    assert calls == []
    opt.step()
    assert calls == ["vj_adamw_step"] * 4
    before = [p.grad.clone() for p in net.parameters()]
    total = clip_grad_norm_(net, 1e-3)                       # torch's clip_grad_norm_: no entry point, clipped in place
    assert calls == ["vj_adamw_step"] * 4
    ref = torch.nn.utils.get_total_norm(before)
    assert torch.allclose(total, ref)
    for b, p in zip(before, net.parameters()):
        assert torch.allclose(p.grad.float(), (b.float() * 1e-3 / (float(ref) + 1e-6)).to(b.dtype).float(), rtol=1e-2)


def test_lone_gradient_outside_a_buffer_is_not_one(calls):
    """A store whose only gradient is a tensor of its own: that gradient agrees with itself on a buffer address, but no
    [total] buffer starts there, so no kernel may be launched on it."""
    from jepa_b200.optim import FlatAdamW
    net, store = _linear_stack()
    for p in net.parameters():
        p.grad = None
    w = net[1].weight
    w.grad = torch.randn(w.shape)
    assert FlatAdamW(net.parameters(), lr=1e-3).unscale_flat_(*_scaler_args()) == [w] and calls == []
    assert store.grad_buffer(net.parameters()) is None
