"""Training the attentive probe on the GPU (-m gpu): gradients of jepa_b200.pooler against the reference's own
(tests/golden/golden_pooler_grad.pt) and against fp64 autograd on the oracle at encoder sizes; determinism; several probe
calls per step; FlatAdamW / FlatGradScaler / clip_grad_norm_ on a probe with a class count that is not a multiple of 4;
and the frozen evaluation's training loop (evals/video_classification_frozen/eval.py:317-373) end to end.
Tolerances are DESIGN section 5's: activations rel-L2 <= 2e-2, gradients <= 3e-2, loss +- 3e-3."""
import copy
import io
import os
import subprocess

import pytest
import torch

from parity_util import TOL_ACT, TOL_GRAD, TOL_LOSS, rel_l2
from test_oracle_cpu import _build_probe, _pooler_fixture
from test_probe_grad_cpu import _grad_fixture, oracle_grads

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CE = torch.nn.CrossEntropyLoss()


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from jepa_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


def bf(t):
    return t.to(torch.bfloat16).float()


def test_native_xattn_binary(dev):
    exe = os.path.join(ROOT, "tests", "native", "test_xattn")
    assert os.path.exists(exe), "run __graft_entry__.build() first"
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "ALL PASSED" in out.stdout, out.stdout[-3000:] + out.stderr[-1000:]


def _train_step_grads(clf, x, labels):
    clf.zero_grad(set_to_none=True)
    logits = clf(x)
    logits.retain_grad()
    loss = CE(logits, labels)
    loss.backward()
    return float(loss.detach()), logits, {n: p.grad for n, p in clf.named_parameters()}


def test_probe_gradients_vs_reference_fixture(dev):
    """hd 64 / 32 / 80 / 128, complete_block on and off: loss, dlogits and every parameter's gradient (proj: None)."""
    for case, gcase in zip(_pooler_fixture()["cases"], _grad_fixture()["cases"]):
        clf = _build_probe(case).to(dev).train()
        x = case["x"].to(dev, torch.bfloat16)
        loss, logits, grads = _train_step_grads(clf, x, gcase["labels"].to(dev))
        cfg = case["cfg"]
        assert abs(loss - gcase["loss"]) < TOL_LOSS, cfg
        assert rel_l2(logits.detach().float().cpu(), gcase["logits"]) < TOL_ACT, cfg
        assert rel_l2(logits.grad.float().cpu(), gcase["dlogits"]) < TOL_GRAD, cfg
        for n, ref in gcase["grads"].items():
            if ref is None:
                assert grads[n] is None, n
                continue
            g = grads[n].float().reshape(-1).cpu()
            assert abs(float(g.norm()) - ref["norm"]) <= TOL_GRAD * ref["norm"], (cfg, n)
            assert rel_l2(g[ref["idx"]], ref["val"]) < TOL_GRAD, (cfg, n)


def _sharpened_classifier(D, H, C, seed, query=20.0, qk=6.0):
    """Perturbed away from the init, with the attention sharpened (the init scale 0.02 gives an almost uniform softmax)."""
    from jepa_b200.pooler import AttentiveClassifier
    torch.manual_seed(seed)
    clf = AttentiveClassifier(embed_dim=D, num_heads=H, depth=1, num_classes=C)
    with torch.no_grad():
        for n, p in clf.named_parameters():
            if n.endswith("bias") or "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
        clf.pooler.query_tokens.mul_(query)
        clf.pooler.cross_attention_block.xattn.q.weight.mul_(qk)
        clf.pooler.cross_attention_block.xattn.kv.weight.mul_(qk)
    return clf


@pytest.mark.parametrize("D,H,S,B", [(1024, 16, 1568, 4), (1280, 16, 392, 3), (1280, 16, 4608, 1), (1024, 16, 12544, 2)])
def test_probe_gradients_encoder_sizes_vs_oracle(dev, D, H, S, B):
    """ViT-L (hd 64) / ViT-H (hd 80) widths at real token counts (K400's 8 x 1568 = 12544 included), 400 classes.
    The fp64 oracle runs on the same device (plain torch float64 tensor algebra) to keep the test short.  The attention is
    sharpened less than in the inference test: there the logits reach |z| ~ 10 and the loss of bf16 logits would be
    judged on their rounding rather than on the backward."""
    clf = _sharpened_classifier(D, H, 400, D + S, query=5.0, qk=3.0)
    x = bf(torch.randn(B, S, D, generator=torch.Generator().manual_seed(S)))
    labels = torch.randint(0, 400, (B,), generator=torch.Generator().manual_seed(B))
    S_ = {k: v.double().to(dev) for k, v in clf.state_dict().items()}
    ref_loss, ref_dl, ref_g = oracle_grads(S_, x.double().to(dev), labels.to(dev), H, True)
    clf = clf.to(dev).train()
    loss, logits, grads = _train_step_grads(clf, x.to(dev, torch.bfloat16), labels.to(dev))
    assert abs(loss - ref_loss) < TOL_LOSS
    assert rel_l2(logits.grad.float().cpu(), ref_dl.float().cpu()) < TOL_GRAD
    for n, g in grads.items():
        if ref_g[n] is None:
            assert g is None, n
            continue
        assert rel_l2(g.float().cpu(), ref_g[n].float().cpu()) < TOL_GRAD, n


def test_pooler_three_queries_vs_oracle(dev):
    """AttentivePooler with nq = 3 at K400's token count: pooled activations and every gradient for an upstream gradient."""
    from jepa_b200.pooler import AttentivePooler
    from oracle import vjepa_oracle as O
    D, H, S, B, nq = 1024, 16, 12544, 2, 3
    torch.manual_seed(3)
    pool = AttentivePooler(num_queries=nq, embed_dim=D, num_heads=H, depth=1)
    with torch.no_grad():
        for n, p in pool.named_parameters():
            if n.endswith("bias") or "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
        pool.query_tokens.mul_(20.0)
        pool.cross_attention_block.xattn.q.weight.mul_(6.0)
        pool.cross_attention_block.xattn.kv.weight.mul_(6.0)
    x = bf(torch.randn(B, S, D, generator=torch.Generator().manual_seed(11)))
    dy = torch.randn(B, nq, D, generator=torch.Generator().manual_seed(12))
    S_ = {k: v.double().to(dev).requires_grad_(True) for k, v in pool.state_dict().items()}
    ref = O.attentive_pooler(S_, x.double().to(dev), H, True, pre="")
    (ref * dy.double().to(dev)).sum().backward()
    pool = pool.to(dev).train()
    out = pool(x.to(dev, torch.bfloat16))
    assert out.shape == (B, nq, D) and out.requires_grad
    assert rel_l2(out.detach().float().cpu(), ref.detach().float().cpu()) < TOL_ACT
    (out * dy.to(dev)).sum().backward()
    for n, p in pool.named_parameters():
        if S_[n].grad is None:
            assert p.grad is None, n
            continue
        assert rel_l2(p.grad.float().cpu(), S_[n].grad.float().cpu()) < TOL_GRAD, n


def test_probe_backward_is_deterministic_and_calls_accumulate(dev):
    clf = _sharpened_classifier(1024, 16, 174, 5).to(dev).train()
    g = torch.Generator().manual_seed(5)
    x1 = bf(torch.randn(4, 1568, 1024, generator=g)).to(dev, torch.bfloat16)
    x2 = bf(torch.randn(4, 1568, 1024, generator=g)).to(dev, torch.bfloat16)
    y = torch.tensor([1, 7, 100, 173], device=dev)
    _train_step_grads(clf, x1, y)
    a = {n: None if p.grad is None else p.grad.clone() for n, p in clf.named_parameters()}
    _train_step_grads(clf, x1, y)
    for n, p in clf.named_parameters():
        assert (p.grad is None) == (a[n] is None), n
        if p.grad is None:
            continue
        if p.dim() > 1:      # weights, query tokens: GEMMs with one CTA per output tile and the atomic-free attention
            assert torch.equal(p.grad, a[n]), n
        else:                # biases / LayerNorm affine: the column-sum reductions add row chunks in arrival order
            assert rel_l2(p.grad, a[n]) < 1e-6, n
    _train_step_grads(clf, x2, y)
    b = {n: None if p.grad is None else p.grad.clone() for n, p in clf.named_parameters()}
    # two classifier calls in one step (eval.py: one per temporal segment, losses summed) -> the summed gradient, in ONE
    # flat buffer; the same when the two losses are back-propagated one after the other
    for joint in (True, False):
        clf.zero_grad(set_to_none=True)
        l1, l2 = CE(clf(x1), y), CE(clf(x2), y)
        if joint:
            (l1 + l2).backward()
        else:
            l1.backward()
            l2.backward()
        base = None
        for n, p in clf.named_parameters():
            if a[n] is None:
                assert p.grad is None, n
                continue
            assert rel_l2(p.grad, a[n] + b[n]) < 1e-5, (joint, n)
            off = p._vj_store.offsets[n][0]
            pb = p.grad.data_ptr() - 4 * off
            assert base is None or pb == base, n
            base = pb


def _param_groups(clf):
    # evals/video_classification_frozen/eval.py:534-544
    return [{"params": [p for n, p in clf.named_parameters() if ("bias" not in n) and (len(p.shape) != 1)]},
            {"params": [p for n, p in clf.named_parameters() if ("bias" in n) or (len(p.shape) == 1)],
             "WD_exclude": True, "weight_decay": 0}]


def test_flat_adamw_on_probe_with_174_classes(dev):
    """SSv2's 174 classes: one flat AdamW launch; proj untouched and stateless; same state entries and values as
    torch.optim.AdamW; a checkpoint of classifier + optimizer resumes the run."""
    from jepa_b200 import _lib
    from jepa_b200.optim import FlatAdamW
    from jepa_b200.step import clip_grad_norm_
    clf = _sharpened_classifier(256, 4, 174, 9).to(dev).train()
    ref = copy.deepcopy(clf)
    opt = FlatAdamW(_param_groups(clf), lr=1e-3, weight_decay=0.05)
    ropt = torch.optim.AdamW(_param_groups(ref), lr=1e-3, weight_decay=0.05)
    proj = clf.pooler.cross_attention_block.xattn.proj.weight
    proj0 = proj.detach().clone()
    g = torch.Generator().manual_seed(9)
    xs = [bf(torch.randn(3, 40, 256, generator=g)).to(dev, torch.bfloat16) for _ in range(4)]
    y = torch.tensor([0, 88, 173], device=dev)

    def step(model, o, x):
        o.zero_grad()
        CE(model(x), y).backward()

    for it in range(3):
        step(clf, opt, xs[it])
        for (n, p), (_, q) in zip(clf.named_parameters(), ref.named_parameters()):
            q.grad = None if p.grad is None else p.grad.clone()
        n_clip = clip_grad_norm_(clf, 1.0)                  # one flat pass, proj contributes nothing
        r_clip = torch.nn.utils.clip_grad_norm_(ref.parameters(), 1.0)
        assert abs(float(n_clip) - float(r_clip)) <= 1e-5 * float(r_clip)
        before = _lib.load().vj_launch_count()
        opt.step()
        # the whole probe in one vj_adamw_flat call: the update kernel and its device step counter
        assert _lib.load().vj_launch_count() - before == 2 and len(opt._flat) == 1
        ropt.step()
    assert torch.equal(proj, proj0) and proj not in opt.state
    sd, rsd = opt.state_dict(), ropt.state_dict()
    assert sorted(sd["state"]) == sorted(rsd["state"])
    for k, st in rsd["state"].items():
        assert set(sd["state"][k]) == set(st) and float(sd["state"][k]["step"]) == float(st["step"])
        for m in ("exp_avg", "exp_avg_sq"):
            assert rel_l2(sd["state"][k][m].cpu(), st[m].cpu()) < 1e-4, (k, m)
    for (n, p), (_, q) in zip(clf.named_parameters(), ref.named_parameters()):
        assert rel_l2(p.detach().cpu(), q.detach().cpu()) < 1e-5, n
    # checkpoint (eval.py's save_checkpoint keeps 'classifier' and 'opt') -> fresh modules resume to the same numbers
    buf = io.BytesIO()
    torch.save({"classifier": clf.state_dict(), "opt": opt.state_dict()}, buf)
    buf.seek(0)
    ck = torch.load(buf, weights_only=False)
    clf2 = _sharpened_classifier(256, 4, 174, 123).to(dev).train()
    clf2.load_state_dict(ck["classifier"])
    opt2 = FlatAdamW(_param_groups(clf2), lr=1e-3, weight_decay=0.05)
    opt2.load_state_dict(ck["opt"])
    step(clf, opt, xs[3]); opt.step()
    step(clf2, opt2, xs[3]); opt2.step()
    for (n, p), (_, q) in zip(clf.named_parameters(), clf2.named_parameters()):
        assert torch.equal(p, q), n


def test_eval_training_loop_fits_separable_set(dev):
    """The reference's training loop, statement for statement, with our encoder, ClipAggregation, classifier, FlatAdamW
    and FlatGradScaler: two temporal segments per clip without attend_across_segments (two classifier calls per step,
    losses summed), GradScaler, clip to 1.0, warmup-cosine LR and cosine WD schedules.  On a fixed separable set the
    training loss falls and the training accuracy reaches 100 %."""
    import torch.nn.functional as F
    from jepa_b200.models import vit_tiny
    from jepa_b200.optim import FlatAdamW, FlatGradScaler
    from jepa_b200.pooler import AttentiveClassifier, ClipAggregation
    from jepa_b200.schedulers import CosineWDSchedule, WarmupCosineSchedule
    torch.manual_seed(0)
    enc = vit_tiny(img_size=64, patch_size=16, num_frames=4, tubelet_size=2, uniform_power=True).to(dev)
    encoder = ClipAggregation(enc, tubelet_size=2, attend_across_segments=False).eval()
    n_cls, n_per, B = 6, 8, 8
    g = torch.Generator().manual_seed(1)
    protos = torch.randn(n_cls, 3, 4, 64, 64, generator=g)
    data = [(c, protos[c] + 0.5 * torch.randn(2, 3, 4, 64, 64, generator=g)) for c in range(n_cls) for _ in range(n_per)]
    classifier = AttentiveClassifier(embed_dim=enc.embed_dim, num_heads=enc.num_heads, depth=1, num_classes=n_cls).to(dev)
    steps, epochs = 40, 1
    optimizer = FlatAdamW(_param_groups(classifier))
    scheduler = WarmupCosineSchedule(optimizer, warmup_steps=3, start_lr=1e-4, ref_lr=1e-3, final_lr=1e-5, T_max=steps)
    wd_scheduler = CosineWDSchedule(optimizer, ref_wd=0.01, final_wd=0.01, T_max=steps)
    scaler = FlatGradScaler()
    classifier.train()
    losses, accs = [], []
    order = torch.randperm(len(data), generator=g)
    for itr in range(steps * epochs):
        idx = [int(order[(itr * B + i) % len(data)]) for i in range(B)]
        labels = torch.tensor([data[i][0] for i in idx], device=dev)
        clips = [[torch.stack([data[i][1][s] for i in idx]).to(dev)] for s in range(2)]   # 2 segments x 1 view
        scheduler.step()
        wd_scheduler.step()
        with torch.no_grad():
            outputs = encoder(clips)
        outputs = [[classifier(ost) for ost in os] for os in outputs]
        loss = sum([sum([CE(ost, labels) for ost in os]) for os in outputs]) / len(outputs) / len(outputs[0])
        with torch.no_grad():
            probs = sum([sum([F.softmax(ost, dim=1) for ost in os]) for os in outputs]) / len(outputs) / len(outputs[0])
            accs.append(100. * float(probs.max(dim=1).indices.eq(labels).sum()) / B)
        scaler.scale(loss).backward()
        scaler.unscale_(optimizer)
        torch.nn.utils.clip_grad_norm_(classifier.parameters(), 1.0)
        scaler.step(optimizer)
        scaler.update()
        optimizer.zero_grad()
        losses.append(float(loss))
    assert sum(losses[-5:]) / 5 < 0.25 * sum(losses[:3]) / 3, losses
    assert accs[-1] == 100.0 and min(accs[-3:]) == 100.0, accs
    assert classifier.pooler.cross_attention_block.xattn.proj.weight.grad is None
