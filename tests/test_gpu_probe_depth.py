"""The attentive probe at depth > 1 on the GPU (-m gpu).

Kernel: vj_query_attn_fwd / _bwd (bf16 and fp16) against fp64 at every head dim and at nq 1, 2, 17, 64 and 128; at
nq = 1 the output is bitwise v and dq = dk = 0 exactly; the backward is bitwise equal over two runs; nq > 128 raises in
the Python wrapper and in the C ABI.  Launches: a depth-1 probe step issues the launches it issued before the Blocks.
Module: AttentivePooler / AttentiveClassifier at depth 2 and 3 (tests/golden/golden_pooler_depth.pt, from the
reference) - output and every parameter gradient against the fixture and the fp64 oracle restatement, in bf16 and under
an fp16 autocast the probe follows; two probe calls of one step add into one flat gradient buffer.
Evaluation: `optimization.probe_depth: 2` trains, saves and resumes end to end."""
import math
import os

import pytest
import torch

from parity_util import rel_l2
from test_gpu_eval import N_ITEMS, _check_run, _eval_cfg, dev, pretrained  # noqa: F401  (fixtures)
from test_probe_depth_cpu import build_case, depth_fixture, oracle_grads

pytestmark = pytest.mark.gpu
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
HEAD_DIMS = (32, 64, 80, 88, 104, 128)
# rel-L2 bounds of the kernel against fp64 (16-bit inputs, fp32 accumulation, 16-bit outputs) and of the whole probe
# (16-bit GEMM operands and activations, fp32 residual stream) against the fp64 oracle
KERNEL_TOL = {BF16: 1e-2, F16: 2e-3}
PROBE_TOL = {BF16: (2e-2, 4e-2), F16: (4e-3, 1e-2)}      # (output, gradients)


def _attn_ref(qkv, dout, B, nq, H, hd, scale):
    """fp64 (out, lse2, dqkv) of softmax(q k^T scale) v per clip and head, from the 16-bit inputs."""
    x = qkv.double().reshape(B, nq, 3, H, hd).permute(2, 0, 3, 1, 4).detach().requires_grad_(True)
    q, k, v = x[0], x[1], x[2]
    s = (q @ k.transpose(-2, -1)) * scale
    out = torch.softmax(s, dim=-1) @ v
    lse2 = torch.logsumexp(s, dim=-1) / math.log(2.0)                 # [B, H, nq]
    out = out.transpose(1, 2).reshape(B * nq, H * hd)
    out.backward(dout.double())
    dqkv = x.grad.permute(1, 3, 0, 2, 4).reshape(B * nq, 3 * H * hd)
    return out.detach(), lse2.permute(0, 2, 1).reshape(B * nq, H), dqkv


def _attn_run(qkv, dout, B, nq, H, hd, scale):
    from jepa_b200 import kernels as Kn
    out = torch.full((B * nq, H * hd), float("nan"), dtype=qkv.dtype, device=qkv.device)
    lse = torch.full((B * nq, H), float("nan"), device=qkv.device)
    Kn.query_attn_fwd(qkv, out, lse, B, nq, H, hd, scale)
    out2 = torch.full_like(out, float("nan"))
    Kn.query_attn_fwd(qkv, out2, None, B, nq, H, hd, scale)
    assert torch.equal(out, out2)
    dqkv = torch.full_like(qkv, float("nan"))
    Kn.query_attn_bwd(qkv, out, dout, lse, dqkv, B, nq, H, hd, scale)
    dqkv2 = torch.full_like(qkv, float("nan"))
    Kn.query_attn_bwd(qkv, out, dout, lse, dqkv2, B, nq, H, hd, scale)
    assert torch.equal(dqkv, dqkv2), "backward is not bitwise reproducible"
    return out, lse, dqkv


@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("nq", [1, 2, 17, 64, 128])
@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_query_attn_kernel_vs_fp64(dev, hd, nq, dt):
    B, H = 3, 2
    D = H * hd
    g = torch.Generator().manual_seed(hd * 1000 + nq)
    qkv = torch.randn(B * nq, 3 * D, generator=g).to(dt).to(dev)
    dout = torch.randn(B * nq, D, generator=g).to(dt).to(dev)
    scale = hd ** -0.5
    out, lse, dqkv = _attn_run(qkv, dout, B, nq, H, hd, scale)
    assert torch.isfinite(out).all() and torch.isfinite(dqkv).all()
    ref_out, ref_lse, ref_d = _attn_ref(qkv, dout, B, nq, H, hd, scale)
    assert rel_l2(out, ref_out) <= KERNEL_TOL[dt], "out"
    assert float((lse.double() - ref_lse).abs().max()) <= 1e-4 * (1 + float(ref_lse.abs().max())), "lse2"
    dq, dk, dv = dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:]
    assert rel_l2(dv, ref_d[:, 2 * D:]) <= KERNEL_TOL[dt], "dv"
    if nq == 1:
        # one key: softmax is exactly 1, so out is v and the scores get no gradient
        assert torch.equal(out, qkv[:, 2 * D:])
        assert torch.count_nonzero(dq) == 0 and torch.count_nonzero(dk) == 0
    else:
        assert rel_l2(dq, ref_d[:, :D]) <= KERNEL_TOL[dt], "dq"
        assert rel_l2(dk, ref_d[:, D:2 * D]) <= KERNEL_TOL[dt], "dk"


def test_query_attn_rejects_more_than_128_tokens(dev):
    from jepa_b200 import _lib
    from jepa_b200 import kernels as Kn
    qkv = torch.zeros(129, 192, dtype=BF16, device=dev)
    with pytest.raises(_lib.VJError, match="128"):
        Kn.query_attn_fwd(qkv, torch.zeros(129, 64, dtype=BF16, device=dev), None, 1, 129, 1, 64, 0.125)


def test_query_attn_entry_point_rejects_more_than_128_tokens(dev):
    """The C ABI's own guard (it sizes the shared memory), past the Python wrapper's check: an error, no launch."""
    from jepa_b200 import _lib
    from jepa_b200.kernels import _p, _s
    qkv = torch.zeros(129, 192, dtype=BF16, device=dev)
    out = torch.zeros(129, 64, dtype=BF16, device=dev)
    lse = torch.zeros(129, 1, device=dev)
    n0 = _lib.load().vj_launch_count()
    for name in ("vj_query_attn_fwd", "vj_query_attn_fwd_f16"):
        with pytest.raises(_lib.VJError, match="at most 128"):
            _lib.call(name, _p(qkv), _p(out), _p(lse), 1, 129, 1, 64, 0.125, _s())
    for name in ("vj_query_attn_bwd", "vj_query_attn_bwd_f16"):
        with pytest.raises(_lib.VJError, match="at most 128"):
            _lib.call(name, _p(qkv), _p(out), _p(out), _p(lse), _p(qkv), 1, 129, 1, 64, 0.125, _s())
    assert _lib.load().vj_launch_count() == n0


def _step_launches(dev, kind, depth, fp16):
    """Library launches (vj_launch_count) of one probe training step - forward, backward, GradScaler step, FlatAdamW -
    at the ViT-L K400 width, after one warm-up step."""
    from jepa_b200 import _lib
    from jepa_b200.optim import FlatAdamW, FlatGradScaler
    from jepa_b200.pooler import AttentiveClassifier, AttentivePooler
    torch.manual_seed(0)
    m = (AttentiveClassifier(embed_dim=1024, num_heads=16, depth=depth, num_classes=400, follow_autocast=fp16)
         if kind == "classifier" else
         AttentivePooler(num_queries=4, embed_dim=1024, num_heads=16, depth=depth, follow_autocast=fp16)).to(dev)
    opt, scaler = FlatAdamW([{"params": list(m.parameters())}], lr=1e-3), FlatGradScaler()
    x = torch.randn(4, 1568, 1024, device=dev)

    def step():
        with torch.autocast("cuda", dtype=F16, enabled=fp16):
            y = m(x)
        scaler.scale(y.float().square().mean()).backward()
        scaler.step(opt)
        scaler.update()
        opt.zero_grad()

    step()
    torch.cuda.synchronize()
    n0 = _lib.load().vj_launch_count()
    step()
    torch.cuda.synchronize()
    return _lib.load().vj_launch_count() - n0


# launches of a depth-1 probe step before the Blocks existed (a6d9f49), (classifier, pooler) x (bf16, fp16)
DEPTH1_LAUNCHES = {("classifier", False): 34, ("classifier", True): 35, ("pooler", False): 36, ("pooler", True): 37}


@pytest.mark.parametrize("fp16", [False, True], ids=["bf16", "fp16_autocast"])
@pytest.mark.parametrize("kind", ["classifier", "pooler"])
def test_step_launches(dev, kind, fp16):
    """depth 1 issues exactly the launches it issued before Blocks existed; every further Block adds the same number."""
    n1, n2, n3 = (_step_launches(dev, kind, d, fp16) for d in (1, 2, 3))
    assert n1 == DEPTH1_LAUNCHES[(kind, fp16)], n1
    assert n3 - n2 == n2 - n1 > 0, (n1, n2, n3)


def _probe_run(dev, case, fp16):
    """(y, {name: grad or None}, module) of sum(y * dy) on the kernels, bf16 or under fp16 autocast."""
    from jepa_b200.pooler import AttentiveClassifier
    m = build_case(case)
    m.follow_autocast = fp16
    if isinstance(m, AttentiveClassifier):
        m.pooler.follow_autocast = fp16
    m = m.to(dev).train()
    x = case["x"].float().to(dev)
    with torch.autocast("cuda", dtype=F16, enabled=fp16):
        y = m(x)
    (y.float() * case["dy"].to(dev)).sum().backward()
    return y.detach().float().cpu(), {n: (None if p.grad is None else p.grad.detach().cpu())
                                      for n, p in m.named_parameters()}, m


@pytest.mark.parametrize("fp16", [False, True], ids=["bf16", "fp16_autocast"])
def test_probe_depth_matches_fixture_and_fp64(dev, fp16):
    tol_y, tol_g = PROBE_TOL[F16 if fp16 else BF16]
    for case in depth_fixture()["cases"]:
        cfg = case["cfg"]
        y, grads, m = _probe_run(dev, case, fp16)
        want_dtype = F16 if fp16 and (case["kind"] == "classifier" or not cfg["complete_block"]) else F32
        with torch.autocast("cuda", dtype=F16, enabled=fp16), torch.no_grad():
            assert m(case["x"].float().to(dev)).dtype == want_dtype, cfg
        S = {k: v.double() for k, v in build_case(case).state_dict().items()}
        y64, g64 = oracle_grads(S, case["x"].double(), case["dy"].double(), case)
        assert rel_l2(y, y64) <= tol_y, (cfg, "y vs fp64")
        assert rel_l2(y, case["y"]) <= tol_y, (cfg, "y vs fixture")
        for n, ref in case["grads"].items():
            if ref is None:
                assert grads[n] is None, n
                continue
            g = grads[n]
            assert torch.isfinite(g).all(), n
            assert rel_l2(g, g64[n]) <= tol_g, (cfg, n, rel_l2(g, g64[n]))
            assert abs(float(g.norm()) - ref["norm"]) <= tol_g * ref["norm"] + 1e-7, (cfg, n)
            assert rel_l2(g.reshape(-1)[ref["idx"].long()], ref["val"]) <= 2 * tol_g + 1e-6, (cfg, n)


def test_two_probe_calls_add_into_one_buffer(dev):
    case = depth_fixture()["cases"][1]          # classifier, depth 3
    m = build_case(case).to(dev).train()
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(case["x"].shape, generator=g).to(dev) for _ in range(2)]
    dys = [torch.randn(case["dy"].shape, generator=g).to(dev) for _ in range(2)]
    single = []
    for x, dy in zip(xs, dys):
        m.zero_grad(set_to_none=True)
        (m(x) * dy).sum().backward()
        single.append({n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None})
    m.zero_grad(set_to_none=True)
    for x, dy in zip(xs, dys):
        (m(x) * dy).sum().backward()
    params = [p for n, p in m.named_parameters() if p.grad is not None]
    assert any(".blocks." in n for n, p in m.named_parameters() if p.grad is not None)
    store = params[0]._vj_store
    assert store.grad_buffer(params) is not None, "the .grads are not slices of one flat buffer"
    for n, p in m.named_parameters():
        if p.grad is None:
            continue
        want = single[0][n] + single[1][n]
        assert float((p.grad - want).abs().max()) <= 1e-5 * float(want.abs().max()) + 1e-8, n


def test_probe_depth_eval_end_to_end(pretrained):
    from evals.scaffold import main as eval_main
    tag = "depth2"
    cfg = _eval_cfg(pretrained, tag, False)
    cfg["optimization"]["probe_depth"] = 2
    torch.manual_seed(0)            # the probe's initial weights do not depend on the tests that ran before
    eval_main("video_classification_frozen", cfg)
    body, ck = _check_run(pretrained, "video_classification_frozen", tag, 2)
    assert [r[0] for r in body] == ["1", "2"]
    # rows are (epoch, training accuracy, validation accuracy); 3 classes: chance is 33 %
    assert float(body[-1][1]) > float(body[0][1]) and float(body[-1][1]) > 50.0, body
    assert float(body[-1][2]) >= 90.0, body
    keys = set(ck["classifier"])
    assert "module.pooler.blocks.0.attn.qkv.weight" in keys and "module.pooler.blocks.0.mlp.fc2.bias" in keys
    assert not any(k.startswith("module.pooler.blocks.1.") for k in keys)
    ipe = N_ITEMS // 8
    assert float(next(iter(ck["opt"]["state"].values()))["step"]) == 2 * ipe

    cfg3 = _eval_cfg(pretrained, tag, False, epochs=3)
    cfg3["optimization"]["probe_depth"] = 2
    cfg3["resume_checkpoint"] = True
    torch.manual_seed(0)
    eval_main("video_classification_frozen", cfg3)
    body, ck3 = _check_run(pretrained, "video_classification_frozen", tag, 3)
    assert [r[0] for r in body] == ["1", "2", "3"]
    assert float(next(iter(ck3["opt"]["state"].values()))["step"]) == 3 * ipe
    assert set(ck3["classifier"]) == keys
