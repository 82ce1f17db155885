"""The attentive probe at depth > 1 on the CPU: construction, initialisation and state-dict layout of AttentivePooler /
AttentiveClassifier with depth - 1 self-attention Blocks, against the UNMODIFIED reference
(tests/golden/golden_pooler_depth.pt, written by tests/golden/make_golden_pooler_depth.py), and the fp64 oracle
restatement the GPU tests compare against."""
import os
import sys

import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def depth_fixture():
    return torch.load(os.path.join(GOLDEN, "golden_pooler_depth.pt"), weights_only=False)


def build_case(case):
    """jepa_b200.pooler's module built exactly like the fixture's reference module (same seed, same perturbation)."""
    from jepa_b200.pooler import AttentiveClassifier, AttentivePooler
    torch.manual_seed(case["seed"])
    m = (AttentiveClassifier if case["kind"] == "classifier" else AttentivePooler)(**case["cfg"])
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("bias") or "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
    return m


def oracle_forward(S, x, case):
    """fp64-capable restatement of the reference's forward from the oracle's pieces: attentive_pooler (depth 1) followed
    by the depth - 1 Blocks (nn.LayerNorm default eps 1e-5, as the probe's norm_layer), then the linear head."""
    from oracle import vjepa_oracle as O
    cfg = case["cfg"]
    pre = "pooler." if case["kind"] == "classifier" else ""
    q = O.attentive_pooler(S, x, cfg["num_heads"], cfg["complete_block"], pre=pre)
    for i in range(cfg["depth"] - 1):
        q = O.block(q, S, f"{pre}blocks.{i}.", cfg["num_heads"], eps=1e-5)
    if case["kind"] == "pooler":
        return q
    return O.linear(q.squeeze(1), S["linear.weight"], S["linear.bias"])


def oracle_grads(S, x, dy, case):
    """(y, {name: gradient of sum(y * dy) or None}) by autograd through oracle_forward."""
    S = {k: v.detach().clone().requires_grad_(True) for k, v in S.items()}
    y = oracle_forward(S, x, case)
    (y * dy).sum().backward()
    return y.detach(), {k: v.grad for k, v in S.items()}


def test_depth_init_and_state_dict_match_reference():
    """Same keys, order and shapes as the reference's state dict, and - draw for draw - the same initial values
    (the reference's _init_weights order and _rescale_blocks with layer_id + 1), for complete_block True and False."""
    sys.path.insert(0, GOLDEN)
    from common import sha16
    for case in depth_fixture()["cases"]:
        sd = build_case(case).state_dict()
        assert list(sd.keys()) == case["keys"], case["cfg"]
        assert {k: tuple(v.shape) for k, v in sd.items()} == case["shapes"]
        for k, v in sd.items():
            assert sha16(v) == case["sha"][k], (case["cfg"], k)
        assert any(".blocks." in "." + k for k in sd)


def test_reference_checkpoint_loads():
    from jepa_b200.pooler import AttentiveClassifier
    ck = depth_fixture()["checkpoint"]
    clf = AttentiveClassifier(**ck["cfg"])
    clf.load_state_dict(ck["state_dict"])          # strict: every pooler.blocks.* key is known, none is missing
    for k, v in clf.state_dict().items():
        assert torch.equal(v, ck["state_dict"][k]), k


def test_oracle_restatement_matches_reference_fixture():
    for case in depth_fixture()["cases"]:
        S = {k: v.double() for k, v in build_case(case).state_dict().items()}
        y, grads = oracle_grads(S, case["x"].double(), case["dy"].double(), case)
        assert float((y.float() - case["y"]).abs().max()) < 2e-5, case["cfg"]
        assert set(grads) == set(case["grads"])
        for n, ref in case["grads"].items():
            if ref is None:                      # the cross-attention's proj: built, never applied
                assert grads[n] is None, n
                continue
            # the fixture is the reference's fp32 autograd: at width 832 its gradients carry ~1e-4 relative rounding
            g = grads[n].reshape(-1)
            assert abs(float(g.norm()) - ref["norm"]) <= 1e-3 * ref["norm"] + 1e-9, n
            assert float((g[ref["idx"].long()].float() - ref["val"]).abs().max()) <= \
                1e-3 * float(ref["val"].abs().max()) + 1e-9, n


def test_too_many_query_tokens_raise():
    from jepa_b200.pooler import AttentivePooler
    AttentivePooler(num_queries=128, embed_dim=64, num_heads=1, depth=2)
    AttentivePooler(num_queries=129, embed_dim=64, num_heads=1, depth=1)     # depth 1 runs no self-attention
    with pytest.raises(NotImplementedError, match="128"):
        AttentivePooler(num_queries=129, embed_dim=64, num_heads=1, depth=2)


def test_deep_probe_without_qkv_bias_raises_for_the_probe():
    from jepa_b200.pooler import AttentivePooler
    AttentivePooler(embed_dim=64, num_heads=1, depth=1, qkv_bias=False)
    with pytest.raises(NotImplementedError, match="AttentivePooler depth > 1 with qkv_bias=False"):
        AttentivePooler(embed_dim=64, num_heads=1, depth=2, qkv_bias=False)


def test_qk_scale_false_means_default():
    from jepa_b200.models import Attention
    assert Attention(64, num_heads=2, qkv_bias=True, qk_scale=False).scale == 32 ** -0.5
    with pytest.raises(NotImplementedError):
        Attention(64, num_heads=2, qkv_bias=True, qk_scale=0.3)


def test_probe_depth_key():
    from evals.video_classification_frozen.eval import read_probe_depth
    assert read_probe_depth({}) == 1
    assert read_probe_depth({"probe_depth": 3}) == 3
    for bad in (0, -1, 1.5, True, "2", None):
        with pytest.raises(ValueError, match="probe_depth"):
            read_probe_depth({"probe_depth": bad})
