"""Pin the oracle's backward for the attentive probe: fp64 autograd through oracle/vjepa_oracle.attentive_classifier
must reproduce the loss, dlogits and every parameter gradient that the UNMODIFIED reference AttentiveClassifier produced
with torch.nn.CrossEntropyLoss (tests/golden/golden_pooler_grad.pt, written by tests/golden/make_golden_pooler_grad.py)."""
import os

import torch

from test_oracle_cpu import _build_probe, _pooler_fixture

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _grad_fixture():
    return torch.load(os.path.join(GOLDEN, "golden_pooler_grad.pt"), weights_only=False)


def oracle_grads(S, x, labels, heads, complete_block):
    """(loss, dlogits, {name: grad or None}) of CrossEntropyLoss(attentive_classifier(S, x)) by autograd on the oracle."""
    from oracle import vjepa_oracle as O
    S = {k: v.detach().clone().requires_grad_(True) for k, v in S.items()}
    logits = O.attentive_classifier(S, x, heads, complete_block)
    logits.retain_grad()
    loss = torch.nn.functional.cross_entropy(logits, labels)
    loss.backward()
    return float(loss.detach()), logits.grad, {k: v.grad for k, v in S.items()}


def test_oracle_probe_gradients_match_reference_fixture():
    fx = _grad_fixture()["cases"]
    for case, gcase in zip(_pooler_fixture()["cases"], fx):
        assert case["cfg"] == gcase["cfg"] and case["seed"] == gcase["seed"]
        S = {k: v.double() for k, v in _build_probe(case).state_dict().items()}
        cfg = case["cfg"]
        loss, dlogits, grads = oracle_grads(S, case["x"].double(), gcase["labels"], cfg["num_heads"], cfg["complete_block"])
        assert abs(loss - gcase["loss"]) < 2e-5, cfg
        assert float((dlogits.float() - gcase["dlogits"]).abs().max()) < 2e-6, cfg
        assert set(grads) == set(gcase["grads"])
        for n, ref in gcase["grads"].items():
            if ref is None:                      # proj: built, never applied by the reference's forward
                assert grads[n] is None, n
                continue
            g = grads[n].reshape(-1)
            assert abs(float(g.norm()) - ref["norm"]) <= 1e-4 * ref["norm"] + 1e-9, n
            assert float((g[ref["idx"]].float() - ref["val"]).abs().max()) <= 1e-4 * float(ref["val"].abs().max()) + 1e-9, n
