"""Several attentive probes on one encoder pass, without a GPU: the `optimization.multihead_kwargs` key (fallbacks,
defaults and every rejected input), the image evaluation reading it through the same helper, and the construction of
the heads - equal initial weights, head 0 bit for bit today's single classifier, and the global torch RNG left where
one classifier leaves it, so that the data pipeline drawing from it next sees the same stream."""
import pytest
import torch

pytestmark = pytest.mark.filterwarnings("ignore:CUDA is not available")

TOP = dict(lr=1e-3, start_lr=2e-4, final_lr=0.0, weight_decay=0.01, warmup=0.5, batch_size=4, use_bfloat16=True)


def _read(heads, **top):
    from evals.video_classification_frozen.eval import read_multihead_kwargs
    opt = dict(TOP, **top)
    if heads is not ...:
        opt["multihead_kwargs"] = heads
    return read_multihead_kwargs(opt)


def test_absent_key_means_one_classifier():
    assert _read(...) is None


def test_fields_fall_back_to_the_top_level_values():
    heads = _read([{}, {"lr": 5e-3, "weight_decay": 0.05}, {"warmup": 0, "final_weight_decay": 0.1, "start_lr": 1}])
    assert len(heads) == 3
    assert heads[0] == dict(lr=1e-3, start_lr=2e-4, final_lr=0.0, weight_decay=0.01, final_weight_decay=1e-6, warmup=0.5)
    assert heads[1] == dict(heads[0], lr=5e-3, weight_decay=0.05)
    assert heads[2] == dict(heads[0], warmup=0.0, final_weight_decay=0.1, start_lr=1.0)
    assert all(type(v) is float for h in heads for v in h.values())
    assert [list(h) for h in heads] == [["lr", "start_lr", "final_lr", "weight_decay", "final_weight_decay", "warmup"]] * 3


def test_final_weight_decay_defaults_to_init_opts_value():
    import inspect
    from evals.video_classification_frozen.eval import init_opt
    assert _read([{}])[0]["final_weight_decay"] == inspect.signature(init_opt).parameters["final_wd"].default == 1e-6


@pytest.mark.parametrize("heads, match", [
    ([{}, {"lr": 1e-3, "momentum": 0.9}], r"multihead_kwargs\[1\].*'momentum'"),
    ([{"lr": "1e-3"}], r"multihead_kwargs\[0\]\.lr"),
    ([{}, {}, {"warmup": None}], r"multihead_kwargs\[2\]\.warmup"),
    ([{"weight_decay": True}], r"multihead_kwargs\[0\]\.weight_decay"),
    ([{"final_lr": float("nan")}], r"multihead_kwargs\[0\]\.final_lr"),
    ([{}, {"start_lr": -1e-4}], r"multihead_kwargs\[1\]\.start_lr.*negative"),
    ([{"final_weight_decay": -0.1}], r"multihead_kwargs\[0\]\.final_weight_decay.*negative"),
    ([{}, [("lr", 1e-3)]], r"multihead_kwargs\[1\].*mapping"),
    ([], r"multihead_kwargs.*non-empty list"),
    ({"lr": 1e-3}, r"multihead_kwargs.*non-empty list"),
    ("lr=1e-3", r"multihead_kwargs.*non-empty list"),
    (None, r"multihead_kwargs.*non-empty list"),
])
def test_rejected_inputs_name_the_head_and_the_key(heads, match):
    with pytest.raises(ValueError, match=match):
        _read(heads)


def test_a_missing_top_level_value_is_named():
    with pytest.raises(ValueError, match=r"multihead_kwargs\[0\]\.lr.*optimization\.lr"):
        _read([{}], lr=None)
    assert _read([{"lr": 2e-3}], lr=None)[0]["lr"] == 2e-3


def test_image_eval_uses_the_same_helpers():
    from evals.image_classification_frozen import eval as ie
    from evals.video_classification_frozen import eval as ve
    assert ie.read_multihead_kwargs is ve.read_multihead_kwargs
    assert ie.build_heads is ve.build_heads and ie.train_heads is ve.train_heads and ie.step_head is ve.step_head


# ------------------------------------------------------------------------------------------------ head construction
def _make():
    from jepa_b200.pooler import AttentiveClassifier
    return AttentiveClassifier(embed_dim=64, num_heads=2, depth=1, num_classes=5)


def _state_equal(a, b):
    sa, sb = a.state_dict(), b.state_dict()
    return list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) and sa[k].dtype == sb[k].dtype for k in sa)


@pytest.mark.parametrize("num_heads", [1, 2, 4])
def test_heads_leave_the_rng_where_one_classifier_does(num_heads):
    from evals.video_classification_frozen.eval import build_heads
    torch.manual_seed(0)
    one = _make()
    want = torch.get_rng_state()
    next_draw = torch.rand(8)
    torch.manual_seed(0)
    heads = build_heads(_make, num_heads)
    assert len(heads) == num_heads
    assert torch.equal(torch.get_rng_state(), want)
    assert torch.equal(torch.rand(8), next_draw)
    assert _state_equal(heads[0], one)


def test_every_head_starts_from_head_zero():
    from evals.video_classification_frozen.eval import build_heads
    torch.manual_seed(3)
    heads = build_heads(_make, 3)
    for h in heads[1:]:
        assert _state_equal(h, heads[0])
        assert all(p.data_ptr() != q.data_ptr() for p, q in zip(h.parameters(), heads[0].parameters()))
    # the heads are independent modules: changing one leaves the others alone
    with torch.no_grad():
        heads[1].linear.weight.add_(1.0)
    assert not torch.equal(heads[1].linear.weight, heads[0].linear.weight)
    assert torch.equal(heads[2].linear.weight, heads[0].linear.weight)


def test_follow_autocast_reaches_every_head():
    from evals.video_classification_frozen.eval import build_heads
    from jepa_b200.pooler import AttentiveClassifier
    heads = build_heads(lambda: AttentiveClassifier(embed_dim=64, num_heads=2, num_classes=3, follow_autocast=True), 3)
    assert all(h.follow_autocast and h.pooler.follow_autocast for h in heads)
