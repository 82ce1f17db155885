"""The frozen evaluations' training loop without a GPU: train_heads (epoch loop, resume, CSV, checkpoint) and both
drivers' run_one_epoch (through run_head_loop) on a stub encoder and a small probe, with init_opt's AdamW and GradScaler
replaced by torch's CPU ones.  Checks both layouts - one classifier as the reference writes it and the
`optimization.multihead_kwargs` lists - resume to the saved epoch, a checkpoint of other heads restarting at epoch 0,
the single-classifier and per-head-list call forms, and N heads ending bitwise where N single runs end."""
import logging

import pytest
import torch
import torch.nn as nn

from evals.image_classification_frozen import eval as ie
from evals.video_classification_frozen import eval as ve
from src.utils.schedulers import CosineWDSchedule, WarmupCosineSchedule

CPU = torch.device("cpu")
B, C, D, STEPS = 4, 3, 16, 3
SETTINGS = [
    ve.one_head(0.01, 2e-3, 1e-2, 1e-4, 0.34),
    dict(lr=5e-3, start_lr=1e-4, final_lr=0.0, weight_decay=0.05, final_weight_decay=0.1, warmup=0.67),
    dict(lr=2e-2, start_lr=5e-3, final_lr=1e-5, weight_decay=0.0, final_weight_decay=0.0, warmup=0.0),
]
REFERENCE_KEYS = {"classifier", "opt", "scaler", "epoch", "batch_size", "world_size", "lr"}
MULTIHEAD_KEYS = {"classifiers", "opts", "scalers", "multihead_kwargs", "epoch", "batch_size", "world_size"}


def _cpu_init_opt(classifier, iterations_per_epoch, start_lr, ref_lr, warmup, num_epochs, wd=1e-6, final_wd=1e-6,
                  final_lr=0.0, use_bfloat16=False):
    """init_opt with torch's AdamW and a CPU GradScaler in place of the flat sm_90a ones."""
    param_groups = [
        {'params': [p for n, p in classifier.named_parameters() if ('bias' not in n) and (len(p.shape) != 1)]},
        {'params': [p for n, p in classifier.named_parameters() if ('bias' in n) or (len(p.shape) == 1)],
         'WD_exclude': True, 'weight_decay': 0},
    ]
    optimizer = torch.optim.AdamW(param_groups)
    T = int(num_epochs * iterations_per_epoch)
    scheduler = WarmupCosineSchedule(optimizer, warmup_steps=int(warmup * iterations_per_epoch), start_lr=start_lr,
                                     ref_lr=ref_lr, final_lr=final_lr, T_max=T)
    wd_scheduler = CosineWDSchedule(optimizer, ref_wd=wd, final_wd=final_wd, T_max=T)
    scaler = torch.amp.GradScaler("cpu", init_scale=2.0 ** 6, growth_interval=2) if use_bfloat16 else None
    return optimizer, scaler, scheduler, wd_scheduler


@pytest.fixture(autouse=True)
def cpu_opt(monkeypatch):
    monkeypatch.setattr(ve, "init_opt", _cpu_init_opt)


class _Patches(nn.Module):
    """A frozen stand-in for the ViT: [N, 3, T, 8, 8] clips or [N, 3, 8, 8] images -> [N, tokens, D]."""
    embed_dim, num_heads = D, 2

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(11)
        self.clip = nn.Parameter(torch.randn(3 * 2 * 16, D, generator=g) / 10, requires_grad=False)
        self.image = nn.Parameter(torch.randn(3 * 16, D, generator=g) / 10, requires_grad=False)

    def forward(self, x):
        if x.dim() == 5:
            N, _, T, _, _ = x.shape
            x = x.reshape(N, 3, T // 2, 2, 2, 4, 2, 4).permute(0, 2, 4, 6, 1, 3, 5, 7)
            return x.reshape(N, -1, 3 * 32) @ self.clip
        x = x.reshape(len(x), 3, 2, 4, 2, 4).permute(0, 2, 4, 1, 3, 5)
        return x.reshape(len(x), 4, 3 * 16) @ self.image


class _Probe(nn.Module):
    def __init__(self):
        super().__init__()
        self.norm = nn.LayerNorm(D)
        self.query = nn.Linear(D, D)
        self.linear = nn.Linear(D, C)

    def forward(self, x):
        return self.linear(torch.tanh(self.query(self.norm(x))).mean(1))


def _setup(kind):
    """(encoder, batches, run_one_epoch of the driver with its loop keywords)."""
    g = torch.Generator().manual_seed(5)
    labels = [torch.randint(0, C, (B,), generator=g) for _ in range(STEPS)]
    if kind == "image":
        batches = [(torch.randn(B, 3, 8, 8, generator=g), labels[i]) for i in range(STEPS)]
        return _Patches(), batches, ie.run_one_epoch
    attend = kind == "video_attend"
    enc = ve.ClipAggregation(_Patches(), tubelet_size=2, attend_across_segments=attend)
    idx = [torch.arange(4).expand(B, 4) + 4 * s for s in range(2)]
    batches = [([[torch.randn(B, 3, 4, 8, 8, generator=g)] for _ in range(2)], labels[i], idx) for i in range(STEPS)]

    def run(**kw):
        return ve.run_one_epoch(num_spatial_views=1, num_temporal_views=2, attend_across_segments=attend, **kw)
    return enc, batches, run


class _Preempted(Exception):
    pass


def _train(tmp_path, kind, settings, multihead, epochs, tag, resume=False, preempt_after=None):
    """train_heads as the drivers call it, optionally stopped once `preempt_after` epochs have been saved; returns
    (classifiers, checkpoint, CSV text)."""
    enc, batches, run = _setup(kind)
    torch.manual_seed(0)
    clfs = ve.build_heads(_Probe, len(settings))
    trained = []

    def run_epoch(training, heads):
        if training:
            if len(trained) == preempt_after:
                raise _Preempted
            trained.append(1)
        return run(device=CPU, training=training, encoder=enc, data_loader=batches, use_bfloat16=True, **heads)
    try:
        ve.train_heads(clfs, settings, run_epoch, multihead=multihead, iterations_per_epoch=STEPS, num_epochs=epochs,
                       use_bfloat16=True, resume_checkpoint=resume, latest_path=str(tmp_path / f"{tag}.pth.tar"),
                       log_file=str(tmp_path / f"{tag}.csv"), device=CPU, rank=0, world_size=1, batch_size=B)
    except _Preempted:
        pass
    return clfs, torch.load(tmp_path / f"{tag}.pth.tar", weights_only=False), (tmp_path / f"{tag}.csv").read_text()


def _rows(csv):
    return [r.split(",") for r in csv.splitlines()]


def _same_state(a, b):
    """Equal nested dicts / lists of tensors and values, tensors bitwise."""
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a, b)
    if isinstance(a, dict):
        return isinstance(b, dict) and list(a) == list(b) and all(_same_state(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(_same_state(x, y) for x, y in zip(a, b))
    return a == b


def test_one_head_keeps_the_reference_layout(tmp_path, caplog):
    caplog.set_level(logging.INFO)
    _, ck, csv = _train(tmp_path, "video", SETTINGS[:1], False, 2, "one")
    assert set(ck) == REFERENCE_KEYS and list(ck) == ["classifier", "opt", "scaler", "epoch", "batch_size",
                                                      "world_size", "lr"]
    assert ck["epoch"] == 2 and ck["batch_size"] == B and ck["world_size"] == 1 and ck["lr"] == SETTINGS[0]["lr"]
    assert all(k.startswith("module.") for k in ck["classifier"]) and ck["scaler"]["scale"] > 0
    rows = _rows(csv)
    assert rows[0] == ["epoch", "loss", "acc"] and [r[0] for r in rows[1:]] == ["1", "2"]
    assert all(len(r) == 3 and len(r[1].split(".")[1]) == 5 for r in rows[1:])
    msgs = [r.getMessage() for r in caplog.records]
    assert not any("head" in m for m in msgs), msgs
    assert sum(m.startswith("[    0] ") and "(loss: " in m for m in msgs) == 4      # train and val, 2 epochs
    assert any(m.startswith("[    2] train: ") and " test: " in m for m in msgs)


def test_one_head_takes_the_top_level_values_unconverted():
    assert ve.one_head(1, None, 2, 0, 3) == dict(lr=2, start_lr=None, final_lr=0, weight_decay=1, final_weight_decay=1e-6,
                                                 warmup=3)
    assert type(ve.one_head(1, 1, 1, 1, 1)["lr"]) is int


def test_heads_keep_the_multihead_layout(tmp_path, caplog):
    caplog.set_level(logging.INFO)
    _, ck, csv = _train(tmp_path, "image", SETTINGS, True, 2, "three")
    assert set(ck) == MULTIHEAD_KEYS and list(ck) == ["classifiers", "opts", "scalers", "multihead_kwargs", "epoch",
                                                      "batch_size", "world_size"]
    assert ck["multihead_kwargs"] == SETTINGS and ck["epoch"] == 2
    assert len(ck["classifiers"]) == len(ck["opts"]) == len(ck["scalers"]) == 3
    rows = _rows(csv)
    assert rows[0] == ["epoch", "head", "loss", "acc"]
    assert [(r[0], r[1]) for r in rows[1:]] == [(str(e), str(k)) for e in (1, 2) for k in range(3)]
    msgs = [r.getMessage() for r in caplog.records]
    assert "Training 3 attentive probes on one encoder pass per batch" in msgs
    assert [m[:16] for m in msgs if m.startswith("[    0] head")] == ["[    0] head 0: ", "[    0] head 1: ",
                                                                        "[    0] head 2: "] * 4
    assert sum(m.startswith("[    2] best of 3 heads: head ") for m in msgs) == 1


@pytest.mark.parametrize("multihead", [False, True], ids=["one_head", "three_heads"])
def test_resume_continues_from_the_saved_epoch(tmp_path, caplog, multihead):
    """A three-epoch run stopped after saving epoch 2 and then resumed trains epoch 3 only and ends bitwise where an
    uninterrupted run ends (weights, optimizer, scaler, the fast-forwarded schedules, the CSV rows)."""
    settings = SETTINGS if multihead else SETTINGS[:1]
    _, straight, straight_csv = _train(tmp_path, "video_attend", settings, multihead, 3, "straight")
    _, saved, _ = _train(tmp_path, "video_attend", settings, multihead, 3, "resumed", preempt_after=2)
    assert saved["epoch"] == 2
    caplog.set_level(logging.INFO)
    caplog.clear()
    _, ck, csv = _train(tmp_path, "video_attend", settings, multihead, 3, "resumed", resume=True)
    msgs = [r.getMessage() for r in caplog.records]
    assert ("loaded optimizers of 3 heads from epoch 2" if multihead else "loaded optimizers from epoch 2") in msgs
    assert [m for m in msgs if m.startswith("Epoch ")] == ["Epoch 3"]
    assert _same_state(ck, straight)
    assert [r for r in _rows(csv) if r[0] != "epoch"] == _rows(straight_csv)[1:]


def test_load_checkpoint_reads_the_reference_layout(tmp_path):
    _train(tmp_path, "video", SETTINGS[:1], False, 2, "ref")
    clf = ve.DistributedDataParallel(_Probe())
    opt, scaler, _, _ = _cpu_init_opt(clf, STEPS, 1e-3, 1e-3, 0, 2, use_bfloat16=True)
    got = ve.load_checkpoint(CPU, str(tmp_path / "ref.pth.tar"), clf, opt, scaler)
    assert got[:3] == (clf, opt, scaler) and got[3] == 2
    ck = torch.load(tmp_path / "ref.pth.tar", weights_only=False)
    assert _same_state(clf.state_dict(), ck["classifier"]) and scaler.get_scale() == ck["scaler"]["scale"]


def test_a_checkpoint_of_other_heads_restarts_at_epoch_zero(tmp_path, caplog):
    _train(tmp_path, "image", SETTINGS, True, 2, "mh")
    other = [dict(h) for h in SETTINGS]
    other[2]["lr"] = 1e-3
    caplog.set_level(logging.INFO)
    caplog.clear()
    _, ck, csv = _train(tmp_path, "image", other, True, 1, "mh", resume=True)
    msgs = [r.getMessage() for r in caplog.records]
    assert any(m.startswith("Encountered exception when loading checkpoint its heads") for m in msgs)
    assert ck["epoch"] == 1 and ck["multihead_kwargs"] == other
    assert [(r[0], r[1]) for r in _rows(csv)[-4:]] == [("epoch", "head"), ("1", "0"), ("1", "1"), ("1", "2")]
    # nor does a one-classifier run read a multi-head checkpoint
    assert ve.load_multihead_checkpoint(CPU, str(tmp_path / "mh.pth.tar"), [ve.DistributedDataParallel(_Probe())],
                                        [None], [None], None) == 0


@pytest.mark.parametrize("kind", ["video", "video_attend", "image"])
def test_single_and_list_call_forms_agree(kind):
    enc, batches, run = _setup(kind)
    out = []
    for listed in (False, True):
        torch.manual_seed(0)
        clf = _Probe()
        opt, scaler, sch, wds = _cpu_init_opt(clf, STEPS, 1e-3, 1e-2, 0.5, 1, wd=0.01, use_bfloat16=True)
        heads = dict(classifier=clf, scaler=scaler, optimizer=opt, scheduler=sch, wd_scheduler=wds)
        if listed:
            heads = {k: [v] for k, v in heads.items()}
        acc = run(device=CPU, training=True, encoder=enc, data_loader=batches, use_bfloat16=True, **heads)
        val = run(device=CPU, training=False, encoder=enc, data_loader=batches, use_bfloat16=True, **heads)
        out.append((acc, val, clf.state_dict(), opt.state_dict()))
    (acc, val, sd, od), (accs, vals, sd1, od1) = out
    assert type(acc) is float and type(val) is float and accs == [acc] and vals == [val]
    assert _same_state(sd, sd1) and _same_state(od, od1)


@pytest.mark.parametrize("kind", ["video", "video_attend", "image"])
def test_heads_end_where_single_runs_end(tmp_path, kind):
    """Three heads with distinct settings on one encoder pass per batch end bitwise where three one-classifier runs with
    those settings end: weights, AdamW moments and steps, GradScaler state, and the CSV accuracies."""
    clfs, ck, csv = _train(tmp_path, kind, SETTINGS, True, 2, "heads")
    rows = _rows(csv)[1:]
    for k, h in enumerate(SETTINGS):
        _, one, one_csv = _train(tmp_path, kind, [h], False, 2, f"single{k}")
        assert _same_state(ck["classifiers"][k], one["classifier"]), (kind, k)
        assert _same_state(ck["opts"][k], one["opt"]) and _same_state(ck["scalers"][k], one["scaler"]), (kind, k)
        assert [r[2:] for r in rows if r[1] == str(k)] == [r[1:] for r in _rows(one_csv)[1:]], (kind, k)
    w = [c.linear.weight for c in clfs]
    assert not torch.equal(w[0], w[1]) and not torch.equal(w[1], w[2])
