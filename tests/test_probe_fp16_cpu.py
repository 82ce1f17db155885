"""The fp16 attentive probe without a GPU: the `optimization.fp16_autocast` key of the evaluation drivers, the argument
checks of the new fp16 entry points (they return < 0 and launch nothing), and the power of the fp16 cross-attention
comparator (tests/xattn16_ref.py) that tests/test_gpu_probe_fp16.py applies to the kernels: on the GPU tests' inputs it
passes an emulation that rounds to fp16 where the kernels round, and rejects known faults."""
import ctypes
import os

import pytest
import torch

import xattn16_ref as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16 = torch.float16


# ------------------------------------------------------------------------------------------------------ config key
@pytest.mark.filterwarnings("ignore:CUDA is not available")
def test_fp16_autocast_key_parsing_and_default():
    from evals.video_classification_frozen.eval import loop_autocast, read_fp16_autocast
    assert read_fp16_autocast({}) is False
    assert read_fp16_autocast({"fp16_autocast": False}) is False
    assert read_fp16_autocast({"fp16_autocast": True}) is True
    for bad in ("true", 1, None):
        with pytest.raises(ValueError, match="fp16_autocast"):
            read_fp16_autocast({"fp16_autocast": bad})
    import contextlib
    assert isinstance(loop_autocast(False, True), contextlib.nullcontext)
    on, off = loop_autocast(True, True), loop_autocast(True, False)    # (without CUDA torch disables both)
    assert isinstance(on, torch.autocast) and on.device == "cuda" and on.fast_dtype == F16
    assert isinstance(off, torch.autocast) and not off._enabled      # use_bfloat16 false: the region is disabled


def test_image_eval_reads_the_same_key():
    from evals.image_classification_frozen import eval as ie
    from evals.video_classification_frozen import eval as ve
    assert ie.read_fp16_autocast is ve.read_fp16_autocast and ie.loop_autocast is ve.loop_autocast


def test_follow_autocast_is_not_state():
    from jepa_b200.pooler import AttentiveClassifier, AttentivePooler
    a = AttentiveClassifier(embed_dim=64, num_heads=2, num_classes=3, follow_autocast=True)
    b = AttentiveClassifier(embed_dim=64, num_heads=2, num_classes=3)
    assert a.follow_autocast and a.pooler.follow_autocast and not b.follow_autocast
    assert list(a.state_dict()) == list(b.state_dict())
    assert [n for n, _ in a.named_parameters()] == [n for n, _ in b.named_parameters()]
    assert AttentivePooler(embed_dim=64, num_heads=2).follow_autocast is False


# ------------------------------------------------------------------------------------------------ ABI argument checks
@pytest.fixture(scope="module")
def lib():
    from jepa_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libvjepa_b200.so is not built")
    return _lib.load()


def _rejects(lib, name, *args):
    n0 = lib.vj_launch_count()
    rc = getattr(lib, name)(*args)
    assert rc < 0, (name, rc)
    assert lib.vj_launch_count() == n0, name
    assert lib.vj_last_error_string().decode().startswith(name), lib.vj_last_error_string()


def test_new_entry_points_reject_bad_arguments(lib):
    A = 1 << 20                       # an aligned fake device address: nothing is dereferenced before the checks
    ws = lib.vj_cross_attn_bwd_workspace(2, 1, 100, 4, 64)
    for name in ("vj_cross_attn_fwd_f16",):
        _rejects(lib, name, None, A, A, 2, 1, 100, 4, 64, 0.125, None)                 # null pointer
        _rejects(lib, name, A, A, A, 0, 1, 100, 4, 64, 0.125, None)                    # empty problem
        _rejects(lib, name, A + 2, A, A, 2, 1, 100, 4, 64, 0.125, None)                # misaligned q
        _rejects(lib, name, A, A, A, 2, 1, 100, 4, 48, 0.125, None)                    # head dim 48
    _rejects(lib, "vj_cross_attn_fwd_lse_f16", A, A, A, None, 2, 1, 100, 4, 64, 0.125, None)     # null lse2
    _rejects(lib, "vj_cross_attn_fwd_lse_f16", A, A, A, A, 2, 1, 100, 4, 96, 0.125, None)        # head dim 96
    bwd = "vj_cross_attn_bwd_f16"
    _rejects(lib, bwd, A, A, A, A, A, A, A, A, ws - 4, 2, 1, 100, 4, 64, 0.125, None)  # workspace too small
    _rejects(lib, bwd, A, A, A, A, A, A, A, None, ws, 2, 1, 100, 4, 64, 0.125, None)   # null workspace
    _rejects(lib, bwd, A, A, A, A, A, A, A, A, ws, 2, 1, 100, 4, 72, 0.125, None)      # head dim 72
    _rejects(lib, bwd, A, A, A, A, A, A, A + 8, A, ws, 2, 1, 100, 4, 64, 0.125, None)  # misaligned dkv
    _rejects(lib, bwd, A, A, A, A, A, A, A, A, 1 << 40, 1, 1, 64 * 65536, 1, 64, 0.125, None)   # too many key chunks
    _rejects(lib, "vj_layernorm_bwd_f16", A, A, A, A, A, None, A, A, A, A, 1 << 30, 16, 100, None)  # D % 8
    _rejects(lib, "vj_layernorm_bwd_f16", A, A, A, A, A, None, A, A, A, A, 1 << 30, 16, 4096, None)  # D > 2048
    _rejects(lib, "vj_layernorm_bwd_f16", None, A, A, A, A, None, A, A, A, A, 1 << 30, 16, 64, None)  # null dy
    _rejects(lib, "vj_colsum_f16", A, A, 100, 12, 16, 0, 0, 0, None)                   # N % 8
    _rejects(lib, "vj_colsum_f16", A, A, 100, 16, 12, 0, 0, 0, None)                   # ld % 8
    _rejects(lib, "vj_colsum_f16", None, A, 100, 16, 16, 0, 0, 0, None)                # null input


def test_header_declares_every_new_entry_point():
    with open(os.path.join(ROOT, "include", "vjepa_b200.h")) as f:
        h = f.read()
    from jepa_b200._lib import SIGNATURES
    for name in ("vj_cross_attn_fwd_f16", "vj_cross_attn_fwd_lse_f16", "vj_cross_attn_bwd_f16", "vj_layernorm_bwd_f16",
                 "vj_colsum_f16"):
        assert f" {name}(" in h and name in SIGNATURES, name
    assert ctypes.c_int == SIGNATURES["vj_colsum_f16"][0]


# ------------------------------------------------------------------------------------------- comparator power
# a slice of the GPU tests' cases: both sides of the backward's key chunk (32 / 64 / 80 / 128 keys at hd 128 / 64 / 80
# / 32), ragged lengths, one and three queries
CASES = [(hd, nq, S) for hd in (32, 64, 80, 128) for nq in (1, 3)
         for S in (1, 7, X.key_chunk(hd) - 1, X.key_chunk(hd), X.key_chunk(hd) + 3, 300)]


def _worst(c, fault=None):
    q, kv, dout = (c[k].to(F16) for k in ("q", "kv", "dout"))
    got = X.emulate(c, fault)
    return X.check(c, *got, X.reference(c, q, kv, dout, got[0]))


def _seed(hd, nq, S):
    return hd * 1000 + nq * 400 + S          # the seeds of test_gpu_probe_fp16.test_cross_attn_f16_vs_fp64_every_residue


def test_comparator_passes_the_kernels_roundings():
    for hd, nq, S in CASES:
        res = _worst(X.make_case(hd, nq, S, _seed(hd, nq, S)))
        assert max(res.values()) <= 0.5, (hd, nq, S, res)
    res = _worst(X.overflow_case())
    assert max(res.values()) <= 0.5, res


@pytest.mark.parametrize("fault", ["bf16", "leak", "drop_chunk"])
def test_comparator_rejects_known_faults(fault):
    """Every case the fault changes is rejected (drop_chunk only changes clips of at least one full key chunk)."""
    changed = 0
    for hd, nq, S in CASES:
        if fault == "drop_chunk" and S < X.key_chunk(hd):
            continue
        changed += 1
        res = _worst(X.make_case(hd, nq, S, _seed(hd, nq, S)), fault)
        assert max(res.values()) > 1.0, (fault, hd, nq, S, res)
    assert changed >= 16


def test_comparator_rejects_a_saturating_store():
    res = _worst(X.overflow_case(), "satfinite")
    assert res["dkv"] == float("inf"), res
