"""Golden fixture of tests/test_gpu_reference.py: the unmodified reference's train-step outputs on the GPU.

tools/ref_gpu.py `step` runs the reference modules (oracle/_ref, copied by oracle/make_ref.sh) on the seeded weights /
clips / masks of tests/parity_util.py, once under bf16 autocast and once in fp32.  This script keeps, per config: both
losses, and for every output / gradient tensor the full-tensor rel-L2 between the two reference runs plus a fixed seeded
sample (sample_index) of both runs' values - small enough to commit, and what the test compares our CUDA step against.

    python tools/ref_gpu.py step --embed-dim 192 --heads 3 --depth 12 --pred-depth 12 --frames 8 --batch 2 \
        --mask-batch 2 --out ref_c1.pt
    python tools/ref_gpu.py step --embed-dim 1024 --heads 16 --depth 2 --pred-depth 2 --frames 16 --batch 1 \
        --mask-batch 32 --out ref_vitl.pt
    python tests/golden/make_golden_reference.py c1_vit_tiny_12+12=ref_c1.pt vitl16_2+2_blocks=ref_vitl.pt \
        -o tests/golden/golden_reference_step.pt
"""
import argparse
import zlib

import torch

N_OUT, N_GRAD = 256, 32   # sampled elements per output tensor / per gradient tensor


def sample_index(numel, key):
    n = N_GRAD if key.startswith(("enc_grad.", "pred_grad.")) else N_OUT
    g = torch.Generator().manual_seed(zlib.crc32(key.encode()))
    return torch.randint(0, numel, (min(n, numel),), generator=g)


def flat_tensors(step):
    """key -> tensor for the outputs (h / z_enc / z lists) and the gradients (enc_grad / pred_grad dicts) of one run."""
    out = {}
    for key in ("h", "z_enc", "z"):
        for i, t in enumerate(step[key]):
            out[f"{key}[{i}]"] = t
    for key in ("enc_grad", "pred_grad"):
        for n, t in step[key].items():
            out[f"{key}.{n}"] = t
    return out


def rel_l2(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def summarize(ref):
    """Per config: keys (sorted), their element counts, the reference's bf16-vs-fp32 rel-L2 per key, and the sampled values of
    both runs concatenated in key order (sample_index(numel, key) elements per key; the bf16 run's kept in bfloat16)."""
    rb, rf = flat_tensors(ref["bf16"]), flat_tensors(ref["fp32"])
    assert set(rb) == set(rf)
    keys = sorted(rf)
    idx = [sample_index(rf[k].numel(), k) for k in keys]
    return dict(loss_bf16=ref["bf16"]["loss_jepa"], loss_fp32=ref["fp32"]["loss_jepa"], keys=keys,
                numel=[rf[k].numel() for k in keys], e_ref=torch.tensor([rel_l2(rb[k], rf[k]) for k in keys], dtype=torch.float64),
                bf16=torch.cat([rb[k].reshape(-1)[i].float() for k, i in zip(keys, idx)]).to(torch.bfloat16),
                fp32=torch.cat([rf[k].reshape(-1)[i].float() for k, i in zip(keys, idx)]),
                dtypes=(ref["bf16"]["h_dtype"], ref["bf16"]["z_enc_dtype"], ref["bf16"]["z_dtype"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("runs", nargs="+", help="name=ref_step.pt")
    ap.add_argument("-o", "--out", required=True)
    a = ap.parse_args()
    golden = {}
    for spec in a.runs:
        name, path = spec.split("=", 1)
        golden[name] = summarize(torch.load(path))
    torch.save(golden, a.out)


if __name__ == "__main__":
    main()
