"""Attention kernels alone at the training step's launch layouts, for one or more builds of libvjepa_b200.so.

    python tools/bench_attn.py LIB [LIB ...] [--launches 50] [--rounds 5]

Each LIB is a path to a libvjepa_b200.so, loaded side by side through ctypes; the first is the baseline.  Layouts (16
heads, seeded random bf16 inputs; padded head lanes are zero):
  target     [1568] x 32, hd 64, forward (the target encoder)
  context    [360] x 32 + [48] x 32, hd 64, forward and backward (the context encoder, both masks in one launch)
  predictor  [1184] x 32 + [1192] x 32, hd 24 -> 32, forward and backward
  vith       [1568] x 24, hd 80 -> 128, forward (ViT-H's encoder)
Timing: CUDA events around `--launches` back-to-back launches after warm-up, mean per launch; the builds take turns in
every one of `--rounds` rounds, first place rotating from round to round, so clock and power drift hit them alike.  The card's name, power limit and the SM clock
nvidia-smi sampled while timing are printed with the numbers.

With two or more builds, every build's O, lse2 and dqkv must be bitwise equal to the first's: at the layouts above and
at every L = 1 ... 385 for hd 24 (-> 32), 64 and 80 (-> 128), sequences [L, 97, L].  The backward of every build gets
the first build's O and lse2.  Exits 1 on any difference.  Writes nothing into the repository.
"""
import argparse
import ctypes
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from tools.bench_offsize import _card  # noqa: E402

P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
H = 16
LAYOUTS = (  # name, sequence lengths, real head dim, kernel head dim, backward too
    ("target", [1568] * 32, 64, 64, False),
    ("context", [360] * 32 + [48] * 32, 64, 64, True),
    ("predictor", [1184] * 32 + [1192] * 32, 24, 32, True),
    ("vith", [1568] * 24, 80, 128, False),
)


class Lib:
    def __init__(self, path):
        self.path = os.path.abspath(path)
        self.so = ctypes.CDLL(self.path)
        self.so.vj_attn_fwd.restype = I
        self.so.vj_attn_fwd.argtypes = [P, P, P, P, I, I, I, I, I, F, P]
        self.so.vj_attn_bwd.restype = I
        self.so.vj_attn_bwd.argtypes = [P, P, P, P, P, P, P, P, I, I, I, I, I, F, P]
        self.so.vj_last_error_string.restype = ctypes.c_char_p

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f"{self.path}: {what} rc={rc}: {self.so.vj_last_error_string().decode()}")

    def fwd(self, pb, out, lse2):
        self._check(self.so.vj_attn_fwd(pb.qkv.data_ptr(), out.data_ptr(), lse2.data_ptr(), pb.cu.data_ptr(), pb.nseq,
                                        pb.max_len, pb.H, pb.hd, pb.T, pb.scale, pb.stream), "vj_attn_fwd")

    def bwd(self, pb, dqkv):
        self._check(self.so.vj_attn_bwd(pb.qkv.data_ptr(), pb.out.data_ptr(), pb.dout.data_ptr(), pb.lse2.data_ptr(),
                                        pb.delta.data_ptr(), dqkv.data_ptr(), None, pb.cu.data_ptr(), pb.nseq,
                                        pb.max_len, pb.H, pb.hd, pb.T, pb.scale, pb.stream), "vj_attn_bwd")


class Problem:
    """Seeded random q, k, v, dO of one launch; padded head lanes (hd_real .. hd) are zero."""

    def __init__(self, lens, hd_real, hd, heads, seed, dev):
        self.nseq, self.max_len, self.T, self.H, self.hd = len(lens), max(lens), sum(lens), heads, hd
        self.scale = 1.0 / math.sqrt(hd_real)
        self.stream = torch.cuda.current_stream(dev).cuda_stream
        cu = [0]
        for n in lens:
            cu.append(cu[-1] + n)
        self.cu = torch.tensor(cu, dtype=torch.int32, device=dev)
        g = torch.Generator(device=dev).manual_seed(seed)
        qkv = torch.randn(self.T, 3, heads, hd, generator=g, device=dev)
        dout = torch.randn(self.T, heads, hd, generator=g, device=dev)
        qkv[..., hd_real:] = 0
        dout[..., hd_real:] = 0
        self.qkv = qkv.to(torch.bfloat16).reshape(self.T, 3 * heads * hd).contiguous()
        self.dout = dout.to(torch.bfloat16).reshape(self.T, heads * hd).contiguous()
        self.delta = torch.empty(heads * self.T, dtype=torch.float32, device=dev)
        self.out = self.lse2 = None

    def new_out(self):
        out = torch.full((self.T, self.H * self.hd), float("nan"), dtype=torch.bfloat16, device=self.qkv.device)
        return out, torch.full((self.H * self.T,), float("nan"), dtype=torch.float32, device=self.qkv.device)

    def new_dqkv(self):
        return torch.full_like(self.qkv, float("nan"))


def _same(a, b):
    return torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                       b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))


def compare(libs, pb, do_bwd):
    """Names of the outputs in which some build differs from libs[0] (bitwise); leaves libs[0]'s O / lse2 in pb."""
    outs = []
    for lib in libs:
        o, l2 = pb.new_out()
        lib.fwd(pb, o, l2)
        outs.append((o, l2))
    pb.out, pb.lse2 = outs[0]
    bad = []
    for k, (o, l2) in enumerate(outs[1:], 1):
        if not _same(o, outs[0][0]):
            bad.append(f"O[{k}]")
        if not _same(l2, outs[0][1]):
            bad.append(f"lse2[{k}]")
    if do_bwd:
        grads = []
        for lib in libs:
            d = pb.new_dqkv()
            lib.bwd(pb, d)
            grads.append(d)
        bad += [f"dqkv[{k}]" for k, d in enumerate(grads[1:], 1) if not _same(d, grads[0])]
    torch.cuda.synchronize()
    return bad


def time_ms(fn, launches):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / launches


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("libs", nargs="+", help="paths of libvjepa_b200.so builds; the first is the baseline")
    ap.add_argument("--launches", type=int, default=50, help="timed launches per (build, round, kernel); at least 20")
    ap.add_argument("--rounds", type=int, default=5, help="rounds in which the builds take turns; at least 3")
    ap.add_argument("--no-sweep", action="store_true", help="skip the L = 1 ... 385 bitwise sweep")
    args = ap.parse_args()
    if args.launches < 20 or args.rounds < 3:
        ap.error("--launches must be at least 20 and --rounds at least 3")
    if not torch.cuda.is_available():
        sys.exit("bench_attn measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    libs = [Lib(p) for p in args.libs]
    failures = []

    problems = {name: Problem(lens, hdr, hd, H, 1000 + i, dev) for i, (name, lens, hdr, hd, _) in enumerate(LAYOUTS)}
    for name, _, _, _, do_bwd in LAYOUTS:
        if len(libs) > 1:
            failures += [f"{name}: {b}" for b in compare(libs, problems[name], do_bwd)]
        else:
            pb = problems[name]
            pb.out, pb.lse2 = pb.new_out()
            libs[0].fwd(pb, pb.out, pb.lse2)

    # kernels to time: (layout, pass); each build writes into its own buffers
    work = []
    for name, lens, hdr, hd, do_bwd in LAYOUTS:
        pb = problems[name]
        bufs = [pb.new_out() for _ in libs]
        work.append((name, "fwd", [lambda lib=lib, pb=pb, b=b: lib.fwd(pb, *b) for lib, b in zip(libs, bufs)]))
        if do_bwd:
            grads = [pb.new_dqkv() for _ in libs]
            work.append((name, "bwd", [lambda lib=lib, pb=pb, d=d: lib.bwd(pb, d) for lib, d in zip(libs, grads)]))
    for _, _, fns in work:   # warm-up: module load, shared-memory attributes, clocks
        for fn in fns:
            for _ in range(5):
                fn()
    torch.cuda.synchronize()

    sampler = ClockSampler(0)
    try:
        ms = {(n, ps, k): [] for n, ps, fns in work for k in range(len(fns))}
        for r in range(args.rounds):
            for n, ps, fns in work:
                # the build timed first after another kernel runs at a different clock: rotate who goes first
                for k in [(r + i) % len(fns) for i in range(len(fns))]:
                    ms[(n, ps, k)].append(time_ms(fns[k], args.launches))
    finally:
        clocks = sampler.stop()

    if len(libs) > 1 and not args.no_sweep:
        for hdr, hd in ((24, 32), (64, 64), (80, 128)):
            for L in range(1, 386):
                pb = Problem([L, 97, L], hdr, hd, 2, L, dev)
                failures += [f"sweep hd {hdr} L {L}: {b}" for b in compare(libs, pb, True)]

    gpu, plimit = _card()
    print(f"# {gpu}, power limit {plimit} W, SM clock while timing: {clocks}")
    print(f"# mean ms per launch over {args.launches} launches; min-max over {args.rounds} alternating rounds")
    result = {"gpu": gpu, "power_limit_w": plimit, "clocks": clocks, "launches": args.launches,
              "rounds": args.rounds, "libs": [lib.path for lib in libs], "kernels": {}}
    for n, ps, fns in work:
        row = []
        for k in range(len(fns)):
            v = ms[(n, ps, k)]
            row.append({"min": round(min(v), 4), "max": round(max(v), 4), "median": round(sorted(v)[len(v) // 2], 4)})
        result["kernels"][f"{n}_{ps}"] = row
        cells = "  ".join(f"[{k}] {r['median']:.4f} ({r['min']:.4f}-{r['max']:.4f})" for k, r in enumerate(row))
        ratio = "" if len(row) < 2 else "  speedup " + " ".join(
            f"{row[0]['median'] / r['median']:.3f}" for r in row[1:])
        print(f"{n:10s} {ps}  {cells}{ratio}")
    if len(libs) > 1:
        result["bitwise_equal"] = not failures
        result["differences"] = failures[:50]
        print(f"# bitwise: {'all equal' if not failures else f'{len(failures)} differences, first: ' + str(failures[:10])}")
    print(json.dumps(result), flush=True)
    sys.exit(1 if failures else 0)


if __name__ == "__main__":
    main()
