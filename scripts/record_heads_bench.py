#!/usr/bin/env python
"""Candidate heads over whole recordings: predict_record(heads=[K models]) against the 1 + K separate predict_record
calls it replaces (the model's and each candidate's), K = 0, 1, 3, 7, in both modes.

Workloads (MyCNN5 geometry, seed-0 weights; the K heads share its conv weights, with seeded LSTM / Linear weights and
their own age_coef):
  (a) [4096, 3, 75000 + 9 x 7500] bf16, W = 75000, S = 7500: 10 windows per recording, tensor cores;
  (b) one 24 h recording at 125 Hz, [1, 3, 10 800 000] bf16, S = 7500: 1431 windows, tensor cores;
  (g) the generic path, [1024, 10, 7200] fp32 at W = 120, S = 12.
Arms, alternating within every round (CUDA events around --steps calls, median of --rounds): ``heads`` (one call) and
``separate`` (1 + K calls).  Every row of the heads call is checked torch.equal to its separate call in the same run
(``rows_equal``).  Prints the card's name, power limit and max SM clock, read in the same run, and one JSON line.
    python scripts/record_heads_bench.py [--steps 3] [--rounds 5] [--only a,b,g] [--ks 0,1,3,7]"""
import argparse
import json
import os
import sys
from dataclasses import replace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import tskd_b200
from oracle import mycnn_torch as O
from record_bench import timed
from slide_heads_bench import card


def family(C, W, K, dev, path="auto"):
    """the seed-0 model and K heads of its front end"""
    ref = O.make_ref(O.stretched(O.ARCH_MYCNN5, C, W), seed=0)
    arch = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W)
    sd = dict(ref.state_dict())
    models = []
    for i in range(K + 1):
        m = tskd_b200.B200MyCNN(replace(arch, age_coef=arch.age_coef if i == 0 else 1e-3 * i), has_out12=ref.arch.has_out12,
                                path=path).to(dev)
        g = torch.Generator().manual_seed(100 + i)
        m.load_state_dict(sd if i == 0 else {k: v if k.startswith(("conv", "affine")) else v + 0.05 * torch.randn(v.shape, generator=g)
                                              for k, v in sd.items()})
        models.append(m)
    return models


def workload(tag, C, W, B, N, S, dtype, path, ks, steps, rounds, dev):
    models = family(C, W, max(ks), dev, path)
    x = tskd_b200.synth.make_windows(B, C, N, "normal", seed=1, dtype=dtype, device=dev)
    age = tskd_b200.synth.make_ages(B, seed=1, device=dev)
    m0 = models[0]
    res = []
    for mode in ("independent", "sequence"):
        for K in ks:
            hs = models[1:1 + K]
            heads = lambda: m0.predict_record(x, S, age, path=path, mode=mode, heads=hs)
            separate = lambda: [m.predict_record(x, S, age, path=path, mode=mode) for m in [m0] + hs]
            out, sep = heads(), separate()
            rows = [out] if K == 0 else list(out)
            equal = all(torch.equal(a, b) for a, b in zip(rows, sep))
            del out, sep
            t = timed({"heads": heads, "separate": separate}, steps, rounds)
            res.append({"workload": tag, "mode": mode, "K": K, "B": B, "N": N, "W": W, "S": S, "path": m0.last_path,
                        "heads_ms": t["heads"]["ms"], "separate_ms": t["separate"]["ms"],
                        "speedup": t["separate"]["ms"] / t["heads"]["ms"], "rows_equal": equal, "rounds": t})
            print(f"{tag} {mode:11s} K={K}: heads {t['heads']['ms']:8.3f} ms  separate {t['separate']['ms']:8.3f} ms  "
                  f"x{res[-1]['speedup']:.2f}  rows_equal={equal}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--only", default="a,b,g")
    ap.add_argument("--ks", default="0,1,3,7")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("record_heads_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = card()
    print(info, flush=True)
    ks = [int(k) for k in args.ks.split(",")]
    only = args.only.split(",")
    out = []
    if "a" in only:
        out += workload("a", 3, 75000, 4096, 75000 + 9 * 7500, 7500, torch.bfloat16, "tensorcore", ks, args.steps, args.rounds, dev)
    if "b" in only:
        out += workload("b-24h", 3, 75000, 1, 10_800_000, 7500, torch.bfloat16, "tensorcore", ks, args.steps, args.rounds, dev)
    if "g" in only:
        out += workload("g-generic", 10, 120, 1024, 7200, 12, torch.float32, "generic", ks, args.steps, args.rounds, dev)
    print(json.dumps({"card": info, "results": out}))
    if not all(r["rows_equal"] for r in out):
        raise SystemExit("a row of predict_record(heads=...) differs from its separate call")


if __name__ == "__main__":
    main()
