#!/usr/bin/env python
"""Check that two builds of libb2cnn compute byte-identical results (needs a GPU).

Runs itself once per library (B2CNN_LIB selects the build; a process loads one), each run computing on the same
inputs, with seed-0 MyCNN5 weights:
  * predict() logits at [--batch, 3, 75000] bf16 (the bench.py workload: the fused streaming kernel, gates out);
  * model.features() at [--feat-batch, 3, 75000] bf16 (the feature-row kernel);
  * one SlidingScorer push after a full window of pushes (the feature-ring kernel), logits and the ring's features;
then compares every array bit for bit.

    python scripts/compare_builds.py --baseline-lib /path/to/parent/libb2cnn.so [--lib /path/to/libb2cnn.so]
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, S, C = 75000, 7500, 3


def dump(path: str, batch: int, feat_batch: int, patients: int) -> None:
    sys.path.insert(0, ROOT)
    import torch

    import tskd_b200
    from oracle import mycnn_torch as O

    dev = "cuda:0"
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W), has_out12=oarch.has_out12).to(dev)
    m.load_state_dict(O.make_ref(oarch, seed=0).state_dict())
    out = {}
    x = tskd_b200.synth.make_windows(batch, C, W, "normal", seed=7, dtype=torch.bfloat16, device=dev)
    ages = tskd_b200.synth.make_ages(batch, seed=7, device=dev)
    out["predict_logits"] = m.predict(x, ages)
    out["predict_path"] = np.array([m.last_path])
    out["features"] = m.features(x[:feat_batch])
    del x
    sc = tskd_b200.SlidingScorer(m, patients, S)
    pages = tskd_b200.synth.make_ages(patients, seed=9, device=dev)
    for i in range(W // S + 1):
        seg = tskd_b200.synth.make_windows(patients, C, S, "normal", seed=200 + i, dtype=torch.bfloat16, device=dev)
        got = sc.push(seg.contiguous(), pages)
    out["slide_logits"] = got
    torch.cuda.synchronize()
    np.savez(path, **{k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in out.items()})


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--baseline-lib", required=True)
    ap.add_argument("--lib", default=None, help="the build under test (default: the package's own lib/libb2cnn.so)")
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--feat-batch", type=int, default=1024)
    ap.add_argument("--patients", type=int, default=1024)
    ap.add_argument("--dump", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump:
        dump(args.dump, args.batch, args.feat_batch, args.patients)
        return 0
    runs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, lib in (("baseline", args.baseline_lib), ("candidate", args.lib)):
            env = dict(os.environ)
            env.pop("B2CNN_LIB", None)
            if lib:
                env["B2CNN_LIB"] = os.path.abspath(lib)
            path = os.path.join(tmp, name + ".npz")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--dump", path, "--batch", str(args.batch),
                                   "--feat-batch", str(args.feat_batch), "--patients", str(args.patients),
                                   "--baseline-lib", "-"], env=env)
            runs[name] = dict(np.load(path))
    ok = True
    for k, a in runs["baseline"].items():
        b = runs["candidate"][k]
        same = a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()
        ok &= same
        extra = "" if a.dtype.kind == "U" else f", max |diff| {np.abs(a.astype(np.float64) - b.astype(np.float64)).max():.3g}" if a.shape == b.shape else ""
        print(f"{k:16s} {str(a.shape):16s} {'byte-identical' if same else 'DIFFERENT'}{extra}  {a.ravel()[:1]}")
    print("all byte-identical" if ok else "builds differ")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
