#!/usr/bin/env python
"""predict_record(mode="sequence"): each recording's windows scored as one LSTM sequence (bin/utils.py run_model).

Workloads (MyCNN5 geometry, seed-0 weights):
  1. run_model's own shape for a cohort: C = 10 fp32, [1024, 10, 17280] (24 h on the 5-second grid), W = S = 120:
     predict_record(mode="sequence") against the only route before it, a Python loop of model(windows_b, age_b) per
     recording on create_batch-style windows copied out of the recording (143 per recording: create_batch drops the
     last full window, so the comparison uses out[:, :-1]);
  2. [4096, 3, 142500] bf16, W = 75000, S = 7500 (10 windows per recording): sequence against independent mode, the
     scan's added cost;
  3. one 24 h recording at 125 Hz, [1, 3, 10 800 000] bf16, S = 7500: a 1431-step scan in one warp.
Arms alternate within every round (CUDA events around --steps calls, median of --rounds).  A torch.profiler run of its
own gives each arm's kernels' device time per call; ``scan_us_per_step`` is head_sequence_kernel's time over n_w.
``max_abs_diff`` is the sequence outputs against model(windows_b, age_b) per recording.  Prints the card's name,
power limit and max SM clock, read in the same run, and one JSON line.
    python scripts/record_sequence_bench.py [--steps 3] [--rounds 5] [--only 1,2,3]"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import tskd_b200
from record_bench import model, timed
from slide_heads_bench import card


def kernel_ms(fn, steps):
    """{kernel name: device ms per call} of fn, from a torch.profiler run"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if not t or e.key.startswith(("cudaLaunch", "cudaMemcpy", "cudaEvent", "cudaStream", "cudaFunc", "cudaMemset")):
            continue
        out[e.key.split("(")[0][:60]] = t / 1e3 / steps
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def loop_windows(m, x, age, S, drop_last):
    """model(windows_b, age_b) per recording on windows copied out of it, [B, n]"""
    W = m.arch.window
    rows = []
    for b in range(x.shape[0]):
        win = x[b].unfold(1, W, S).permute(1, 0, 2)
        if drop_last:
            win = win[:-1]
        rows.append(m(win.contiguous(), age[b:b + 1]))
    return torch.stack(rows)


def scan_row(tag, m, x, age, S, steps, rounds, drop_last, loop_arm):
    W = m.arch.window
    B, N = x.shape[0], x.shape[2]
    n_w = (N - W) // S + 1
    seq = m.predict_record(x, S, age, mode="sequence")
    path = m.last_path
    ref = loop_windows(m, x, age, S, drop_last)
    diff = float((seq[:, :ref.shape[1]] - ref).abs().max())
    del ref
    arms = {"sequence": lambda: m.predict_record(x, S, age, mode="sequence")}
    if loop_arm:
        arms["loop"] = lambda: loop_windows(m, x, age, S, drop_last)
    else:
        arms["independent"] = lambda: m.predict_record(x, S, age)
    res = timed(arms, steps, rounds)
    kern = {"sequence": kernel_ms(arms["sequence"], max(1, steps))}
    if not loop_arm:
        kern["independent"] = kernel_ms(arms["independent"], max(1, steps))
    scan = next((v for k, v in kern["sequence"].items() if "head_sequence_kernel" in k), float("nan"))
    return {"workload": tag, "B": B, "C": x.shape[1], "N": N, "W": W, "S": S, "n_w": n_w, "dtype": str(x.dtype), "path": path,
            "arms": res, "kernel_ms": kern, "scan_ms": scan, "scan_us_per_step": scan * 1e3 / n_w, "max_abs_diff": diff}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--only", default="1,2,3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("record_sequence_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    only = set(a.only.split(","))
    rows = []
    if "1" in only:
        m = model(10, 120, dev)
        x = tskd_b200.synth.make_windows(1024, 10, 17280, "physio", seed=1, dtype=torch.float32, device=dev)
        age = tskd_b200.synth.make_ages(1024, seed=1, device=dev)
        rows.append(scan_row("1-run_model-1024x17280", m, x, age, 120, 1, a.rounds, True, True))
        del m, x
    if only & {"2", "3"}:
        m = model(3, 75000, dev)
        if "2" in only:
            x = tskd_b200.synth.make_windows(4096, 3, 142500, "normal", seed=2, dtype=torch.bfloat16, device=dev)
            age = tskd_b200.synth.make_ages(4096, seed=2, device=dev)
            rows.append(scan_row("2-4096x10", m, x, age, 7500, a.steps, a.rounds, False, False))
            del x
            torch.cuda.empty_cache()
        if "3" in only:
            x = tskd_b200.synth.make_windows(1, 3, 10_800_000, "normal", seed=3, dtype=torch.bfloat16, device=dev)
            rows.append(scan_row("3-24h", m, x, torch.tensor([63.0], device=dev), 7500, a.steps, a.rounds, False, False))
    for r in rows:
        arms = ", ".join(f"{k} {v['ms']:.3f} ms" for k, v in r["arms"].items())
        print(f"  {r['workload']} ({r['path']}): {arms}; scan {r['scan_ms'] * 1e3:.1f} us = {r['scan_us_per_step']:.3f} us/step; "
              f"max |seq - loop| {r['max_abs_diff']:.3e}", file=sys.stderr)
        for arm, k in r["kernel_ms"].items():
            print(f"    {arm}: " + ", ".join(f"{n} {v * 1e3:.1f} us" for n, v in k.items()), file=sys.stderr)
    print(json.dumps({"metric": "predict_record(mode='sequence')", "card": c, "rows": rows}))


if __name__ == "__main__":
    main()
