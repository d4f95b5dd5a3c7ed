#!/usr/bin/env python
"""SlidingScorer(mode="sequence"): what carrying each patient's LSTM state from push to push costs next to an
independent scorer, and what it replaces.  Seed-0 weights.

  1. tensor-core path, MyCNN5 geometry, C = 3, W = 75000, S = 7500 (600 s sliding by 60 s at 125 Hz), bf16, padded
     rows ([P, 3, 7504][:, :, :7500] views), P = 1024 and 4096: a push of an independent and of a sequence scorer;
  2. generic path, [4096, 10, 120] fp32, S = 12 (the reference's 600 s window sliding by 60 s at 5 s samples): the same
     two arms;
  3. the workaround sequence mode replaces: predict_record(mode="sequence") over each patient's whole history after
     1 h (60 pushes, 51 windows) at P = 1024, against one sequence push;
  4. in a torch.profiler run of its own per arm, the device time per push of the head kernels (the step kernel in
     sequence mode, the reduction and head kernels in independent mode) and of all kernels.

Arms alternate within every round (CUDA events over --steps calls, median of --rounds).  Prints one JSON line with the
card's name, power limit and max SM clock, read in the same run.
    python scripts/slide_sequence_bench.py [--steps 20] [--warmup 3] [--rounds 5]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import tskd_b200
from oracle import mycnn_torch as O


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown", "max_sm_clock": "unknown"}


def model(C, W, path, dev):
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W), has_out12=oarch.has_out12, path=path).to(dev)
    m.load_state_dict(O.make_ref(oarch, seed=0).state_dict())
    return m


def timed(arms, steps, warmup, rounds):
    """median ms per call of each arm; the arms alternate within every round"""
    for f in arms.values():
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    ms = {a: [] for a in arms}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for a, f in arms.items():
            e0.record()
            for _ in range(steps):
                f()
            e1.record()
            torch.cuda.synchronize()
            ms[a].append(e0.elapsed_time(e1) / steps)
    return {a: {"ms": statistics.median(v), "ms_rounds": v} for a, v in ms.items()}


HEAD_KERNELS = ("slide_seq_step_kernel", "head_reduce_independent_kernel", "reduce_gates_kernel", "head_independent_kernel")


def kernel_ms(fn, steps):
    """device ms per call of fn: the head kernels and all kernels, from a torch.profiler run of its own"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {"head": 0.0, "all": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if not t or e.key.startswith(("cudaLaunch", "cudaMemcpy", "cudaEvent", "cudaStream", "cudaFunc")):
            continue
        out["all"] += t
        if any(n in e.key for n in HEAD_KERNELS):
            out["head"] += t
    return {g: v / 1e3 / steps for g, v in out.items()}


def ward(m, P, S, dtype, path, steps, warmup, rounds, dev, pad=0):
    """an independent and a sequence scorer pushed with the same segments once every window is complete"""
    C, W = m.arch.in_channels, m.arch.window
    sc = {mode: tskd_b200.SlidingScorer(m, P, S, dtype=dtype, path=path, mode=mode) for mode in ("independent", "sequence")}
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    segs = [torch.empty(P, C, S + pad, dtype=dtype, device=dev)[:, :, :S] for _ in range(2)]
    for j, s in enumerate(segs):
        s.copy_(tskd_b200.synth.make_windows(P, C, S, "normal", seed=300 + j, dtype=dtype, device=dev))
    for t in range(-(-W // S)):
        for s in sc.values():
            s.push(segs[t % 2], ages)
    arms = {mode: (lambda s: lambda: s.push(segs[0], ages))(s) for mode, s in sc.items()}
    res = timed(arms, steps, warmup, rounds)
    prof = {mode: kernel_ms(f, steps) for mode, f in arms.items()}
    out = {"P": P, "C": C, "W": W, "S": S, "dtype": str(dtype), "path": sc["sequence"].path, "arms": res, "device_ms_per_push": prof,
           "sequence_over_independent": res["sequence"]["ms"] / res["independent"]["ms"],
           "lstm_state_bytes_per_push": 2 * 256 * P}
    for s in sc.values():
        s.close()
    return out


def workaround(m, P, S, n_push, steps, warmup, rounds, dev):
    """predict_record(mode="sequence") over the whole history after n_push pushes against one sequence push"""
    C, W = m.arch.in_channels, m.arch.window
    N = n_push * S
    x = tskd_b200.synth.make_windows(P, C, N, "normal", seed=5, dtype=torch.bfloat16, device=dev)
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    sc = tskd_b200.SlidingScorer(m, P, S, mode="sequence")
    for t in range(n_push):
        out = sc.push(x[:, :, t * S:(t + 1) * S], ages)
    rec = m.predict_record(x, S, ages, mode="sequence")
    err = float((rec[:, -1] - out).abs().max())
    seg = x[:, :, :S]
    arms = {"predict_record_history": lambda: m.predict_record(x, S, ages, mode="sequence"), "sequence_push": lambda: sc.push(seg, ages)}
    res = timed(arms, max(steps // 4, 2), warmup, rounds)
    sc.close()
    return {"P": P, "pushes": n_push, "history_samples": N, "windows": rec.shape[1], "arms": res,
            "record_over_push": res["predict_record_history"]["ms"] / res["sequence_push"]["ms"],
            "max_abs_diff_last_window": err}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    m5 = model(3, 75000, "auto", dev)
    res = {"tensorcore": [ward(m5, P, 7500, torch.bfloat16, "tensorcore", a.steps, a.warmup, a.rounds, dev, pad=4) for P in (1024, 4096)]}
    mg = model(10, 120, "generic", dev)
    res["generic"] = [ward(mg, 4096, 12, torch.float32, "generic", a.steps, a.warmup, a.rounds, dev)]
    del mg
    res["workaround"] = workaround(m5, 1024, 7500, 60, a.steps, a.warmup, a.rounds, dev)
    for r in res["tensorcore"] + res["generic"]:
        print(f"{r['path']} P={r['P']}: independent {r['arms']['independent']['ms']:.4f} ms, sequence {r['arms']['sequence']['ms']:.4f} ms "
              f"({r['sequence_over_independent']:.3f}x); head kernels {json.dumps(r['device_ms_per_push'])}", file=sys.stderr)
    w = res["workaround"]
    print(f"workaround P={w['P']} after {w['pushes']} pushes: predict_record {w['arms']['predict_record_history']['ms']:.3f} ms vs "
          f"push {w['arms']['sequence_push']['ms']:.4f} ms", file=sys.stderr)
    print(json.dumps({"metric": "SlidingScorer sequence mode", "card": c, **res}))


if __name__ == "__main__":
    main()
