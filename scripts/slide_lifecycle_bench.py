#!/usr/bin/env python
"""Per-patient lifecycle of the sliding-window scorer (SlidingScorer.admit / discharge): what an admission with a full
history costs, and what the per-patient masking adds to a push.  MyCNN5 geometry, C = 3, W = 75000, S = 7500 (600 s
sliding by 60 s at 125 Hz), bf16, seed-0 weights.

  * admission: ``admit(all P, history [P, 3, 75000])`` next to ``model.features()`` on the same batch, which computes
    the same features into a [P, L] buffer (CUDA events over --steps calls, the two arms alternating, median of
    --rounds);
  * push: a scorer that never used the lifecycle next to one that admitted a patient (so every push also runs the
    masking kernel), the same segments (rows padded to 7504 samples), alternating, at each --patients P.

Prints one JSON line with the card's name, power limit and max SM clock, read in the same run.
    python scripts/slide_lifecycle_bench.py [--admit-patients 4096] [--patients 1024 4096] [--steps 20] [--rounds 3]"""
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

W, S, C = 75000, 7500, 3


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown", "max_sm_clock": "unknown"}


def model(dev):
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W), has_out12=oarch.has_out12).to(dev)
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


def admission(m, P, steps, warmup, rounds, dev):
    hist = tskd_b200.synth.make_windows(P, C, W, "normal", seed=7, dtype=torch.bfloat16, device=dev)
    sc = tskd_b200.SlidingScorer(m, P, S)
    idx = list(range(P))
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    res = timed({"admit": lambda: sc.admit(idx, hist), "model_features": lambda: m.features(hist)}, steps, warmup, rounds)
    # the admitted windows score at the next push: parity against predict() on the histories
    sc.admit(idx, hist)
    seg = tskd_b200.synth.make_windows(P, C, S, "normal", seed=8, dtype=torch.bfloat16, device=dev)
    got = sc.push(seg, ages)
    want = m.predict(torch.cat([hist[:, :, S:], seg], dim=2), ages)
    sc.close()
    L = m.arch.l_out
    return {"P": P, "arms": res, "admit_over_features": res["admit"]["ms"] / res["model_features"]["ms"],
            "scatter_bytes": 2 * P * L * 4,
            "parity_vs_predict": float(((got - want).abs().max() / want.abs().max().clamp_min(1e-6)).item())}


def pushes(m, P, steps, warmup, rounds, dev):
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    segs = []
    for i in range(4):
        buf = torch.empty(P, C, S + 4, dtype=torch.bfloat16, device=dev)[:, :, :S]
        buf.copy_(tskd_b200.synth.make_windows(P, C, S, "normal", seed=100 + i, dtype=torch.bfloat16, device=dev))
        segs.append(buf)
    plain, live = tskd_b200.SlidingScorer(m, P, S), tskd_b200.SlidingScorer(m, P, S)
    live.admit([0], tskd_b200.synth.make_windows(1, C, W, "normal", seed=9, dtype=torch.bfloat16, device=dev))
    k = {"plain": 0, "masked": 0}

    def push(name, sc):
        def f():
            out = sc.push(segs[k[name] % 4], ages)
            k[name] += 1
            return out
        return f

    arms = {"plain": push("plain", plain), "masked": push("masked", live)}
    for _ in range(10):                          # both scorers past their first window
        a, b = arms["plain"](), arms["masked"]()
    same = bool(torch.equal(a[1:], b[1:]))       # patient 0 was readmitted in the masked scorer
    res = timed(arms, steps, warmup, rounds)
    plain.close(); live.close()
    return {"P": P, "arms": res, "masking_ms": res["masked"]["ms"] - res["plain"]["ms"], "other_patients_bit_identical": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--admit-patients", type=int, default=4096)
    ap.add_argument("--patients", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slide_lifecycle_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    m = model(dev)
    adm = admission(m, a.admit_patients, a.steps, a.warmup, a.rounds, dev)
    print(f"admit P={adm['P']}: {adm['arms']['admit']['ms']:.3f} ms, model.features {adm['arms']['model_features']['ms']:.3f} ms "
          f"(x{adm['admit_over_features']:.2f}); parity {adm['parity_vs_predict']:.2e}", file=sys.stderr)
    torch.cuda.empty_cache()
    out = []
    for P in a.patients:
        r = pushes(m, P, a.steps * 5, a.warmup, a.rounds, dev)
        print(f"push P={P}: plain {r['arms']['plain']['ms']:.3f} ms, masked {r['arms']['masked']['ms']:.3f} ms "
              f"(+{r['masking_ms'] * 1e3:.1f} us); others bit-identical {r['other_patients_bit_identical']}", file=sys.stderr)
        out.append(r)
    print(json.dumps({"metric": "SlidingScorer lifecycle, [P, 3, 75000] bf16, stride 7500, MyCNN5 geometry", "card": c,
                      "admission": adm, "push": out}))


if __name__ == "__main__":
    main()
