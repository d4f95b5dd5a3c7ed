#!/usr/bin/env python
"""Export and import of SlidingScorer patients (SlidingScorer.export / restore): what moving a whole ward's state
costs, next to re-admitting the same patients from their raw histories.  W = 75000, S = 7500 (600 s sliding by 60 s
at 125 Hz), seed-0 weights, every patient with a complete window.

  * tensor-core path, MyCNN5 geometry, C = 3, bf16, --tc-patients P: ``export(all P)``, ``restore(all P)`` into a
    second scorer, and ``admit(all P, history [P, 3, 75000])`` (CUDA events over --steps calls, the arms alternating,
    median of --rounds);
  * generic path, C = 10, bf16, --generic-patients P: ``export`` and ``restore``.

The algorithmic bytes are the features (4 P L, read and written) and the tails (4 P C T, read and written); their
share of the H100 SXM data-sheet bandwidth, 3.35 TB/s, is given per arm.  The timed calls include their small
pageable host-to-device copy of the indices (and the counts).  Prints one JSON line with the card's name, power limit
and max SM clock, read in the same run.
    python scripts/slide_state_bench.py [--tc-patients 4096] [--generic-patients 1024] [--steps 10] [--rounds 3]"""
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

W, S = 75000, 7500
PEAK_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown", "max_sm_clock": "unknown"}


def model(C, path, dev):
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W), has_out12=oarch.has_out12,
                            path="generic" if path == "generic" else "auto").to(dev)
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


def ward(C, P, path, steps, warmup, rounds, dev, with_admit):
    m = model(C, path, dev)
    src, dst = tskd_b200.SlidingScorer(m, P, S, path=path), tskd_b200.SlidingScorer(m, P, S, path=path)
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    for t in range(W // S):                                   # every window complete
        src.push(tskd_b200.synth.make_windows(P, C, S, "normal", seed=200 + t, dtype=torch.bfloat16, device=dev), ages)
    idx = list(range(P))
    state = src.export(idx)
    arms = {"export": lambda: src.export(idx), "restore": lambda: dst.restore(idx, state)}
    hist = None
    if with_admit:
        hist = tskd_b200.synth.make_windows(P, C, W, "normal", seed=7, dtype=torch.bfloat16, device=dev)
        arms["admit_full_history"] = lambda: dst.admit(idx, hist)
    res = timed(arms, steps, warmup, rounds)
    # the restored ward scores as the source: same segment, bit-identical logits
    dst.restore(idx, state)
    seg = tskd_b200.synth.make_windows(P, C, S, "normal", seed=300, dtype=torch.bfloat16, device=dev)
    same = bool(torch.equal(src.push(seg, ages), dst.push(seg, ages)))
    L, T = m.arch.l_out, src._state_fields["tail_len"]
    nbytes = 2 * 4 * P * (L + C * T)                          # features and tails, each read once and written once
    out = {"C": C, "P": P, "path": src.path, "L": L, "T": T, "arms": res, "state_bytes_per_patient": 4 * (L + C * T),
           "algorithmic_bytes": nbytes, "restored_logits_bit_identical": same}
    for a in ("export", "restore"):
        out[f"{a}_share_of_3.35TBps"] = nbytes / (res[a]["ms"] * 1e-3) / PEAK_BPS
    if with_admit:
        out["admit_over_restore"] = res["admit_full_history"]["ms"] / res["restore"]["ms"]
        out["history_bytes_per_patient"] = 2 * C * W
    src.close(); dst.close()
    del hist, state
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tc-patients", type=int, default=4096)
    ap.add_argument("--generic-patients", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slide_state_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    res = []
    for C, P, path in ((3, a.tc_patients, "tensorcore"), (10, a.generic_patients, "generic")):
        r = ward(C, P, path, a.steps, a.warmup, a.rounds, dev, with_admit=path == "tensorcore")
        arms = ", ".join(f"{k} {v['ms']:.3f} ms" for k, v in r["arms"].items())
        print(f"{path} C={C} P={P}: {arms}; {r['algorithmic_bytes'] / 1e6:.0f} MB, export "
              f"{100 * r['export_share_of_3.35TBps']:.0f} %, restore {100 * r['restore_share_of_3.35TBps']:.0f} % of 3.35 TB/s; "
              f"bit-identical {r['restored_logits_bit_identical']}", file=sys.stderr)
        res.append(r)
    print(json.dumps({"metric": "SlidingScorer export / restore, W = 75000, S = 7500, bf16", "card": c, "wards": res}))


if __name__ == "__main__":
    main()
