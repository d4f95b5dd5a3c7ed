#!/usr/bin/env python
"""Heads with shorter windows over one SlidingScorer's features (set_heads(..., shorter_windows=True)): risk over the
last 60 s, 300 s and 600 s of a 125 Hz waveform from one scorer, next to one scorer per window.  W = 75000, S = 7500
(600 s sliding by 60 s), MyCNN5 geometry, C = 3, bf16, --patients P, padded rows ([P, 3, 7504][:, :, :7500] views).
M0 has seed-0 weights at W; the heads at W_k = 7500, 37500 and 75000 have M0's conv weights and seeded LSTM / Linear
weights (their W_ih has L_k = L_out(W_k) columns).

Arms, alternating within every round (CUDA events over --steps pushes, median of --rounds):
  * ``push``: the scorer without heads;
  * ``heads_<W_k>``: ``push(heads=True)`` with the one head at W_k (its cost over ``push`` is what the head adds);
  * ``heads_all``: ``push(heads=True)`` with the three heads;
  * ``separate_<W_k>``: a scorer of the head's model at its own window W_k, pushed with the same segments;
  * ``separate_all``: the scorer of M0 and the three separate scorers.
In the same run every row of ``heads_all`` is checked with torch.equal against its separate scorer, and a torch.profiler
run of its own gives the device time of the projection and head kernels per push.  Prints one JSON line with the card's
name, power limit and max SM clock, read in the same run.
    python scripts/slide_horizons_bench.py [--patients 4096] [--steps 20] [--rounds 3]"""
import argparse
import json
import os
import statistics
import sys
from dataclasses import replace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import tskd_b200
from oracle import mycnn_torch as O
from slide_heads_bench import card, kernel_ms, timed

W, S, C = 75000, 7500, 3
HEAD_WINDOWS = (7500, 37500, 75000)


def models(dev):
    """M0 at W and one model per head window with M0's conv weights"""
    base = O.stretched(O.ARCH_MYCNN5, C, W)
    sd0 = O.make_ref(base, seed=0).state_dict()
    conv = {k: v for k, v in sd0.items() if k.startswith("conv")}
    out = []
    for i, Wk in enumerate((W,) + HEAD_WINDOWS):
        sd = dict(sd0) if i == 0 else {**O.make_ref(replace(base, window=Wk), seed=100 + i).state_dict(), **conv}
        m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, Wk), has_out12=base.has_out12).to(dev)
        m.load_state_dict(sd)
        out.append(m)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--patients", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slide_horizons_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    P = a.patients
    ms = models(dev)
    m0, hm = ms[0], ms[1:]
    base = tskd_b200.SlidingScorer(m0, P, S)
    one = {}
    for Wk, m in zip(HEAD_WINDOWS, hm):
        one[Wk] = tskd_b200.SlidingScorer(m0, P, S)
        one[Wk].set_heads([m], shorter_windows=True)
    allh = tskd_b200.SlidingScorer(m0, P, S)
    allh.set_heads(hm, shorter_windows=True)
    sep = {Wk: tskd_b200.SlidingScorer(m, P, S) for Wk, m in zip(HEAD_WINDOWS, hm)}
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    Sp = (S + 7) // 8 * 8
    segs = [torch.empty(P, C, Sp, dtype=torch.bfloat16, device=dev)[:, :, :S] for _ in range(2)]
    for j, s in enumerate(segs):
        s.copy_(tskd_b200.synth.make_windows(P, C, S, "normal", seed=300 + j, dtype=torch.bfloat16, device=dev))
    scs = [base, allh] + list(one.values()) + list(sep.values())
    for t in range(W // S):                                                    # every window complete
        for sc in scs:
            sc.push(segs[t % 2], ages)
    got = allh.push(segs[1], ages, heads=True)
    want = [base.push(segs[1], ages)] + [sep[Wk].push(segs[1], ages) for Wk in HEAD_WINDOWS]
    same = {str(wr): bool(torch.equal(got[i], want[i])) for i, wr in enumerate((W,) + HEAD_WINDOWS)}
    arms = {"push": lambda: base.push(segs[0], ages)}
    for Wk in HEAD_WINDOWS:
        arms[f"heads_{Wk}"] = (lambda sc: lambda: sc.push(segs[0], ages, heads=True))(one[Wk])
        arms[f"separate_{Wk}"] = (lambda sc: lambda: sc.push(segs[0], ages))(sep[Wk])
    arms["heads_all"] = lambda: allh.push(segs[0], ages, heads=True)
    arms["separate_all"] = lambda: [sc.push(segs[0], ages) for sc in [base] + list(sep.values())]
    res = timed(arms, a.steps, a.warmup, a.rounds)
    prof = {"push": kernel_ms(lambda: base.push(segs[0], ages), a.steps),
            "heads_all": kernel_ms(lambda: allh.push(segs[0], ages, heads=True), a.steps)}
    for Wk in HEAD_WINDOWS:
        prof[f"heads_{Wk}"] = kernel_ms(lambda: one[Wk].push(segs[0], ages, heads=True), a.steps)
    added = {str(Wk): res[f"heads_{Wk}"]["ms"] - res["push"]["ms"] for Wk in HEAD_WINDOWS}
    for k, v in res.items():
        print(f"  {k}: {v['ms']:.3f} ms ({', '.join(f'{x:.3f}' for x in v['ms_rounds'])})", file=sys.stderr)
    print(f"  a head adds (ms over push): {json.dumps(added)}", file=sys.stderr)
    print(f"  device ms per push: {json.dumps(prof)}", file=sys.stderr)
    print(f"  rows torch.equal to separate scorers: {same}", file=sys.stderr)
    print(json.dumps({"metric": "SlidingScorer heads with shorter windows, W = 75000, S = 7500, bf16", "card": c, "P": P,
                      "L": m0.arch.l_out, "head_windows": HEAD_WINDOWS, "L_k": [m.arch.l_out for m in hm], "arms": res,
                      "head_added_ms": added, "device_ms_per_push": prof, "rows_equal_to_separate_scorers": same}))
    for sc in scs:
        sc.close()


if __name__ == "__main__":
    main()
