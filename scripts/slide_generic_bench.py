#!/usr/bin/env python
"""The generic path of the sliding-window scorer (SlidingScorer(..., path="auto") on a model the tensor-core scorer
cannot hold) against scoring whole windows with predict().  Seed-0 weights; the arms alternate within every round and
each arm's time is the median over --rounds of the mean over --steps calls (CUDA events).

  * trigger: MyCNN5 geometry (the shipped MyCNN5.pth), C = 10, W = 120, S = 12 (600 s every 60 s on the 5 s grid), P
    patients, fp32: one push against one predict() of the [P, 10, 120] windows, which runs the one-launch batch kernel;
  * waveform: C = 10, W = 75000, S = 7500 (600 s sliding by 60 s at 125 Hz), P patients, bf16: one push against
    predict() on the full windows (the generic front end + head), and against a shift of the window buffer by S samples
    followed by predict().

Prints one JSON line with the card's name, power limit and max SM clock, read in the same run.
    python scripts/slide_generic_bench.py [--trigger-patients 4096] [--wave-patients 1024] [--steps 20] [--rounds 5]"""
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


def model(C, W, dev):
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


def scorer_arm(sc, segs, ages):
    k = [0]

    def f():
        out = sc.push(segs[k[0] % len(segs)], ages)
        k[0] += 1
        return out
    return f


def trigger(P, steps, warmup, rounds, dev):
    C, W, S = 10, 120, 12
    m = model(C, W, dev)
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    stream = tskd_b200.synth.make_windows(P, C, W + 4 * S, "physio", seed=3, device=dev)
    segs = [stream[:, :, W + i * S:W + (i + 1) * S] for i in range(4)]
    win = stream[:, :, 4 * S:].contiguous()                             # the window after the last of the four segments
    sc = tskd_b200.SlidingScorer(m, P, S, torch.float32, path="auto")
    assert sc.path == "generic"
    for i in range(W // S):
        sc.push(stream[:, :, i * S:(i + 1) * S], ages)
    for s in segs:
        got = sc.push(s, ages)
    want = m.predict(win, ages)
    route = (m.last_path, m.gpu_launches)
    res = timed({"push": scorer_arm(sc, segs, ages), "predict_batch": lambda: m.predict(win, ages)}, steps, warmup, rounds)
    sc.close()
    return {"P": P, "C": C, "W": W, "S": S, "dtype": "fp32", "predict_route": list(route), "arms": res,
            "push_over_predict": res["push"]["ms"] / res["predict_batch"]["ms"],
            "max_abs_diff_vs_batch_kernel": float((got - want).abs().max())}


def waveform(P, steps, warmup, rounds, dev):
    C, W, S = 10, 75000, 7500
    m = model(C, W, dev)
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    bf = torch.bfloat16
    segs = [tskd_b200.synth.make_windows(P, C, S, "normal", seed=100 + i, dtype=bf, device=dev) for i in range(4)]
    sc = tskd_b200.SlidingScorer(m, P, S, bf, path="auto")
    assert sc.path == "generic"
    bufs = [tskd_b200.synth.make_windows(P, C, W, "normal", seed=7, dtype=bf, device=dev), torch.empty(P, C, W, dtype=bf, device=dev)]
    for i in range(W // S):
        sc.push(bufs[0][:, :, i * S:(i + 1) * S], ages)
    got = sc.push(segs[0], ages)
    k = [0]

    def shift_predict():
        a, b = bufs[k[0] % 2], bufs[(k[0] + 1) % 2]
        b[:, :, :W - S].copy_(a[:, :, S:])
        b[:, :, W - S:].copy_(segs[k[0] % 4])
        k[0] += 1
        return m.predict(b, ages)
    want = shift_predict()                                              # the same window the push just scored
    route = (m.last_path, m.gpu_launches)
    bit_identical = bool(torch.equal(got, want))
    win = bufs[1]
    res = timed({"push": scorer_arm(sc, segs, ages), "predict_full": lambda: m.predict(win, ages),
                 "shift_and_predict": shift_predict}, steps, warmup, rounds)
    sc.close()
    return {"P": P, "C": C, "W": W, "S": S, "dtype": "bf16", "predict_route": list(route), "arms": res,
            "predict_over_push": res["predict_full"]["ms"] / res["push"]["ms"],
            "shift_and_predict_over_push": res["shift_and_predict"]["ms"] / res["push"]["ms"],
            "logits_bit_identical_to_predict": bit_identical}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trigger-patients", type=int, default=4096)
    ap.add_argument("--wave-patients", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slide_generic_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    t = trigger(a.trigger_patients, a.steps * 10, a.warmup, a.rounds, dev)
    print(f"trigger P={t['P']}: push {t['arms']['push']['ms'] * 1e3:.1f} us, predict (batch kernel) "
          f"{t['arms']['predict_batch']['ms'] * 1e3:.1f} us (x{t['push_over_predict']:.2f})", file=sys.stderr)
    torch.cuda.empty_cache()
    w = waveform(a.wave_patients, a.steps, a.warmup, a.rounds, dev)
    print(f"waveform P={w['P']}: push {w['arms']['push']['ms']:.3f} ms, predict {w['arms']['predict_full']['ms']:.3f} ms "
          f"(x{w['predict_over_push']:.2f}), shift + predict {w['arms']['shift_and_predict']['ms']:.3f} ms "
          f"(x{w['shift_and_predict_over_push']:.2f}); bit-identical {w['logits_bit_identical_to_predict']}", file=sys.stderr)
    print(json.dumps({"metric": "SlidingScorer generic path vs predict(), MyCNN5 geometry, C = 10", "card": c,
                      "trigger": t, "waveform": w}))


if __name__ == "__main__":
    main()
