#!/usr/bin/env python
"""Sliding-window scoring of long waveforms: SlidingScorer (one push of the new samples per trigger) against today's
alternative on the same streams -- predict() on the full [P, 3, W] windows, alone and together with the shift copy that
produces them.  MyCNN5 geometry, C = 3, W = 75000, S = 7500 (600 s sliding by 60 s at 125 Hz), bf16, seed-0 weights.

Per P: ms per trigger and windows/s of each arm (CUDA events over --steps triggers, the three arms alternating in
blocks, median of --rounds), the scorer's split between front end and projection + head (the library's stage events,
in a separate profiled pass), the scorer once more with contiguous 7500-sample segments (15000-byte rows, which the
library first copies into aligned staging rows), the algorithmic bytes per trigger from shapes with the HBM-bound fraction (3.35 TB/s,
H100 SXM data sheet), and the in-run parity of the scorer's logits against predict() on the same windows.  The main
scorer arm pushes segments row-padded to 7504 samples (16-byte rows), which stream without a staging copy.
    python scripts/slide_bench.py [--patients 1024 4096] [--steps 50] [--warmup 5]"""
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

HBM_BPS = 3.35e12
W, S, C = 75000, 7500, 3


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown", "max_sm_clock": "unknown"}


def run(P, steps, warmup, rounds, dev):
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W), has_out12=oarch.has_out12).to(dev)
    m.load_state_dict(O.make_ref(oarch, seed=0).state_dict())
    L = m.arch.l_out
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    segs, csegs = [], []
    for i in range(4):                      # a pool of distinct segments, pushed in turn
        c = tskd_b200.synth.make_windows(P, C, S, "normal", seed=100 + i, dtype=torch.bfloat16, device=dev).contiguous()
        buf = torch.empty(P, C, S + 4, dtype=torch.bfloat16, device=dev)[:, :, :S]
        buf.copy_(c)
        segs.append(buf)                    # rows padded to 7504 samples: 16-byte aligned, streamed in place
        csegs.append(c)                     # contiguous 7500-sample rows (15000 bytes): staged by the library
    wins = [torch.zeros(P, C, W, dtype=torch.bfloat16, device=dev) for _ in range(2)]
    cur = [0]

    def shift(seg):                         # today's producer: the window buffer moves by S and takes the new samples
        src, dst = wins[cur[0]], wins[cur[0] ^ 1]
        dst[:, :, :W - S].copy_(src[:, :, S:])
        dst[:, :, W - S:].copy_(seg)
        cur[0] ^= 1

    sc = tskd_b200.SlidingScorer(m, P, S)
    k = [0]

    def push(pool=segs):
        out = sc.push(pool[k[0] % 4], ages)
        k[0] += 1
        return out

    # fill: 10 pushes, the window buffer kept in step for the parity check
    for _ in range(10):
        shift(segs[k[0] % 4])
        got = push()
    want = m.predict(wins[cur[0]], ages)
    parity = float(((got - want).abs().max() / want.abs().max().clamp_min(1e-6)).item())

    arms = {"scorer_push": push, "scorer_push_contiguous": lambda: push(csegs), "predict_full_windows": lambda: m.predict(wins[cur[0]], ages),
            "shift_copy_and_predict": lambda: (shift(segs[k[0] % 4]), m.predict(wins[cur[0]], ages))}
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
    res = {a: {"ms_per_trigger": statistics.median(v), "windows_per_s": P / statistics.median(v) * 1e3, "ms_rounds": v}
           for a, v in ms.items()}

    # stage split of a push (separate pass: the stage events synchronise)
    m.set_profile(True)
    fe, hd = [], []
    for _ in range(10):
        push()
        fe.append(m.last_stage_ms(0)); hd.append(m.last_stage_ms(1))
    m.set_profile(False)

    tiles = max(4, ((L + 32) // 33 + 4 + 5) // 6)                 # the streaming kernels' position ranges (csrc/b2cnn_tc.cu)
    ranges = (L + 6 * tiles - 5) // (6 * tiles - 4)
    # new samples + ring read + new features + range partials written and read + tails read and written
    b_push = P * C * S * 2 + P * L * 4 + P * (S // 4) * 4 + 2 * ranges * P * 64 * 4 + P * C * 24 * 4 * 2
    b_pred = P * C * W * 2
    b_shift = 2 * P * C * W * 2
    res["scorer_push"].update(front_end_ms=statistics.median(fe), projection_head_ms=statistics.median(hd),
                              bytes_per_trigger=b_push, hbm_bound_fraction=b_push / HBM_BPS * 1e3 / res["scorer_push"]["ms_per_trigger"])
    res["scorer_push_contiguous"].update(bytes_per_trigger=b_push + 2 * P * C * S * 2,
                                         hbm_bound_fraction=(b_push + 2 * P * C * S * 2) / HBM_BPS * 1e3 / res["scorer_push_contiguous"]["ms_per_trigger"])
    res["predict_full_windows"].update(bytes_per_trigger=b_pred,
                                       hbm_bound_fraction=b_pred / HBM_BPS * 1e3 / res["predict_full_windows"]["ms_per_trigger"])
    res["shift_copy_and_predict"].update(bytes_per_trigger=b_pred + b_shift,
                                         hbm_bound_fraction=(b_pred + b_shift) / HBM_BPS * 1e3 / res["shift_copy_and_predict"]["ms_per_trigger"])
    sc.close()
    return {"P": P, "parity_vs_predict": parity,
            "speedup_vs_predict": res["predict_full_windows"]["ms_per_trigger"] / res["scorer_push"]["ms_per_trigger"],
            "speedup_vs_shift_and_predict": res["shift_copy_and_predict"]["ms_per_trigger"] / res["scorer_push"]["ms_per_trigger"],
            "arms": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--patients", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slide_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    out = []
    for P in a.patients:
        r = run(P, a.steps, a.warmup, a.rounds, dev)
        s, p, sp = r["arms"]["scorer_push"], r["arms"]["predict_full_windows"], r["arms"]["shift_copy_and_predict"]
        sc_ = r["arms"]["scorer_push_contiguous"]
        print(f"P={P}: scorer {s['ms_per_trigger']:.3f} ms/trigger (contiguous rows {sc_['ms_per_trigger']:.3f}; front end {s['front_end_ms']:.3f} + projection/head "
              f"{s['projection_head_ms']:.3f}), predict {p['ms_per_trigger']:.3f}, shift+predict {sp['ms_per_trigger']:.3f}; "
              f"x{r['speedup_vs_predict']:.2f} vs predict; parity {r['parity_vs_predict']:.2e}", file=sys.stderr)
        out.append(r)
    print(json.dumps({"metric": "sliding-window scoring [P, 3, 75000] bf16, stride 7500, MyCNN5 geometry", "card": c,
                      "results": out}))


if __name__ == "__main__":
    main()
