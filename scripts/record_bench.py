#!/usr/bin/env python
"""Every sliding window of whole recordings (B200MyCNN.predict_record) against the two other ways to score them.

Workloads (MyCNN5 geometry, seed-0 weights):
  (a) [4096, 3, 75000 + 9 x 7500] bf16, W = 75000, S = 7500: 10 windows per recording;
  (b) one 24 h recording at 125 Hz, [1, 3, 10 800 000] bf16, S = 7500: 1431 windows;
  (c) (a) at the 40 % overlap stride of bin/utils.py's create_batch, S = 45000: 2 windows per recording;
  (d) the generic path, [1024, 10, 120 x 60] fp32 at W = 120 with S = 72 and S = 12.
Arms, alternating within every round (CUDA events around --steps calls, median of --rounds):
  * ``record``: predict_record(x, S);
  * ``predict``: the windows copied out of the recording (in chunks of at most 4096 windows of W = 75000) and scored
    by predict(); at (d) the whole [B n_w, 10, 120] batch at once (the one-launch batch kernel);
  * ``scorer`` ((a) to (c)): a tensor-core SlidingScorer with P = B, reset and fed the recording's S-sample segments
    (19 pushes at (a), 1440 at (b), 3 at (c), where its windows end at multiples of S, not at W + w S).
A torch.profiler run of its own splits predict_record's device time into front end (staging, front end, exact
re-computation) and projection + head; ``bound_ms`` is the algorithmic bytes (the recording read once, the scores
written once) over 3.35 TB/s.  ``max_abs_diff`` compares the arms' scores of the same windows.  Prints the card's
name, power limit and max SM clock, read in the same run, and one JSON line.
    python scripts/record_bench.py [--steps 3] [--rounds 3] [--only a,b,c,d]"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import tskd_b200
from oracle import mycnn_torch as O
from slide_heads_bench import card

HBM = 3.35e12
FRONT = ("record_stage_kernel", "tc_stream_kernel", "tc_compact_flags_kernel", "frontend_kernel", "frontend_any_kernel")
PROJ_HEAD = ("slide_record_proj_kernel", "record_proj_kernel", "record_age_kernel", "head_reduce_independent_kernel",
             "reduce_gates_kernel", "head_independent_kernel")


def model(C, W, dev):
    ref = O.make_ref(O.stretched(O.ARCH_MYCNN5, C, W), seed=0)
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W), has_out12=ref.arch.has_out12).to(dev)
    m.load_state_dict(ref.state_dict())
    return m


def timed(arms, steps, rounds):
    for f in arms.values():
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


def split_ms(fn, steps):
    """device ms per call of predict_record: front end, projection + head, all"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {"front_end": 0.0, "projection_head": 0.0, "all": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if not t or e.key.startswith(("cudaLaunch", "cudaMemcpy", "cudaEvent", "cudaStream", "cudaFunc")):
            continue
        out["all"] += t
        if any(n in e.key for n in FRONT):
            out["front_end"] += t
        elif any(n in e.key for n in PROJ_HEAD):
            out["projection_head"] += t
    return {k: v / 1e3 / steps for k, v in out.items()}


def tc_workload(tag, m, B, N, S, steps, rounds, dev):
    C, W = m.arch.in_channels, m.arch.window
    x = tskd_b200.synth.make_windows(B, C, N, "normal", seed=1, dtype=torch.bfloat16, device=dev)
    age = tskd_b200.synth.make_ages(B, seed=1, device=dev)
    n_w = (N - W) // S + 1
    per = max(1, 4096 // B)                                         # windows per recording per predict() chunk
    buf = torch.empty(B * per, C, W, dtype=torch.bfloat16, device=dev)
    ages_rep = age.repeat_interleave(per)
    pred_out = torch.empty(B, n_w, device=dev)

    def predict_arm():
        for w0 in range(0, n_w, per):
            k = min(per, n_w - w0)
            v = buf[:B * k].view(B, k, C, W)
            v.copy_(x.unfold(2, W, S)[:, :, w0:w0 + k].permute(0, 2, 1, 3))
            pred_out[:, w0:w0 + k] = m.predict(buf[:B * k], ages_rep[:B * k] if per > 1 else age).view(B, k)
        return pred_out

    sc = tskd_b200.SlidingScorer(m, B, S, torch.bfloat16)
    n_push = N // S

    def scorer_arm():
        sc.reset()
        outs = []
        for n in range(1, n_push + 1):
            got = sc.push(x[:, :, (n - 1) * S:n * S], age)
            if got is not None:
                outs.append(got)
        return outs

    rec = m.predict_record(x, S, age)
    pred = predict_arm().clone()
    diff = {"record_vs_predict": float((rec - pred).abs().max())}
    if W % S == 0:
        sco = torch.stack(scorer_arm(), 1)
        diff["record_vs_scorer"] = float((rec - sco).abs().max())
    res = timed({"record": lambda: m.predict_record(x, S, age), "predict": predict_arm, "scorer": scorer_arm}, steps, rounds)
    split = split_ms(lambda: m.predict_record(x, S, age), max(1, steps))
    sc.close()
    nbytes = B * C * N * 2 + B * n_w * 4
    return {"workload": tag, "B": B, "N": N, "W": W, "S": S, "n_w": n_w, "pushes": n_push, "arms": res, "record_device_ms": split,
            "bytes": nbytes, "bound_ms": nbytes / HBM * 1e3, "max_abs_diff": diff}


def generic_workload(S, steps, rounds, dev):
    m = model(10, 120, dev)
    B, C, W, N = 1024, 10, 120, 120 * 60
    x = tskd_b200.synth.make_windows(B, C, N, "normal", seed=2, dtype=torch.float32, device=dev)
    age = tskd_b200.synth.make_ages(B, seed=2, device=dev)
    n_w = (N - W) // S + 1
    ages_rep = age.repeat_interleave(n_w)

    def predict_arm():
        win = x.unfold(2, W, S).permute(0, 2, 1, 3).reshape(B * n_w, C, W)
        return m.predict(win, ages_rep)

    rec = m.predict_record(x, S, age, path="generic")
    pred = predict_arm()
    last = m.last_path
    diff = float((rec.reshape(-1) - pred).abs().max())
    res = timed({"record": lambda: m.predict_record(x, S, age, path="generic"), "predict": predict_arm}, steps, rounds)
    split = split_ms(lambda: m.predict_record(x, S, age, path="generic"), max(1, steps))
    nbytes = B * C * N * 4 + B * n_w * 4
    return {"workload": f"d-generic-S{S}", "B": B, "N": N, "W": W, "S": S, "n_w": n_w, "predict_path": last, "arms": res,
            "record_device_ms": split, "bytes": nbytes, "bound_ms": nbytes / HBM * 1e3, "max_abs_diff": {"record_vs_predict": diff}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default="a,b,c,d")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("record_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    only = set(a.only.split(","))
    rows = []
    if only & {"a", "b", "c"}:
        m = model(3, 75000, dev)
        if "a" in only:
            rows.append(tc_workload("a-4096x10", m, 4096, 75000 + 9 * 7500, 7500, a.steps, a.rounds, dev))
        if "b" in only:
            rows.append(tc_workload("b-24h", m, 1, 10_800_000, 7500, 1, a.rounds, dev))
        if "c" in only:
            rows.append(tc_workload("c-4096-overlap40", m, 4096, 75000 + 9 * 7500, 45000, a.steps, a.rounds, dev))
        del m
        torch.cuda.empty_cache()
    if "d" in only:
        for S in (72, 12):
            rows.append(generic_workload(S, a.steps, a.rounds, dev))
    for r in rows:
        arms = ", ".join(f"{k} {v['ms']:.3f} ms" for k, v in r["arms"].items())
        print(f"  {r['workload']}: {arms}; record device {json.dumps({k: round(v, 3) for k, v in r['record_device_ms'].items()})}; "
              f"bound {r['bound_ms']:.3f} ms; diff {r['max_abs_diff']}", file=sys.stderr)
    print(json.dumps({"metric": "predict_record against predict() and SlidingScorer", "card": c, "rows": rows}))


if __name__ == "__main__":
    main()
