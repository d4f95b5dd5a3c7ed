#!/usr/bin/env python
"""The sequence-mode LSTM state across calls: predict_record(mode="sequence", state=..., return_state=True) and
SlidingScorer.admit(..., lstm=...).

Workloads (MyCNN5 geometry, C = 3, W = 75000, S = 7500 -- 600 s windows every 60 s at 125 Hz -- seed-0 weights, bf16):
  1. 24 h in chunks: [B, 3, 10 800 000] for B = 1 and 256: one call against 24 chained calls of one hour of windows
     each (60 windows; the last chunk 51), each chunk re-reading the W - S overlap with the one before.  Reports each
     arm's workspace and, computed from the workspace queries and the device's free memory (not measured), the largest
     cohort B each arm can score with the whole recording on the device, and the largest a chunked backtest can score
     when only the current hour is on the device.
  2. Warm-start admission: P patients with 12 h of stay.  Arm "backtest": 12 chained hourly calls over the P stays
     (every hour scores the same [P, 3, 1 h + W - S] tensor: the time does not depend on the values), then
     admit(history, lstm) of all P patients and one live push.  Today's remedy for live scores equal to a backtest
     re-scores the whole history at every push: its cost per push is the backtest's 12 hourly calls again, as the
     numbers below state (it grows with the stay; the push after a warm-started admission does not).
  3. TBPTT: B200Trainer.step_record at [64, 3, N] bf16 recordings of 40 windows (N = W + 39 S), one step over the whole
     recordings against 4 chained steps of 10 windows each (state=..., return_state=True), Adam on: time per step and
     the workspace of each (b2cnn_train_workspace_bytes_record).
Arms alternate within every round (CUDA events around --steps calls, median of --rounds).  Prints the card's name, power
limit, max SM clock and current SM clock, read in the same run, and one JSON line.
    python scripts/record_state_bench.py [--steps 2] [--rounds 5] [--only 1,2,3] [--patients 1024]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import tskd_b200
from record_bench import model, timed
from slide_heads_bench import card
from tskd_b200 import capi
from tskd_b200.trainer import B200Trainer

W, S, C, FS = 75000, 7500, 3, 125
DAY = 24 * 3600 * FS
HOUR_W = 3600 * FS // S                                   # windows per hour: 60


def sm_clock():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def ws_bytes(m, B, N):
    lib, h = m._ensure_handle()
    return int(lib.b2cnn_record_workspace_bytes_ex(h, B, N, N, S, capi.DTYPE_BF16, capi.PATH_AUTO, capi.MODE_SEQUENCE))


def chunks(n_w):
    """[(first window, last window + 1)] of the hourly chunks"""
    return [(w0, min(w0 + HOUR_W, n_w)) for w0 in range(0, n_w, HOUR_W)]


def chained(m, x, age, n_w):
    s, outs = None, []
    for w0, w1 in chunks(n_w):
        o, s = m.predict_record(x[:, :, w0 * S:(w1 - 1) * S + W], S, age, mode="sequence", state=s, return_state=True)
        outs.append(o)
    return torch.cat(outs, dim=1), s


def day_row(m, B, steps, rounds, dev):
    N = DAY
    n_w = (N - W) // S + 1
    per_rec = C * N * 2
    hour_N = (HOUR_W - 1) * S + W
    ws_one, ws_hour = ws_bytes(m, B, N), ws_bytes(m, B, hour_N)
    ws_one_1, ws_hour_1 = ws_bytes(m, 1, N), ws_bytes(m, 1, hour_N)
    free, _ = torch.cuda.mem_get_info(dev)
    row = {"workload": f"24h-B{B}", "B": B, "N": N, "W": W, "S": S, "n_w": n_w, "chunks": len(chunks(n_w)),
           "workspace_bytes": {"one_call": ws_one, "hourly_chunk": ws_hour},
           "largest_B_computed": {"one_call": free // (per_rec + ws_one_1), "chunked_whole_stay_on_device": free // (per_rec + ws_hour_1),
                                  "chunked_hour_on_device": free // (C * hour_N * 2 + ws_hour_1)}}
    if B * per_rec + max(ws_one, ws_hour) > free * 0.9:
        row["arms"] = "not run: the input and the one-call workspace exceed the free device memory"
        return row
    x = tskd_b200.synth.make_windows(B, C, N, "normal", seed=5, dtype=torch.bfloat16, device=dev, chunk=8)
    age = tskd_b200.synth.make_ages(B, seed=5, device=dev)
    one, s_one = m.predict_record(x, S, age, mode="sequence", return_state=True)
    ch, s_ch = chained(m, x, age, n_w)
    row["path"] = m.last_path
    row["bit_identical"] = bool(torch.equal(one, ch) and torch.equal(s_one, s_ch))
    del one, ch
    arms = {"one_call": lambda: m.predict_record(x, S, age, mode="sequence", return_state=True),
            "24_hourly_calls": lambda: chained(m, x, age, n_w)}
    row["arms"] = timed(arms, steps, rounds)
    row["chunked_over_one_call"] = row["arms"]["24_hourly_calls"]["ms"] / row["arms"]["one_call"]["ms"]
    del x
    torch.cuda.empty_cache()
    return row


def warm_row(m, P, steps, rounds, dev):
    hours = 12
    hour_N = (HOUR_W - 1) * S + W
    x = tskd_b200.synth.make_windows(P, C, hour_N, "normal", seed=6, dtype=torch.bfloat16, device=dev)
    age = tskd_b200.synth.make_ages(P, seed=6, device=dev)
    hist = x[:, :, hour_N - W:].contiguous()
    live = tskd_b200.synth.make_windows(P, C, S, "normal", seed=7, dtype=torch.bfloat16, device=dev)
    sc = tskd_b200.SlidingScorer(m, P, S, dtype=torch.bfloat16, mode="sequence")
    idx = list(range(P))

    def backtest():
        s = None
        for _ in range(hours):
            _, s = m.predict_record(x, S, age, mode="sequence", state=s, return_state=True)
        return s

    state = backtest()
    arms = {"backtest_12h": backtest,
            "admit_lstm": lambda: sc.admit(idx, hist, lstm=state),
            "push": lambda: sc.push(live, age=age)}
    sc.admit(idx, hist, lstm=state)
    res = timed(arms, steps, rounds)
    warm = res["backtest_12h"]["ms"] + res["admit_lstm"]["ms"]
    return {"workload": f"warm-start-P{P}-12h", "P": P, "hours": hours, "path": sc.path, "arms": res,
            "warm_start_once_ms": warm, "push_after_warm_start_ms": res["push"]["ms"],
            "remedy_per_push_ms": res["backtest_12h"]["ms"] + res["push"]["ms"],
            "note": "remedy_per_push re-scores the 12 h history at every push (the backtest's calls again) and grows with the stay"}


def tbptt_row(steps, rounds, dev):
    B, n_w, n_chunks = 64, 40, 4
    N = W + (n_w - 1) * S
    per = n_w // n_chunks
    n_chunk = W + (per - 1) * S
    m = model(C, W, dev)
    tr = B200Trainer(m, lr=1e-6)
    x = tskd_b200.synth.make_windows(B, C, N, "normal", seed=8, dtype=torch.bfloat16, device=dev)
    age = tskd_b200.synth.make_ages(B, seed=8, device=dev)
    y = (torch.rand(B * n_w, device=dev) > 0.5).float()
    yc = y.reshape(B, n_w)

    def whole():
        tr.step_record(x, S, age, y)

    def tbptt():
        s = None
        for c in range(n_chunks):
            _, s = tr.step_record(x[:, :, c * per * S:c * per * S + n_chunk], S, age, yc[:, c * per:(c + 1) * per].reshape(-1), state=s,
                                  return_state=True)

    res = timed({"whole_recording": whole, "4_chained_chunks": tbptt}, steps, rounds)

    def ws(n, k):
        cts = (ctypes.c_int64 * B)(*([k] * B))
        return int(tr._lib.b2cnn_train_workspace_bytes_record(ctypes.byref(tr._cfg), B, n, S, cts, capi.MODE_SEQUENCE))
    return {"workload": f"tbptt-{B}x{N}", "B": B, "N": N, "n_w": n_w, "chunks": n_chunks, "arms": res,
            "per_chunk_step_ms": res["4_chained_chunks"]["ms"] / n_chunks,
            "workspace_bytes": {"whole_recording": ws(N, n_w), "chunk": ws(n_chunk, per)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--only", default="1,2,3")
    ap.add_argument("--patients", type=int, default=1024)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("record_state_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    only = set(a.only.split(","))
    m = model(C, W, dev)
    rows = []
    if "1" in only:
        for B in (1, 256):
            rows.append(day_row(m, B, a.steps, a.rounds, dev))
            r = rows[-1]
            if isinstance(r["arms"], dict):
                print(f"  {r['workload']} ({r['path']}): one call {r['arms']['one_call']['ms']:.2f} ms, 24 hourly calls "
                      f"{r['arms']['24_hourly_calls']['ms']:.2f} ms (x{r['chunked_over_one_call']:.3f}), bit-identical "
                      f"{r['bit_identical']}", file=sys.stderr)
            print(f"    workspace {r['workspace_bytes']}, largest B (computed) {r['largest_B_computed']}", file=sys.stderr)
    if "2" in only:
        r = warm_row(m, a.patients, a.steps, a.rounds, dev)
        rows.append(r)
        print(f"  {r['workload']} ({r['path']}): backtest {r['arms']['backtest_12h']['ms']:.2f} ms + admit "
              f"{r['arms']['admit_lstm']['ms']:.2f} ms once, then push {r['push_after_warm_start_ms']:.3f} ms; remedy "
              f"{r['remedy_per_push_ms']:.2f} ms per push", file=sys.stderr)
    if "3" in only:
        del m
        torch.cuda.empty_cache()
        r = tbptt_row(a.steps, a.rounds, dev)
        rows.append(r)
        print(f"  {r['workload']}: whole {r['arms']['whole_recording']['ms']:.2f} ms, 4 chained chunks "
              f"{r['arms']['4_chained_chunks']['ms']:.2f} ms ({r['per_chunk_step_ms']:.2f} ms per chunk step); workspace "
              f"{r['workspace_bytes']}", file=sys.stderr)
    c["sm_clock_after"] = sm_clock()
    print(f"SM clock after the run: {c['sm_clock_after']}", file=sys.stderr)
    print(json.dumps({"metric": "sequence-mode LSTM state across calls", "card": c, "rows": rows}))


if __name__ == "__main__":
    main()
