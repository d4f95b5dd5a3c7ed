"""Many patients' window sequences per training step (seq_lengths) against what it replaces.

Arms, each timed with CUDA events over --steps iterations after --warmup:
  seq_step        B200Trainer.step(..., seq_lengths=[n] * N): one fused call, the LSTM scans run one CTA per sequence
  loop_autograd   the same gradient today: one B200TrainableMyCNN forward per sequence under autograd, the losses summed
                  (each BCE sum divided by B, so the total is the batch mean), one backward, one torch.optim.Adam step
  single_step     the single-sequence step at the same B (today's sequence mode), for context
  predict_seq     predict(mode="sequence", seq_lengths=...) against predict_loop, one predict per sequence
Shapes: [2048,10,120] as 64 x 32 and 256 x 8 sequences, [256,3,75000] as 16 x 16.  --profile instead prints a
torch.profiler split of the scan kernels and the new reduction (run it on its own: tracing slows the host).

Prints one JSON line with the card's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tskd_b200  # noqa: E402
from tskd_b200.trainer import B200Trainer  # noqa: E402

SHAPES = [(10, 120, 64, 32), (10, 120, 256, 8), (3, 75000, 16, 16)]      # C, W, N sequences, n windows each


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def model_for(C, W, trainable=False):
    arch = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W)
    torch.manual_seed(0)
    cls = tskd_b200.B200TrainableMyCNN if trainable else tskd_b200.B200MyCNN
    return cls(arch).to("cuda")


def batch(C, W, B):
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(B, C, W, device="cuda", generator=g)
    age = torch.rand(B, device="cuda", generator=g) * 60 + 20
    y = (torch.rand(B, device="cuda", generator=g) > 0.5).float()
    return x, age, y


def run(args):
    out = {"card": card(), "steps": args.steps, "warmup": args.warmup, "arms": []}
    for C, W, N, n in SHAPES:
        B = N * n
        lens = [n] * N
        steps = max(2, args.steps // 10) if W > 1000 else args.steps
        x, age, y = batch(C, W, B)
        m = model_for(C, W)
        tr = B200Trainer(m, dropout=0.1)
        masks = tr.draw_masks(B)
        arm = {"shape": [B, C, W], "n_seq": N, "seq_len": n}
        arm["seq_step_ms"] = timed(lambda: tr.step(x, age, y, masks=masks, seq_lengths=lens), steps, args.warmup)
        arm["single_step_ms"] = timed(lambda: tr.step(x, age, y, masks=masks), steps, args.warmup)
        mt = model_for(C, W, trainable=True)
        mt.train()
        opt = torch.optim.Adam(mt.parameters(), lr=1e-3)
        crit = nn.BCEWithLogitsLoss(reduction="sum")

        def loop():
            opt.zero_grad()
            loss = 0.0
            for s in range(N):
                sl = slice(s * n, (s + 1) * n)
                loss = loss + crit(mt(x[sl], age[sl]), y[sl]) / B
            loss.backward()
            opt.step()

        arm["loop_autograd_ms"] = timed(loop, steps, args.warmup)
        arm["predict_seq_ms"] = timed(lambda: m.predict(x, age, mode="sequence", seq_lengths=lens), steps, args.warmup)
        arm["predict_loop_ms"] = timed(lambda: [m.predict(x[s * n:(s + 1) * n], age[s * n:(s + 1) * n], mode="sequence")
                                                for s in range(N)], steps, args.warmup)
        out["arms"].append(arm)
    return out


def profile_split(args):
    from torch.profiler import ProfilerActivity, profile
    out = {"card": card(), "profile": []}
    for C, W, N, n in SHAPES[:2] + [(10, 120, 1, 2048)]:
        B = N * n
        x, age, y = batch(C, W, B)
        tr = B200Trainer(model_for(C, W), dropout=0.1)
        masks = tr.draw_masks(B)
        lens = [n] * N
        for _ in range(3):
            tr.step(x, age, y, masks=masks, seq_lengths=lens)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                tr.step(x, age, y, masks=masks, seq_lengths=lens)
            torch.cuda.synchronize()
        tot = {}
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
                tot[e.key] = e.device_time_total / args.steps
        pick = lambda s: sum(v for k, v in tot.items() if s in k)
        out["profile"].append({"shape": [B, C, W], "n_seq": N, "lstm_fwd_us": pick("train_lstm_fwd"), "lstm_bwd_us": pick("train_lstm_bwd"),
                               "head_reduce_us": pick("train_head_reduce"), "all_kernels_us": sum(tot.values())})
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_seq_bench.py needs a CUDA device")
    print(json.dumps(profile_split(a) if a.profile else run(a)))
