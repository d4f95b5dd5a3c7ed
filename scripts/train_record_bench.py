"""Training on whole recordings (B200Trainer.step_record, mycnn_train_record_forward) against what it replaces: the
windows cut out of the recordings as copies, then B200Trainer.step(..., seq_lengths=...) / mycnn_train_forward.

Arms, each timed with CUDA events over --steps iterations after --warmup (a tenth of --steps at the waveform shape):
  record_step      one fused step_record call
  cut_step         step(seq_lengths = the counts) on windows already cut; cut_copy is the cut itself, timed on its own
  record_autograd  mycnn_train_record_forward + BCEWithLogitsLoss + backward (records and parameters)
  cut_autograd     mycnn_train_forward on the cut windows + the same loss + backward (windows and parameters)
Workloads: (a) [256,3,142500] fp32, W = 75000, S = 7500, 10 windows each; (b) [64,10,10416], W = 120, S = 72 (the 40 %
overlap of create_batch), 144 windows each; (c) gaps, S = 2W, [256,10,4680], 20 windows each.  Also printed: the
record workspace against the cut copies' bytes plus the cut path's workspace.  --profile instead prints a torch.profiler
split of both fused steps (run it on its own: tracing slows the host).

Prints one JSON line with the card's name and power limit."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tskd_b200  # noqa: E402
from tskd_b200 import capi  # noqa: E402
from tskd_b200.autograd import cut_record_windows  # noqa: E402
from tskd_b200.trainer import B200Trainer  # noqa: E402

WORKLOADS = [("a", 3, 75000, 256, 142500, 7500), ("b", 10, 120, 64, 10416, 72), ("c", 10, 120, 256, 120 + 19 * 240, 240)]


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


def setup(C, W, B, N, S, trainable=False):
    arch = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W)
    torch.manual_seed(0)
    m = (tskd_b200.B200TrainableMyCNN if trainable else tskd_b200.B200MyCNN)(arch).to("cuda")
    g = torch.Generator(device="cuda").manual_seed(1)
    rec = torch.randn(B, C, N, device="cuda", generator=g)
    n_w = (N - W) // S + 1
    counts = [n_w] * B
    age = torch.rand(B, device="cuda", generator=g) * 60 + 20
    y = (torch.rand(B * n_w, device="cuda", generator=g) > 0.5).float()
    return m, rec, counts, age, y


def run(args):
    out = {"card": card(), "steps": args.steps, "warmup": args.warmup, "arms": []}
    for name, C, W, B, N, S in WORKLOADS:
        steps = max(2, args.steps // 10) if W > 1000 else args.steps
        m, rec, counts, age, y = setup(C, W, B, N, S)
        M = sum(counts)
        tr = B200Trainer(m, dropout=0.1)
        m1, m2 = tr.draw_masks(B, N)
        arm = {"workload": name, "records": [B, C, N], "W": W, "S": S, "windows": M}
        arm["record_step_ms"] = timed(lambda: tr.step_record(rec, S, age, y, masks=(m1, m2)), steps, args.warmup)
        cut = lambda: cut_record_windows(rec, W, S, counts, m.arch.pool_s, m1, m2)
        arm["cut_copy_ms"] = timed(cut, steps, args.warmup)
        x, c1, c2 = cut()
        age_w = age.repeat_interleave(M // B)
        arm["cut_step_ms"] = timed(lambda: tr.step(x, age_w, y, masks=(c1, c2), seq_lengths=counts), steps, args.warmup)
        cfg = capi.make_config(m.arch, 0)
        lib = capi.load_library()
        cts = (ctypes.c_int64 * B)(*counts)
        arm["record_workspace_bytes"] = int(lib.b2cnn_train_workspace_bytes_record(ctypes.byref(cfg), B, N, S, cts, capi.MODE_SEQUENCE))
        arm["cut_copy_bytes"] = 4 * (x.numel() + (c1.numel() + c2.numel() if c1 is not None else 0))
        arm["cut_workspace_bytes"] = int(lib.b2cnn_train_workspace_bytes_seq(ctypes.byref(cfg), M, (ctypes.c_int64 * B)(*counts), B))
        del x, c1, c2
        torch.cuda.empty_cache()
        mt, _, _, _, _ = setup(C, W, B, N, S, trainable=True)
        mt.train()
        crit = nn.BCEWithLogitsLoss()
        named = dict(mt.named_parameters())
        params = [named[k] for k in tskd_b200.arch.BLOB_KEYS]
        recg = rec.clone().requires_grad_()

        def rec_ag():
            for q in params:
                q.grad = None
            recg.grad = None
            z = tskd_b200.mycnn_train_record_forward(recg, S, age, params, mt.arch, "sequence", m1, m2, counts)
            crit(z, y).backward()

        arm["record_autograd_ms"] = timed(rec_ag, steps, args.warmup)
        x, c1, c2 = cut()
        xg = x.requires_grad_()

        def cut_ag():
            for q in params:
                q.grad = None
            xg.grad = None
            z = tskd_b200.mycnn_train_forward(xg, age_w, params, mt.arch, "sequence", c1, c2, seq_lengths=counts)
            crit(z, y).backward()

        arm["cut_autograd_ms"] = timed(cut_ag, steps, args.warmup)
        del x, xg, c1, c2, recg
        torch.cuda.empty_cache()
        out["arms"].append(arm)
    return out


def profile_split(args):
    from torch.profiler import ProfilerActivity, profile
    out = {"card": card(), "profile": []}
    for name, C, W, B, N, S in WORKLOADS:
        m, rec, counts, age, y = setup(C, W, B, N, S)
        M = sum(counts)
        tr = B200Trainer(m, dropout=0.1)
        m1, m2 = tr.draw_masks(B, N)
        x, c1, c2 = cut_record_windows(rec, W, S, counts, m.arch.pool_s, m1, m2)
        age_w = age.repeat_interleave(M // B)
        steps = 2 if W > 1000 else args.steps
        for label, fn in (("record", lambda: tr.step_record(rec, S, age, y, masks=(m1, m2))),
                          ("cut", lambda: tr.step(x, age_w, y, masks=(c1, c2), seq_lengths=counts))):
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(steps):
                    fn()
                torch.cuda.synchronize()
            tot = {}
            for e in prof.key_averages():
                if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
                    tot[e.key] = e.device_time_total / steps
            pick = lambda s: sum(v for k, v in tot.items() if s in k)
            out["profile"].append({"workload": name, "path": label, "conv_fwd_us": pick("train_conv_fwd"), "conv_bwd_us": pick("train_conv_bwd"),
                                   "fold_us": pick("train_dfeat_fold"), "dfeat_us": pick("train_dfeat("),
                                   "scans_us": pick("train_lstm_fwd") + pick("train_lstm_bwd"), "all_kernels_us": sum(tot.values())})
        del x, c1, c2
        torch.cuda.empty_cache()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_record_bench.py needs a CUDA device")
    print(json.dumps(profile_split(a) if a.profile else run(a)))
