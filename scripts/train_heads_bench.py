"""K candidate heads on one frozen front end per training step (B200HeadTrainer) against what it replaces.

Arms at K in {1, 2, 4, 8}, each the time of one training step of all K heads:
  heads      B200HeadTrainer(model, K heads).step: the conv forward once, the K heads' scans side by side
  separate   K B200HeadTrainer(model, [head]).step calls, one after another
  autograd   K frozen-conv B200TrainableMyCNN steps (conv1 / conv2 requires_grad False) under autograd, each with
             BCEWithLogitsLoss and torch.optim.Adam: what a sweep of K candidates costs without this class
Workloads: [4096, 3, 75000] fp32 windows, sequence mode, dropout 0.1; [256, 10, 120] windows, sequence mode; and
step_record over [64, 3, 142500] recordings at stride 7500, sequence mode.  Each round times every arm once with CUDA
events, the arms alternating; the result is the median over --rounds rounds after --warmup.

Prints one JSON line with the card's name, power limit and maximum SM clock."""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tskd_b200  # noqa: E402
from tskd_b200.arch import BLOB_KEYS  # noqa: E402

DEV = torch.device("cuda", 0)
HEAD_KEYS = BLOB_KEYS[BLOB_KEYS.index("lstm.weight_ih_l0"):]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def candidates(m, K):
    g = torch.Generator().manual_seed(K)
    out = []
    for _ in range(K):
        h = copy.deepcopy(m)
        with torch.no_grad():
            sd = h.state_dict()
            for k in HEAD_KEYS:
                sd[k].add_(0.01 * torch.randn(sd[k].shape, generator=g).to(DEV))
        out.append(h)
    return out


def autograd_step(tm, opt, fwd, y):
    opt.zero_grad(set_to_none=True)
    z = fwd(tm)
    nn.BCEWithLogitsLoss()(z.reshape(-1), y).backward()
    opt.step()


def run(name, arch, K, batch, rounds, warmup, record=None):
    m = tskd_b200.B200MyCNN(arch).to(DEV)
    heads = candidates(m, K)
    x, age, y, masks = batch
    multi = tskd_b200.B200HeadTrainer(m, heads, dropout=0.1)
    single = [tskd_b200.B200HeadTrainer(m, [copy.deepcopy(h)], dropout=0.1) for h in heads]
    trainables = []
    for h in heads:
        tm = tskd_b200.B200TrainableMyCNN(arch).to(DEV)
        tm.load_state_dict(h.state_dict())
        tm.conv1.requires_grad_(False)
        tm.conv2.requires_grad_(False)
        named = dict(tm.named_parameters())
        trainables.append((tm, torch.optim.Adam([named[k] for k in HEAD_KEYS], lr=1e-3), [named[k] for k in BLOB_KEYS]))
    if record is None:
        step = lambda t: t.step(x, age, y, masks=masks)
        fwd = lambda p: (lambda tm: tskd_b200.mycnn_train_forward(x, age, p, arch, "sequence", *masks))
    else:
        S = record
        step = lambda t: t.step_record(x, S, age, y, masks=masks)
        fwd = lambda p: (lambda tm: tskd_b200.mycnn_train_record_forward(x, S, age, p, arch, "sequence", *masks))
    arms = {
        "heads": lambda: step(multi),
        "separate": lambda: [step(t) for t in single],
        "autograd": lambda: [autograd_step(tm, opt, fwd(p), y) for tm, opt, p in trainables],
    }
    times = {k: [] for k in arms}
    for r in range(warmup + rounds):
        for k, fn in arms.items():
            t = timed(fn)
            if r >= warmup:
                times[k].append(t)
    med = {k: round(statistics.median(v), 3) for k, v in times.items()}
    out = {"workload": name, "K": K, **{f"{k}_ms": v for k, v in med.items()},
           "speedup_vs_separate": round(med["separate"] / med["heads"], 2), "speedup_vs_autograd": round(med["autograd"] / med["heads"], 2)}
    print(json.dumps(out), file=sys.stderr, flush=True)
    del multi, single, trainables
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--workloads", default="long,short,record")
    a = ap.parse_args()
    ks = [int(k) for k in a.ks.split(",")]
    g = torch.Generator(device=DEV).manual_seed(0)
    preset = tskd_b200.ARCH_PRESETS["mycnn5"]
    results = []
    for w in a.workloads.split(","):
        if w == "long":
            arch, B = preset.with_shape(3, 75000), 4096
        elif w == "short":
            arch, B = preset, 256
        else:
            arch, B, N, S = preset.with_shape(3, 7500), 64, 142500, 7500
        if w == "record":
            x = torch.randn(B, 3, N, device=DEV, generator=g)
            n_w = (N - arch.window) // S + 1
            age = torch.full((B,), 60.0, device=DEV)
            y = (torch.rand(B * n_w, device=DEV, generator=g) > 0.9).float()
            masks = tskd_b200.autograd.draw_masks(arch.with_shape(3, N), B, 0.1, DEV, g)
            batch, record = (x, age, y, masks), S
        else:
            x = torch.randn(B, arch.in_channels, arch.window, device=DEV, generator=g)
            age = torch.full((B,), 60.0, device=DEV)
            y = (torch.rand(B, device=DEV, generator=g) > 0.9).float()
            batch, record = (x, age, y, tskd_b200.autograd.draw_masks(arch, B, 0.1, DEV, g)), None
        for K in ks:
            results.append(run(f"{w}[{B},{arch.in_channels},{N if w == 'record' else arch.window}]", arch, K, batch, a.rounds, a.warmup, record))
        del batch, x
        torch.cuda.empty_cache()
    name, power, clock = card()
    print(json.dumps({"card": name, "power_limit": power, "max_sm_clock": clock, "rounds": a.rounds, "results": results}))


if __name__ == "__main__":
    main()
