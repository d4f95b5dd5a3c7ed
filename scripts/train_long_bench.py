#!/usr/bin/env python
"""ms per training step at the waveform window [B,3,75000] fp32 (L_out = 18745, the tiled training kernels of
csrc/b2cnn_train.cu): B200Trainer.step (one fused call) and the autograd loop on B200TrainableMyCNN with
torch.optim.Adam, with every parameter trained and with conv1 / conv2 frozen, in both batch modes; predict() on the
same windows beside them; then a torch.profiler run of its own for the per-kernel split of one fused step.
CUDA events after warm-up.  Needs a GPU; prints the card, its power limit and max SM clock, then one JSON line.

    python scripts/train_long_bench.py [--batches 256,4096] [--steps 5] [--no-profile]"""
import argparse, collections, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch import nn
import tskd_b200
from tskd_b200.trainer import B200Trainer

ap = argparse.ArgumentParser()
ap.add_argument("--batches", default="256,4096")
ap.add_argument("--window", type=int, default=75000)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--no-profile", action="store_true")
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("train_long_bench.py measures on a GPU; none found")
dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card, flush=True)


def timed(fn, n):
    fn(); fn()                                           # warm-up: module loads, attributes, allocator
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / n, 3)


arch = tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(3, args.window)
out = {}
for B in [int(b) for b in args.batches.split(",")]:
    x = torch.randn(B, 3, args.window, device=dev)
    age = torch.rand(B, device=dev) * 60 + 20
    y = (torch.rand(B, device=dev) > 0.5).float()
    res = {}
    for mode in ("sequence", "independent"):
        m = tskd_b200.B200MyCNN(arch).to(dev)
        tr = B200Trainer(m, lr=1e-5, mode=mode, dropout=0.1)
        res[f"fused_step_ms_{mode}"] = timed(lambda: tr.step(x, age, y), args.steps)
        del tr
        am = tskd_b200.B200TrainableMyCNN(arch).to(dev).train()
        am.batch_mode = mode
        crit = nn.BCEWithLogitsLoss()
        for frozen in (False, True):
            am.conv1.requires_grad_(not frozen); am.conv2.requires_grad_(not frozen)
            opt = torch.optim.Adam([p for p in am.parameters() if p.requires_grad], lr=1e-5)

            def body():
                opt.zero_grad(); crit(am(x, age), y).backward(); opt.step()
            res[f"autograd_adam_ms_{mode}{'_frozen_conv' if frozen else ''}"] = timed(body, args.steps)
        am.eval()
        with torch.no_grad():
            res[f"predict_fp32_ms_{mode}"] = timed(lambda: m.predict(x, age, mode=mode), args.steps)
        del am, m
    out[f"B{B}"] = res
    if not args.no_profile:                               # a run of its own: tracing slows the host
        from torch.profiler import ProfilerActivity, profile
        m = tskd_b200.B200MyCNN(arch).to(dev)
        tr = B200Trainer(m, lr=1e-5, mode="sequence", dropout=0.1)
        tr.step(x, age, y); torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            tr.step(x, age, y); torch.cuda.synchronize()
        split = collections.Counter()
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and "b2cnn::train_" in e.name:
                split[e.name.split("b2cnn::")[1].split("(")[0].split("<")[0]] += e.device_time_total / 1e3
        res["kernel_ms_fused_sequence"] = {k: round(v, 3) for k, v in split.most_common()}
        del tr, m
    del x
    torch.cuda.empty_cache()
print(json.dumps({"metric": f"training step [B,3,{args.window}] fp32, dropout 0.1, Adam", "card": card, "results": out}))
