#!/usr/bin/env python
"""ms per training step (row f4) at the reference's training shape [B,10,120]: B200Trainer.step on the GPU (one fused call),
the same loop body (bin/utils.py:200-208: zero_grad, forward in train() mode, BCEWithLogitsLoss, backward, Adam.step) on
B200TrainableMyCNN with torch autograd and torch.optim.Adam on the GPU, and on the oracle module with torch on this box's
CPU threads.  Prints one JSON line."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch import nn
import tskd_b200
from tskd_b200.trainer import B200Trainer
from oracle import mycnn_torch as O

out = {}
for B in (32, 256, 2048):
    arch = tskd_b200.ARCH_PRESETS["mycnn5"]
    m = tskd_b200.B200MyCNN(arch).to("cuda:0")
    tr = B200Trainer(m, dropout=0.1)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 10, 120, generator=g); age = torch.rand(B, generator=g) * 60 + 20; y = (torch.rand(B, generator=g) > 0.5).float()
    xd, ad, yd = x.cuda(), age.cuda(), y.cuda()
    for _ in range(5):
        tr.step(xd, ad, yd)
    torch.cuda.synchronize()
    n = 50
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(n):
        tr.step(xd, ad, yd)
    ev1.record(); torch.cuda.synchronize()
    gpu_ms = ev0.elapsed_time(ev1) / n
    am = tskd_b200.B200TrainableMyCNN(arch).to("cuda:0").train()
    aopt = torch.optim.Adam(am.parameters(), lr=1e-3); crit = nn.BCEWithLogitsLoss()
    def gpu_body():
        aopt.zero_grad(); loss = crit(am(xd, ad), yd); loss.backward(); aopt.step()
    for _ in range(5):
        gpu_body()
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(n):
        gpu_body()
    ev1.record(); torch.cuda.synchronize()
    autograd_ms = ev0.elapsed_time(ev1) / n
    ref = O.make_ref(O.ARCH_MYCNN5, seed=0); ref.train()
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3); crit = nn.BCEWithLogitsLoss()
    def body():
        opt.zero_grad(); loss = crit(ref(x, age), y); loss.backward(); opt.step()
    for _ in range(3):
        body()
    k = max(3, int(200 / B) + 3)
    t0 = time.perf_counter()
    for _ in range(k):
        body()
    cpu_ms = (time.perf_counter() - t0) / k * 1e3
    out[f"B{B}"] = {"gpu_ms_per_step": round(gpu_ms, 4), "gpu_autograd_adam_ms_per_step": round(autograd_ms, 4), "cpu_torch_ms_per_step": round(cpu_ms, 3), "cpu_threads": torch.get_num_threads()}
print(json.dumps({"metric": "training step [B,10,120], sequence semantics, dropout 0.1, Adam", "results": out}))
