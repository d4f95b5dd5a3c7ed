#!/usr/bin/env python
"""BASELINE.json configs[3]: architectures {MyCNN3/4-arch (k1=5, pool(2,2)), MyCNN5-arch (k1=10,
pool(3,2))} x W in {7500, 37500, 75000}, B=1024, C=3, bf16 and fp32, one GPU.  One JSON line per
case: windows/s, the dominant stage's duration and its fraction of the measured HBM roofline.
Also the production shape [1,10,120] fp32 latency.   python scripts/sweep.py > profiles/<tag>.jsonl"""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import tskd_b200

dev = torch.device("cuda", 0)
peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"] \
    if os.path.exists(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else 6650.0


from oracle import mycnn_torch as O      # the checker of the `parity` figure every cell carries (never the thing timed)


def run(kind, C, W, B, dtype, steps=10, warm=3, path="auto", padded_rows=False):
    """padded_rows: the producer writes the batch into B200MyCNN.empty_windows() (rows padded to 16 bytes) instead of a
    contiguous tensor -- for W % 8 != 0 (7500, 37500) that is what lets TMA stream the windows without a staging copy."""
    arch = tskd_b200.ARCH_PRESETS[kind].with_shape(C, W)
    torch.manual_seed(0)
    m = tskd_b200.B200MyCNN(arch, has_out12=(kind == "mycnn5"), path=path).to(dev)
    x = tskd_b200.synth.make_windows(B, C, W, "normal", seed=1234, dtype=dtype, device=dev)
    if padded_rows:
        xp = m.empty_windows(B, dtype=dtype)
        xp.copy_(x)
        x = xp
    ages = tskd_b200.synth.make_ages(B, seed=1234, device=dev)
    m.set_profile(True)
    for _ in range(warm):
        y = m.predict(x, ages)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        y = m.predict(x, ages)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    k_ms = m.last_stage_ms(0)
    esz = 2 if dtype == torch.bfloat16 else 4
    nw = sum(v.numel() for k, v in m.state_dict().items() if k in tskd_b200.arch.BLOB_KEYS)
    alg = B * (C * W * esz + 4) + nw * 4
    # parity of this cell: 16 of its windows through the CPU oracle, per-element relative error of the logits
    ref = O.make_ref(O.stretched(O.ARCHS[kind], C, W), seed=0)
    ref.load_state_dict({k: v.cpu() for k, v in m.state_dict().items() if k in ref.state_dict()})
    idx = torch.linspace(0, B - 1, 16).round().long()
    want = O.ref_independent(ref, x[idx.to(dev)].float().cpu(), ages[idx.to(dev)].cpu()).double()
    got = y[idx.to(dev)].cpu().double()
    den = torch.maximum(want.abs(), 1e-2 * want.abs().max())
    parity = float(((got - want).abs() / den).max())
    return {"arch": kind, "C": C, "W": W, "B": B, "dtype": str(dtype).replace("torch.", ""), "path": m.last_path,
            "rows": "padded to 16 B by the producer" if padded_rows else "contiguous", "parity_max_rel": parity, "parity_n": 16,
            "ms_per_step": ms, "windows_per_s": B / ms * 1e3, "front_stage_ms": k_ms, "head_ms": m.last_stage_ms(1),
            "algorithmic_bytes": alg, "hbm_frac_front_stage": alg / (k_ms * 1e-3) / 1e9 / peak, "hbm_frac_step": alg / (ms * 1e-3) / 1e9 / peak,
            "launches": m.gpu_launches, "finite": bool(torch.isfinite(y).all())}


if __name__ == "__main__":
    for kind in ("mycnn3", "mycnn5"):
        for W in (7500, 37500, 75000):
            for dtype in (torch.bfloat16, torch.float32):
                print(json.dumps(run(kind, 3, W, 1024, dtype)), flush=True)
                if dtype == torch.bfloat16 and W % 8:
                    print(json.dumps(run(kind, 3, W, 1024, dtype, padded_rows=True)), flush=True)
    # production shape, batched: all patients of a trigger in one launch ([P,10,120], one warp per window)
    for P in (256, 4096, 32768):
        arch = tskd_b200.ARCH_PRESETS["mycnn5"]
        torch.manual_seed(0)
        m = tskd_b200.B200MyCNN(arch).to(dev)
        x = tskd_b200.synth.make_windows(P, 10, 120, "physio", seed=7, dtype=torch.float32, device=dev)
        ages = tskd_b200.synth.make_ages(P, seed=7, device=dev)
        for _ in range(5):
            y = m.predict(x, ages)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(50):
            y = m.predict(x, ages)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 50
        ref = O.make_ref(O.ARCH_MYCNN5, seed=0)
        ref.load_state_dict({k: v.cpu() for k, v in m.state_dict().items() if k in ref.state_dict()})
        want = O.ref_independent(ref, x[:64].cpu(), ages[:64].cpu()).double()
        den = torch.maximum(want.abs(), 1e-2 * want.abs().max())
        print(json.dumps({"arch": "mycnn5", "shape": [P, 10, 120], "dtype": "float32", "ms_per_step": ms, "windows_per_s": P / ms * 1e3,
                          "launches": m.gpu_launches, "hbm_frac_step": P * 4804 / (ms * 1e-3) / 1e9 / peak,
                          "parity_max_rel": float(((y[:64].cpu().double() - want).abs() / den).max()), "parity_n": 64,
                          "logits_head": [float(v) for v in y[:3].cpu()], "oracle_head": [float(v) for v in want[:3]],
                          "note": "short_batch_kernel: one warp per window, one launch per trigger for all patients"}), flush=True)
    # production shape: MyCNN5 [1,10,120] fp32, latency per call (host-side call overhead included)
    arch = tskd_b200.ARCH_PRESETS["mycnn5"]
    m = tskd_b200.B200MyCNN(arch).to(dev)
    x = torch.randn(1, 10, 120, device=dev); a = torch.tensor([65.0], device=dev)
    for _ in range(20):
        m(x, a)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(2000):
        m(x, a)
    torch.cuda.synchronize(); dt = (time.perf_counter() - t0) / 2000
    print(json.dumps({"arch": "mycnn5", "shape": [1, 10, 120], "dtype": "float32", "us_per_call": dt * 1e6, "calls_per_s": 1 / dt,
                      "path": m.last_path, "launches": m.gpu_launches, "note": "python call + ctypes + 4 kernel launches, device-resident input"}))
    xh = torch.randn(1, 10, 120).double().numpy()
    t0 = time.perf_counter()
    for _ in range(500):
        y = m(torch.from_numpy(xh).float(), torch.tensor([65.0]))     # predictStream.py:155-157 with host tensors
    dt = (time.perf_counter() - t0) / 500
    print(json.dumps({"arch": "mycnn5", "shape": [1, 10, 120], "dtype": "float64->float32 host tensors", "us_per_call": dt * 1e6,
                      "note": "as predictStream.py:155-160 calls it: host numpy in, host result out (H2D + D2H + sync per call)"}))
