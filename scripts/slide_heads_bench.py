#!/usr/bin/env python
"""Extra heads over one SlidingScorer's features (SlidingScorer.set_heads / push(heads=True)): what shadow-scoring K
heads costs, next to K + 1 separate scorers that each run the front end.  W = 75000, S = 7500 (600 s sliding by 60 s
at 125 Hz), seed-0 weights for M0; head i has M0's conv weights and seeded LSTM / Linear weights.

  * tensor-core path, MyCNN5 geometry, C = 3, bf16, --tc-patients P, padded rows ([P, 3, 7504][:, :, :7500] views);
  * generic path, C = 10, bf16, --generic-patients P.

Arms, alternating within every round (CUDA events over --steps pushes, median of --rounds): ``push()`` of a scorer
without heads, ``push(heads=True)`` with K = 1, 3, 7, and K + 1 separate scorers pushed with the same samples.  Then,
in a separate torch.profiler run per K, the device time of the projection kernel and of the head kernels per push.
The algorithmic bytes of the tensor-core projection are the ring (4 L P, read once per CTA pair of heads), each row's
packed W_ih chunks (read once; every patient tile re-reads them, mostly from L2: reported apart) and the partials
(4 n_ranges P 64 per row, written); their share of the H100 SXM data-sheet bandwidth, 3.35 TB/s, is given per K.
Prints one JSON line with the card's name, power limit and max SM clock, read in the same run.
    python scripts/slide_heads_bench.py [--tc-patients 4096] [--generic-patients 1024] [--steps 20] [--rounds 3]"""
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

W, S = 75000, 7500
KS = (1, 3, 7)
PEAK_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown", "max_sm_clock": "unknown"}


def models(C, path, dev, n):
    """M0 (seed-0 weights) and n - 1 heads with its conv weights and other LSTM / Linear weights"""
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    sd = O.make_ref(oarch, seed=0).state_dict()
    out = []
    for i in range(n):
        g = torch.Generator().manual_seed(100 + i)
        sdi = sd if i == 0 else {k: v if k.startswith("conv") else v + 0.05 * torch.randn(v.shape, generator=g) for k, v in sd.items()}
        m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W), has_out12=oarch.has_out12,
                                path="generic" if path == "generic" else "auto").to(dev)
        m.load_state_dict(sdi)
        out.append(m)
    return out


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


def kernel_ms(fn, steps):
    """device ms per call of fn by kernel group, from a torch.profiler run of its own"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    groups = {"projection": ("slide_ring_proj_kernel", "ring_proj_kernel"),
              "heads": ("head_reduce_independent_kernel", "reduce_gates_kernel", "head_independent_kernel")}
    out = {g: 0.0 for g in groups}
    out["all"] = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if not t or e.key.startswith(("cudaLaunch", "cudaMemcpy", "cudaEvent", "cudaStream", "cudaFunc")):
            continue
        out["all"] += t
        for g, names in groups.items():
            if any(n in e.key for n in names):
                out[g] += t
    return {g: v / 1e3 / steps for g, v in out.items()}


def ward(C, P, path, steps, warmup, rounds, dev):
    ms = models(C, path, dev, 1 + max(KS))
    sep = [tskd_b200.SlidingScorer(m, P, S, path=path) for m in ms]           # separate scorers, one per model
    base = tskd_b200.SlidingScorer(ms[0], P, S, path=path)                    # no heads
    withk = {}
    for K in KS:
        withk[K] = tskd_b200.SlidingScorer(ms[0], P, S, path=path)
        withk[K].set_heads(ms[1:1 + K])
    ages = tskd_b200.synth.make_ages(P, seed=1, device=dev)
    Sp = (S + 7) // 8 * 8
    segs = [torch.empty(P, C, Sp, dtype=torch.bfloat16, device=dev)[:, :, :S] for _ in range(2)]
    for j, s in enumerate(segs):
        s.copy_(tskd_b200.synth.make_windows(P, C, S, "normal", seed=300 + j, dtype=torch.bfloat16, device=dev))
    scs = sep + [base] + list(withk.values())
    for t in range(W // S):                                                   # every window complete
        for sc in scs:
            sc.push(segs[t % 2], ages)
    # bit identity on the timed shape: row i of push(heads=True) equals the separate scorer of model i
    want = [sc.push(segs[1], ages) for sc in sep]
    base.push(segs[1], ages)
    same = all(torch.equal(sc.push(segs[1], ages, heads=True), torch.stack(want[:1 + K])) for K, sc in withk.items())
    arms = {"push": lambda: base.push(segs[0], ages)}
    for K in KS:
        arms[f"push_heads_k{K}"] = (lambda sc: lambda: sc.push(segs[0], ages, heads=True))(withk[K])
        arms[f"separate_{K + 1}"] = (lambda n: lambda: [sep[i].push(segs[0], ages) for i in range(n)])(K + 1)
    res = timed(arms, steps, warmup, rounds)
    prof = {"k0": kernel_ms(lambda: base.push(segs[0], ages), steps)}
    for K in KS:
        prof[f"k{K}"] = kernel_ms(lambda: withk[K].push(segs[0], ages, heads=True), steps)
    L = ms[0].arch.l_out
    out = {"C": C, "P": P, "path": base.path, "L": L, "arms": res, "device_ms_per_push": prof,
           "heads_bit_identical_to_separate_scorers": bool(same)}
    for K in KS:
        out[f"k{K}_over_separate"] = res[f"push_heads_k{K}"]["ms"] / res[f"separate_{K + 1}"]["ms"]
        out[f"k{K}_extra_over_push"] = res[f"push_heads_k{K}"]["ms"] / res["push"]["ms"] - 1
    if path == "tensorcore":
        ring = 4 * L * ((P + 3) // 4 * 4)
        tiles = (P + 127) // 128
        nt = max(((L + 32) // 33 + 4 + 5) // 6, 4)                          # TcState: tiles, features, chunks per CTA
        fpc = 6 * nt - 4
        ranges = (L + fpc - 1) // fpc
        wpack = ranges * ((3 * nt + 7) // 8) * 6144
        part = 4 * ranges * P * 64
        for K in (0,) + KS:
            rows = 1 + K
            pairs = 1 if K == 0 else (rows + 1) // 2
            nbytes = ring * pairs + rows * (wpack + part)
            t = prof[f"k{K}"]["projection"]
            out[f"projection_k{K}"] = {"ms": t, "algorithmic_bytes": nbytes, "ring_bytes": ring * pairs,
                                       "wih_chunk_bytes": rows * wpack, "partial_bytes": rows * part,
                                       "wih_chunk_rereads_per_tile_bytes": rows * tiles * wpack,
                                       "share_of_3.35TBps": nbytes / (t * 1e-3) / PEAK_BPS if t else None}
        out["head_bytes_tensorcore"] = (3345 * 4 + 255) // 256 * 256 + (4 * L * 64 + 255) // 256 * 256 + wpack + part
    for sc in scs:
        sc.close()
    del ms, sep, withk, segs
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tc-patients", type=int, default=4096)
    ap.add_argument("--generic-patients", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slide_heads_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}", file=sys.stderr)
    res = []
    for C, P, path in ((3, a.tc_patients, "tensorcore"), (10, a.generic_patients, "generic")):
        r = ward(C, P, path, a.steps, a.warmup, a.rounds, dev)
        arms = ", ".join(f"{k} {v['ms']:.3f} ms" for k, v in r["arms"].items())
        print(f"{path} C={C} P={P}: {arms}", file=sys.stderr)
        print(f"  device ms per push: {json.dumps(r['device_ms_per_push'])}", file=sys.stderr)
        for K in (0,) + KS:
            pr = r.get(f"projection_k{K}")
            if pr:
                print(f"  projection K={K}: {pr['ms']:.3f} ms, {pr['algorithmic_bytes'] / 1e6:.0f} MB, "
                      f"{100 * pr['share_of_3.35TBps']:.0f} % of 3.35 TB/s", file=sys.stderr)
        print(f"  rows bit-identical to separate scorers: {r['heads_bit_identical_to_separate_scorers']}", file=sys.stderr)
        res.append(r)
    print(json.dumps({"metric": "SlidingScorer extra heads, W = 75000, S = 7500, bf16", "card": c, "wards": res}))


if __name__ == "__main__":
    main()
