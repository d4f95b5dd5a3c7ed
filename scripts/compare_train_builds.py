#!/usr/bin/env python
"""Check that two built checkouts train byte-identically where scripts/compare_builds.py does not look (needs a GPU).

Runs itself once per checkout (each process imports tskd_b200 and its lib/libb2cnn.so from that checkout's tree, so the
Python trainers are compared along with the library), each run on the same seeded inputs and masks:
  * B200HeadTrainer with K = 3 heads (one of them the model), sequence mode, pos_weight 2: three .step calls at
    [64, 10, 120] with seq_lengths, then three .step_record calls over [4, 10, 480] recordings at stride 40 with
    ragged window counts;
  * B200Trainer.step_record, sequence mode: three steps over the same recordings, then three more carrying the LSTM
    state from chunk to chunk (state / return_state);
saving every step's losses, and after each trainer's last step its gradients and every head's parameters.  Then it
compares every array bit for bit and prints each array's status.

    python scripts/compare_train_builds.py --baseline-root /path/to/parent/checkout [--root /path/to/candidate]
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dump(path: str, root: str) -> None:
    sys.path.insert(0, root)
    import torch

    import tskd_b200
    from tskd_b200.arch import BLOB_KEYS

    dev = "cuda:0"
    arch = tskd_b200.ARCH_PRESETS["mycnn5"]
    g = torch.Generator(device=dev).manual_seed(21)

    def model(seed):
        torch.manual_seed(seed)
        return tskd_b200.B200MyCNN(arch).to(dev)

    def masks(a, B):
        return tskd_b200.autograd.draw_masks(a, B, 0.1, dev, g)

    out = {}
    base = model(0)
    heads = [model(1), model(2), base]
    for h in heads[:2]:                                   # every head shares the model's front end
        h.load_state_dict({**h.state_dict(), **{k: v for k, v in base.state_dict().items() if k.startswith("conv")}})
    tr = tskd_b200.B200HeadTrainer(base, heads, lr=[1e-3, 3e-4, 1e-4], pos_weight=2.0)
    B, lens = 64, [20, 1, 30, 13]
    for i in range(3):
        x = torch.randn(B, 10, 120, device=dev, generator=g)
        age = torch.rand(B, device=dev, generator=g) * 60 + 20
        y = (torch.rand(B, device=dev, generator=g) > 0.5).float()
        out[f"heads_step{i}_loss"] = tr.step(x, age, y, masks=masks(arch, B), seq_lengths=lens)
    N, S, counts = 480, 40, [10, 0, 4, 7]
    rarch = arch.with_shape(10, N)
    for i in range(3):
        rec = torch.randn(4, 10, N, device=dev, generator=g)
        age = torch.rand(4, device=dev, generator=g) * 60 + 20
        y = (torch.rand(sum(counts), device=dev, generator=g) > 0.5).float()
        out[f"heads_record{i}_loss"] = tr.step_record(rec, S, age, y, window_counts=counts, masks=masks(rarch, 4))
    for h, grads in enumerate(tr.grads()):
        out.update({f"heads_grad{h}_{k}": v.clone() for k, v in grads.items()})
    for h, m in enumerate(heads):
        sd = m.state_dict()
        out.update({f"heads_param{h}_{k}": sd[k].clone() for k in BLOB_KEYS})

    m = model(5)
    tr = tskd_b200.B200Trainer(m, mode="sequence")
    state = None
    for i in range(6):
        rec = torch.randn(4, 10, N, device=dev, generator=g)
        age = torch.rand(4, device=dev, generator=g) * 60 + 20
        y = (torch.rand(sum(counts), device=dev, generator=g) > 0.5).float()
        if i < 3:
            out[f"record{i}_loss"] = tr.step_record(rec, S, age, y, window_counts=counts, masks=masks(rarch, 4))
        else:
            loss, state = tr.step_record(rec, S, age, y, window_counts=counts, masks=masks(rarch, 4), state=state, return_state=True)
            out[f"record{i}_loss"], out[f"record{i}_state"] = loss, state
    out.update({f"record_grad_{k}": v.clone() for k, v in tr.grads().items()})
    sd = m.state_dict()
    out.update({f"record_param_{k}": sd[k].clone() for k in BLOB_KEYS})
    torch.cuda.synchronize()
    np.savez(path, **{k: v.detach().reshape(-1).cpu().numpy() for k, v in out.items()})


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--baseline-root", required=True, help="a checkout of the baseline, built")
    ap.add_argument("--root", default=ROOT, help="the checkout under test, built (default: this one)")
    ap.add_argument("--dump", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump:
        dump(args.dump, os.path.abspath(args.root))
        return 0
    runs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, root in (("baseline", args.baseline_root), ("candidate", args.root)):
            env = dict(os.environ)
            env.pop("B2CNN_LIB", None)
            path = os.path.join(tmp, name + ".npz")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--dump", path, "--root", os.path.abspath(root),
                                   "--baseline-root", "-"], env=env)
            runs[name] = dict(np.load(path))
    ok = runs["baseline"].keys() == runs["candidate"].keys()
    for k, a in runs["baseline"].items():
        b = runs["candidate"].get(k)
        same = b is not None and a.shape == b.shape and a.tobytes() == b.tobytes()
        ok &= same
        print(f"{k:48s} {str(a.shape):10s} {'byte-identical' if same else 'DIFFERENT'}  {a[:1]}")
    print("all byte-identical" if ok else "builds differ")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
