#!/usr/bin/env python
"""Check that two builds of libb2cnn compute byte-identical results (needs a GPU).

Runs itself once per library (B2CNN_LIB selects the build; a process loads one), each run computing on the same
inputs, with seed-0 MyCNN5 weights:
  * predict() logits at [--batch, 3, 75000] bf16 (the bench.py workload: the fused streaming kernel, gates out);
  * model.features() at [--feat-batch, 3, 75000] bf16 (the feature-row kernel);
  * one SlidingScorer push after a full window of pushes (the feature-ring kernel), logits and the ring's features;
  * push(heads=True) with three heads, one of a shorter window (the ring projection with two rows per CTA, its
    padding row, and one row alone), and export() of a few patients;
  * a tensor-core scorer at W = 7502 (phase 2, so an admission's history is staged): a full-history admit of three
    patients, then one push;
  * a generic-path scorer (C = 10, bf16) after a full window of pushes;
  * predict_record() on the tensor-core and generic paths, independent and sequence modes;
  * training: one B200Trainer.step (sequence, dropout masks given) at [2048, 10, 120] and at [256, 3, 75000], with the
    loss, the gradients and the updated parameters; and one autograd forward and backward at [257, 10, 120] with the
    logits, every parameter gradient, d x and d age; and the dropout masks B200Trainer(seed=0).draw_masks(64) and
    B200TrainableMyCNN.draw_masks(64) after torch.manual_seed(0);
then compares every array bit for bit and prints each array's status and max |diff|.

    python scripts/compare_builds.py --baseline-lib /path/to/parent/libb2cnn.so [--lib /path/to/libb2cnn.so]
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, S, C = 75000, 7500, 3


def dump(path: str, batch: int, feat_batch: int, patients: int) -> None:
    sys.path.insert(0, ROOT)
    import torch

    import tskd_b200
    from oracle import mycnn_torch as O

    dev = "cuda:0"
    oarch = O.stretched(O.ARCH_MYCNN5, C, W)
    m = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, W), has_out12=oarch.has_out12).to(dev)
    m.load_state_dict(O.make_ref(oarch, seed=0).state_dict())
    out = {}
    x = tskd_b200.synth.make_windows(batch, C, W, "normal", seed=7, dtype=torch.bfloat16, device=dev)
    ages = tskd_b200.synth.make_ages(batch, seed=7, device=dev)
    out["predict_logits"] = m.predict(x, ages)
    out["predict_path"] = np.array([m.last_path])
    out["features"] = m.features(x[:feat_batch])
    del x
    sc = tskd_b200.SlidingScorer(m, patients, S)
    pages = tskd_b200.synth.make_ages(patients, seed=9, device=dev)
    for i in range(W // S + 1):
        seg = tskd_b200.synth.make_windows(patients, C, S, "normal", seed=200 + i, dtype=torch.bfloat16, device=dev)
        got = sc.push(seg.contiguous(), pages)
    out["slide_logits"] = got
    out["slide_features"] = sc.features()

    # heads: rows 0-2 share the window W (a pair and a padded pair), row 3 has a shorter one and runs alone
    conv = {k: v for k, v in m.state_dict().items() if k.startswith("conv")}
    heads = []
    for i, Wk in enumerate((W, W, W // 2)):
        ha = O.stretched(O.ARCH_MYCNN5, C, Wk)
        hm = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, Wk), has_out12=ha.has_out12).to(dev)
        sd = O.make_ref(ha, seed=20 + i).state_dict()
        sd.update(conv)
        hm.load_state_dict(sd)
        heads.append(hm)
    sc.set_heads(heads, shorter_windows=True)
    seg = tskd_b200.synth.make_windows(patients, C, S, "normal", seed=300, dtype=torch.bfloat16, device=dev)
    out["heads_logits"] = sc.push(seg.contiguous(), pages, heads=True)
    st = sc.export([0, 5, 17, patients - 1])
    out["export_features"], out["export_tail"], out["export_seen"] = st["features"], st["tail"], st["seen"]
    del sc, heads

    # admission with a full history at phase 2: staged before the tensor-core front end
    Wa, Sa, Pa = 7502, 1876, 64
    aa = O.stretched(O.ARCH_MYCNN5, C, Wa)
    ma = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(C, Wa), has_out12=aa.has_out12).to(dev)
    ma.load_state_dict(O.make_ref(aa, seed=1).state_dict())
    sa = tskd_b200.SlidingScorer(ma, Pa, Sa)
    aages = tskd_b200.synth.make_ages(Pa, seed=10, device=dev)
    for i in range(Wa // Sa + 1):
        sa.push(tskd_b200.synth.make_windows(Pa, C, Sa, "normal", seed=400 + i, dtype=torch.bfloat16, device=dev), aages)
    sa.admit([3, 10, 40], tskd_b200.synth.make_windows(3, C, Wa, "normal", seed=410, dtype=torch.bfloat16, device=dev))
    out["admit_logits"] = sa.push(tskd_b200.synth.make_windows(Pa, C, Sa, "normal", seed=411, dtype=torch.bfloat16, device=dev),
                                  aages)
    out["admit_features"] = sa.features()
    del sa

    # the generic path: 10 channels have no tensor-core kernel
    Wg, Sg, Pg, Cg = 1200, 120, 256, 10
    ag = O.stretched(O.ARCH_MYCNN5, Cg, Wg)
    mg = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(Cg, Wg), has_out12=ag.has_out12).to(dev)
    mg.load_state_dict(O.make_ref(ag, seed=2).state_dict())
    sg = tskd_b200.SlidingScorer(mg, Pg, Sg, path="generic")
    gages = tskd_b200.synth.make_ages(Pg, seed=11, device=dev)
    for i in range(Wg // Sg + 1):
        got = sg.push(tskd_b200.synth.make_windows(Pg, Cg, Sg, "normal", seed=500 + i, dtype=torch.bfloat16, device=dev), gages)
    out["generic_slide_logits"] = got
    out["generic_slide_features"] = sg.features()
    del sg

    # whole recordings
    rec = tskd_b200.synth.make_windows(4, C, 4 * W, "normal", seed=600, dtype=torch.bfloat16, device=dev)
    recg = tskd_b200.synth.make_windows(8, Cg, 20 * Wg, "normal", seed=601, dtype=torch.bfloat16, device=dev)
    for mode in ("independent", "sequence"):
        out[f"record_tc_{mode}"] = m.predict_record(rec, S, 60.0, path="tensorcore", mode=mode)
        out[f"record_generic_{mode}"] = mg.predict_record(recg, Sg, 60.0, path="generic", mode=mode)
    del m, mg, rec, recg

    # training
    from tskd_b200.arch import BLOB_KEYS
    from tskd_b200.trainer import B200Trainer

    def train_inputs(Ct, Wt, Bt, seed):
        ta = O.stretched(O.ARCH_MYCNN5, Ct, Wt)
        g = torch.Generator(device=dev).manual_seed(seed)
        xt = torch.randn(Bt, Ct, Wt, generator=g, device=dev)
        at = torch.rand(Bt, generator=g, device=dev) * 60 + 20
        yt = (torch.rand(Bt, generator=g, device=dev) > 0.5).float()
        m1 = torch.bernoulli(torch.full((Bt, ta.c_mid, ta.p1), 0.9, device=dev), generator=g) / 0.9
        m2 = torch.bernoulli(torch.full((Bt, ta.l_out), 0.9, device=dev), generator=g) / 0.9
        return ta, xt, at, yt, m1, m2

    for Ct, Wt, Bt in ((10, 120, 2048), (3, 75000, 256)):
        ta, xt, at, yt, m1, m2 = train_inputs(Ct, Wt, Bt, 12)
        tm = tskd_b200.B200MyCNN(tskd_b200.ARCH_PRESETS["mycnn5"].with_shape(Ct, Wt), has_out12=ta.has_out12).to(dev)
        tm.load_state_dict(O.make_ref(ta, seed=3).state_dict())
        tr = B200Trainer(tm, mode="sequence", dropout=0.1)
        tag = f"train_step_{Bt}x{Ct}x{Wt}"
        out[tag + "_loss"] = tr.step(xt, at, yt, masks=(m1, m2)).reshape(1)
        out.update({f"{tag}_grad_{k}": v.clone() for k, v in tr.grads().items()})
        sd = tm.state_dict()
        out.update({f"{tag}_param_{k}": sd[k].clone() for k in BLOB_KEYS})
        del tr, tm, xt
    ta, xt, at, _, m1, m2 = train_inputs(10, 120, 257, 13)
    sd = O.make_ref(ta, seed=4).state_dict()
    params = [sd[k].to(dev).clone().requires_grad_() for k in BLOB_KEYS]
    xt.requires_grad_()
    at.requires_grad_()
    z = tskd_b200.mycnn_train_forward(xt, at, params, tskd_b200.ARCH_PRESETS["mycnn5"], "sequence", m1, m2)
    z.backward(torch.randn(257, generator=torch.Generator(device=dev).manual_seed(14), device=dev))
    tag = "train_autograd_257x10x120"
    out[tag + "_z"] = z.detach()
    out.update({f"{tag}_grad_{k}": p.grad for k, p in zip(BLOB_KEYS, params)})
    out[tag + "_dx"], out[tag + "_dage"] = xt.grad, at.grad
    # dropout masks: the trainer's seeded generator, and torch's default generator under autograd
    dm = tskd_b200.B200TrainableMyCNN(tskd_b200.ARCH_PRESETS["mycnn5"]).to(dev)
    out["masks_trainer_mask1"], out["masks_trainer_mask2"] = B200Trainer(dm, seed=0).draw_masks(64)
    torch.manual_seed(0)
    out["masks_autograd_mask1"], out["masks_autograd_mask2"] = dm.draw_masks(64)
    torch.cuda.synchronize()
    np.savez(path, **{k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in out.items()})


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--baseline-lib", required=True)
    ap.add_argument("--lib", default=None, help="the build under test (default: the package's own lib/libb2cnn.so)")
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--feat-batch", type=int, default=1024)
    ap.add_argument("--patients", type=int, default=1024)
    ap.add_argument("--dump", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump:
        dump(args.dump, args.batch, args.feat_batch, args.patients)
        return 0
    runs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, lib in (("baseline", args.baseline_lib), ("candidate", args.lib)):
            env = dict(os.environ)
            env.pop("B2CNN_LIB", None)
            if lib:
                env["B2CNN_LIB"] = os.path.abspath(lib)
            path = os.path.join(tmp, name + ".npz")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--dump", path, "--batch", str(args.batch),
                                   "--feat-batch", str(args.feat_batch), "--patients", str(args.patients),
                                   "--baseline-lib", "-"], env=env)
            runs[name] = dict(np.load(path))
    ok = True
    for k, a in runs["baseline"].items():
        b = runs["candidate"][k]
        same = a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()
        ok &= same
        extra = "" if a.dtype.kind == "U" else f", max |diff| {np.abs(a.astype(np.float64) - b.astype(np.float64)).max():.3g}" if a.shape == b.shape else ""
        print(f"{k:56s} {str(a.shape):16s} {'byte-identical' if same else 'DIFFERENT'}{extra}  {a.ravel()[:1]}")
    print("all byte-identical" if ok else "builds differ")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
