"""Instruction census of the bf16 streaming kernel's main loop (no GPU needed).

Compiles csrc/b2cnn_tc.cu for sm_90a (or reads an already built object with --object), disassembles one
tc_stream_kernel instance (default: the flagship, MyCNN5 C=3, 3 weight pieces, gates out) and prints

  * the instructions of its main loop per 8-position block, by class, with the projection (every 8th block) apart;
  * the registers each role uses (the highest register it names; setmaxnreg gives the limit), spills and stack;
  * every warpgroup wait ptxas injected (C7517), and the R2UR / warpgroup waits inside the loop.

The main loop is the backward branch whose body holds the most conv1 HGMMA.64x32; its blocks per iteration are
those HGMMAs / (2 row halves x C x SPLITS).  A projection is the code a forward branch skips around a run of
HGMMA.64x64.

    python scripts/sass_census.py                   # compile b2cnn_tc.cu, flagship instance
    python scripts/sass_census.py --object time-series-kafka-demo_b200/lib/obj/b2cnn_tc.o
    python scripts/sass_census.py --c 1 --splits 2 --out 0
"""
from __future__ import annotations

import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "time-series-kafka-demo_b200", "csrc")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")

CLASSES = [
    ("epilogue float", ("FFMA", "FMNMX", "MUFU", "FADD", "FMUL", "F2FP", "FSEL", "FSETP", "FCHK")),
    ("HGMMA", ("HGMMA",)),
    ("shared memory", ("LDS", "STS", "LDSM")),
    ("global memory", ("LDG", "STG", "LD", "ST", "ATOM", "ATOMS", "RED")),
    ("integer / moves", ("IMAD", "LOP3", "MOV", "LEA", "ISETP", "IADD3", "S2R", "SHF", "SEL", "PRMT", "IABS", "IMNMX",
                         "R2UR", "CS2R", "S2UR", "VIADD", "IADD", "ISCADD", "P2R", "R2P", "PLOP3", "SGXT", "BMSK", "POPC",
                         "FLO", "BREV", "LDC", "VOTE", "SHFL", "I2F", "F2I")),
    ("uniform datapath", ("U",)),
    ("barriers, mbarrier, branches", ("BAR", "SYNCS", "BRA", "WARPGROUP", "MEMBAR", "FENCE", "WARPSYNC", "BSSY", "BSYNC",
                                      "EXIT", "NOP", "CCTL", "DEPBAR", "ELECT", "YIELD", "RET", "CALL", "BPT")),
]

INS_RE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")


def classify(op: str) -> str:
    base = op.split(".")[0]
    for name, prefixes in CLASSES:
        if name == "uniform datapath":
            if base.startswith("U") and base not in ("UNKNOWN",):
                return name
            continue
        if base in prefixes:
            return name
    return "other"


def parse_sass(text: str):
    """-> [(addr, opcode, full text)] of the first function in `text`, predicate guards stripped"""
    out = []
    for m in INS_RE.finditer(text):
        addr, body = int(m.group(1), 16), m.group(2).strip()
        if body.startswith("@"):
            body = body.split(None, 1)[1]
        op = body.split()[0]
        out.append((addr, op, body))
    return out


def branch_target(body: str):
    m = re.search(r"\bBRA(?:\.\S+)?\s+(?:`?\(?[!]?U?P\d,\s*)?(0x[0-9a-f]+)", body)
    return int(m.group(1), 16) if m else None


def census(ins, C: int, splits: int):
    idx = {a: i for i, (a, _, _) in enumerate(ins)}
    per_block_mma = 2 * C * splits
    # the main loop: backward branch with the most conv1 HGMMAs in its body
    best = None
    for i, (a, op, body) in enumerate(ins):
        if not op.startswith("BRA"):
            continue
        t = branch_target(body)
        if t is None or t >= a or t not in idx:
            continue
        lo = idx[t]
        if any(o.startswith("EXIT") for _, o, _ in ins[lo:i]):
            continue            # an out-of-line mbarrier retry jumping back, not a loop
        n32 = sum(1 for _, o, b in ins[lo:i + 1] if o.startswith("HGMMA") and "64x32x16" in o)
        if n32 and (best is None or n32 > best[2] or (n32 == best[2] and i - lo > best[1] - best[0])):
            best = (lo, i, n32)
    if best is None:
        raise SystemExit("no loop with conv1 HGMMAs found")
    lo, hi, n32 = best
    body = ins[lo:hi + 1]
    blocks = n32 // per_block_mma
    # projections: the code a forward branch skips around each run of HGMMA.64x64
    runs = []
    for k, (_, op, _) in enumerate(body):
        if op.startswith("HGMMA") and "64x64x16" in op:
            if runs and k - runs[-1][1] <= 64:
                runs[-1][1] = k
            else:
                runs.append([k, k])
    proj = []
    for r0, r1 in runs:
        span = None
        for k in range(r0, -1, -1):
            a, op, b = body[k]
            if op.startswith("BRA"):
                t = branch_target(b)
                if t is not None and t > body[r1][0] and t <= body[-1][0] and (span is None or idx[t] - lo > span[1]):
                    span = (k + 1, idx[t] - lo)
        if span:
            proj.append(span)
    in_proj = set()
    for s0, s1 in proj:
        in_proj.update(range(s0, s1))
    main = [body[k] for k in range(len(body)) if k not in in_proj]
    projc = [body[k] for k in sorted(in_proj)]
    return body, blocks, main, projc, len(proj)


def table(rows, blocks, title):
    cnt = collections.Counter(classify(op) for _, op, _ in rows)
    ops = collections.defaultdict(collections.Counter)
    for _, op, _ in rows:
        ops[classify(op)][op.split(".")[0]] += 1
    print(title)
    tot = 0
    for name, _ in CLASSES + [("other", ())]:
        if cnt[name]:
            top = ", ".join(f"{o} {n / blocks:g}" for o, n in ops[name].most_common(8))
            print(f"  {name:32s} {cnt[name] / blocks:7.1f}   ({top})")
            tot += cnt[name]
    print(f"  {'total':32s} {tot / blocks:7.1f}")
    return cnt


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--object", help="read this built object / cubin instead of compiling b2cnn_tc.cu")
    ap.add_argument("--c", type=int, default=3)
    ap.add_argument("--splits", type=int, default=3)
    ap.add_argument("--arch", type=int, default=0)
    ap.add_argument("--out", type=int, default=1, help="0 features, 1 gates, 2 ring")
    ap.add_argument("--nvcc", default=os.path.join(CUDA, "bin", "nvcc"))
    args = ap.parse_args()
    fn = f"_ZN5b2cnn16tc_stream_kernelILi{args.c}ELi{args.splits}ELi{args.arch}ELb0ELi{args.out}EEEv14CUtensorMap_stNS_13TcFusedParamsE"

    with tempfile.TemporaryDirectory() as tmp:
        ptxas_log = None
        obj = args.object
        if obj is None:
            obj = os.path.join(tmp, "b2cnn_tc.cubin")
            r = subprocess.run([args.nvcc, "-cubin", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                                "-Xptxas", "-v", "-o", obj, os.path.join(CSRC, "b2cnn_tc.cu")],
                               cwd=CSRC, capture_output=True, text=True)
            if r.returncode != 0:
                sys.stderr.write(r.stderr)
                return 1
            ptxas_log = r.stderr
        cuobjdump = os.path.join(CUDA, "bin", "cuobjdump")
        sass = subprocess.run([cuobjdump, "-sass", "-fun", fn, obj], capture_output=True, text=True, check=True).stdout
        res = subprocess.run([cuobjdump, "-res-usage", "-fun", fn, obj], capture_output=True, text=True, check=True).stdout

    ins = parse_sass(sass)
    if not ins:
        print(f"{fn} not found", file=sys.stderr)
        return 1
    print(f"{fn}\n")
    body, blocks, main_, projc, nproj = census(ins, args.c, args.splits)
    print(f"main loop 0x{body[0][0]:x}-0x{body[-1][0]:x}: {len(body)} instructions, {blocks} block(s) per iteration, "
          f"{nproj} projection site(s) ({len(projc)} instructions)\n")
    table(main_, blocks, "per 8-position block, projection excluded:")
    if nproj:
        print()
        table(projc, nproj, "per projection (once every 8 blocks):")
        print(f"\n  average per block: {(len(main_) / blocks) + len(projc) / nproj / 8:.1f}")

    r2ur = sum(1 for _, op, _ in body if op.startswith("R2UR"))
    waits = [(a, b) for a, op, b in body if op.startswith("WARPGROUP.DEPBAR")]
    bars = [(a, b) for a, op, b in body if op.startswith("BAR.SYNC")]
    # the source waits once per block (it retires the block's conv1 and the projection issued a block earlier) and
    # passes one warpgroup barrier per block (the a1 exchange): any more waits are ptxas's
    print(f"\nin the loop: R2UR {r2ur}, warpgroup waits {len(waits)} (the source's: {blocks}), "
          f"named barriers {len(bars)} (the source's: {blocks})")

    # registers per role: setmaxnreg limits and the highest register each role's code names
    # (a role's code ends at the next setmaxnreg or the function's last EXIT: the mbarrier retry loops ptxas moves
    # out of line come after it)
    roles = [(a, op, b) for a, op, b in ins if op.startswith("USETMAXREG")]
    if roles:
        starts = sorted(a for a, _, _ in roles)
        last_exit = max(a for a, op, _ in ins if op.startswith("EXIT"))
        for a, op, b in roles:
            lim = int(re.search(r"(0x[0-9a-f]+)\s*$", b).group(1), 16)
            end = min([s for s in starts if s > a] + [last_exit + 1])
            regs = [int(x) for aa, _, bb in ins if a <= aa < end for x in re.findall(r"\bR(\d+)\b", bb)]
            role = "consumer" if "TRY_ALLOC" in op else "producer"
            print(f"{role}: setmaxnreg {lim}, highest register R{max(regs) if regs else 0}")
    m = re.search(r"REG:(\d+)\s+STACK:(\d+)\s+SHARED:(\d+)\s+LOCAL:(\d+)", res)
    if m:
        print(f"launch: {m.group(1)} registers, stack {m.group(2)} B, local {m.group(4)} B")
    if ptxas_log is not None:
        blk = ptxas_log.split(f"Compiling entry function '{fn}'")
        if len(blk) > 1:
            sp = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", blk[1])
            if sp:
                print(f"ptxas: stack frame {sp.group(1)} B, spill stores {sp.group(2)} B, spill loads {sp.group(3)} B")
        inj = [ln for ln in ptxas_log.splitlines() if "C7517" in ln and f"'{fn}'" in ln]
        ser = [ln for ln in ptxas_log.splitlines() if "C7515" in ln or ("serializ" in ln and fn in ln)]
        print(f"ptxas injected warpgroup waits: {len(inj)}")
        for ln in inj:
            print("  " + re.sub(r" by compiler.*", "", ln.split("info    : ")[-1]))
        print(f"ptxas serialized wgmma messages: {len(ser)}")
        for ln in ser:
            print("  " + ln)
    else:
        print("ptxas messages (injected waits, spills): only when compiling (drop --object)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
