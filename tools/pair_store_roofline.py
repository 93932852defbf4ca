"""Write ceiling of the headline's coefficient store pattern (developer tool, not the benchmark).

The headline (1 048 576 trajectories x 16 segments, N = 10, r = 4, D = 3, fp64) writes a [B][K*D*N] coefficient
tensor of 4.03 GB per solve, one 240-byte segment of a row at a time.  In one process this times, at that size:

  fill       a plain device write of the whole tensor (the write ceiling);
  copy       a device copy into it from a tensor of the same size (bytes read + bytes written);
  fill240    the same tensor written as 240-byte pieces (one segment): the even segments of every row, then the odd
             ones, by two strided fills; every odd piece starts and ends 16 bytes into a 32-byte sector;
  fill480    the same with 480-byte pieces (two segments, every piece on a sector boundary);
  copy240,   the same two patterns by strided copies from a contiguous source (bytes written only);
  copy480
  solve      the headline solve (Solver.solve_linear, default route), bytes = Problem.bytes_per_trajectory * B,

alternating them in every round (CUDA events around --reps launches after one untimed launch).  Each line gives the
median over the rounds in GB/s, the spread of the round values, and the share of the plain-write figure.  The card
name, power limit and SM clock are read in the same run.

  python tools/pair_store_roofline.py [--rounds 5] [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import mav_trajectory_generation_b200 as m  # noqa: E402
from quick_bench import synth  # noqa: E402

N, R, K, D, B = 10, 4, 16, 3, 1048576


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power, max_clock, clock = [x.strip() for x in q.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=max_clock, sm_clock_at_start=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("pair_store_roofline.py needs a CUDA device")

    dev = torch.device("cuda:0")
    info = card()
    row = K * D * N
    out = torch.empty((B, row), device=dev, dtype=torch.float64)
    src = torch.ones((B, row), device=dev, dtype=torch.float64)
    half = torch.ones((B, K // 2, D * N), device=dev, dtype=torch.float64)
    out_bytes = out.numel() * 8
    seg = out.view(B, K, D * N)        # pieces of one segment, 240 bytes
    pair = out.view(B, K // 2, 2 * D * N)  # pieces of two segments, 480 bytes
    pair_src = half.view(B, K // 4, 2 * D * N)

    prob = m.Problem(N, R, K, D)
    solver = m.Solver(0)
    times, dfix = synth(N, K, D, B, dev)
    coeffs = out.view(B, K, D, N)

    cases = {
        "fill": (lambda: out.fill_(1.0), out_bytes),
        "copy": (lambda: out.copy_(src), 2 * out_bytes),
        "fill240": (lambda: (seg[:, 0::2].fill_(1.0), seg[:, 1::2].fill_(2.0)), out_bytes),
        "fill480": (lambda: (pair[:, 0::2].fill_(1.0), pair[:, 1::2].fill_(2.0)), out_bytes),
        "copy240": (lambda: (seg[:, 0::2].copy_(half), seg[:, 1::2].copy_(half)), out_bytes),
        "copy480": (lambda: (pair[:, 0::2].copy_(pair_src), pair[:, 1::2].copy_(pair_src)), out_bytes),
        "solve": (lambda: solver.solve_linear(prob, times, dfix, coeffs=coeffs), prob.bytes_per_trajectory * B),
    }
    per = {k: [] for k in cases}
    names = list(cases)
    for rnd in range(args.rounds):
        for name in (names if rnd % 2 == 0 else names[::-1]):
            fn, nbytes = cases[name]
            fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            per[name].append(nbytes * args.reps / (e0.elapsed_time(e1) * 1e-3) / 1e9)
    info["sm_clock_at_end"] = card()["sm_clock_at_start"]

    def med(v):
        v = sorted(v)
        return v[len(v) // 2]

    ceiling = med(per["fill"])
    rows = []
    for name in names:
        g = med(per[name])
        rows.append(dict(case=name, gb_s=round(g, 1), spread_gb_s=round(max(per[name]) - min(per[name]), 1),
                         share_of_fill=round(g / ceiling, 4)))
    lines = ["%s, power limit %s, max SM clock %s, SM clock %s at start and %s at end; %d rounds of %d launches"
             % (info["name"], info["power_limit"], info["max_sm_clock"], info["sm_clock_at_start"],
                info["sm_clock_at_end"], args.rounds, args.reps), "",
             "| case | GB/s | spread GB/s | share of fill |", "|---|---|---|---|"]
    for r in rows:
        lines.append("| %s | %.1f | %.1f | %.3f |" % (r["case"], r["gb_s"], r["spread_gb_s"], r["share_of_fill"]))
    table = "\n".join(lines)
    print(table)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pair_store_roofline.md"), "w") as f:
            f.write(table + "\n")
        with open(os.path.join(args.out, "pair_store_roofline.json"), "w") as f:
            json.dump(dict(card=info, rows=rows, rounds=per), f, indent=1)


if __name__ == "__main__":
    main()
