"""Forced-configuration sweep of the chunked kernel K3 (developer tool, not the benchmark).

Times K3 (N = 10, r = 4, D = 3) at K = 8, 12, 16, 50 and 100 over
  * C: vertex blocks per lane kept in shared memory (--cs, default 2 to 6),
  * warps per SM, from 4 up to the most that fit, as one-warp CTAs (W = 1) and as four-warp CTAs (W = 4),
  * pairs per SM of the paired form (W = 2: twisted_chunked_pair_kernel, which the default route launches), from 2
    up to the most that fit,
  * L2 cache hints on the streamed inputs and coefficient stores on and off (--hints, default both),
in one process.  Every configuration is timed in each of --rounds rounds (the order alternates between rounds), with
CUDA events around --steps solves after --warmup solves; the line of a configuration gives the median of its round
medians and the spread of the round medians.  `same` says whether its coefficients are bitwise equal to those of the
first configuration of the same K.  The card name and power limit are read in the same run.

  python tools/k3_sweep.py [--ks 8,16,50,100] [--cs 2,3,4,5,6] [--ws 1,4,2] [--hints 0,1] [--rounds 3] [--out DIR]
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

N, R, D = 10, 4, 3
BATCH = {8: 1048576, 12: 1048576, 16: 1048576, 50: 246272, 100: 113664}
SMEM_PER_SM = 228 * 1024  # H100; every CTA also reserves 1 KB
MAX_WARPS_BY_REGS = 8     # K3 at N = 10, D = 3 uses 248-250 registers per thread


def k3_smem(C, W, K):
    """Dynamic shared memory of K3 at N = 10, D = 3 (ChunkedLayout<10, 3, 3, W>::bytes, ring depth 3; W = 2:
    ChunkedPairLayout<10, 3, 3>::bytes)"""
    h, slots = N // 2, 25
    pro = 2 * D + (h - 1) * D + 1
    if W == 2:  # two staging buffers of two segments per row; mbarriers; tile input buffer; final-segment inputs,
        # handoff, times, blocks
        tile = 8 * 16 * (K + D * (2 * h + K - 1))
        region = (D + (h - 1) * D + 1) + h * D + C
        return 4 * 32 * (D * h * 16) + 256 + tile + 32 * 8 * (region + C * slots)
    region = 3 * (1 + D) + C + D + 1
    return 32 * W * (D * h * 16 + 8 * (region + max(C * slots, pro)))


def max_warps(C, W, K):
    return min(MAX_WARPS_BY_REGS, SMEM_PER_SM // (k3_smem(C, W, K) + 1024) * W)


def configs(K, cs, ws, hint_modes):
    nmax = (K + 1) // 2 - 1
    out = []
    for C in cs:
        if C > nmax:
            continue
        for hints in hint_modes:
            if 1 in ws:
                for w in range(4, max_warps(C, 1, K) + 1):
                    out.append(dict(C=C, W=1, warps=w, hints=hints))
            if 4 in ws:
                for w in range(4, max_warps(C, 4, K) + 1, 4):
                    out.append(dict(C=C, W=4, warps=w, hints=hints))
        if 2 in ws:  # the paired form runs without hints
            for w in range(4, max_warps(C, 2, K) + 1, 2):
                out.append(dict(C=C, W=2, warps=w, hints=0))
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(0), power_limit="unknown (%s)" % e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="8,16,50,100")
    ap.add_argument("--cs", default="2,3,4,5,6")
    ap.add_argument("--ws", default="1,4,2", help="CTA forms: 1 and 4 warps, 2 = warp pairs")
    ap.add_argument("--hints", default="0,1")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    dev = torch.device("cuda:0")
    s = m.Solver(0)
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    rows = []
    for K in [int(k) for k in args.ks.split(",")]:
        B = BATCH[K]
        prob = m.Problem(N, R, K, D)
        times, dfix = synth(N, K, D, B, dev)
        out = torch.empty((B, K, D, N), device=dev, dtype=torch.float64)
        cfgs = configs(K, [int(c) for c in args.cs.split(",")], [int(w) for w in args.ws.split(",")],
                       [int(x) for x in args.hints.split(",")])
        per = [[] for _ in cfgs]
        same = [True] * len(cfgs)
        ref = None

        def run(cf):
            # the paired form is the default route's; the one-warp and four-warp forms are forced
            s.set_option(m.capi.OPT_WAYPOINT_VARIANT, 0 if cf["W"] == 2 else 5)
            s.set_option(m.capi.OPT_CHUNK_BLOCKS, cf["C"])
            s.set_option(m.capi.OPT_CHUNK_WARPS, 0 if cf["W"] == 2 else cf["W"])
            s.set_option(m.capi.OPT_CTAS_PER_SM, cf["warps"])
            s.set_option(m.capi.OPT_L2_HINTS, cf["hints"])
            s.solve_linear(prob, times, dfix, coeffs=out)

        for rnd in range(args.rounds):
            order = list(range(len(cfgs)))
            if rnd % 2:
                order.reverse()
            for i in order:
                for _ in range(args.warmup):
                    run(cfgs[i])
                torch.cuda.synchronize()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
                ev[0].record()
                for j in range(args.steps):
                    run(cfgs[i])
                    ev[j + 1].record()
                torch.cuda.synchronize()
                ms = sorted(ev[j].elapsed_time(ev[j + 1]) for j in range(args.steps))
                per[i].append(ms[len(ms) // 2])
                if ref is None:
                    ref = out.clone()
                elif not torch.equal(out.view(torch.int64), ref.view(torch.int64)):
                    same[i] = False
        for i, cf in enumerate(cfgs):
            r = sorted(per[i])
            med = r[len(r) // 2]
            row = dict(K=K, B=B, **cf, ms=round(med, 4), spread_ms=round(r[-1] - r[0], 4),
                       traj_per_s=round(B / (med * 1e-3)), same=same[i])
            rows.append(row)
            print(json.dumps(row), flush=True)
        del out, ref, times, dfix
        torch.cuda.empty_cache()
    for key in ("WAYPOINT_VARIANT", "CHUNK_BLOCKS", "CHUNK_WARPS", "CTAS_PER_SM", "L2_HINTS"):
        s.set_option(getattr(m.capi, "OPT_" + key), 0)

    lines = ["%s, power limit %s" % (info.get("name"), info.get("power_limit")), "",
             "| K | C | W | warps/SM | L2 hints | ms | spread ms | traj/s | same |",
             "|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        lines.append("| %d | %d | %d | %d | %s | %.3f | %.3f | %.3g | %s |" % (
            r["K"], r["C"], r["W"], r["warps"], "on" if r["hints"] else "off", r["ms"], r["spread_ms"],
            r["traj_per_s"], "yes" if r["same"] else "NO"))
    table = "\n".join(lines)
    print(table)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "k3_sweep.md"), "w") as f:
            f.write(table + "\n")
        with open(os.path.join(args.out, "k3_sweep.json"), "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
