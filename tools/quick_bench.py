"""Developer timing loop (NOT the contract bench): device-resident synthetic batch, CUDA events.

Arguments select configs (C3 C2 C4 K50 K100), waypoint variants (v5 = the chunked kernel K3) and K3's resident
vertex blocks per lane (chunk=2; 0 = auto), e.g. `python tools/quick_bench.py C3 K50 v5 chunk=1`.  frac_hbm is the
algorithmic traffic over the 3350 GB/s of the H100 SXM data sheet."""
import json
import sys
import os

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import mav_trajectory_generation_b200 as m


def synth(N, K, D, B, dev, seed=0):
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    pos = (torch.rand((B, K + 1, D), generator=g, device=dev, dtype=torch.float64) * 20.0 - 10.0)
    dist = (pos[:, 1:] - pos[:, :-1]).norm(dim=2).clamp_min(0.2)
    v, a = 3.0, 5.0
    times = dist / v * 2 * (1.0 + 6.5 * v / a * torch.exp(-dist / v * 2))
    h = N // 2
    nf = 2 * h + K - 1
    dfix = torch.zeros((B, D, nf), device=dev, dtype=torch.float64)
    dfix[:, :, 0] = pos[:, 0]
    dfix[:, :, h:h + K - 1] = pos[:, 1:K].transpose(1, 2)
    dfix[:, :, h + K - 1] = pos[:, K]
    return times.contiguous(), dfix.contiguous()


def main():
    dev = torch.device("cuda:0")
    s = m.Solver(0)
    cfgs = [("C3", 10, 4, 16, 3, 262144), ("C2", 10, 4, 8, 3, 65536), ("C4", 8, 3, 4, 3, 1048576),
            ("K50", 10, 4, 50, 3, 246272), ("K100", 10, 4, 100, 3, 113664)]
    cfgs = [c for c in cfgs if c[0] in sys.argv[1:]] or cfgs
    variants = [int(a[1:]) for a in sys.argv[1:] if a.startswith("v")] or [0]
    chunks = [int(a[len("chunk="):]) for a in sys.argv[1:] if a.startswith("chunk=")] or [0]
    for variant, chunk in [(v, c) for v in variants for c in chunks]:
        s.set_option(m.capi.OPT_WAYPOINT_VARIANT, variant)
        s.set_option(m.capi.OPT_CHUNK_BLOCKS, chunk)
        for name, N, r, K, D, B in cfgs:
            prob = m.Problem(N, r, K, D)
            times, dfix = synth(N, K, D, B, dev)
            out = torch.empty((B, K, D, N), device=dev, dtype=torch.float64)
            for _ in range(3):
                s.solve_linear(prob, times, dfix, coeffs=out)
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(11)]
            ev[0].record()
            for i in range(10):
                s.solve_linear(prob, times, dfix, coeffs=out)
                ev[i + 1].record()
            torch.cuda.synchronize()
            ms = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(10))
            med = ms[len(ms) // 2]
            rate = B / (med * 1e-3)
            gbs = rate * prob.bytes_per_trajectory / 1e9
            print(json.dumps(dict(variant=variant, chunk=chunk, cfg=name, K=K, B=B, ms=round(med, 4),
                                  traj_per_s=round(rate), GBs=round(gbs, 1), frac_hbm=round(gbs / 3350.0, 4),
                                  finite=bool(torch.isfinite(out).all().item()))))


if __name__ == "__main__":
    main()
