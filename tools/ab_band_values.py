#!/usr/bin/env python
"""A/B of the band stream's value tables (context option "band_values") on laplace_matrix(Float64, N, 3).

Builds the operator once, then alternates band_values 0 and 1 over several rounds; each round times, with the context
timer, 50 mul! launches and one fixed 200-iteration cg! (reltol 0, the benchmark's step) per mode.  Checks that the two
modes' outputs (y of mul!, cg!'s residual history and x) are bitwise equal and writes the per-round times as JSON.

    python tools/ab_band_values.py --grid 512 --rounds 5 --out ab_band_values.json
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--spmv", type=int, default=50, help="mul! launches per round and mode")
    ap.add_argument("--iters", type=int, default=200, help="cg! iterations per round and mode")
    ap.add_argument("--out", default="ab_band_values.json")
    args = ap.parse_args()

    import iterativesolvers_jl_b200 as isb
    ctx = isb.default_context()
    N = args.grid
    A = isb.B200CSR.laplacian(N, 3, np.float64, ctx=ctx)
    n = A.m_local
    uniform, value_bytes = A.band_values
    rng = np.random.default_rng(1234321)
    b_host = rng.standard_normal(n)
    b_host /= np.linalg.norm(b_host)
    b = isb.DeviceArray.from_numpy(ctx, b_host)
    xin = isb.DeviceArray.from_numpy(ctx, rng.standard_normal(n))
    y = isb.DeviceArray.zeros(ctx, n)
    x = isb.DeviceArray.zeros(ctx, n)
    L = isb.lib()

    def run(mode):
        ctx.set_option("band_values", mode)
        A.mul_(y, xin)   # warm (first launch sets the kernel's shared-memory attribute)
        ctx.timer_start()
        for _ in range(args.spmv):
            A.mul_(y, xin)
        spmv_ms = ctx.timer_stop() / args.spmv
        ys = y.numpy()
        L.b200_fill(ctx._h, n, 0.0, x._p, 0)
        ctx.timer_start()
        _, h = isb.cg_(x, A, b, initially_zero=True, maxiter=args.iters, reltol=0.0, _fixed_iterations=True, log=True)
        cg_ms = ctx.timer_stop()
        return spmv_ms, cg_ms, ys, np.array(h["resnorm"]), x.numpy()

    rounds = []
    ref = {}
    for r in range(args.rounds):
        rec = {"round": r}
        for mode in ((0, 1) if r % 2 == 0 else (1, 0)):
            spmv_ms, cg_ms, ys, hist, xs = run(mode)
            rec[f"spmv_ms_{mode}"] = spmv_ms
            rec[f"cg_ms_{mode}"] = cg_ms
            rec[f"cg_it_per_s_{mode}"] = args.iters / (cg_ms * 1e-3)
            outs = (ys, hist, xs)
            if mode in ref:
                assert all(np.array_equal(a.view(np.uint8), c.view(np.uint8)) for a, c in zip(outs, ref[mode]))
            ref[mode] = outs
        assert all(np.array_equal(a.view(np.uint8), c.view(np.uint8)) for a, c in zip(ref[0], ref[1])), \
            "band_values 0 and 1 differ"
        rounds.append(rec)
        print(json.dumps(rec), flush=True)
    ctx.set_option("band_values", 1)

    def summary(key):
        v = np.array([rec[key] for rec in rounds])
        return {"min": float(v.min()), "median": float(np.median(v)), "max": float(v.max())}

    out = {"grid": N, "n": n, "nnz": A.nnz, "uniform_tiles": uniform, "value_bytes": value_bytes,
           "spmv_launches_per_round": args.spmv, "cg_iters_per_round": args.iters, "bitwise_equal": True,
           "rounds": rounds, **{k: summary(k) for k in ("spmv_ms_0", "spmv_ms_1", "cg_ms_0", "cg_ms_1")}}
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({k: out[k] for k in ("uniform_tiles", "value_bytes", "spmv_ms_0", "spmv_ms_1", "cg_ms_0", "cg_ms_1")}))
    A.close()


if __name__ == "__main__":
    main()
