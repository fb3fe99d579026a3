#!/usr/bin/env python
"""bench_configs.py -- single-GPU throughput of the other BASELINE.json configs (not the driver's bench):

    gmres     configs[2]: gmres!(restart=30) on advection_dominated(N=256), fp64, CGS and DGKS, fixed maxiter
    lobpcg    configs[4]: lobpcg block=16 on laplace_matrix(Float32, 256, 3), fixed number of steps
    minres    minres! on laplace_matrix(Float64, 256, 3), fixed maxiter
    bicgstabl bicgstabl!(l=2) on advection_dominated(N=256), fixed max_mv_products
    cg256     configs[1]: cg! on laplace_matrix(Float64, 256, 3)
    widen     SURVEY 8(f) item 4: qmr!, lsqr!, lsmr!, idrs!(s=8) on laplace_matrix(Float64, N, 3), fixed iteration counts
              (adjoint operator built by the device transpose)
    cg2d      configs[0]: cg! on laplace_matrix(Float64, 128, 2) (n = 16 384), reltol = sqrt(eps): solves/s and microseconds per
              iteration with the persistent cooperative kernel (default) and with the three-launch streaming iteration
    scattered y = A x (mul!) on CSR operators WITHOUT stencil structure, 7 nonzeros per row: columns uniform over all n, and
              columns within a band of +-2^16 around the diagonal -- what the L1/L2 gather of x costs when the x-window argument
              of the stencil case (DESIGN section 3) does not apply
    general   the general (callback-operator) engines of DESIGN sections 11 / 16 next to the tuned ones: cg!, minres! on
              laplace_matrix(Float64, N, 3), gmres!(30, CGS), bicgstabl!(2) on advection_dominated(N); the operator goes
              through the b200_linop interface with the library's own SpMV thunk (no host code inside the iteration)
    complex   (command line only) ComplexF64 operators built on the host from laplace_matrix(Float64, N, 3)'s CSC arrays:
              gmres!(30, CGS) on the shifted Helmholtz operator -Laplace - k^2 I + i sigma I, and cg! on the Hermitian
              positive-definite L + I + i S (S the antisymmetric central difference in x, coefficient 1/4); fixed
              iteration counts; one JSON line each with it/s, the complex SpMV's ms per launch and its GB/s
    large     (command line only) an operator above 2^31 nonzeros: laplace_matrix(Float64, 680, 3) built on the device
              (2 198 249 600 nonzeros, 8-byte row offsets): cg! it/s and mul!'s ms per launch and GB/s.  Prints a
              "skipped" record instead when the GPU has too little free memory (about 47 GiB are needed)
    ilu       (command line only) the ILU(0) preconditioner (DESIGN section 22): cg! on laplace_matrix(Float64, N, 3) with
              Jacobi and with ILU(0); gmres!(30, CGS) and bicgstabl!(2) on advection_dominated(N) with Identity and with
              ILU(0); each to the default reltol (the unpreconditioned runs capped).  Per record: iterations, time to
              solution, factorization time, ms per ldiv!, levels per sweep, bytes of each triangular solve, card and power

Each line is a JSON object with iterations/s, per-kernel-class CUDA-event times recorded inside the run
(b200_ctx_profile_*), the algorithmic bytes (SURVEY.md section 8d) and the achieved fraction of the measured
HBM peak.  Used for profiles/ (ncu launch lists are taken with the same commands).
"""
import argparse
import ctypes as C
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def peak():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0                        # H100 SXM data sheet, 3.35 TB/s HBM3


def prof_reset(L, ctx):
    L.b200_ctx_profile_enable(ctx._h, 1)
    for s in range(4):
        L.b200_ctx_profile_read(ctx._h, s, None, None, 1)


def prof_read(L, ctx):
    out = {}
    names = ["spmv_class", "vector_with_reduction", "vector_no_reduction", "other"]
    for s in range(4):
        t, c = C.c_double(), C.c_int64()
        L.b200_ctx_profile_read(ctx._h, s, C.byref(t), C.byref(c), 1)
        out[names[s]] = {"total_ms": t.value, "launches": c.value}
    L.b200_ctx_profile_enable(ctx._h, 0)
    return out


class _Clocks:
    """nvidia-smi clocks / throttle reasons around the LAST (timed) repetition of a config (bench.ClockSampler)."""

    def __init__(self, enabled=True, device=0):
        self.s, self.device, self.enabled = None, device, enabled

    def start(self):
        if self.enabled:
            from bench import ClockSampler
            self.s = ClockSampler(self.device)
            self.s.start()

    def stop(self):
        out = self.s.stop() if self.s else None
        self.s = None
        return out


def run(which, grid=256, iters=None, orth="cgs", reps=2, ctx=None, clocks=True, solves=1):
    """one config on cuda:<ctx.device>; returns the JSON-able record (see the module docstring)."""
    args = argparse.Namespace(which=which, grid=grid, iters=iters, orth=orth, reps=reps, solves=solves)
    import iterativesolvers_jl_b200 as isb
    ctx = ctx or isb.default_context()
    L = isb.lib()
    clk = _Clocks(clocks)
    N = args.grid
    n = N ** 3
    nnz = 7 * N ** 3 - 6 * N ** 2
    pk = peak()
    rng = np.random.default_rng(1234321)
    out = {"config": args.which, "grid": N, "n": n, "nnz": nnz, "peak_gbs": pk}

    if args.which in ("gmres", "bicgstabl"):
        cp, rv, nz, shape, b = isb.advection_dominated(N, 1000.0, base=1)
        A = isb.B200CSR.from_csc_arrays(cp, rv, nz, shape, base=1, ctx=ctx)
        del cp, rv, nz
        bd = isb.DeviceArray.from_numpy(ctx, b)
        xd = isb.DeviceArray.zeros(ctx, n)
    if args.which == "gmres":
        restart = 30
        iters = args.iters or 90
        V = 8
        spmv_b = nnz * 12 + (n + 1) * 4 + 2 * n * V
        # per cycle of `restart` inner iterations: sum_k (B_spmv + (2k+5) n V) + restart solution update + init!
        cyc = sum(spmv_b + (2 * k + 5) * n * V for k in range(1, restart + 1)) + (restart + 2) * n * V + spmv_b + 6 * n * V
        for rep in range(args.reps + 1):
            L.b200_fill(ctx._h, n, 0.0, xd._p, 0)
            if rep == 1:
                prof_reset(L, ctx)
            ctx.sync()
            if rep == args.reps:
                clk.start()
            t0 = time.perf_counter()
            x, h = isb.gmres_(xd, A, bd, restart=restart, maxiter=iters, orth_meth=args.orth, initially_zero=True,
                              log=True, reltol=0.0)
            ctx.sync()
            dt = time.perf_counter() - t0
        out["clocks"] = clk.stop()
        pr = prof_read(L, ctx)
        out.update({"solver": f"gmres!(restart=30, orth_meth={args.orth})", "iters": h.niters, "seconds": dt,
                    "iters_per_s": h.niters / dt, "mvps": h.mvps, "resnorm_first_last": [float(h["resnorm"][0]), float(h["resnorm"][-1])],
                    "algorithmic_gb_per_cycle": cyc / 1e9,
                    "achieved_gbs": cyc * (h.niters / restart) / dt / 1e9, "profile": pr})
    elif args.which == "bicgstabl":
        l = 2
        mv = args.iters or 80
        rsh = isb.DeviceArray.from_numpy(ctx, rng.random(n))
        for rep in range(args.reps + 1):
            L.b200_fill(ctx._h, n, 0.0, xd._p, 0)
            if rep == 1:
                prof_reset(L, ctx)
            ctx.sync()
            if rep == args.reps:
                clk.start()
            t0 = time.perf_counter()
            x, h = isb.bicgstabl_(xd, A, bd, l, max_mv_products=mv, initial_zero=True, log=True, reltol=0.0, r_shadow=rsh)
            ctx.sync()
            dt = time.perf_counter() - t0
        out["clocks"] = clk.stop()
        pr = prof_read(L, ctx)
        # algorithmic bytes of one outer iteration (reference src/bicgstabl.jl:88-131, every operation reading its operands
        # once): BiCG part, step j: two dots with r_shadow (2n each), us[:,1:j] update (3jn), rs[:,1:j] update (3jn), x update
        # (3n), two products; MR part: the Gram pass over rs (l+1)n and the three gemv updates (2l+6)n
        V = 8
        spmv_b = nnz * 12 + (n + 1) * 4 + 2 * n * V
        per_outer = (3 * l * l + 13 * l + 7) * n * V + 2 * l * spmv_b
        out.update({"solver": "bicgstabl!(l=2)", "outer_iters": h.niters, "mvps": h.mvps, "seconds": dt,
                    "mv_products_per_s": h.mvps / dt, "algorithmic_gb_per_outer_iteration": per_outer / 1e9,
                    "achieved_gbs": per_outer * h.niters / dt / 1e9, "profile": pr})
    elif args.which in ("minres", "cg256"):
        A = isb.B200CSR.laplacian(N, 3, np.float64, ctx=ctx)
        b = rng.standard_normal(n)
        b /= np.linalg.norm(b)
        bd = isb.DeviceArray.from_numpy(ctx, b)
        xd = isb.DeviceArray.zeros(ctx, n)
        iters = args.iters or 200
        V = 8
        per_it = nnz * 12 + (n + 1) * 4 + (14 if args.which == "minres" else 11) * n * V
        for rep in range(args.reps + 1):
            L.b200_fill(ctx._h, n, 0.0, xd._p, 0)
            if rep == 1:
                prof_reset(L, ctx)
            ctx.sync()
            if rep == args.reps:
                clk.start()
            t0 = time.perf_counter()
            if args.which == "minres":
                x, h = isb.minres_(xd, A, bd, maxiter=iters, initially_zero=True, log=True, reltol=0.0)
            else:
                x, h = isb.cg_(xd, A, bd, maxiter=iters, initially_zero=True, log=True, reltol=0.0, _fixed_iterations=True)
            ctx.sync()
            dt = time.perf_counter() - t0
        out["clocks"] = clk.stop()
        pr = prof_read(L, ctx)
        out.update({"solver": args.which, "iters": h.niters, "seconds": dt, "iters_per_s": h.niters / dt,
                    "algorithmic_gb_per_iter": per_it / 1e9, "achieved_gbs": per_it * h.niters / dt / 1e9,
                    "profile": pr})
    elif args.which == "widen":
        A = isb.B200CSR.laplacian(N, 3, np.float64, ctx=ctx)
        t0 = time.perf_counter()
        At = A.adjoint()
        ctx.sync()
        out["transpose_seconds"] = time.perf_counter() - t0
        b = rng.standard_normal(n)
        b /= np.linalg.norm(b)
        bd = isb.DeviceArray.from_numpy(ctx, b)
        xd = isb.DeviceArray.zeros(ctx, n)
        iters = args.iters or 100
        V = 8
        s_dim = 8
        Pd = isb.DeviceArray.from_numpy(ctx, np.asfortranarray(rng.random((n, s_dim))))
        spmv_b = nnz * 12 + (n + 1) * 4 + 2 * n * V
        # IDR(s): vector passes of one cycle of s direction steps + the polynomial step (csrc/idrs_core.h)
        cyc = (s_dim + 1) * n * V                                                         # D
        for k in range(1, s_dim + 1):
            cyc += (2 * (s_dim - k + 1) + 2) * n * V + spmv_b                             # V, S
            if k == 1:
                cyc += (1 + s_dim) * n * V                                                # new column of M
            else:
                cyc += 2 * n * V + (k - 2) * 7 * n * V + (6 + s_dim - k + 1) * n * V      # first dot, updates, last update
            cyc += 6 * n * V                                                              # X
        cyc += spmv_b + 2 * n * V + 5 * n * V                                             # S, O, X' (Identity)
        per_it = {"qmr": 2 * spmv_b + 21 * n * V, "lsqr": 2 * spmv_b + 14 * n * V, "lsmr": 2 * spmv_b + 16 * n * V,
                  "idrs": cyc / (s_dim + 1)}
        res = {}
        for name in ("qmr", "lsqr", "lsmr", "idrs"):
            for rep in range(args.reps + 1):
                L.b200_fill(ctx._h, n, 0.0, xd._p, 0)
                if rep == 1:
                    prof_reset(L, ctx)
                ctx.sync()
                if rep == args.reps:
                    clk.start()
                t0 = time.perf_counter()
                if name == "qmr":
                    x, h = isb.qmr_(xd, A, bd, maxiter=iters, initially_zero=True, log=True, reltol=0.0)
                elif name == "lsqr":
                    x, h = isb.lsqr_(xd, A, bd, maxiter=iters, log=True, atol=0.0, btol=0.0, conlim=0.0)
                elif name == "lsmr":
                    x, h = isb.lsmr_(xd, A, bd, maxiter=iters, log=True, atol=0.0, btol=0.0, conlim=0.0)
                else:
                    x, h = isb.idrs_(xd, A, bd, s=s_dim, P=Pd, maxiter=iters, log=True, reltol=0.0)
                ctx.sync()
                dt = time.perf_counter() - t0
            ck = clk.stop()
            pr = prof_read(L, ctx)
            key = "resnorm" if name in ("qmr", "idrs", "lsqr") else "rnorm"
            res[name] = {"clocks": ck, "iters": h.iters, "seconds": dt, "iters_per_s": h.iters / dt,
                         "algorithmic_gb_per_iter": per_it[name] / 1e9,
                         "achieved_gbs": per_it[name] * h.iters / dt / 1e9,
                         "frac_of_measured_peak": per_it[name] * h.iters / dt / 1e9 / pk,
                         "first_last": [float(h[key][0]), float(h[key][-1])], "profile": pr}
        out["solvers"] = res
    elif args.which == "cg2d":
        from oracle import oracle as _orc        # generator only (this script is a bench tool, like bench.py's CPU arm)
        O = _orc.laplace_matrix(np.float64, 128, 2, base=1)
        A = isb.B200CSR.from_csc_arrays(O.colptr, O.rowval, O.nzval, O.shape, base=1, ctx=ctx)
        b = np.random.default_rng(1234321).standard_normal(O.n)
        b /= np.linalg.norm(b)
        bd = isb.DeviceArray.from_numpy(ctx, b)
        xd = isb.DeviceArray.zeros(ctx, O.n)
        res = {}
        solves = args.iters or 200
        for mode in (1, 0):
            L.b200_ctx_set_option(ctx._h, b"cg_persistent", mode)
            for rep in range(2):
                if rep == 1:
                    clk.start()
                ctx.sync()
                t0 = time.perf_counter()
                its = 0
                for _ in range(solves):
                    L.b200_fill(ctx._h, O.n, 0.0, xd._p, 0)
                    isb.cg_(xd, A, bd, initially_zero=True)
                    its += int(isb.cg_.last_result.iters)
                ctx.sync()
                dt = time.perf_counter() - t0
            res["persistent" if mode else "three_launches"] = {
                "clocks": clk.stop(), "solves_per_s": solves / dt, "iterations_per_solve": its / solves,
                "us_per_iteration": dt / its * 1e6, "iterations_per_s": its / dt}
        L.b200_ctx_set_option(ctx._h, b"cg_persistent", 1)
        out.update({"solver": "cg! 5-pt 2-D Poisson 128^2 fp64 (configs[0])", "grid": 128, "n": O.n, "nnz": int(A.nnz), "engines": res,
                    "speedup": res["persistent"]["iterations_per_s"] / res["three_launches"]["iterations_per_s"]})
    elif args.which == "scattered":
        V = 8
        per_row = 7
        res = {}
        rowptr = (np.arange(n + 1, dtype=np.int64) * per_row).astype(np.int32)
        xs = isb.DeviceArray.from_numpy(ctx, rng.standard_normal(n))
        ys = isb.DeviceArray(ctx, n)
        for name, band in (("banded_2^16", 1 << 16), ("uniform", None)):
            rows = np.repeat(np.arange(n, dtype=np.int64), per_row - 1)
            if band is None:
                off = rng.integers(0, n, rows.size, dtype=np.int64)
            else:
                off = np.clip(rows + rng.integers(-band, band + 1, rows.size, dtype=np.int64), 0, n - 1)
            cols = np.empty((n, per_row), dtype=np.int32)
            cols[:, 0] = np.arange(n, dtype=np.int32)
            cols[:, 1:] = off.reshape(n, per_row - 1)
            del rows, off
            cols.sort(axis=1)
            vals = rng.standard_normal(n * per_row)
            A = isb.B200CSR.from_csr_slab(rowptr, cols.reshape(-1), vals, n, 0, 0, None, ctx)
            del cols, vals
            spmv_b = A.nnz * 12 + (n + 1) * 4 + 2 * n * V
            reps = args.iters or 50
            for rep in range(2):
                if rep == 1:
                    clk.start()
                ctx.sync()
                t0 = time.perf_counter()
                for _ in range(reps):
                    A.mul_(ys, xs)
                ctx.sync()
                dt = (time.perf_counter() - t0) / reps
            res[name] = {"clocks": clk.stop(), "nnz": int(A.nnz), "ms_per_spmv": dt * 1e3,
                         "algorithmic_gb": spmv_b / 1e9, "achieved_gbs": spmv_b / dt / 1e9,
                         "frac_of_measured_peak": spmv_b / dt / 1e9 / pk}
            A.close()
        # the stencil operator of the same size for comparison
        A = isb.B200CSR.laplacian(N, 3, np.float64, ctx=ctx)
        spmv_b = A.nnz * 12 + (n + 1) * 4 + 2 * n * V
        reps = args.iters or 50
        for rep in range(2):
            ctx.sync()
            t0 = time.perf_counter()
            for _ in range(reps):
                A.mul_(ys, xs)
            ctx.sync()
            dt = (time.perf_counter() - t0) / reps
        res["laplace_7pt"] = {"nnz": int(A.nnz), "ms_per_spmv": dt * 1e3, "algorithmic_gb": spmv_b / 1e9,
                              "achieved_gbs": spmv_b / dt / 1e9, "frac_of_measured_peak": spmv_b / dt / 1e9 / pk}
        out["operators"] = res
    elif args.which == "general":
        V = 8
        spmv_b = nnz * 12 + (n + 1) * 4 + 2 * n * V
        iters = args.iters or 90
        res = {}
        Alap = isb.B200CSR.laplacian(N, 3, np.float64, ctx=ctx)
        b = rng.standard_normal(n)
        b /= np.linalg.norm(b)
        bd = isb.DeviceArray.from_numpy(ctx, b)
        xd = isb.DeviceArray.zeros(ctx, n)
        sh = isb.DeviceArray.from_numpy(ctx, rng.random(n))
        restart = 30
        gm_cyc = sum(spmv_b + (2 * k + 5) * n * V for k in range(1, restart + 1)) + (restart + 2) * n * V + spmv_b + 6 * n * V
        runs = {   # name -> (callable(operator) -> history, algorithmic bytes per iteration of the TUNED engine, matrix)
            "cg": (lambda op: isb.cg_(xd, op, bd, maxiter=iters, initially_zero=True, log=True, reltol=0.0)[1],
                   spmv_b + 10 * n * V, "lap"),
            "minres": (lambda op: isb.minres_(xd, op, bd, maxiter=iters, initially_zero=True, log=True, reltol=0.0)[1],
                       spmv_b + 13 * n * V, "lap"),
            "gmres": (lambda op: isb.gmres_(xd, op, bd, restart=restart, maxiter=iters, orth_meth="cgs", initially_zero=True,
                                            log=True, reltol=0.0)[1], gm_cyc / restart, "adv"),
            "bicgstabl": (lambda op: isb.bicgstabl_(xd, op, bd, 2, max_mv_products=4 * (iters // 4), initial_zero=True,
                                                    r_shadow=sh, log=True, reltol=0.0)[1], None, "adv"),
        }
        Aadv = None
        for name, (fn, per_it, mat) in runs.items():
            if mat == "adv" and Aadv is None:
                cp, rv, nz, shape, badv = isb.advection_dominated(N, 1000.0, base=1)
                Aadv = isb.B200CSR.from_csc_arrays(cp, rv, nz, shape, base=1, ctx=ctx)
                del cp, rv, nz
                bd.upload(badv)
            A = Alap if mat == "lap" else Aadv
            entry = {}
            for kind, op in (("tuned", A), ("general", isb.B200LinearOperator.from_csr(A))):
                for rep in range(args.reps + 1):
                    L.b200_fill(ctx._h, n, 0.0, xd._p, 0)
                    ctx.sync()
                    if rep == args.reps:
                        clk.start()
                    t0 = time.perf_counter()
                    h = fn(op)
                    ctx.sync()
                    dt = time.perf_counter() - t0
                units = h.mvps if name == "bicgstabl" else h.iters
                entry[kind] = {"clocks": clk.stop(), "units": int(units), "seconds": dt, "units_per_s": units / dt,
                               "last_resnorm": float(h["resnorm"][-1]) if len(h["resnorm"]) else None}
                if per_it:
                    entry[kind]["achieved_gbs_on_tuned_bytes"] = per_it * units / dt / 1e9
                    entry[kind]["frac_of_measured_peak"] = per_it * units / dt / 1e9 / pk
            entry["unit"] = "mv-products" if name == "bicgstabl" else "iterations"
            entry["general_over_tuned"] = entry["general"]["units_per_s"] / entry["tuned"]["units_per_s"]
            res[name] = entry
        out["solvers"] = res
    else:  # lobpcg
        bs = 16
        A = isb.B200CSR.laplacian(N, 3, np.float32, ctx=ctx)
        X0 = rng.random((n, bs), dtype=np.float32)
        steps = args.iters or 10
        V = 4
        per_step = nnz * (V + 4) + (n + 1) * 4 + 26 * n * bs * V        # SURVEY 8d ideal
        # `solves` timed solves of `steps` steps each (fp32 LOBPCG without soft locking breaks down -- CholQR PosDefException, in
        # the reference's own arithmetic too -- when it is driven for many tens of steps at this size, so the horizon stays
        # short and the sample is made long enough for the clock sampler by repetition); X0 is restored on the device
        solves = max(1, getattr(args, "solves", 1) or 1)
        X0d = isb.DeviceArray.from_numpy(ctx, X0)
        Xd = isb.DeviceArray(ctx, X0.shape, np.float32)
        dt = 0.0
        for rep in range(args.reps + solves):
            isb._lib.check(L.b200_copy(ctx._h, n * bs, X0d._p, Xd._p, 1))
            if rep == args.reps:
                prof_reset(L, ctx)
                clk.start()
            ctx.sync()
            t0 = time.perf_counter()
            r = isb.lobpcg(A, False, Xd, maxiter=steps, _fixed_iterations=True)
            ctx.sync()
            if rep >= args.reps:
                dt += time.perf_counter() - t0
        out["clocks"] = clk.stop()
        steps_total = steps * solves
        pr = prof_read(L, ctx)
        out.update({"solver": "lobpcg(block=16, fp32, smallest)", "steps": steps, "solves": solves, "seconds": dt,
                    "steps_per_s": steps_total / dt,
                    "lambda_min": float(np.min(r.lam)), "max_resnorm": float(np.max(r.residual_norms)),
                    "algorithmic_gb_per_step_ideal": per_step / 1e9, "achieved_gbs_vs_ideal_bytes": per_step * steps_total / dt / 1e9,
                    "frac_of_measured_peak": per_step * steps_total / dt / 1e9 / pk,
                    "profile": pr})
    if "achieved_gbs" in out:
        out["frac_of_measured_peak"] = out["achieved_gbs"] / pk
    return out


def gpu_name_power(device=0):
    """the GPU's name and power limit (W) as nvidia-smi reports them: part of every number this script prints"""
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit_w": q[1] if len(q) > 1 else None}
    except Exception:
        return {"gpu": None, "power_limit_w": None}


def complex_operators(N, k2=0.5, sigma=0.5):
    """ComplexF64 CSC arrays (colptr, rowval, nzval) of the shifted Helmholtz operator -Laplace - k^2 I + i sigma I and of
    the Hermitian positive-definite L + I + i S, from laplace_matrix(Float64, N, 3) (0-based)."""
    import iterativesolvers_jl_b200 as isb
    colptr, rowval, nz, shape = isb.laplace_matrix(np.float64, N, 3, base=0)
    col = np.repeat(np.arange(shape[1], dtype=np.int64), np.diff(colptr))
    diag = rowval == col
    helm = nz.astype(np.complex128)
    helm[diag] += -k2 + 1j * sigma
    hpd = nz.astype(np.complex128)
    hpd[diag] += 1.0
    hpd[col == rowval + 1] += 0.25j          # A[r, r+1] = -1 + i/4, A[r+1, r] = -1 - i/4: x-neighbours (stride 1)
    hpd[col == rowval - 1] -= 0.25j
    del col, diag
    return colptr, rowval, helm, hpd, shape


def run_complex(grid=256, iters=None, reps=2, ctx=None):
    """the `complex` workloads: two records (gmres!(30) CGS on the Helmholtz operator, cg! on the HPD operator)"""
    import iterativesolvers_jl_b200 as isb
    ctx = ctx or isb.default_context()
    L = isb.lib()
    N = grid
    n = N ** 3
    colptr, rowval, helm, hpd, shape = complex_operators(N)
    nnz = int(colptr[-1])
    V = 16
    spmv_b = nnz * (V + 4) + (n + 1) * 4 + 2 * n * V          # algorithmic bytes of one complex SpMV
    gpu = gpu_name_power(ctx.device)
    rng = np.random.default_rng(1234321)
    b = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) / math.sqrt(2 * n)
    bd = isb.DeviceArray.from_numpy(ctx, b)
    xd = isb.DeviceArray.zeros(ctx, n, np.complex128)
    out = []
    for name, vals in (("gmres", helm), ("cg", hpd)):
        A = isb.B200CSR.from_csc_arrays(colptr, rowval, vals, shape, base=0, ctx=ctx)
        it = iters or (90 if name == "gmres" else 200)
        for rep in range(reps + 1):
            L.b200_fill(ctx._h, n, 0.0, xd._p, isb._lib.CF64)
            if rep == reps:
                prof_reset(L, ctx)
            ctx.sync()
            t0 = time.perf_counter()
            if name == "gmres":
                x, h = isb.gmres_(xd, A, bd, restart=30, maxiter=it, orth_meth="cgs", initially_zero=True, log=True,
                                  reltol=0.0)
            else:
                x, h = isb.cg_(xd, A, bd, maxiter=it, initially_zero=True, log=True, reltol=0.0)
            ctx.sync()
            dt = time.perf_counter() - t0
        pr = prof_read(L, ctx)
        sp_ms = pr["spmv_class"]["total_ms"] / max(pr["spmv_class"]["launches"], 1)
        out.append({"config": "complex", "solver": "gmres!(restart=30, orth_meth=cgs), ComplexF64 Helmholtz" if name == "gmres"
                    else "cg!, ComplexF64 Hermitian positive definite", "grid": N, "n": n, "nnz": nnz, **gpu,
                    "iters": h.niters, "seconds": dt, "iters_per_s": h.niters / dt,
                    "resnorm_first_last": [float(h["resnorm"][0]), float(h["resnorm"][-1])],
                    "spmv_ms_per_launch": sp_ms, "spmv_bytes": spmv_b, "spmv_gbs": spmv_b / (sp_ms * 1e-3) / 1e9,
                    "spmv_frac_of_3350_gbs": spmv_b / (sp_ms * 1e-3) / 1e9 / 3350.0, "profile": pr})
        A.close()
    return out


def run_large(grid=680, iters=None, reps=2, ctx=None):
    """the `large` workload: cg! and mul! on laplace_matrix(Float64, grid, 3) with 8-byte row offsets"""
    import torch
    import iterativesolvers_jl_b200 as isb
    n = grid ** 3
    nnz = n + 6 * (grid - 1) * grid * grid
    V = 8
    free, _ = torch.cuda.mem_get_info(0)
    need = nnz * (V + 4) + (n + 1) * 8 + 6 * n * V          # operator + cg!'s x, b, r, u, c and mul!'s y
    gpu = gpu_name_power(0)
    if need > 0.95 * free:
        return {"config": "large", "grid": grid, "skipped": f"needs {need / 2**30:.1f} GiB of free device memory, "
                f"{free / 2**30:.1f} GiB are free", **gpu}
    ctx = ctx or isb.default_context()
    L = isb.lib()
    A = isb.B200CSR.laplacian(grid, 3, np.float64, ctx=ctx)
    kind, sbytes = C.c_int(), C.c_int64()
    L.b200_csr_stream_kind(A._h, C.byref(kind), C.byref(sbytes))
    _, value_b = A.band_values
    csr_b = nnz * (V + 4) + (n + 1) * 8 + 2 * n * V           # algorithmic bytes of one SpMV (SURVEY 8d, 8-byte offsets)
    read_b = value_b + sbytes.value + 2 * n * V               # what the chosen form reads: values, its structure, x, y
    rng = np.random.default_rng(1234321)
    b = rng.standard_normal(n)
    b /= np.linalg.norm(b)
    bd = isb.DeviceArray.from_numpy(ctx, b)
    del b
    xd = isb.DeviceArray.zeros(ctx, n, np.float64)
    yd = isb.DeviceArray.zeros(ctx, n, np.float64)
    it = iters or 200
    for rep in range(reps + 1):
        L.b200_fill(ctx._h, n, 0.0, xd._p, isb._lib.F64)
        ctx.sync()
        t0 = time.perf_counter()
        x, h = isb.cg_(xd, A, bd, maxiter=it, initially_zero=True, log=True, reltol=0.0)
        ctx.sync()
        dt = time.perf_counter() - t0
    K = 50
    A.mul_(yd, bd)
    ctx.timer_start()
    for _ in range(K):
        A.mul_(yd, bd)
    spmv_ms = ctx.timer_stop() / K
    rec = {"config": "large", "solver": "cg! and mul!, laplace_matrix(Float64, 680, 3), 8-byte row offsets", "grid": grid,
           "n": n, "nnz": A.nnz, "index_bytes": A.index_bytes, "stream_kind": kind.value, **gpu,
           "iters": h.niters, "seconds": dt, "iters_per_s": h.niters / dt,
           "resnorm_first_last": [float(h["resnorm"][0]), float(h["resnorm"][-1])],
           "spmv_ms_per_launch": spmv_ms, "spmv_bytes_algorithmic": csr_b, "spmv_bytes_read": read_b,
           "spmv_gbs_algorithmic": csr_b / (spmv_ms * 1e-3) / 1e9, "spmv_gbs_read": read_b / (spmv_ms * 1e-3) / 1e9}
    A.close()
    return rec


def _ilu_record(isb, ctx, P, n, V=8, applies=20):
    """ms per ldiv! (CUDA events over `applies` back-to-back applies), levels and algorithmic bytes of each triangular
    solve.  Forward: L's values and column indices, and per row its row offset, diagonal position, schedule entry and
    ready flag (16 B), x read, y written, y gathered once; backward: U's strictly upper part likewise plus u_ii."""
    xd = isb.DeviceArray.from_numpy(ctx, np.random.default_rng(3).standard_normal(n))
    yd = isb.DeviceArray(ctx, n)
    P.ldiv_(yd, xd)
    ctx.sync()
    ctx.timer_start()
    for _ in range(applies):
        P.ldiv_(yd, xd)
    ms = ctx.timer_stop() / applies
    fwd_b = P.nnz_lower * (V + 4) + n * (16 + 3 * V)
    bwd_b = P.nnz_upper * (V + 4) + n * (16 + 4 * V)
    return {"ldiv_ms": ms, "levels_forward": P.levels[0], "levels_backward": P.levels[1],
            "forward_solve_bytes": fwd_b, "backward_solve_bytes": bwd_b,
            "ldiv_gbs_on_algorithmic_bytes": (fwd_b + bwd_b) / (ms * 1e-3) / 1e9}


def run_ilu(grid=256, ctx=None, gmres_maxiter=3000, bicgstabl_max_mv=6000):
    """the `ilu` workloads: cg! (Jacobi vs ILU(0)) on laplace_matrix(Float64, N, 3); gmres!(30) CGS and bicgstabl!(2)
    (Identity vs ILU(0)) on advection_dominated(N); each to the default reltol, with caps on the unpreconditioned runs"""
    import iterativesolvers_jl_b200 as isb
    ctx = ctx or isb.default_context()
    N = grid
    n = N ** 3
    gpu = gpu_name_power(ctx.device)
    rng = np.random.default_rng(1234321)
    out = []

    def timed(fn):
        ctx.sync()
        t0 = time.perf_counter()
        r = fn()
        ctx.sync()
        return r, time.perf_counter() - t0

    def factor(A):
        P, dt = timed(lambda: isb.ILU0Prec(A))
        return P, dt

    A = isb.B200CSR.laplacian(N, 3, np.float64, ctx=ctx)
    b = rng.standard_normal(n)
    b /= np.linalg.norm(b)
    bd = isb.DeviceArray.from_numpy(ctx, b)
    xd = isb.DeviceArray.zeros(ctx, n)
    P, t_fact = factor(A)
    runs = {}
    for name, Pl in (("jacobi", isb.JacobiPrec(A.diag())), ("ilu0", P)):
        for rep in range(2):
            isb.lib().b200_fill(ctx._h, n, 0.0, xd._p, 0)
            (x, h), dt = timed(lambda: isb.cg_(xd, A, bd, Pl=Pl, initially_zero=True, log=True))
        runs[name] = {"iters": h.niters, "converged": h.isconverged, "seconds": dt,
                      "final_resnorm": float(h["resnorm"][-1])}
    out.append({"config": "ilu", "solver": "cg!, laplace_matrix(Float64, %d, 3), default reltol" % N, "grid": N, "n": n,
                "nnz": int(A.nnz), **gpu, "runs": runs, "ilu0_factor_seconds": t_fact, **_ilu_record(isb, ctx, P, n),
                "ilu0_over_jacobi_time": runs["ilu0"]["seconds"] / runs["jacobi"]["seconds"]})
    P.close()
    del P, A
    cp, rv, nz, shape, badv = isb.advection_dominated(N, 1000.0, base=1)
    A = isb.B200CSR.from_csc_arrays(cp, rv, nz, shape, base=1, ctx=ctx)
    del cp, rv, nz
    bd.upload(badv)
    P, t_fact = factor(A)
    sh = isb.DeviceArray.from_numpy(ctx, rng.random(n))
    rec = _ilu_record(isb, ctx, P, n)
    for solver in ("gmres", "bicgstabl"):
        runs = {}
        for name, Pl in (("identity", None), ("ilu0", P)):
            for cap in ((30, 8), (gmres_maxiter, bicgstabl_max_mv)):        # a short warm-up run, then the timed one
                isb.lib().b200_fill(ctx._h, n, 0.0, xd._p, 0)
                if solver == "gmres":
                    (x, h), dt = timed(lambda: isb.gmres_(xd, A, bd, Pl=Pl, restart=30, orth_meth="cgs", maxiter=cap[0],
                                                          initially_zero=True, log=True))
                else:
                    (x, h), dt = timed(lambda: isb.bicgstabl_(xd, A, bd, 2, Pl=Pl, max_mv_products=cap[1],
                                                              initial_zero=True, r_shadow=sh, log=True))
            runs[name] = {"iters": h.niters, "mvps": h.mvps, "converged": h.isconverged, "seconds": dt,
                          "final_resnorm": float(h["resnorm"][-1]) if len(h["resnorm"]) else None}
        out.append({"config": "ilu", "solver": ("gmres!(restart=30, CGS)" if solver == "gmres" else "bicgstabl!(l=2)")
                    + ", advection_dominated(%d), default reltol" % N, "grid": N, "n": n, "nnz": int(A.nnz), **gpu,
                    "caps": {"gmres_maxiter": gmres_maxiter, "bicgstabl_max_mv_products": bicgstabl_max_mv},
                    "runs": runs, "ilu0_factor_seconds": t_fact, **rec,
                    "ilu0_over_identity_time": runs["ilu0"]["seconds"] / runs["identity"]["seconds"]})
    P.close()
    return out


def _amg_record(isb, ctx, P, n, applies=20):
    """the hierarchy (rows and nonzeros per level, operator complexity), the setup split, and ms per ldiv! from CUDA
    events over `applies` back-to-back applies.  The fine level's share is measured with torch.profiler: a V-cycle of
    L levels is 5 (L - 1) + 1 launches in a fixed order, of which the first three and the last two are the fine level's."""
    xd = isb.DeviceArray.from_numpy(ctx, np.random.default_rng(3).standard_normal(n))
    yd = isb.DeviceArray(ctx, n)
    P.ldiv_(yd, xd)
    ctx.sync()
    ctx.timer_start()
    for _ in range(applies):
        P.ldiv_(yd, xd)
    ms = ctx.timer_stop() / applies
    rec = {"level_rows": P.level_rows, "level_nnz": P.level_nnz, "operator_complexity": P.operator_complexity,
           "setup_seconds": P.setup_seconds, "setup_seconds_total": sum(P.setup_seconds.values()), "ldiv_ms": ms,
           "launches_per_ldiv": 5 * (len(P.level_rows) - 1) + 1}
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        L = rec["launches_per_ldiv"]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                P.ldiv_(yd, xd)
            ctx.sync()
            torch.cuda.synchronize()
        ks = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and "Memcpy" not in e.name and "Memset" not in e.name), key=lambda e: e.time_range.start)
        if len(ks) == 5 * L and L > 1:
            fine = total = 0.0
            for c in range(5):
                grp = ks[c * L:(c + 1) * L]
                us = [e.time_range.end - e.time_range.start for e in grp]
                fine += sum(us[:3]) + sum(us[-2:])
                total += sum(us)
            rec["fine_level_kernel_ms"] = fine / 5 / 1e3
            rec["fine_level_share_of_kernel_time"] = fine / total
    except Exception as e:                                    # the share is reported when the profiler can give it
        rec["fine_level_share_error"] = repr(e)
    return rec


def run_amg(grid=256, ctx=None, gmres_maxiter=3000):
    """the `amg` workloads: cg! (Jacobi vs smoothed-aggregation AMG) on laplace_matrix(Float64, N, 3) and gmres!(30) CGS
    (Identity vs AMG, with a cap) on advection_dominated(N), each to the default reltol.  Setup is timed apart from the
    solve; the solve is timed on its second run."""
    import iterativesolvers_jl_b200 as isb
    ctx = ctx or isb.default_context()
    N = grid
    n = N ** 3
    gpu = gpu_name_power(ctx.device)
    rng = np.random.default_rng(1234321)
    out = []

    def timed(fn):
        ctx.sync()
        t0 = time.perf_counter()
        r = fn()
        ctx.sync()
        return r, time.perf_counter() - t0

    A = isb.B200CSR.laplacian(N, 3, np.float64, ctx=ctx)
    b = rng.standard_normal(n)
    b /= np.linalg.norm(b)
    bd = isb.DeviceArray.from_numpy(ctx, b)
    xd = isb.DeviceArray.zeros(ctx, n)
    P, t_setup = timed(lambda: isb.SmoothedAggregationPrec(A))
    runs = {}
    for name, Pl in (("jacobi", isb.JacobiPrec(A.diag())), ("amg", P)):
        for rep in range(2):
            isb.lib().b200_fill(ctx._h, n, 0.0, xd._p, 0)
            (x, h), dt = timed(lambda: isb.cg_(xd, A, bd, Pl=Pl, initially_zero=True, log=True))
        runs[name] = {"iters": h.niters, "converged": h.isconverged, "seconds": dt,
                      "final_resnorm": float(h["resnorm"][-1])}
    rec = _amg_record(isb, ctx, P, n)
    out.append({"config": "amg", "solver": "cg!, laplace_matrix(Float64, %d, 3), default reltol" % N, "grid": N, "n": n,
                "nnz": int(A.nnz), **gpu, "runs": runs, "amg_setup_wall_seconds": t_setup, **rec,
                "amg_over_jacobi_solve_time": runs["amg"]["seconds"] / runs["jacobi"]["seconds"],
                "amg_setup_plus_solve_over_jacobi": (t_setup + runs["amg"]["seconds"]) / runs["jacobi"]["seconds"]})
    P.close()
    del P, A
    cp, rv, nz, shape, badv = isb.advection_dominated(N, 1000.0, base=1)
    A = isb.B200CSR.from_csc_arrays(cp, rv, nz, shape, base=1, ctx=ctx)
    del cp, rv, nz
    bd.upload(badv)
    P, t_setup = timed(lambda: isb.SmoothedAggregationPrec(A))
    runs = {}
    for name, Pl in (("identity", None), ("amg", P)):
        for cap in (30, gmres_maxiter):                                     # a short warm-up run, then the timed one
            isb.lib().b200_fill(ctx._h, n, 0.0, xd._p, 0)
            (x, h), dt = timed(lambda: isb.gmres_(xd, A, bd, Pl=Pl, restart=30, orth_meth="cgs", maxiter=cap,
                                                  initially_zero=True, log=True))
        runs[name] = {"iters": h.niters, "converged": h.isconverged, "seconds": dt,
                      "final_resnorm": float(h["resnorm"][-1]) if len(h["resnorm"]) else None}
    rec = _amg_record(isb, ctx, P, n)
    out.append({"config": "amg", "solver": "gmres!(restart=30, CGS), advection_dominated(%d), default reltol" % N,
                "grid": N, "n": n, "nnz": int(A.nnz), **gpu, "caps": {"gmres_maxiter": gmres_maxiter}, "runs": runs,
                "amg_setup_wall_seconds": t_setup, **rec,
                "amg_over_identity_solve_time": runs["amg"]["seconds"] / runs["identity"]["seconds"]})
    P.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("which", choices=["gmres", "lobpcg", "minres", "bicgstabl", "cg256", "widen", "general", "scattered", "cg2d",
                                      "complex", "large", "ilu", "amg"])
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--iters", type=int, default=None)
    ap.add_argument("--orth", default="cgs")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--no-clocks", action="store_true")
    ap.add_argument("--solves", type=int, default=1, help="lobpcg: timed solves of --iters steps each")
    args = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    if args.which == "large":
        print(json.dumps(run_large(680 if args.grid == 256 else args.grid, args.iters, args.reps)))
        return
    if args.which == "complex":
        for rec in run_complex(args.grid, args.iters, args.reps):
            print(json.dumps(rec))
        return
    if args.which == "ilu":
        for rec in run_ilu(args.grid):
            print(json.dumps(rec), flush=True)
        return
    if args.which == "amg":
        for rec in run_amg(args.grid):
            print(json.dumps(rec), flush=True)
        return
    print(json.dumps(run(args.which, args.grid, args.iters, args.orth, args.reps, clocks=not args.no_clocks, solves=args.solves)))


if __name__ == "__main__":
    main()
