#!/usr/bin/env python
"""The reference's own benchmark suite (examples/benchmarks.rs: 24 scenarios, "Speedup vs. realtime") on the CUDA engine, next to
the CPU port of the reference renderer on the same box.

    python tools/reference_benchmarks.py --seconds 120 --graphs 32 --out reference_benchmarks.json

For every scenario: `graphs` identical contexts are rendered as ONE batch on the GPU (kernel time from the engine's CUDA events,
median of `--steps` runs after a warm-up) and the same scenario is rendered by the oracle (a) as one context on one core — what
`cargo run --release --example benchmarks` measures — and (b) as `graphs` contexts over all cores.  "x realtime" = rendered audio
seconds per wall second, summed over the batch.  The first graph of the batch is compared with the oracle (max |diff|).
The oracle is used here as the checker and as the timed CPU baseline only (tools/, like bench.py's cpu_baseline leg)."""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120.0, help="the reference's DURATION (benchmarks.rs:71)")
    ap.add_argument("--graphs", type=int, default=32)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--only", type=str, default="")
    ap.add_argument("--out", type=str, default="")
    args = ap.parse_args()

    import __graft_entry__ as ge
    pkg = ge.build()
    import benchmark_scenarios as BS
    import conftest  # noqa: F401  (oracle loader lives next to the tests)
    so = os.path.join(ROOT, "oracle", "_build", "liboracle.so")
    oracle = pkg.context.Backend(pkg.Api(ctypes.CDLL(so), "wao_"))
    eng = pkg.Engine(0)
    cores = os.cpu_count() or 1
    rows = []
    for name, build in BS.SCENARIOS:
        if args.only and args.only.lower() not in name.lower():
            continue
        row = {"scenario": name}
        try:
            ctxs = [build(pkg, eng.backend, args.seconds) for _ in range(args.graphs)]
            ch, length, sr = ctxs[0]._channels, ctxs[0]._length, ctxs[0]._sample_rate
            audio_s = length / sr
            t0 = time.perf_counter()
            batch = pkg.Batch(ctxs)
            row["prepare_ms"] = (time.perf_counter() - t0) * 1e3
            batch.run()
            batch.sync()
            ms = []
            for _ in range(args.steps):
                batch.run()
                batch.sync()
                ms.append(batch.stats().last_run_ms)
            gpu_ms = float(np.median(ms))
            st = batch.stats()
            got = batch.fetch().reshape(args.graphs, ch, length)[0].copy()
            batch.destroy()
            del ctxs
            row.update({"channels": ch, "frames": length, "sample_rate": sr, "graphs": args.graphs, "gpu_ms_per_batch": gpu_ms,
                        "gpu_x_realtime": args.graphs * audio_s / (gpu_ms * 1e-3), "kernel_launches": int(st.kernel_launches_per_run),
                        "chunks": int(st.chunks)})
            # CPU: one context on one core (the reference benchmark's own measurement), then the batch over all cores
            n_cpu = min(args.graphs, cores)
            octx = [build(pkg, oracle, args.seconds) for _ in range(n_cpu)]
            arr1 = (ctypes.c_void_p * 1)(octx[0]._g)
            ref = np.empty((1, ch, length), np.float32)
            secs = ctypes.c_double()
            oracle.api.check(oracle.api.render_many(arr1, 1, ref.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), 1, ctypes.byref(secs)))
            row["cpu_1core_ms"] = secs.value * 1e3
            row["cpu_1core_x_realtime"] = audio_s / secs.value
            row["max_abs_diff"] = float(np.abs(got.astype(np.float64) - ref[0]).max())
            row["ref_abs_max"] = float(np.abs(ref[0]).max())
            if n_cpu > 1:
                arr = (ctypes.c_void_p * (n_cpu - 1))(*[c._g for c in octx[1:]])
                many = np.empty((n_cpu - 1, ch, length), np.float32)
                oracle.api.check(oracle.api.render_many(arr, n_cpu - 1, many.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), n_cpu - 1, ctypes.byref(secs)))
                row["cpu_allcores_x_realtime"] = (n_cpu - 1) * audio_s / secs.value
                row["cpu_threads"] = n_cpu - 1
            row["gpu_over_cpu_1core"] = row["gpu_x_realtime"] / row["cpu_1core_x_realtime"]
        except Exception as e:  # a scenario the engine refuses is reported, not hidden
            row["error"] = "%s: %s" % (type(e).__name__, e)
        rows.append(row)
        print(json.dumps(row), flush=True)
    eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump({"seconds": args.seconds, "graphs": args.graphs, "steps": args.steps, "host_cores": cores, "rows": rows}, open(args.out, "w"), indent=1)
        md = ["| scenario | ch x s | GPU ms / %d graphs | GPU x realtime | CPU port 1 core x realtime | CPU all cores x realtime | GPU / 1 core | max diff |" % args.graphs,
              "|---|---|---|---|---|---|---|---|"]
        for r in rows:
            if "error" in r:
                md.append("| %s | | | | | | | %s |" % (r["scenario"], r["error"]))
            else:
                md.append("| %s | %d x %.1f | %.2f | %.0f | %.0f | %s | %.0f | %.1e |" % (
                    r["scenario"], r["channels"], r["frames"] / r["sample_rate"], r["gpu_ms_per_batch"], r["gpu_x_realtime"], r["cpu_1core_x_realtime"],
                    ("%.0f" % r["cpu_allcores_x_realtime"]) if "cpu_allcores_x_realtime" in r else "-", r["gpu_over_cpu_1core"], r["max_abs_diff"]))
        open(os.path.splitext(args.out)[0] + ".md", "w").write("\n".join(md) + "\n")


if __name__ == "__main__":
    main()
