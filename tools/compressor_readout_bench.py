"""Compressor reduction read-outs (wae_compressor_set_readouts) and analyser byte read-outs (wae_analyser_set_byte_readouts) on the GPU.

- 1000 stereo graphs of 10 s (oscillator -> DynamicsCompressorNode -> destination): median run + sync with a reduction read-out every
  quantum (3750 per graph) and without the declaration.
- The analyser bench's shape (tools/analyser_readout_bench.py: oscillator -> biquad -> analyser of fftSize 2048 -> destination, a
  frequency read-out every 1024 frames): median run + sync with the float rows alone and with byte rows added.

Medians after a warm-up run.  Prints one JSON line with the card's name and power limit, read in the same call."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    import __graft_entry__ as entry
    pkg = entry.load_package()
    sr, fft_size, hop = 48000.0, 2048, 1024
    length = int(args.seconds * sr)
    eng = pkg.Engine(0)

    def compressors(declare):
        ctxs, nodes = [], []
        quanta = length // 128
        for g in range(args.graphs):
            c = pkg.OfflineAudioContext(2, length, sr, eng.backend)
            o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=110.0 + g)
            d = c.create_dynamics_compressor(threshold=-30.0)
            o.connect(d)
            d.connect(c.destination())
            o.start()
            if declare:
                d.set_readouts((np.arange(1, quanta + 1) * 128 - 0.5) / sr)
            ctxs.append(c)
            nodes.append(d)
        return pkg.context.Batch(ctxs), nodes

    def analysers(byte):
        ctxs, nodes = [], []
        times = np.arange(1, length // hop + 1) * hop / sr
        for g in range(args.graphs):
            c = pkg.OfflineAudioContext(2, length, sr, eng.backend)
            o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=110.0 + g)
            bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=2000.0, q=1.0)
            a = c.create_analyser(fft_size=fft_size)
            o.connect(bq)
            bq.connect(a)
            a.connect(c.destination())
            o.start()
            a.set_readouts(times)
            if byte:
                a.set_byte_readouts(frequency=True)
            ctxs.append(c)
            nodes.append(a)
        return pkg.context.Batch(ctxs), nodes

    def timed(b):
        b.run()
        b.sync()
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            b.run()
            b.sync()
            ts.append(time.perf_counter() - t0)
        return float(np.median(ts)) * 1e3

    res = {"card": card(), "graphs": args.graphs, "seconds": args.seconds, "reps": args.reps}
    for name, declare in (("compressor_run_ms_without", False), ("compressor_run_ms_with_readouts", True)):
        b, nodes = compressors(declare)
        res[name] = timed(b)
        if declare:
            res["compressor_readout_shape"] = list(b.compressor_readouts(nodes[0]).shape)
            torch.cuda.synchronize()
        b.destroy()
    for name, byte in (("analyser_run_ms_float_rows", False), ("analyser_run_ms_float_and_byte_rows", True)):
        b, nodes = analysers(byte)
        res[name] = timed(b)
        if byte:
            res["byte_readout_shape"] = list(b.analyser_readouts(nodes[0], byte=True).shape)
            torch.cuda.synchronize()
        b.destroy()
    eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
