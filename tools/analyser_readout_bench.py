"""Analyser read-outs at declared render times (wae_analyser_set_readouts) on the GPU: 1000 stereo graphs of 10 s (oscillator -> biquad ->
analyser -> destination), one analyser each (fftSize 2048), a read-out every 1024 frames (469 per graph, frequency data).  Median time
of run + sync with and without the declaration, and torch.stft of the rendered output (the same hop and window length) as a point of
reference.  Prints one JSON line with the card's name and power limit."""
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
    times = np.arange(1, length // hop + 1) * hop / sr
    eng = pkg.Engine(0)

    def make(declare):
        ctxs = []
        for g in range(args.graphs):
            c = pkg.OfflineAudioContext(2, length, sr, eng.backend)
            o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=110.0 + g)
            bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=2000.0, q=1.0)
            a = c.create_analyser(fft_size=fft_size)
            o.connect(bq)
            bq.connect(a)
            a.connect(c.destination())
            o.start()
            if declare:
                a.set_readouts(times)
            ctxs.append(c)
        return pkg.context.Batch(ctxs)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return float(np.median(ts)) * 1e3

    res = {"card": card(), "graphs": args.graphs, "seconds": args.seconds, "fft_size": fft_size, "readouts_per_graph": len(times)}
    for name, declare in (("run_ms_without", False), ("run_ms_with_readouts", True)):
        b = make(declare)

        def run():
            b.run()
            b.sync()
        res[name] = timed(run)
        if declare:
            view = b.analyser_readouts(b.contexts[0]._readout_nodes[next(iter(b.contexts[0]._readout_nodes))])
            res["readout_shape"] = list(view.shape)
        else:
            out = b.output_tensor()
            win = torch.blackman_window(fft_size, device=out.device)
            res["torch_stft_ms"] = timed(lambda: torch.stft(out.mean(1), fft_size, hop_length=hop, window=win, return_complex=True).abs())
        b.destroy()
    eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
