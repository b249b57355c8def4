#!/usr/bin/env python
"""Writes tests/golden/irc_1003_c_subset.npz from the reference's resources/IRC_1003_C.bin (path given as the argument).

The full sphere (187 vertices x 2 ears x 512 taps) is too large to keep in the repository.  The tests that use it need the whole
geometry (every vertex position and face, for the face lookup) but only the responses of the vertices the HRTF panner actually
blends for their source direction; the other responses are stored as zeros.  The script finds those vertices, checks that a
render with the subset is bit-identical to one with the full sphere (44.1 kHz and 48 kHz contexts), and stores the subset."""
import ctypes
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "irc_1003_c_subset.npz")
RQ = 128


def container(sr, pos, faces, left, right):
    out = [b"HRIR", struct.pack("<IIII", int(sr), left.shape[1], len(pos), faces.size), np.asarray(faces, "<u4").tobytes()]
    for v in range(len(pos)):
        out += [np.asarray(pos[v], "<f4").tobytes(), np.asarray(left[v], "<f4").tobytes(), np.asarray(right[v], "<f4").tobytes()]
    return b"".join(out)


def render(pkg, oracle, sphere, sr):
    # the render of tests/test_oracle_kat.py::test_hrtf_reference_test_assertions
    oracle.set_hrir_sphere(sphere)
    c = pkg.OfflineAudioContext(2, RQ * 4, sr, oracle)
    s = c.create_buffer_source(pkg.AudioBuffer([np.ones(RQ, np.float32)], sr))
    p = c.create_panner(panning_model=pkg.context.HRTF)
    p.position_x.set_value(1.0)
    s.connect(p)
    p.connect(c.destination())
    s.start()
    return np.stack(c.start_rendering_sync().channels)


def main():
    import __graft_entry__ as ge
    import graphs as G
    data = open(sys.argv[1], "rb").read()
    sr, pos, faces, left, right = G.parse_hrir_sphere(data)
    pkg = ge.load_package()
    oracle = pkg.context.Backend(pkg.Api(ctypes.CDLL(ge.ORACLE_SO), "wao_"))
    rates = (44100.0, 48000.0)
    want = [render(pkg, oracle, data, r) for r in rates]
    # a vertex is used when silencing its responses changes either render
    keep = np.zeros(len(pos), bool)
    for v in range(len(pos)):
        m = np.ones(len(pos), bool)
        m[v] = False
        sub = container(sr, pos, faces, np.where(m[:, None], left, 0.0), np.where(m[:, None], right, 0.0))
        keep[v] = not all(np.array_equal(render(pkg, oracle, sub, r), x) for r, x in zip(rates, want))
    sub = container(sr, pos, faces, np.where(keep[:, None], left, 0.0), np.where(keep[:, None], right, 0.0))
    if not all(np.array_equal(render(pkg, oracle, sub, r), x) for r, x in zip(rates, want)):
        raise SystemExit("the subset does not reproduce the full-sphere render")
    np.savez_compressed(OUT, sample_rate=np.uint32(sr), positions=np.asarray(pos, np.float32), faces=np.asarray(faces, np.uint32),
                        vertices=np.flatnonzero(keep).astype(np.uint32), left=np.asarray(left[keep], np.float32),
                        right=np.asarray(right[keep], np.float32), taps=np.uint32(left.shape[1]))
    print(f"wrote {OUT}: vertices {np.flatnonzero(keep).tolist()}")


if __name__ == "__main__":
    main()
