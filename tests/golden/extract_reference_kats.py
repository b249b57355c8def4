#!/usr/bin/env python
"""Extracts known-answer vectors from the reference's own #[test]s into tests/golden/reference_kats.json.

Usage: python tests/golden/extract_reference_kats.py <checkout of the reference>.  The JSON is committed, so the tests do
not need the reference's sources.  Only numeric literals of test tables are read — no reference code is copied.
  - biquad frequency responses, Chrome/Firefox values  (src/node/biquad_filter.rs:1000-1412)
  - un-normalised biquad coefficients for f0=2000, Q=1, gain=3 @44.1k (src/node/iir_filter.rs:611-755)
  - IIR magnitude response vs scipy                      (src/node/iir_filter.rs:757-800)
"""
import json
import os
import re
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "reference"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_kats.json")
NUM = r"-?\d[\d_]*\.?[\d_]*(?:[eE]-?\d+)?"


def floats(block):
    return [float(x.replace("_", "")) for x in re.findall(NUM, block)]


def main():
    out = {}
    src = open(os.path.join(REF, "src/node/biquad_filter.rs")).read()
    resp = {}
    for m in re.finditer(r"fn test_frequency_responses_(\w+)\(\)\s*\{(.*?)\n    \}", src, re.S):
        name, body = m.group(1), m.group(2)
        if name.startswith("arguments"):
            continue
        d = {}
        for key in ("frequency", "q", "gain"):
            d[key] = float(re.search(r"let %s = (%s);" % (key, NUM), body).group(1))
        d["freqs"] = floats(re.search(r"let freqs = \[(.*?)\];", body, re.S).group(1))
        d["mags"] = floats(re.search(r"let expected_mags = \[(.*?)\];", body, re.S).group(1))
        d["phases"] = floats(re.search(r"let expected_phases = \[(.*?)\];", body, re.S).group(1))
        d["tol"] = 1e-6
        d["source"] = "src/node/biquad_filter.rs test_frequency_responses_" + name
        resp[name] = d
    out["biquad_frequency_response"] = resp

    src = open(os.path.join(REF, "src/node/iir_filter.rs")).read()
    body = re.search(r"fn test_output_against_biquad\(\)(.*?)\n    #\[test\]", src, re.S).group(1)
    coefs = {}
    for m in re.finditer(r"// (\w+)\n\s*let a0 = (%s);\s*let a1 = (%s);\s*let a2 = (%s);\s*let b0 = (%s);\s*let b1 = (%s);\s*let b2 = (%s);"
                         % ((NUM,) * 6), body):
        coefs[m.group(1)] = {"a": [float(m.group(i)) for i in (2, 3, 4)], "b": [float(m.group(i)) for i in (5, 6, 7)]}
    out["biquad_unnormalised_coefs"] = {"frequency": 2000.0, "q": 1.0, "gain": 3.0, "sample_rate": 44100.0, "types": coefs,
                                        "source": "src/node/iir_filter.rs:605-755 test_output_against_biquad"}
    body = re.search(r"fn tests_get_frequency_response\(\)(.*?)\n    #\[test\]", src, re.S).group(1)
    out["iir_frequency_response"] = {
        "ref_mag": floats(re.search(r"let ref_mag = \[(.*?)\];", body, re.S).group(1)),
        "feedforward": floats(re.search(r"let feedforward = vec!\[(.*?)\];", body, re.S).group(1)),
        "feedback": floats(re.search(r"let feedback = vec!\[(.*?)\];", body, re.S).group(1)),
        "frequency_hz": floats(re.search(r"let frequency_hz = \[(.*?)\];", body, re.S).group(1)),
        "sample_rate": 44100.0, "source": "src/node/iir_filter.rs:757-800 tests_get_frequency_response (scipy)"}
    json.dump(out, open(OUT, "w"), indent=1)
    print("wrote", OUT, {k: len(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
