#!/usr/bin/env python
"""Which of the reference's own #[test]s are restated in tests/ ?  Needs a checkout of the reference (first argument); writes
tests/REFERENCE_TESTS.md.  A reference test counts as restated when one of our test files cites a line range of its source file that
contains the test function (citations look like `param.rs:1814-1872`, or `:1874-1899` after the file was named), or names the function."""
import glob
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = sys.argv[1] if len(sys.argv) > 1 else "reference"
# the files SURVEY.md section 8 puts on the path (+ the integration tests that render offline)
FILES = ["src/param.rs", "src/node/audio_buffer_source.rs", "src/node/oscillator.rs", "src/node/scheduled_source.rs", "src/analysis.rs", "src/buffer.rs",
         "src/node/convolver.rs", "src/node/iir_filter.rs", "src/node/delay.rs", "src/context/offline.rs", "src/node/biquad_filter.rs", "src/render/quantum.rs",
         "src/periodic_wave.rs", "src/node/waveshaper.rs", "tests/offline.rs", "src/spatial.rs", "src/render/graph.rs", "tests/mixing.rs",
         "src/node/dynamics_compressor.rs", "src/node/panner.rs", "src/node/stereo_panner.rs", "src/node/constant_source.rs", "src/node/channel_splitter.rs",
         "src/node/channel_merger.rs", "src/node/analyser.rs", "tests/denormals.rs", "src/node/gain.rs", "src/node/audio_node.rs"]
# tests of the control plane (events, constructors / accessors of the Rust API, thread-safety of futures): outside the render path
CONTROL = re.compile(r"ended_event|onended|onstatechange|oncomplete|thread_safe|thread_safety|concurrency|_async$|clones_in_sync|synchronicity|"
                     r"default_and_accessors|default_build|build_with|default_options|user_defined_options|constructor|after_closed|playing_some_file|"
                     r"while_dropped|test_pool|lifecycle|release_orphaned|test_active|media_element")


# tests of Rust-side API surface that has no counterpart behind the C boundary, with the reason
NOT_APPLICABLE = {
    "test_frequency_response_arguments": "Rust slice-length assert: the C ABI passes ONE length for the three arrays (include/wae.h)",
    "test_frequency_response_arguments_2": "Rust slice-length assert: the C ABI passes ONE length for the three arrays (include/wae.h)",
    "test_channel_data_get_set": "AudioBuffer accessor (host container API, stays in the Rust crate)",
    "test_invalid_copy_from_channel": "AudioBuffer accessor (host container API, stays in the Rust crate)",
    "test_copy_from_channel": "AudioBuffer accessor (host container API, stays in the Rust crate)",
    "test_invalid_copy_to_channel": "AudioBuffer accessor (host container API, stays in the Rust crate)",
    "test_copy_to_channel": "AudioBuffer accessor (host container API, stays in the Rust crate)",
    "test_invalid_get_channel_data": "AudioBuffer accessor (host container API, stays in the Rust crate)",
    "render_twice_panics": "context state machine: stays in the Rust shim (INTEGRATION.md)",
    "test_audiobuffer_channels": "AudioRenderQuantum channel-count bookkeeping without samples to compare; the mixing tables themselves are restated",
    "test_audiobuffer_mix_speakers_all": "AudioRenderQuantum channel-count bookkeeping without samples to compare; the mixing tables themselves are restated",
}


def citations():
    """{file basename: [(lo, hi, our test file)]} + the text of all our tests"""
    cites, text = {}, ""
    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "*.py"))):
        src = open(path).read()
        text += src
        cur = None
        for m in re.finditer(r"(?:(\w+\.rs))?:(\d+)(?:\s*-\s*(\d+))?", src):
            if m.group(1):
                cur = m.group(1)
            if cur is None:
                continue
            lo = int(m.group(2))
            hi = int(m.group(3)) if m.group(3) else lo
            if hi < lo or hi - lo > 4000:
                continue
            cites.setdefault(cur, []).append((lo, hi, os.path.basename(path)))
    return cites, text


def main():
    cites, text = citations()
    rows, tot, done, ctrl = [], 0, 0, 0
    for f in FILES:
        p = os.path.join(REF, f)
        if not os.path.exists(p):
            continue
        lines = open(p).read().split("\n")
        base = os.path.basename(f)
        for i, ln in enumerate(lines):
            if ln.strip() != "#[test]":
                continue
            j = i + 1
            while j < len(lines) and not re.search(r"\bfn\s+\w+", lines[j]):
                j += 1
            name = re.search(r"\bfn\s+(\w+)", lines[j]).group(1)
            fn_line = j + 1
            # the test body: up to the next line that starts a new item at the same indentation
            hit = None
            for lo, hi, ours in cites.get(base, []):
                if lo <= fn_line <= hi or (lo == hi and abs(lo - fn_line) <= 2):
                    hit = ours
                    break
            if hit is None and (name in text or re.sub("^test_", "", name) in text):
                hit = "(by name)"
            tot += 1
            if hit:
                done += 1
                status = "restated: " + hit
            elif name in NOT_APPLICABLE:
                ctrl += 1
                status = "n/a: " + NOT_APPLICABLE[name]
            elif CONTROL.search(name):
                ctrl += 1
                status = "control plane (not on the render path)"
            else:
                status = "NOT restated"
            rows.append((f, fn_line, name, status))
    out = ["# The reference's own tests on the path, and where they are restated", "",
           "Generated by `tools/reference_test_map.py` from the citations in `tests/*.py` (a reference test counts as restated when one of our test files",
           "cites a line range of its source file that contains it, or names it).  Files: the ones SURVEY.md section 8 puts on the path.", "",
           f"**{tot} reference tests: {done} restated, {ctrl} control plane or not applicable behind a C boundary (events, constructors / accessors of the",
           f"Rust API, thread safety — each with its reason), {tot - done - ctrl} not restated.**", "", "| reference file | line | test | status |", "|---|---|---|---|"]
    for f, ln, name, status in rows:
        out.append(f"| {f} | {ln} | `{name}` | {status} |")
    open(os.path.join(ROOT, "tests", "REFERENCE_TESTS.md"), "w").write("\n".join(out) + "\n")
    print(tot, done, ctrl, tot - done - ctrl)
    for f, ln, name, status in rows:
        if status == "NOT restated":
            print(" ", f, ln, name)


if __name__ == "__main__":
    main()
