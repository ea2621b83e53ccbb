#!/usr/bin/env python3
"""Mechanical provenance of tests/golden/pairing_kats.json: the reference's Tate pairing values and its kzg::check cases.

Every integer vector of the JSON is located in the cited source file of a checkout of the reference's Rust sources
(path in RONK_REFERENCE) as a contiguous run of its numeric literals, with the same literal stream as
extract_reference_kats.py (type parameters, const-generic sizes and suffixes stripped).  A vector that cannot be found
is an error.  The check cases' expectations (true / false / panic) are the reference's behaviour as restated by
tests/pairing_oracle.c; tests/test_pairing_oracle.py checks them.

Run:  RONK_REFERENCE=<checkout> python tests/golden/extract_pairing_kats.py     (exit code 1 on any unlocated vector)
It is run by hand when the JSON changes; the test suite does not depend on the reference's sources."""
from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import extract_reference_kats as ek  # noqa: E402

JSON_PATH = os.path.join(HERE, "pairing_kats.json")


def main():
    if not os.path.isdir(os.path.join(ek.REF, "src")):
        sys.exit("set RONK_REFERENCE to a checkout of the reference's sources")
    with open(JSON_PATH) as f:
        kats = json.load(f)
    problems, located = [], 0
    streams = {}

    def locate(label, vec, rel):
        nonlocal located
        if rel not in streams:
            streams[rel] = ek.number_stream(ek.read(rel))
        vec = [int(v) for v in vec]
        if ek.contains_run(streams[rel], vec):
            located += 1
        else:
            problems.append(f"{label}: {vec} not found in {rel}")

    for i, t in enumerate(kats["tate"]):
        for key in ("p", "q", "expected"):
            locate(f"tate[{i}].{key}", t[key], "src/curve/pairing.rs")
    tests = "src/kzg/tests.rs"
    for c in kats["check"]:
        locate(f"check.{c['test']}.coeffs", c["coeffs"], tests)
    for test in ("e2e", "invalid_check", "fake_proof"):   # the rstest points, in case order
        locate(f"check.{test}.points", [c["point"] for c in kats["check"] if c["test"] == test], tests)
    locate("check.invalid_check.value", [c["value"] for c in kats["check"] if c["test"] == "invalid_check"][:1], tests)
    pp = kats["pairing_params"]
    locate("pairing_params.point", [pp["point"]], tests)
    locate("pairing_params.q", ek.point_literals(pp["q"])[0], tests)
    print(json.dumps({"located": located, "problems": problems}, indent=1))
    return 1 if problems else 0


if __name__ == "__main__":
    sys.exit(main())
