#!/usr/bin/env python3
"""Mechanical provenance of tests/golden/poseidon_kats.json: the reference's Poseidon parameters, constants, known
answer and sponge case shapes (src/hashes/poseidon/tests/{constants,mod}.rs).

Everything is parsed from a checkout of the reference's Rust sources (path in RONK_REFERENCE) with the literal parser of
extract_reference_kats.py: the constant vectors as the numeric literal stream of their `let` blocks, the four
parameters from their `pub const` lines, the sponge cases from the `#[case(...)]` tables above each test function.
Each entry carries the file:line it was read from.  The sponge cases are checked against arkworks on random inputs in
the reference, so they fix shapes (sizes, repeat counts), not output words.

Run:  RONK_REFERENCE=<checkout> python tests/golden/extract_poseidon_kats.py            (check: exit code 1 on a mismatch)
      RONK_REFERENCE=<checkout> python tests/golden/extract_poseidon_kats.py --write    (rewrite the JSON from the parse)
It is run by hand when the JSON changes; the test suite does not depend on the reference's sources."""
from __future__ import annotations

import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import extract_reference_kats as ek  # noqa: E402

JSON_PATH = os.path.join(HERE, "poseidon_kats.json")
CONSTANTS = "src/hashes/poseidon/tests/constants.rs"
TESTS = "src/hashes/poseidon/tests/mod.rs"
SPONGE_TESTS = {   # test function → names of its #[case] columns
    "poseidon_sponge_single_absorb_squeeze": ["absorb_size", "squeeze_size"],
    "poseidon_sponge_multiple_absorb_single_squeeze": ["absorb_size", "absorb_time", "squeeze_size"],
    "poseidon_sponge_multiple_absorb_multiple_squeeze": ["absorb_size", "absorb_time", "squeeze_size", "squeeze_time"],
    "poseidon_sponge_multiple_absorb_vs_one_time_absorb": ["absorb_size", "absorb_time", "squeeze_size"],
}


def line_of(src: str, pos: int) -> int:
    return src.count("\n", 0, pos) + 1


def parse():
    consts, tests = ek.read(CONSTANTS), ek.read(TESTS)
    out = {"field": 101, "field_src": "src/algebra/field/prime/mod.rs (PlutoBaseField)"}
    for name in ("ALPHA", "WIDTH", "NUM_F", "NUM_P"):
        m = re.search(r"pub const " + name + r": usize = (\d+);", consts)
        out[name.lower()] = int(m.group(1))
        out[name.lower() + "_src"] = f"{CONSTANTS}:{line_of(consts, m.start())}"
    for name in ("rc16", "mds16"):
        start = consts.index(f"let {name}")
        end = consts.index("];", start)
        body = consts[consts.index("vec![", start) + len("vec!["):end]
        if name == "rc16":
            out[name] = ek.number_stream(body)
        else:
            out[name] = [ek.number_stream(row) for row in re.findall(r"vec!\[([^\]]*)\]", body)]
        out[name + "_src"] = f"{CONSTANTS}:{line_of(consts, start)}-{line_of(consts, end)}"
    m = re.search(r"fn hash\(.*?PlutoBaseField::new\((\d+)\)", tests, re.S)
    out["hash_zero"] = {"state": [0] * out["width"], "expected": int(m.group(1)),
                        "src": f"{TESTS}:{line_of(tests, m.start())}-{line_of(tests, m.end())}"}
    cases = []
    for fn, cols in SPONGE_TESTS.items():
        pos = tests.index(f"fn {fn}(")
        for case in ek.rstest_cases(tests, fn):
            cases.append({"test": fn, **{c: v for c, (_, v) in zip(cols, case)}, "src": f"{TESTS}:{line_of(tests, pos)}"})
    out["sponge_cases"] = cases
    m = re.search(r"fn rate\(\) -> usize \{ (\d+) \}", tests)
    out["rate"] = int(m.group(1))
    out["rate_src"] = f"{TESTS}:{line_of(tests, m.start())}"
    return out


def main():
    if not os.path.isdir(os.path.join(ek.REF, "src")):
        sys.exit("set RONK_REFERENCE to a checkout of the reference's sources")
    parsed = parse()
    if "--write" in sys.argv:
        with open(JSON_PATH, "w") as f:
            json.dump(parsed, f, indent=1)
            f.write("\n")
        print(f"wrote {JSON_PATH}")
        return 0
    with open(JSON_PATH) as f:
        have = json.load(f)
    problems = [k for k in sorted(set(parsed) | set(have)) if parsed.get(k) != have.get(k)]
    print(json.dumps({"keys": len(parsed), "problems": problems}, indent=1))
    return 1 if problems else 0


if __name__ == "__main__":
    sys.exit(main())
