#!/usr/bin/env python3
"""Mechanical provenance of tests/golden/sha_merkle_kats.json: the reference's SHA-256 known answers
(src/hashes/sha.rs, the `#[case]` table of `test_sha256`) and its Merkle-tree tests (src/tree/merkle.rs, `mod tests`):
each test's leaf lists, the level counts it asserts, the index it opens, the value it proves and the sibling it zeroes.

Everything is parsed from a checkout of the reference's Rust sources (path in RONK_REFERENCE), and each entry carries
the file:line it was read from.

Run:  RONK_REFERENCE=<checkout> python tests/golden/extract_sha_merkle_kats.py            (check: exit code 1 on a mismatch)
      RONK_REFERENCE=<checkout> python tests/golden/extract_sha_merkle_kats.py --write    (rewrite the JSON from the parse)
It is run by hand when the JSON changes; the test suite does not depend on the reference's sources."""
from __future__ import annotations

import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
JSON_PATH = os.path.join(HERE, "sha_merkle_kats.json")
SHA = "src/hashes/sha.rs"
MERKLE = "src/tree/merkle.rs"


def line_of(src: str, pos: int) -> int:
    return src.count("\n", 0, pos) + 1


def parse_sha(src: str):
    start = src.index("fn test_sha512")
    end = src.index("fn test_sha256")
    cases = []
    for m in re.finditer(r'#\[case\(\s*b"((?:[^"\\]|\\.)*)",\s*"([0-9a-f]{64})"\s*,?\s*\)\]', src[start:end]):
        a, b = line_of(src, start + m.start()), line_of(src, start + m.end())
        cases.append({"input": m.group(1), "digest": m.group(2), "src": f"{SHA}:{a}" + (f"-{b}" if b != a else "")})
    return cases


def parse_merkle(src: str):
    mod = src.index("mod tests")
    tests = {}
    fns = list(re.finditer(r"#\[test\]\s*(#\[should_panic\]\s*)?fn (\w+)\(\)", src[mod:]))
    for k, f in enumerate(fns):
        s = mod + f.start()
        e = mod + fns[k + 1].start() if k + 1 < len(fns) else src.rindex("}")  # the last test ends before the module
        body = src[s:e]
        t = {"should_panic": bool(f.group(1)), "src": f"{MERKLE}:{line_of(src, s)}-{line_of(src, src.rindex("}", s, e))}"}
        t["trees"] = [re.findall(r'"([^"]*)"\.to_string\(\)', v.group(1))
                      for v in re.finditer(r"vec!\[(.*?)\]", body, re.S)]
        if m := re.search(r"tree\.hashes\.len\(\),\s*(\d+)\)", body):
            t["levels"] = int(m.group(1))
        sizes = {int(a): int(b) for a, b in re.findall(r"tree\.hashes\[(\d+)\]\.len\(\),\s*(\d+)\)", body)}
        if sizes:
            t["level_sizes_root_first"] = [sizes[i] for i in range(len(sizes))]
        if m := re.search(r"get_proof\((\d+)\)", body):
            t["index"] = int(m.group(1))
        if m := re.search(r'prove\("([^"]*)"\.to_string\(\)', body):
            t["value"] = m.group(1)
        if m := re.search(r"proof\.0\[(\d+)\]\.0 = \[0u8; 32\]", body):
            t["zeroed_sibling"] = int(m.group(1))
        tests[f.group(2)] = t
    return tests


def parse(ref: str):
    with open(os.path.join(ref, SHA)) as f:
        sha = f.read()
    with open(os.path.join(ref, MERKLE)) as f:
        merkle = f.read()
    return {"sha256": parse_sha(sha), "merkle_tests": parse_merkle(merkle)}


def main() -> int:
    ref = os.environ.get("RONK_REFERENCE")
    if not ref:
        print("set RONK_REFERENCE to a checkout of the reference", file=sys.stderr)
        return 2
    got = parse(ref)
    if "--write" in sys.argv:
        with open(JSON_PATH, "w") as f:
            json.dump(got, f, indent=1)
            f.write("\n")
        return 0
    with open(JSON_PATH) as f:
        want = json.load(f)
    if got != want:
        print("sha_merkle_kats.json differs from the reference's sources", file=sys.stderr)
        return 1
    print("sha_merkle_kats.json matches")
    return 0


if __name__ == "__main__":
    sys.exit(main())
