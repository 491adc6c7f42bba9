#!/usr/bin/env python
"""Regenerates tests/golden/reference_runs_receiver.json from the reference built with other receiver constants:

    make -C oracle ref                                  # the unmodified reference (and _ref/build/version.h)
    python tests/golden/make_receiver_golden.py         # REFERENCE=<dir>: the sources, as for oracle/Makefile

For every (clock lock T1/C1, S1; access-code errors T1/C1, S1) of tests/receiver_cases.py VARIANTS the four constant
lines of the reference's rtl_wmbus.c -- opts_CLOCK_LOCK_THRESHOLD_T1_C1 / _S1 (:865-866), ACCESS_CODE_T1_C1_ERRORS /
ACCESS_CODE_S1_ERRORS (:99, :103) -- are substituted into a copy under oracle/_ref/variants/, which is compiled with
the flags oracle/Makefile uses for the reference (its `make release` line).  Every substitution must match exactly once
and the copy may differ from the original in no other line, or the script stops: an upstream edit cannot produce an
unmodified binary under a variant's name.  The output holds, per variant, the lines (TIMESTAMP blanked) for the
captures of receiver_cases.cases(), and the sha256 of the synthetic ones, which the tests generate by seed."""
import json
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import orc  # noqa: E402
import receiver_cases as rc  # noqa: E402


def _makefile_reference():
    """the reference source directory oracle/Makefile builds from (its `REFERENCE ?=` line)"""
    for line in open(os.path.join(ROOT, "oracle", "Makefile")):
        if line.startswith("REFERENCE") and "?=" in line:
            return line.split("?=", 1)[1].strip()
    sys.exit("oracle/Makefile names no REFERENCE")


REFERENCE = os.environ.get("REFERENCE") or _makefile_reference()
OUT = os.path.join(ROOT, "oracle", "_ref")
CONSTANTS = [("opts_CLOCK_LOCK_THRESHOLD_T1_C1", "2"), ("opts_CLOCK_LOCK_THRESHOLD_S1", "2"),
             ("ACCESS_CODE_T1_C1_ERRORS", "0u"), ("ACCESS_CODE_S1_ERRORS", "0u")]


def build_variant(lock, errors):
    src = open(os.path.join(REFERENCE, "rtl_wmbus.c")).read()
    values = [str(lock[0]), str(lock[1]), f"{errors[0]}u", f"{errors[1]}u"]
    for (name, old), new in zip(CONSTANTS, values):
        pat = re.compile(rf"^(static const unsigned {name} = ){re.escape(old)};", re.M)
        src, n = pat.subn(rf"\g<1>{new};", src)
        if n != 1:
            sys.exit(f"substitution of {name} matched {n} times in {REFERENCE}/rtl_wmbus.c")
    orig = open(os.path.join(REFERENCE, "rtl_wmbus.c")).read().split("\n")
    changed = sum(a != b for a, b in zip(orig, src.split("\n")))
    if len(orig) != len(src.split("\n")) or changed != sum(v != o for v, (_, o) in zip(values, CONSTANTS)):
        sys.exit(f"variant {lock} {errors} differs from the reference in other lines than the four constants")
    os.makedirs(os.path.join(OUT, "variants"), exist_ok=True)
    base = os.path.join(OUT, "variants", "rtl_wmbus_" + rc.variant_name(lock, errors))
    with open(base + ".c", "w") as f:
        f.write(src)
    subprocess.run(["gcc", "-DNDEBUG", "-O3", "-std=gnu99", f"-I{REFERENCE}/include", f"-I{REFERENCE}", f"-I{OUT}",
                    "-o", base, base + ".c", "-lm"], check=True)
    return base


def main():
    assert os.path.exists(os.path.join(OUT, "build", "version.h")), "run `make -C oracle ref` first"
    out = {"lines": {}, "capture_sha256": {}}
    caps = {name: rc.capture(name) for name, _ in rc.cases()}
    for name, cu8 in caps.items():
        out["capture_sha256"][name] = orc.capture_sha(cu8)
    for lock, errors in rc.VARIANTS:
        v = rc.variant_name(lock, errors)
        exe = build_variant(lock, errors)
        out["lines"][v] = {}
        for name, flags in rc.cases():
            r = subprocess.run([exe] + flags.split(), input=caps[name].tobytes(), capture_output=True, check=True)
            out["lines"][v][f"{name}|{flags}"] = [orc.blank_ts(l) for l in r.stdout.decode().split("\n") if l]
        print(v, {k: len(x) for k, x in out["lines"][v].items()})
    json.dump(out, open(rc.FIXTURE, "w"), indent=0, sort_keys=True)


if __name__ == "__main__":
    main()
