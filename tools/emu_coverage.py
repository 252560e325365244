"""Which lines of the kernel sources a pytest selection runs, on the SIMT emulator (tests/emu_lib.py).

Builds the emulator with --coverage under its own library name (ARMADA_EMU_COVERAGE=1; the plain emulator library is
left alone), runs the selection against it and prints, per armada_b200/csrc/*.inc file, the lines that carry code and
never ran, a line counting as run when any template instantiation ran it.

    python tools/emu_coverage.py [--lines armada_pass.inc:424,3739-3757 ...] -- [pytest arguments]

--lines also reports, for each range given, which of its lines ran.  The default selection is the non-GPU suite."""
from __future__ import annotations

import argparse
import collections
import glob
import gzip
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
os.environ["ARMADA_EMU_COVERAGE"] = "1"
import emu_lib  # noqa: E402  (reads ARMADA_EMU_COVERAGE)


def ranges(lines):
    out, start, prev = [], None, None
    for n in sorted(lines):
        if start is None:
            start = prev = n
        elif n == prev + 1:
            prev = n
        else:
            out.append((start, prev))
            start = prev = n
    if start is not None:
        out.append((start, prev))
    return ", ".join(str(a) if a == b else f"{a}-{b}" for a, b in out)


def line_counts(gcda: str):
    """{source file: {line: count}} over every function (template instantiation) that contains the line."""
    out = subprocess.run(["gcov", "--json-format", "--stdout", "--object-directory", os.path.dirname(gcda), gcda],
                         cwd=ROOT, check=True, capture_output=True).stdout
    if out[:2] == b"\x1f\x8b":
        out = gzip.decompress(out)
    counts = collections.defaultdict(dict)
    for doc in out.decode().splitlines():
        if not doc.strip():
            continue
        for f in json.loads(doc)["files"]:
            name = os.path.basename(f["file"])
            for ln in f["lines"]:
                n = ln["line_number"]
                counts[name][n] = max(counts[name].get(n, 0), ln["count"])
    return counts


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lines", nargs="*", default=[], help="FILE:A[-B][,C[-D]…]: report these lines")
    ap.add_argument("pytest_args", nargs="*", default=["-m", "not gpu", "tests"])
    args = ap.parse_args()
    emu_lib.build()
    for f in glob.glob(os.path.join(emu_lib.EMU_DIR, "*.gcda")):
        os.remove(f)
    rc = subprocess.run([sys.executable, "-m", "pytest", "-p", "no:cacheprovider", *args.pytest_args], cwd=ROOT).returncode
    gcda = glob.glob(emu_lib.EMU_LIB + "*.gcda")
    if not gcda:
        print("no coverage data: the selection loaded no emulator library", file=sys.stderr)
        return 1
    counts = line_counts(gcda[0])
    print(f"\npytest exit status {rc}; lines of armada_b200/csrc/*.inc that never ran:")
    for name in sorted(n for n in counts if n.endswith(".inc")):
        never = [n for n, c in counts[name].items() if c == 0]
        print(f"  {name} ({len(never)} of {len(counts[name])} lines): {ranges(never) or '-'}")
    for spec in args.lines:
        name, rs = spec.split(":")
        want = set()
        for r in rs.split(","):
            a, _, b = r.partition("-")
            want.update(range(int(a), int(b or a) + 1))
        have = counts.get(name, {})
        code = [n for n in sorted(want) if n in have]
        ran = [n for n in code if have[n] > 0]
        print(f"  {name}:{rs}: ran {ranges(ran) or '-'}; never ran {ranges(set(code) - set(ran)) or '-'}")
    return rc


if __name__ == "__main__":
    sys.exit(main())
