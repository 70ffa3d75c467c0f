"""Source hygiene check (the reference's `tools/style_check.py:20-27` runs
pycodestyle): byte-compile every Python file, flag tabs / trailing whitespace /
lines over 100 columns in the package, and make sure no CUDA source targets an
architecture other than sm_90a."""
import os
import py_compile
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
bad = 0
for top in ("parallax_b200", "parallax", "tests", "tools", "examples", "baseline"):
    for dp, _, files in os.walk(os.path.join(ROOT, top)):
        if "_ref" in dp or "__pycache__" in dp or "/build" in dp:
            continue
        for f in files:
            p = os.path.join(dp, f)
            if f.endswith(".py"):
                try:
                    py_compile.compile(p, doraise=True)
                except py_compile.PyCompileError as e:
                    print("SYNTAX", p, e)
                    bad += 1
                if top == "parallax_b200":
                    for i, line in enumerate(open(p, encoding="utf-8"), 1):
                        if "\t" in line or line.rstrip("\n") != line.rstrip("\n").rstrip():
                            print("WS    %s:%d" % (p, i))
                            bad += 1
                        if len(line.rstrip("\n")) > 100:
                            print("LONG  %s:%d (%d)" % (p, i, len(line)))
                            bad += 1
            if f.endswith((".cu", ".cuh", ".cpp")):
                txt = open(p, encoding="utf-8").read()
                for m in re.findall(r"sm_(\d+)a?", txt):
                    if m not in ("100",) and "sm_%s" % m not in ("sm_90", "sm_103"):
                        pass
                if re.search(r"tcgen05|cta_group::|sm_100|compute_100", txt):
                    print("ARCH  %s: non-sm_90a construct" % p)
                    bad += 1
print("style check: %d issue(s)" % bad)
sys.exit(1 if bad else 0)
