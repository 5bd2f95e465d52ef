#!/usr/bin/env bash
# Branch coverage of the butteraugli metric's value-dependent branches under the float-input corpus
# of tests/test_metric_inputs.py.
#
# Builds the CPU port (oracle/Makefile.port: the same ba_math.h and kernels.h bodies the CUDA kernels
# run) with --coverage at -O0 into a temporary directory, runs the CPU half of the module against
# that build (GB200_PORT_LIB), and prints for every value-dependent branch of ba_math.h and of the
# per-pixel functors of kernels.h how often each of its arcs ran.  -O0 keeps every `if` and `?:` a
# branch of its own; the results must still equal the reference bit for bit, or the tests fail.
#
# The fused CUDA epilogues (fused_kernels.cuh: EpiHf's copy of the SameNoiseLevels clamp, and the
# epilogues that call maximum_clamp, malta_diff and mask_lut_eval) cannot be measured this way.  They
# get the same values at the same stage of the chain as the port's functors, so the port's coverage
# stands in for theirs; the GPU half of the module checks that they compute the same bits.
#
# Uses only the repository's own code.  Needs g++, gcov, python3 with numpy and pytest.  The tests
# run on one thread of an unoptimised build: a full run takes about 25 minutes, most of it the
# 1080x1920 case (-k "not 1080x1920" leaves it out).
#   tools/metric_branch_coverage.sh [extra pytest arguments]
set -euo pipefail
ROOT="$(cd "$(dirname "${BASH_SOURCE[0]}")/.." && pwd)"
TMP="$(mktemp -d)"
trap 'rm -rf "$TMP"' EXIT

# -O0 comes after Makefile.port's -O2 and wins; --coverage in CXX reaches the compile and the link
echo 'CXXFLAGS += -O0 -w' > "$TMP/coverage.mk"
make -s -C "$ROOT/oracle" -f Makefile.port -f "$TMP/coverage.mk" OUT="$TMP" CXX="g++ --coverage" \
  -j "$(nproc)" "$TMP/libguetzli_port.so" >/dev/null

cd "$ROOT"
# one thread: the coverage counters are shared by all threads, and OpenMP workers contending for them
# make the run many times slower
GB200_PORT_LIB="$TMP/libguetzli_port.so" OMP_NUM_THREADS=1 python3 -m pytest tests/test_metric_inputs.py -m "not gpu" -q \
  -p no:cacheprovider "$@" | tail -3

(cd "$TMP" && gcov --json-format --branch-probabilities --branch-counts "$TMP"/*.gcda >/dev/null 2>&1)
python3 - "$TMP" "$ROOT/guetzli_b200/csrc" <<'EOF'
import collections, glob, gzip, json, os, re, sys
tmp, csrc = sys.argv[1:]
# (file, line) -> per-arc counts, summed over the translation units that instantiate the line
arcs = collections.defaultdict(list)
for path in glob.glob(os.path.join(tmp, "*.gcov.json.gz")):
    for f in json.load(gzip.open(path))["files"]:
        name = os.path.basename(f["file"])
        if name not in ("ba_math.h", "kernels.h"):
            continue
        for ln in f["lines"]:
            counts = [b["count"] for b in ln.get("branches", []) if not b.get("throw")]
            if not counts:
                continue
            have = arcs[(name, ln["line_number"])]
            have.extend([0] * (len(counts) - len(have)))
            for i, c in enumerate(counts):
                have[i] += c

# (label, file, function whose body holds the line, the line's text); the arcs of each line are
# listed in gcov's order, two per condition
BRANCHES = [
    ("gamma_poly: yq == 0", "ba_math.h", "gamma_poly", r"if \(yq == 0\.0\)"),
    ("remove_range_around_zero: x > w, x < -w", "ba_math.h", "remove_range_around_zero", r"return x > w"),
    ("amplify_range_around_zero: x > w, x < -w", "ba_math.h", "amplify_range_around_zero", r"return x > w"),
    ("maximum_clamp: v >= maxval", "ba_math.h", "maximum_clamp", r"if \(v >= maxval\)"),
    ("maximum_clamp: v < -maxval", "ba_math.h", "maximum_clamp", r"else if \(v < -maxval\)"),
    ("malta_diff: v0 < 0", "ba_math.h", "malta_diff", r"if \(v0 < 0\)"),
    ("malta_diff: v0 < 0 and r1 > -too_small", "ba_math.h", "malta_diff", r"if \(r1 > -too_small\)"),
    ("malta_diff: v0 < 0 and r1 < -too_big", "ba_math.h", "malta_diff", r"else if \(r1 < -too_big\)"),
    ("malta_diff: v0 >= 0 and r1 < too_small", "ba_math.h", "malta_diff", r"if \(r1 < too_small\)"),
    ("malta_diff: v0 >= 0 and r1 > too_big", "ba_math.h", "malta_diff", r"else if \(r1 > too_big\)"),
    ("malta_diff: an objective applies", "ba_math.h", "malta_diff", r"if \(has\)"),
    ("malta_diff: diff < 0", "ba_math.h", "malta_diff", r"if \(diff < 0\)"),
    ("mask_lut_eval: ix < 0", "ba_math.h", "mask_lut_eval", r"if \(ix < 0\)"),
    ("mask_lut_eval: baseix >= 511 (top clamp)", "ba_math.h", "mask_lut_eval", r"if \(baseix >= 511\)"),
    ("NoisePre: v0 > maxclamp (85.7)", "kernels.h", "struct NoisePre", r"if \(v0 > maxclamp\)"),
    ("NoisePre: v1 > maxclamp (85.7)", "kernels.h", "struct NoisePre", r"if \(v1 > maxclamp\)"),
    ("CombineAndSqrt: v < 1e-4 (linear) or sqrt", "kernels.h", "struct CombineAndSqrt", r"out\[o\] = \(v < "),
]
print(f"{'branch':46s} {'line':>10s}  arc counts")
missing = []
for label, name, func, pattern in BRANCHES:
    lines = open(os.path.join(csrc, name)).read().split("\n")
    start = next(i for i, t in enumerate(lines) if func in t and ("(" in t or "{" in t))
    ln = next(i for i in range(start, len(lines)) if re.search(pattern, lines[i])) + 1
    counts = arcs.get((name, ln))
    if counts is None:
        missing.append(label)
        print(f"{label:46s} {name}:{ln:<4d}  never reached")
        continue
    print(f"{label:46s} {name}:{ln:<4d}  {counts}{'' if all(counts) else '   <- an arc never ran'}")
if missing:
    sys.exit(f"no coverage data for: {missing}")
EOF
